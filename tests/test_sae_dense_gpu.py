"""Dense ReLU + L1 training step and ghost grads (csrc/sae_dense.cu, vit_prisma/b200/sae_dense.py) against the reference
fixtures (tests/golden/sae_tiny_{d,e,f}.pt: torch autograd + torch.optim.Adam on the unmodified reference module) and, at a
size that reaches the wgmma GEMMs, against the pinned oracle."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle.sae_oracle import lr_multiplier, new_adam_state, sae_train_step  # noqa: E402
from tests.util import assert_close, load_golden, rel_err  # noqa: E402


def _data(gold):
    g = torch.Generator().manual_seed(gold["data_seed"])
    n, d = gold["batch"] * gold["n_steps"], gold["d_in"]
    return torch.randn(n, d, generator=g) * 2.0 + torch.randn(d, generator=g)


def _engine(p, k, norm, l1, impl=None):
    from vit_prisma.b200 import _lib as L
    from vit_prisma.b200.sae_dense import SaeDenseStepEngine
    from vit_prisma.b200.sae_engine import unit_norm_rows_
    eng = SaeDenseStepEngine(p["W_enc"].t().contiguous().cuda(), p["W_dec"].clone().cuda(), p["b_enc"].clone().cuda(), p["b_dec"].clone().cuda(),
                             k=max(k, 1), normalize_activations=norm, max_grad_norm=1.0, l1_coefficient=l1,
                             gemm_impl={None: L.GEMM_AUTO, "simt": L.GEMM_SIMT, "tc": L.GEMM_AUTO}[impl])
    unit_norm_rows_(eng.W_dec)
    eng.refresh_lo()
    return eng


def test_glue_kernels_match_torch():
    from vit_prisma.b200 import sae_dense as D
    g = torch.Generator().manual_seed(0)
    x = torch.randn(77, 133, generator=g).cuda()
    xt, lo = D.transpose(x)
    assert torch.equal(xt, x.t().contiguous())
    hi = (xt.view(torch.int32) & -8192).view(torch.float32)                 # what a tf32 wgmma reads of the value
    # lo plane = (x - hi) rounded to the nearest tf32: low 13 mantissa bits clear, within half a tf32 ulp of the exact remainder
    assert int((lo.view(torch.int32) & 8191).abs().max()) == 0
    assert float((lo - (xt - hi)).abs().max()) <= float((xt - hi).abs().max()) * 2.0 ** -11
    assert rel_err(D.colsum(x), x.sum(0)) < 1e-6
    v = torch.randn(77, generator=g).cuda()
    assert rel_err(D.gemv_rows(x, v), v @ x) < 1e-6
    acc = torch.ones(133, device="cuda")
    D.colsum(x, out=acc, accumulate=True)
    assert rel_err(acc, 1 + x.sum(0)) < 1e-6


@pytest.mark.parametrize("tag", ["d", "e", "f"])
def test_dense_and_ghost_steps_match_reference_golden(tag):
    """d: ReLU + L1; e: TopK + ghost grads (112-122 dead features from step 2); f: ReLU + L1 + ghost grads (77 dead)."""
    gold = load_golden(f"sae_tiny_{tag}.pt")
    data = _data(gold)
    eng = _engine(gold["init"], gold["k"], gold["norm"], gold["l1_coefficient"])
    F = gold["d_sae"]
    since_fired, act_freq = torch.zeros(F, device="cuda"), torch.zeros(F, device="cuda")
    B = gold["batch"]
    for s, rec in enumerate(gold["steps"]):
        x = data[s * B:(s + 1) * B].cuda()
        lr = gold["lr"] * lr_multiplier(s, gold["warm_up_steps"], gold["total_steps"], gold["lr_end"])
        if gold["act"] == "relu":
            eng.train_step_dense(x, lr, since_fired, act_freq, use_ghost_grads=gold["use_ghost_grads"],
                                 dead_feature_window=gold["dead_feature_window"], want_out=True)
        else:
            eng.train_step_topk_ghost(x, lr, since_fired, act_freq, gold["dead_feature_window"])
            assert torch.equal(eng.idx.cpu().long(), rec["topk_idx"]), f"step {s}: TopK indices differ from the reference"
        t = eng.loss_terms(B)
        # the ghost term divides by elements of (G - r)^2 / rcn that can be ~1e-6: fp32 round-off is amplified (the reference's own
        # autograd and the pinned oracle agree to ~1e-4 there, tests/test_oracle_golden.py), hence the wider bars with dead features
        tol = 2e-3 if rec["n_dead"] else 1e-4
        if gold["use_ghost_grads"]:
            assert eng.last_n_dead == rec["n_dead"]
            assert abs(t["ghost"] - rec["ghost"]) <= 1e-4 * abs(rec["ghost"]), (s, t["ghost"], rec["ghost"])
        if gold["act"] == "relu":
            assert abs(t["l1"] - rec["l1"]) <= 1e-4 * abs(rec["l1"]), (s, t["l1"], rec["l1"])
        assert abs(t["mse"] - rec["mse"]) <= 1e-4 * abs(rec["mse"]), (s, t["mse"], rec["mse"])
        assert abs(t["loss"] - rec["loss"]) <= 1e-4 * abs(rec["loss"]), (s, t["loss"], rec["loss"])
        assert abs(t["l0"] - rec["l0"]) < 1e-4
        assert abs(t["grad_norm"] - rec["grad_norm"]) <= tol * rec["grad_norm"], (s, t["grad_norm"], rec["grad_norm"])
        assert_close(eng.sae_out.cpu(), rec["sae_out"], 1e-4, f"step {s} sae_out")
        if "raw_grads" in rec:
            assert_close(eng.gW_dec.cpu(), rec["raw_grads"]["W_dec"], tol, f"step {s} dL/dW_dec")
            assert_close(eng.gW_encT.t().cpu(), rec["raw_grads"]["W_enc"], tol, f"step {s} dL/dW_enc")
            assert_close(eng.gb_enc.cpu(), rec["raw_grads"]["b_enc"], tol, f"step {s} dL/db_enc")
            assert_close(eng.gb_dec.cpu(), rec["raw_grads"]["b_dec"], tol, f"step {s} dL/db_dec")
        if "params_after" in rec:
            ref = rec["params_after"]
            ptol = 2e-3 if gold["use_ghost_grads"] else 1e-4
            ref_dec = ref["W_dec"] / ref["W_dec"].norm(dim=1, keepdim=True)   # the reference renormalises at its next step
            assert_close(eng.W_dec.cpu(), ref_dec, ptol, f"step {s} W_dec")
            assert_close(eng.W_encT.t().cpu(), ref["W_enc"], ptol, f"step {s} W_enc")
            assert_close(eng.b_dec.cpu(), ref["b_dec"], ptol, f"step {s} b_dec")
    assert torch.equal(since_fired.cpu(), gold["since_fired"])
    assert torch.equal(act_freq.cpu(), gold["act_freq"])


@pytest.mark.parametrize("ghost,impl", [(False, "tc"), (True, "simt"), (True, "tc")])
def test_dense_step_midsize_matches_oracle(ghost, impl):
    """d=256, F=2048, 512 tokens: every product takes the wgmma 3xTF32 GEMM ("tc") or the exact-fp32 FFMA kernel ("simt");
    three steps against the pinned oracle.  The ghost loss is ill-conditioned by construction (it divides by elements of
    (G - r)^2 / rcn + 1e-6): torch fp32 vs fp64 differ by 6e-4 on these gradients, the FFMA route stays within 3e-3, and the
    tensor-core route -- whose accumulation rounds toward zero, ~1e-5 on hidden_pre / sae_out -- within 6e-2 on the worst
    element of a dead feature's gradient row, while loss values, the live features and the no-ghost step keep the 2e-4 bar."""
    d, F, rows, l1 = 256, 2048, 512, 2e-3
    g = torch.Generator().manual_seed(5)
    p = {"W_enc": torch.randn(d, F, generator=g) / math.sqrt(d), "W_dec": torch.randn(F, d, generator=g), "b_enc": 0.01 * torch.randn(F, generator=g),
         "b_dec": 0.1 * torch.randn(d, generator=g)}
    if ghost:
        p["b_enc"][::7] = -6.0                                               # 6 sigma below zero: silent, dead after the first step, exp(h) ~ 2e-3
    xs = [torch.randn(rows, d, generator=g) * 2.0 + torch.randn(d, generator=g) for _ in range(3)]
    eng = _engine(p, 0, "layer_norm", l1, impl)
    ref_p = {k: v.clone() for k, v in p.items()}
    state = new_adam_state(ref_p)
    sf_ref, af_ref = torch.zeros(F), torch.zeros(F)
    sf, af = torch.zeros(F, device="cuda"), torch.zeros(F, device="cuda")
    ever_flipped = torch.zeros(F, dtype=torch.bool)
    for s, x in enumerate(xs):
        if ghost and s > 0:
            # every step starts from the oracle's state: with an ill-conditioned loss two fp32 trajectories separate by O(lr) per
            # step on a few elements, and the next step's ghost gradient is compared on those very elements
            ref_p["W_dec"] /= ref_p["W_dec"].norm(dim=1, keepdim=True)
            eng.W_encT.copy_(ref_p["W_enc"].t()); eng.W_dec.copy_(ref_p["W_dec"]); eng.b_enc.copy_(ref_p["b_enc"]); eng.b_dec.copy_(ref_p["b_dec"])
            eng.refresh_lo()
            for name, m, v in (("W_dec", eng.m_dec, eng.v_dec), ("b_enc", eng.m_be, eng.v_be), ("b_dec", eng.m_bd, eng.v_bd)):
                m.copy_(state[name]["m"]); v.copy_(state[name]["v"])
            eng.m_enc.copy_(state["W_enc"]["m"].t()); eng.v_enc.copy_(state["W_enc"]["v"].t())
            sf.copy_(sf_ref); af.copy_(af_ref)
        out = sae_train_step(ref_p, state, x, 0, 1e-3, s + 1, since_fired=sf_ref, act_freq=af_ref, act="relu", l1_coefficient=l1,
                             use_ghost_grads=ghost, dead_feature_window=0)
        eng.train_step_dense(x.cuda(), 1e-3, sf, af, use_ghost_grads=ghost, dead_feature_window=0, want_out=True)
        t = eng.loss_terms(rows)
        tol = (6e-2 if impl == "tc" else 3e-3) if (ghost and out["n_dead"]) else 2e-4
        assert abs(t["mse"] - out["mse"].item()) <= 1e-4 * out["mse"].item()
        assert abs(t["l1"] - out["l1"].item()) <= 1e-4 * out["l1"].item()
        if ghost:
            assert eng.last_n_dead == out["n_dead"] and (s == 0 or out["n_dead"] > 100)
            assert abs(t["ghost"] - out["ghost"].item()) <= 2e-4 * out["ghost"].item()
        assert abs(t["grad_norm"] - out["grad_norm"].item()) <= tol * out["grad_norm"].item()
        # a pre-activation within the GEMM round-off of zero (about one in 10^6 here) may land on the other side of the ReLU:
        # its whole d_hidden entry then differs.  Such features are counted, bounded, and left out of the element-wise check.
        flipped = ((eng.last_acts.cpu() > 0) != (out["fwd"]["feature_acts"] > 0)).any(0)
        assert int(flipped.sum()) <= 8, f"{int(flipped.sum())} features with a ReLU sign flip"
        keep = ~flipped
        ever_flipped |= flipped
        assert_close(eng.gW_dec.cpu(), out["raw_grads"]["W_dec"], tol, f"step {s} dL/dW_dec")
        assert_close(eng.gW_encT.t().cpu()[:, keep], out["raw_grads"]["W_enc"][:, keep], tol, f"step {s} dL/dW_enc")
        assert_close(eng.gb_enc.cpu()[keep], out["raw_grads"]["b_enc"][keep], tol, f"step {s} dL/db_enc")
        assert_close(eng.gb_dec.cpu(), out["raw_grads"]["b_dec"], max(tol, 2e-3 if flipped.any() else tol), f"step {s} dL/db_dec")
    keep = ~ever_flipped
    assert torch.equal(sf.cpu()[keep], sf_ref[keep]) and torch.equal(af.cpu()[keep], af_ref[keep])
    # Adam's m / (sqrt(v) + eps) turns a 1e-9 absolute difference on a near-zero gradient element into a fraction of lr:
    # the bar on the parameters is a third of one learning-rate step relative to max |W_enc| (~0.28), the gradients above are the sharp check
    assert_close(eng.W_encT.t().cpu()[:, keep], ref_p["W_enc"][:, keep], (1e-2 if impl == "tc" else 3e-3) if ghost else 1.2e-3, "W_enc after 3 steps")


def test_forward_tuple_reports_ghost_loss():
    """StandardSparseAutoencoder.forward in training mode with cfg.use_ghost_grads: 7-tuple with the ghost term (sae.py:609-614)."""
    from vit_prisma.sae.config import VisionModelSAERunnerConfig
    from vit_prisma.sae.sae import StandardSparseAutoencoder
    gold = load_golden("sae_tiny_e.pt")
    cfg = VisionModelSAERunnerConfig(d_in=gold["d_in"], expansion_factor=8, activation_fn_str="topk", activation_fn_kwargs={"k": gold["k"]},
                                     _device="cuda", _dtype="float32", normalize_activations=gold["norm"], use_ghost_grads=True,
                                     dead_feature_window=1, log_to_wandb=False, n_checkpoints=0, checkpoint_path="/tmp/unused")
    sae = StandardSparseAutoencoder(cfg)
    sae.load_state_dict({k: v.cuda() for k, v in gold["init"].items()})
    sae.train()
    sae.set_decoder_norm_to_unit_norm()
    x = _data(gold)[:gold["batch"]].cuda()
    out = sae(x, torch.zeros(gold["d_sae"], dtype=torch.bool, device="cuda"))
    rec = gold["steps"][0]
    assert abs(out[3].item() - rec["mse"]) <= 1e-4 * rec["mse"]
    assert abs(out[5].item() - rec["ghost"]) <= 1e-4 * rec["ghost"]
    assert abs(out[2].item() - rec["loss"]) <= 1e-4 * rec["loss"]
