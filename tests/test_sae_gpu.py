"""TopK-SAE path on the GPU vs the oracle and the reference-generated goldens (GPU only).

Bars (north_star): reconstructions within 1e-4 relative (fp32); TopK indices bit-exact."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle.sae_oracle import lr_multiplier, new_adam_state, sae_forward, sae_train_step  # noqa: E402
from tests.util import assert_close, load_golden, rel_err  # noqa: E402


def _L():
    from vit_prisma.b200 import _lib
    return _lib


def _data(gold):
    g = torch.Generator().manual_seed(gold["data_seed"])
    n, d = gold["batch"] * gold["n_steps"], gold["d_in"]
    return torch.randn(n, d, generator=g) * 2.0 + torch.randn(d, generator=g)


# ---------------------------------------------------------------------------- top-k kernel
@pytest.mark.parametrize("rows,F,k", [(5, 256, 4), (64, 2048, 32), (33, 24576, 32), (16, 49152, 64), (8, 98304, 32), (7, 1000, 8)])
def test_topk_matches_torch(rows, F, k):
    from vit_prisma.b200.sae_engine import topk_support
    g = torch.Generator().manual_seed(F + k)
    x = torch.randn(rows, F, generator=g)
    ref = torch.topk(x, k, dim=-1)
    idx, val = topk_support(x.cuda(), k)
    assert torch.equal(idx.cpu().long(), ref.indices), "TopK indices must be bit-exact (same order as torch.topk)"
    assert torch.equal(val.cpu(), ref.values)


def test_topk_ties_and_negative_rows():
    from vit_prisma.b200.sae_engine import topk_dense, topk_support
    x = torch.zeros(3, 512)
    x[1] = -1.0
    x[2, 7] = 5.0
    idx, val = topk_support(x.cuda(), 4)
    assert idx[0].tolist() == [0, 1, 2, 3]                     # ties resolve to the lowest indices
    assert idx[2].tolist()[0] == 7 and val[2, 0].item() == 5.0
    dense = topk_dense(x.cuda(), 4)                             # relu of selected values: all-negative row -> zeros
    assert dense[1].abs().sum().item() == 0 and dense[2, 7].item() == 5.0 and dense.shape == (3, 512)


# ---------------------------------------------------------------------------- fused encoder -> TopK (csrc/sae_fused.cu)
def _fused_case(rows, d, F, k, seed, scale_rows=None, w_scale=None, b_scale=0.01, **kw):
    from vit_prisma.b200.sae_engine import SaeStepEngine
    g = torch.Generator().manual_seed(seed)
    W_encT = torch.randn(F, d, generator=g) / math.sqrt(d)
    if w_scale is not None:
        W_encT = W_encT * w_scale[:, None]
    W_dec = torch.randn(F, d, generator=g)
    W_dec /= W_dec.norm(dim=1, keepdim=True)
    b_enc = b_scale * torch.randn(F, generator=g)
    x = torch.randn(rows, d, generator=g) * 2.0 + torch.randn(d, generator=g)
    if scale_rows is not None:
        x = x * scale_rows[:, None]
    eng = SaeStepEngine(W_encT.cuda(), W_dec.cuda(), b_enc.cuda(), torch.zeros(d).cuda(), k=k, normalize_activations="none", encoder="fused", **kw)
    eng.encode_topk(x.cuda())
    torch.cuda.synchronize()
    hp = x.double() @ W_encT.double().t() + b_enc.double()                 # what sae.py:568 computes, in float64
    return eng, hp


def _check_against_float64(eng, hp, k):
    ref = torch.topk(hp, k, dim=-1)
    idx, val = eng.idx.cpu().long(), eng.val.cpu()
    same = (idx == ref.indices).all(dim=1)
    gap = torch.topk(hp, k + 1, dim=-1).values
    srt = ref.values
    # rows where two of the top k+1 float64 values are closer than fp32 round-off of the dot product may legitimately swap
    near = ((srt[:, :-1] - srt[:, 1:]).abs().min(dim=1).values < 2e-6 * hp.abs().max()) | ((gap[:, k - 1] - gap[:, k]).abs() < 2e-6 * hp.abs().max())
    assert bool((same | near).all()), f"{(~(same | near)).sum().item()} rows differ from the float64 top-k beyond near-ties"
    assert same.float().mean().item() > 0.98
    ok = same
    assert rel_err(val[ok], ref.values[ok].float()) < 2e-6                 # re-scored values are fp32-exact, not tf32
    assert bool((val[:, :-1] >= val[:, 1:]).all()), "values must come out sorted descending"
    cnt = torch.zeros(hp.shape[1]).index_add_(0, idx.flatten(), torch.ones(idx.numel()))
    assert torch.equal(eng.feat_count.cpu(), cnt)


@pytest.mark.parametrize("rows,d,F,k,c_keep", [(300, 128, 2048, 8, 8), (257, 768, 24576, 32, 8), (129, 768, 24576, 32, 6), (64, 1024, 65536, 32, 4),
                                               (130, 100, 1280, 16, 8)])
def test_fused_encode_topk_matches_float64_topk(rows, d, F, k, c_keep):
    eng, hp = _fused_case(rows, d, F, k, seed=rows + F, c_keep=c_keep)
    _check_against_float64(eng, hp, k)
    if F >= 2048:
        assert eng.fallback_rows() <= max(2, rows // 50), f"{eng.fallback_rows()} of {rows} rows took the exact path on Gaussian data"


def test_fused_encode_topk_adversarial_rows_take_the_exact_path():
    """Cases the approximate pass cannot settle: constant rows (every value ties: lowest indices win), all winners inside one
    128-feature segment (more than c_keep of them: saturation), and rows with a huge norm next to tiny ones (loose error bound)."""
    from vit_prisma.b200.sae_engine import SaeStepEngine
    d, F, k = 64, 1024, 16
    W_encT = torch.zeros(F, d)
    eng = SaeStepEngine(W_encT.cuda(), torch.eye(F, d).cuda().contiguous(), torch.zeros(F).cuda(), torch.zeros(d).cuda(), k=k,
                        normalize_activations="none", encoder="fused")
    eng.encode_topk(torch.randn(5, d).cuda())
    assert eng.idx.cpu().tolist() == [list(range(k))] * 5 and eng.fallback_rows() == 5
    # winners clustered in features 256..383: saturation of that segment
    w_scale = torch.ones(F)
    w_scale[256:384] = 50.0
    eng2, hp2 = _fused_case(40, d, F, k, seed=3, w_scale=w_scale, b_scale=0.0)
    hp2_abs = hp2                                                             # winners = largest of the boosted block (sign-dependent)
    _check_against_float64(eng2, hp2_abs, k)
    assert eng2.fallback_rows() >= 20
    # mixed row norms: the bound scales per row
    sr = torch.ones(64)
    sr[::2] = 1e3
    eng3, hp3 = _fused_case(64, 128, 4096, 8, seed=9, scale_rows=sr)
    _check_against_float64(eng3, hp3, 8)


# ---------------------------------------------------------------------------- engine vs reference goldens
def _engine_from(p, k, norm, impl, **kw):
    from vit_prisma.b200.sae_engine import SaeStepEngine
    W_encT = p["W_enc"].t().contiguous().cuda()
    return SaeStepEngine(W_encT, p["W_dec"].clone().cuda(), p["b_enc"].clone().cuda(), p["b_dec"].clone().cuda(), k=k,
                         normalize_activations=norm, max_grad_norm=1.0, gemm_impl=impl, **kw)


@pytest.mark.parametrize("tag", ["a", "b", "c"])
@pytest.mark.parametrize("impl", ["simt", "tc", "fused"])
def test_train_steps_match_reference_golden(tag, impl):
    """6 optimizer steps driven by the step engine vs torch autograd + torch.optim.Adam on the reference module.  ``fused`` is the
    default encoder route (tf32 candidate GEMM + exact re-scoring): at d_sae = 256 / 512 every 128-feature segment is saturated, so
    these runs also drive its exact path on every row."""
    L = _L()
    gold = load_golden(f"sae_tiny_{tag}.pt")
    data = _data(gold)
    if impl == "fused":
        eng = _engine_from(gold["init"], gold["k"], gold["norm"], L.GEMM_AUTO)
        assert eng.encoder == "fused"
    else:
        eng = _engine_from(gold["init"], gold["k"], gold["norm"], L.GEMM_SIMT if impl == "simt" else L.GEMM_TC)
        assert eng.encoder == "dense"
    from vit_prisma.b200.sae_engine import unit_norm_rows_
    unit_norm_rows_(eng.W_dec)
    eng.refresh_lo()
    since_fired = torch.zeros(gold["d_sae"], device="cuda")
    act_freq = torch.zeros(gold["d_sae"], device="cuda")
    B = gold["batch"]
    for s, rec in enumerate(gold["steps"]):
        x = data[s * B:(s + 1) * B].cuda()
        lr = gold["lr"] * lr_multiplier(s, gold["warm_up_steps"], gold["total_steps"], gold["lr_end"])
        eng.train_step(x, lr, since_fired=since_fired, act_freq=act_freq, want_out=True)
        sc = eng.scalars_dict()
        assert torch.equal(eng.idx.cpu().long(), rec["topk_idx"]), f"step {s}: TopK indices differ from the reference"
        assert abs(sc["mse"] - rec["mse"]) <= 1e-4 * abs(rec["mse"]), (s, sc["mse"], rec["mse"])
        assert abs(sc["grad_norm"] - rec["grad_norm"]) <= 1e-4 * rec["grad_norm"], (s, sc["grad_norm"], rec["grad_norm"])
        assert abs(sc["l0"] - rec["l0"]) < 1e-5
        assert_close(eng.sae_out.cpu(), rec["sae_out"], 1e-4, f"step {s} sae_out")
        if "raw_grads" in rec:
            assert_close(eng.gW_dec.cpu(), rec["raw_grads"]["W_dec"], 1e-4, "dL/dW_dec")
            assert_close(eng.gW_encT.t().cpu(), rec["raw_grads"]["W_enc"], 1e-4, "dL/dW_enc")
            assert_close(eng.gb_enc.cpu(), rec["raw_grads"]["b_enc"], 1e-4, "dL/db_enc")
            assert_close(eng.gb_dec.cpu(), rec["raw_grads"]["b_dec"], 1e-4, "dL/db_dec")
        if "params_after" in rec:
            ref = rec["params_after"]
            ref_dec = ref["W_dec"] / ref["W_dec"].norm(dim=1, keepdim=True)   # the reference renormalises at its next step
            assert_close(eng.W_dec.cpu(), ref_dec, 1e-4, f"step {s} W_dec")
            assert_close(eng.W_encT.t().cpu(), ref["W_enc"], 1e-4, f"step {s} W_enc")
            assert_close(eng.b_enc.cpu(), ref["b_enc"], 1e-4 if ref["b_enc"].abs().max() > 1e-3 else 1e-2, f"step {s} b_enc")
            assert_close(eng.b_dec.cpu(), ref["b_dec"], 1e-4, f"step {s} b_dec")
    assert torch.equal(since_fired.cpu(), gold["since_fired"])
    assert torch.equal(act_freq.cpu(), gold["act_freq"])


def test_engine_forward_matches_oracle_midsize():
    """d=768, F=768*8, k=32, 512 tokens: above the size where the 128x128 wgmma tiles and the 24-per-thread TopK kick in."""
    L = _L()
    from vit_prisma.b200.sae_engine import SaeStepEngine, unit_norm_rows_
    d, F, k, rows = 768, 768 * 8, 32, 512
    g = torch.Generator().manual_seed(3)
    p = {"W_enc": torch.randn(d, F, generator=g) / math.sqrt(d), "W_dec": torch.randn(F, d, generator=g), "b_enc": 0.01 * torch.randn(F, generator=g),
         "b_dec": torch.randn(d, generator=g)}
    p["W_dec"] /= p["W_dec"].norm(dim=1, keepdim=True)
    x = torch.randn(rows, d, generator=g) * 2.0 + torch.randn(d, generator=g)
    ref = sae_forward(p, x, k)
    for impl in (L.GEMM_SIMT, L.GEMM_TC):
        eng = SaeStepEngine(p["W_enc"].t().contiguous().cuda(), p["W_dec"].clone().cuda(), p["b_enc"].clone().cuda(), p["b_dec"].clone().cuda(), k=k, gemm_impl=impl)
        out, idx, val = eng.forward(x.cuda())
        assert rel_err(eng.hidden_pre.cpu(), ref["hidden_pre"]) < 2e-5
        same = (idx.cpu().long() == ref["idx"]).all(dim=1)
        # rows whose k-th / (k+1)-th pre-activations are closer than the GEMM round-off may legitimately swap
        gap = torch.topk(ref["hidden_pre"], k + 1, dim=-1).values
        near_tie = (gap[:, k - 1] - gap[:, k]).abs() < 1e-5 * ref["hidden_pre"].abs().max()
        assert bool((same | near_tie).all()), f"impl {impl}: {(~same).sum().item()} rows differ beyond near-ties"
        assert same.float().mean().item() > 0.99
        assert_close(out.cpu(), ref["sae_out"], 1e-4, "sae_out")
        assert abs(eng.scalars_dict()["mse"] - ref["mse"].item()) <= 1e-4 * ref["mse"].item()


def test_hot_features_split_lists_match_oracle_gradients():
    """A decoder bias far from the data makes a few features win TopK on (almost) every token -- the regime of real
    activations.  Their per-feature lists (hundreds of tokens) take the split-across-warps path of pb_sae_backward."""
    L = _L()
    from oracle.sae_oracle import sae_grads
    from vit_prisma.b200.sae_engine import SaeStepEngine
    import ctypes as C
    d, F, k, rows = 64, 1024, 16, 768
    g = torch.Generator().manual_seed(11)
    p = {"W_enc": torch.randn(d, F, generator=g) / math.sqrt(d), "W_dec": torch.randn(F, d, generator=g), "b_enc": torch.zeros(F),
         "b_dec": 3.0 * torch.randn(d, generator=g)}
    p["W_dec"] /= p["W_dec"].norm(dim=1, keepdim=True)
    x = torch.randn(rows, d, generator=g) * 2.0 + torch.randn(d, generator=g)
    fwd = sae_forward(p, x, k)
    counts = torch.bincount(fwd["idx"].reshape(-1), minlength=F)
    assert int(counts.max()) > 256, "test premise: at least one hot feature"
    ref = sae_grads(p, x, fwd)
    eng = SaeStepEngine(p["W_enc"].t().contiguous().cuda(), p["W_dec"].clone().cuda(), p["b_enc"].clone().cuda(), p["b_dec"].clone().cuda(), k=k,
                        gemm_impl=L.GEMM_SIMT)
    xs = x.cuda()
    eng.encode_topk(xs)
    eng.scalars.zero_()
    eng.step_count = 1
    s = eng._desc(xs, training=True, lr=1e-3)
    L.check(L.get_lib().pb_sae_decode(C.byref(s), torch.cuda.current_stream().cuda_stream))
    L.check(L.get_lib().pb_sae_backward(C.byref(s), torch.cuda.current_stream().cuda_stream))
    assert torch.equal(eng.idx.cpu().long(), fwd["idx"])
    assert_close(eng.gW_dec.cpu(), ref["W_dec"], 1e-4, "dL/dW_dec")
    assert_close(eng.gW_encT.t().cpu(), ref["W_enc"], 1e-4, "dL/dW_enc")
    assert_close(eng.gb_enc.cpu(), ref["b_enc"], 1e-4, "dL/db_enc")
    assert_close(eng.gb_dec.cpu(), ref["b_dec"], 1e-4, "dL/db_dec")
    assert torch.equal(eng.fired.cpu(), (fwd["feature_acts"] > 0).float().sum(0))
    norm_ref = math.sqrt(sum((v.double() ** 2).sum().item() for v in ref.values()))
    assert abs(eng.scalars_dict()["grad_norm"] - norm_ref) <= 1e-4 * norm_ref


# ---------------------------------------------------------------------------- module / trainer surface
def _cfg(**kw):
    from vit_prisma.sae.config import VisionModelSAERunnerConfig
    base = dict(d_in=64, expansion_factor=8, activation_fn_str="topk", activation_fn_kwargs={"k": 8}, _device="cuda", n_checkpoints=0,
                log_to_wandb=False, b_dec_init_method="mean", train_batch_size=256, lr_warm_up_steps=5, checkpoint_path="/tmp/prisma_b200_ckpt")
    base.update(kw)
    return VisionModelSAERunnerConfig(**base)


def test_module_forward_routes_agree_and_match_oracle():
    from vit_prisma.sae.sae import StandardSparseAutoencoder
    torch.manual_seed(0)
    sae = StandardSparseAutoencoder(_cfg())
    sae.b_dec.data.normal_()
    x = torch.randn(4, 10, 64, device="cuda") * 2 + 1
    out = sae(x)                                                   # sparse route
    assert len(out) == 7 and out[0].shape == x.shape and out[1].shape == (4, 10, 512) and out[4] is None
    p = {k: v.detach().cpu().contiguous() for k, v in sae.state_dict().items()}
    ref = sae_forward(p, x.reshape(-1, 64).cpu(), 8)
    assert_close(out[0].reshape(-1, 64).cpu(), ref["sae_out"], 1e-4, "sae_out")
    assert_close(out[1].reshape(-1, 512).cpu(), ref["feature_acts"], 1e-4, "feature_acts")
    assert abs(out[3].item() - ref["mse"].item()) <= 1e-4 * ref["mse"].item()
    seen = []
    sae.add_hook("hook_hidden_pre", lambda t, hook: seen.append(tuple(t.shape)))   # any hook -> dense / hooked route
    out_h = sae(x)
    sae.reset_hooks()
    assert seen == [(4, 10, 512)]
    assert_close(out_h[0].cpu(), out[0].cpu(), 1e-5, "hooked vs sparse sae_out")
    assert abs(out_h[3].item() - out[3].item()) <= 1e-5 * abs(out[3].item())
    sae_in, feats = sae.encode(x)
    assert torch.equal(feats, out_h[1]) and sae.decode(feats).shape == x.shape
    sd = sae.state_dict()
    assert sd["W_enc"].shape == (64, 512) and sd["W_dec"].shape == (512, 64)


def test_trainer_runs_and_learns_on_synthetic_activations():
    from vit_prisma.sae.train_sae import VisionSAETrainer
    from vit_prisma.sae.training.activations_store import SyntheticActivationsStore
    cfg = _cfg(num_epochs=1, lr=2e-3)
    torch.manual_seed(0)
    store = SyntheticActivationsStore(cfg, pool_tokens=1 << 14, seed=1)
    trainer = VisionSAETrainer(cfg, model=None, dataset=None, activations_store=store)
    act_freq, since_fired, n_frac, opt, sched = trainer.initialize_training_variables()
    trainer.initialize_geometric_medians()
    losses = []
    for step in range(60):
        loss, mse, l1, l0, act_freq, since_fired, n_frac = trainer.train_step(
            trainer.sparse_coder, opt, sched, act_freq, since_fired, n_frac, store.next_batch(), step, step * cfg.train_batch_size)
        losses.append(mse.item())
    assert l1 is None and n_frac == 60 * 256
    assert losses[-1] < 0.7 * losses[0], (losses[0], losses[-1])
    norms = trainer.sparse_coder.W_dec.data.norm(dim=1)
    assert torch.allclose(norms, torch.ones_like(norms), atol=1e-5)
    assert abs(l0.item() - 8.0) < 1e-3 and float(act_freq.sum()) > 0
