"""Gated SAE step (vit_prisma/b200/sae_gated.py, csrc/sae_dense.cu pb_gated_*) against the reference fixtures
(tests/golden/sae_gated_{g,h}.pt: autograd + torch.optim.Adam on the unmodified GatedSparseAutoencoder) and, at a size that takes
the wgmma GEMMs, against the pinned oracle."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle.sae_oracle import GATED_PARAMS, gated_train_step, lr_multiplier, new_adam_state  # noqa: E402
from tests.util import assert_close, load_golden  # noqa: E402


def _engine(p, norm, l1, impl=None):
    from vit_prisma.b200 import _lib as L
    from vit_prisma.b200.sae_engine import unit_norm_rows_
    from vit_prisma.b200.sae_gated import SaeGatedStepEngine
    c = lambda t: t.clone().cuda()  # noqa: E731
    eng = SaeGatedStepEngine(p["W_enc"].t().contiguous().cuda(), c(p["W_dec"]), c(p["b_gate"]), c(p["r_mag"]), c(p["b_mag"]), c(p["b_dec"]),
                             l1_coefficient=l1, normalize_activations=norm, max_grad_norm=1.0,
                             gemm_impl=L.GEMM_SIMT if impl == "simt" else L.GEMM_AUTO)
    unit_norm_rows_(eng.W_dec)
    eng.refresh_lo()
    return eng


def _grads(eng):
    return dict(W_enc=eng.gW_encT.t().cpu(), b_gate=eng.gb_enc.cpu(), r_mag=eng.gr_mag.cpu(), b_mag=eng.gb_mag.cpu(), W_dec=eng.gW_dec.cpu(),
                b_dec=eng.gb_dec.cpu())


def _params(eng):
    return dict(W_enc=eng.W_encT.t().cpu(), b_gate=eng.b_gate.cpu(), r_mag=eng.r_mag.cpu(), b_mag=eng.b_mag.cpu(), W_dec=eng.W_dec.cpu(),
                b_dec=eng.b_dec.cpu())


@pytest.mark.parametrize("tag", ["g", "h"])
def test_gated_steps_match_reference_golden(tag):
    gold = load_golden(f"sae_gated_{tag}.pt")
    g = torch.Generator().manual_seed(gold["data_seed"])
    n, d = gold["batch"] * gold["n_steps"], gold["d_in"]
    data = torch.randn(n, d, generator=g) * 2.0 + torch.randn(d, generator=g)
    eng = _engine({k: gold["init"][k] for k in GATED_PARAMS}, gold["norm"], gold["l1_coefficient"])
    F, B = gold["d_sae"], gold["batch"]
    since_fired, act_freq = torch.zeros(F, device="cuda"), torch.zeros(F, device="cuda")
    for s, rec in enumerate(gold["steps"]):
        x = data[s * B:(s + 1) * B].cuda()
        lr = gold["lr"] * lr_multiplier(s, gold["warm_up_steps"], gold["total_steps"], gold["lr_end"])
        eng.train_step_gated(x, lr, since_fired, act_freq, want_out=True)
        t = eng.loss_terms(B)
        for name in ("loss", "mse", "l1", "aux"):
            assert abs(t[name] - rec[name]) <= 1e-4 * abs(rec[name]), (s, name, t[name], rec[name])
        assert abs(t["l0"] - rec["l0"]) < 1e-4
        assert abs(t["grad_norm"] - rec["grad_norm"]) <= 2e-4 * rec["grad_norm"], (s, t["grad_norm"], rec["grad_norm"])
        assert_close(eng.sae_out.cpu(), rec["sae_out"], 1e-4, f"step {s} sae_out")
        assert torch.equal(eng.last_acts.cpu() > 0, rec["feature_acts"] > 0), f"step {s}: active set differs"
        assert_close(eng.last_acts.cpu(), rec["feature_acts"], 1e-4, f"step {s} feature_acts")
        if "raw_grads" in rec:
            for name, got in _grads(eng).items():
                assert_close(got, rec["raw_grads"][name], 2e-4, f"step {s} dL/d{name}")
        if "params_after" in rec:
            ref = dict(rec["params_after"])
            ref["W_dec"] = ref["W_dec"] / ref["W_dec"].norm(dim=1, keepdim=True)   # the reference renormalises at its next step
            for name, got in _params(eng).items():
                assert_close(got, ref[name], 2e-3, f"step {s} {name}")   # Adam amplifies near-zero gradient elements (see test_sae_dense_gpu)
    assert torch.equal(since_fired.cpu(), gold["since_fired"])
    assert torch.equal(act_freq.cpu(), gold["act_freq"])


@pytest.mark.parametrize("impl", ["simt", "tc"])
def test_gated_step_midsize_matches_oracle(impl):
    """d=256, F=2048, 512 tokens: all seven products on the wgmma 3xTF32 GEMM ("tc") or the exact FFMA kernel ("simt")."""
    d, F, rows, l1 = 256, 2048, 512, 2e-3
    g = torch.Generator().manual_seed(9)
    p = {"W_enc": torch.randn(d, F, generator=g) / math.sqrt(d), "W_dec": torch.randn(F, d, generator=g), "b_gate": 0.05 * torch.randn(F, generator=g),
         "r_mag": 0.1 * torch.randn(F, generator=g), "b_mag": 0.05 * torch.randn(F, generator=g), "b_dec": 0.1 * torch.randn(d, generator=g)}
    x = torch.randn(rows, d, generator=g) * 2.0 + torch.randn(d, generator=g)
    eng = _engine(p, "layer_norm", l1, impl)
    ref_p = {k: v.clone() for k, v in p.items()}
    out = gated_train_step(ref_p, new_adam_state(ref_p), x, 1e-3, 1, "layer_norm", l1)
    eng.train_step_gated(x.cuda(), 1e-3, None, None, want_out=True)
    t = eng.loss_terms(rows)
    for name in ("loss", "mse", "l1", "aux"):
        assert abs(t[name] - out[name].item()) <= 1e-4 * abs(out[name].item()), (name, t[name], out[name].item())
    # pre-activations within the GEMM round-off of zero may land on the other side of a gate / ReLU: count, bound, exclude
    flipped = ((eng.last_acts.cpu() > 0) != (out["feature_acts"] > 0)).any(0)
    assert int(flipped.sum()) <= 8
    keep = ~flipped
    got = _grads(eng)
    tol = 3e-4
    assert_close(got["W_dec"][keep], out["raw_grads"]["W_dec"][keep], tol, "dL/dW_dec")
    assert_close(got["W_enc"][:, keep], out["raw_grads"]["W_enc"][:, keep], tol, "dL/dW_enc")
    for name in ("b_gate", "r_mag", "b_mag"):
        assert_close(got[name][keep], out["raw_grads"][name][keep], tol, f"dL/d{name}")
    assert_close(got["b_dec"], out["raw_grads"]["b_dec"], 2e-3 if flipped.any() else tol, "dL/db_dec")
    assert abs(t["grad_norm"] - out["grad_norm"].item()) <= 1e-3 * out["grad_norm"].item()


@pytest.mark.parametrize("variant", ["relu", "relu_ghost", "topk_ghost", "gated"])
def test_trainer_steps_every_variant_on_synthetic_activations(variant):
    """VisionSAETrainer.train_step (train_sae.py:278-411) dispatches to the dense / ghost / gated engines and the loss goes down."""
    from vit_prisma.sae.config import VisionModelSAERunnerConfig
    from vit_prisma.sae.train_sae import VisionSAETrainer
    from vit_prisma.sae.training.activations_store import SyntheticActivationsStore
    kw = dict(d_in=64, expansion_factor=8, _device="cuda", n_checkpoints=0, log_to_wandb=False, b_dec_init_method="mean", train_batch_size=256,
              lr_warm_up_steps=5, checkpoint_path="/tmp/prisma_b200_ckpt", lr=2e-3, l1_coefficient=1e-3, num_epochs=1)
    if variant.startswith("relu"):
        kw.update(activation_fn_str="relu", activation_fn_kwargs={})
    elif variant == "topk_ghost":
        kw.update(activation_fn_str="topk", activation_fn_kwargs={"k": 8})
    else:
        kw.update(activation_fn_str="relu", activation_fn_kwargs={}, architecture="gated")
    if variant.endswith("ghost"):
        kw.update(use_ghost_grads=True, dead_feature_window=2)
    cfg = VisionModelSAERunnerConfig(**kw)
    torch.manual_seed(0)
    store = SyntheticActivationsStore(cfg, pool_tokens=1 << 14, seed=1)
    trainer = VisionSAETrainer(cfg, model=None, dataset=None, activations_store=store)
    act_freq, since_fired, n_frac, opt, sched = trainer.initialize_training_variables()
    trainer.initialize_geometric_medians()
    losses = []
    for step in range(40):
        loss, mse, l1, l0, act_freq, since_fired, n_frac = trainer.train_step(
            trainer.sparse_coder, opt, sched, act_freq, since_fired, n_frac, store.next_batch(), step, step * cfg.train_batch_size)
        losses.append(float(loss))
    assert all(math.isfinite(v) for v in losses)
    assert losses[-1] < 0.9 * losses[0], (variant, losses[0], losses[-1])
    assert (l1 is None) == (variant == "topk_ghost")
    norms = trainer.sparse_coder.W_dec.data.norm(dim=1)
    assert torch.allclose(norms, torch.ones_like(norms), atol=1e-5)
    assert n_frac == 40 * 256 and float(act_freq.sum()) > 0


def test_gated_module_forward_tuple_and_trainer_dispatch():
    """GatedSparseAutoencoder.forward returns the reference's 7-tuple (sae.py:753-761); step_engine() is the gated engine."""
    from vit_prisma.b200.sae_gated import SaeGatedStepEngine
    from vit_prisma.sae.config import VisionModelSAERunnerConfig
    from vit_prisma.sae.sae import GatedSparseAutoencoder
    gold = load_golden("sae_gated_g.pt")
    cfg = VisionModelSAERunnerConfig(d_in=gold["d_in"], expansion_factor=8, activation_fn_str="relu", architecture="gated",
                                     l1_coefficient=gold["l1_coefficient"], _device="cuda", _dtype="float32", normalize_activations=gold["norm"],
                                     log_to_wandb=False, n_checkpoints=0, checkpoint_path="/tmp/unused")
    sae = GatedSparseAutoencoder(cfg)
    sae.load_state_dict({k: v.cuda() for k, v in gold["init"].items()})
    sae.set_decoder_norm_to_unit_norm()
    assert isinstance(sae.step_engine(), SaeGatedStepEngine)
    g = torch.Generator().manual_seed(gold["data_seed"])
    data = torch.randn(gold["batch"] * gold["n_steps"], gold["d_in"], generator=g) * 2.0 + torch.randn(gold["d_in"], generator=g)
    out = sae(data[:gold["batch"]].cuda())
    rec = gold["steps"][0]
    assert len(out) == 7 and float(out[5]) == 0.0
    for i, name in ((2, "loss"), (3, "mse"), (4, "l1"), (6, "aux")):
        assert abs(float(out[i]) - rec[name]) <= 1e-4 * abs(rec[name]), (name, float(out[i]), rec[name])
    assert_close(out[0].cpu(), rec["sae_out"], 1e-4, "sae_out")
    assert_close(out[1].cpu(), rec["feature_acts"], 1e-4, "feature_acts")
