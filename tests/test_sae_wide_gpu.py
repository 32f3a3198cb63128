"""SAEs on activations wider than 1536 (1536 < d_in <= 8192, d_in % 4 == 0): the residual streams of the large towers (bigG 1664,
EVA02-E 1792, gigantic 1920) and MLP neurons (mlp.hook_post, d_in = d_mlp up to 8192), against the float64 oracle.

Past 1536 the row kernels of the step take their wide forms (csrc/sae.cu section 8): k_sae_prep_wide, k_sae_decode_wide,
k_sae_adam_rows_wide and k_unit_rows_wide give one row to the 256 threads of a CTA, CHUNKS in {2, 4, 6, 8} float4 per thread for
d_in up to 2048, 4096, 6144, 8192 (wide_chunks_for in csrc/sae_optim.cuh), with the sums over the row in shared memory; the
per-feature gradients (k_sae_grads_wide, k_sae_grads_long_wide) walk d_in in 1024-column slices.  WIDTHS take every instance full
and with idle threads: 1540 (a second chunk and a second slice of 129 float4 each; d % 8 != 0, so the fused route reads tf32
operands), 1664 / 1792 / 1920 (the towers), 2048 (CHUNKS 2 full), 3072 (CHUNKS 4, last chunk idle), 4096, 5120 (CHUNKS 6, last
chunk idle), 6144, 7680 (CHUNKS 8, warps 4-7 idle in the last chunk, a half slice) and 8192, the ceiling.  Every width runs three
steps on both encoder routes (fused and GEMM_TC dense), with the checks of tests/test_sae_step_widths_gpu.py.  The wide widths
are also the first GPU runs of the fused encoder's select / fallback phases past d = 1536.

The dense route's 3xTF32 GEMM has K = d_in; 1e-4 is asserted up to K = 8192 as below 1536.  Every other step engine (dense ReLU,
ghost grads with ReLU and TopK, Gated, both Transcoders) takes two steps at 2048 x 4096 through the helper of
tests/test_sae_dense_steps_gpu.py.  The module surface (sparse and hooked forward, unit-norm decoder, save / load) runs at
d_in 3072, and so does a dtype="bfloat16" module trained through VisionSAETrainer.train_step: fp32 masters within 1e-4 of the
float64 oracle, the exported bf16 parameters equal to the masters rounded once, hence within one bf16 rounding of the oracle.
VisionActivationsStore + VisionSAETrainer train on blocks.1.mlp.hook_post of a small HookedViT with d_mlp 2048.

Refusals: every step engine refuses d_in 8196 when it is built, before it allocates anything, and the C entry points refuse 8196
and 2050 themselves (PB_EUNSUPPORTED, message naming 8192) before any launch, leaving their operands untouched.  The data-parallel
engine refuses d_in > 1536 at construction, before any peer allocation.

The file runs in about 125 s on an H100 80GB HBM3 (700 W); its process peaks at 9.0 GB of resident host memory, most of it the
float64 oracle's d_in x d_sae matrices at the widest cases.
"""
import contextlib
import io

import pytest
import torch

from oracle.sae_oracle import new_adam_state, sae_forward, sae_train_step
from tests import test_sae_dense_steps_gpu as dense_steps
from tests.test_sae_step_widths_gpu import NORMS, _init, _steps_match_oracle
from tests.util import assert_close, load_golden, rel_err

pytestmark = pytest.mark.gpu

WIDTHS = (1540, 1664, 1792, 1920, 2048, 3072, 4096, 5120, 6144, 7680, 8192)
K = 16


def _shape(d):
    """(d_sae, rows) of a width case: the float64 oracle holds six d x d_sae matrices, so d_sae shrinks as d_in grows."""
    return (4096, 300) if d <= 3072 else (2048, 256)


CASES = [(d, route, NORMS[(j + r) % 3], j % 2 == r) for j, d in enumerate(WIDTHS) for r, route in enumerate(("fused", "dense"))]


@pytest.mark.parametrize("d,route,norm,clip", CASES)
def test_wide_three_steps_match_float64_oracle(d, route, norm, clip):
    F, rows = _shape(d)
    _steps_match_oracle(d, F, K, route, norm, clip, rows, 3, seed=1000 * d + (route == "dense"))


# ------------------------------------------------------------------------------------------------ every other step engine
@pytest.mark.parametrize("kind", dense_steps.ENGINES)
def test_wide_dense_engines_match_float64_oracle(kind):
    d, F, rows = 2048, 4096, 256
    ghost = kind.endswith("ghost")
    nd = dense_steps._axis_a_dead(F) if ghost else 0
    norm = dense_steps.NORMS[dense_steps.ENGINES.index(kind) % (2 if ghost else 3)]
    exp = dense_steps._routes(kind, d, F, rows, nd)
    dense_steps._steps_match_oracle(kind, d, F, rows, norm, 2, seed=2048 + dense_steps.ENGINES.index(kind), nd=nd, expect=exp)


# ------------------------------------------------------------------------------------------------ module surface
def _cfg(**kw):
    from vit_prisma.sae.config import VisionModelSAERunnerConfig
    base = dict(d_in=3072, expansion_factor=4, activation_fn_str="topk", activation_fn_kwargs={"k": K}, _device="cuda", n_checkpoints=0,
                log_to_wandb=False, b_dec_init_method="mean", train_batch_size=256, lr_warm_up_steps=5, checkpoint_path="/tmp/prisma_b200_ckpt")
    base.update(kw)
    with contextlib.redirect_stdout(io.StringIO()):
        return VisionModelSAERunnerConfig(**base)


def test_wide_module_forward_routes_unit_norm_and_round_trip(tmp_path):
    from vit_prisma.sae.sae import SparseAutoencoder, StandardSparseAutoencoder
    d, F = 3072, 12288
    torch.manual_seed(0)
    sae = StandardSparseAutoencoder(_cfg())
    assert sae.W_enc.shape == (d, F)
    norms = sae.W_dec.data.norm(dim=1)
    assert torch.allclose(norms, torch.ones_like(norms), atol=1e-5), "decoder rows not unit-norm after construction"
    sae.b_dec.data.normal_()
    x = torch.randn(2, 40, d, device="cuda") * 2 + 1
    out = sae(x)                                                   # sparse route
    assert out[0].shape == x.shape and out[1].shape == (2, 40, F)
    p = {k: v.detach().cpu().contiguous() for k, v in sae.state_dict().items()}
    ref = sae_forward(p, x.reshape(-1, d).cpu(), K)
    assert_close(out[0].reshape(-1, d).cpu(), ref["sae_out"], 1e-4, "sae_out")
    assert_close(out[1].reshape(-1, F).cpu(), ref["feature_acts"], 1e-4, "feature_acts")
    assert abs(out[3].item() - ref["mse"].item()) <= 1e-4 * ref["mse"].item()
    seen = []
    sae.add_hook("hook_hidden_pre", lambda t, hook: seen.append(tuple(t.shape)))   # any hook -> hooked route
    out_h = sae(x)
    sae.reset_hooks()
    assert seen == [(2, 40, F)]
    assert_close(out_h[0].cpu(), out[0].cpu(), 1e-5, "hooked vs sparse sae_out")
    sae_in, feats = sae.encode(x)
    assert torch.equal(feats, out_h[1])
    assert_close(sae.decode(feats).reshape(-1, d).cpu(), ref["sae_out"], 1e-4, "decode(encode(x))")
    # set_decoder_norm_to_unit_norm on rows of every scale
    with torch.no_grad():
        sae.W_dec.data.mul_(torch.rand(F, 1, device="cuda") * 10 + 0.1)
    want = sae.W_dec.data.double().cpu()
    want /= want.norm(dim=1, keepdim=True)
    sae.set_decoder_norm_to_unit_norm()
    assert rel_err(sae.W_dec.data, want) <= 1e-6
    # save_model -> load_from_pretrained
    path = str(tmp_path / "wide.pt")
    sae.save_model(path)
    loaded = SparseAutoencoder.load_from_pretrained(path)
    assert type(loaded) is StandardSparseAutoencoder
    sa, sb = sae.state_dict(), loaded.state_dict()
    assert list(sa) == list(sb) and all(torch.equal(sa[k].cpu(), sb[k].cpu()) for k in sa)
    loaded = loaded.to("cuda")
    assert torch.equal(loaded(x)[0], sae(x)[0])


def test_wide_bf16_module_trains_on_fp32_masters_and_exports_bf16():
    """dtype="bfloat16" at d_in 3072 through VisionSAETrainer.train_step, as tests/test_sae_bf16_gpu.py does at d_in 64: the step
    engine trains fp32 masters (unit-norm rows through k_unit_rows_wide before the first step, Adam through k_sae_adam_rows_wide)
    and the module's bf16 parameters are the masters rounded once.  The float64 oracle starts from the same bf16 values.  Bars: the
    loss and the masters within 1e-4 of the oracle; every exported parameter bitwise equal to its master rounded to bf16, and so
    within one bf16 rounding (2^-8 relative) plus that 1e-4 of the oracle."""
    from vit_prisma.sae.train_sae import VisionSAETrainer
    d, F, k, rows, lr = 3072, 6144, K, 256, 1e-3
    scfg = _cfg(expansion_factor=F // d, _dtype="bfloat16", train_batch_size=rows, lr=lr, lr_warm_up_steps=1, lr_scheduler_name="constant",
                b_dec_init_method="zeros", checkpoint_path="/tmp/prisma_b200_unused")
    with contextlib.redirect_stdout(io.StringIO()):
        trainer = VisionSAETrainer(scfg, model=None, dataset=None, activations_store=object())
    sae = trainer.sparse_coder
    assert sae.low_precision and all(v.dtype == torch.bfloat16 for v in sae.state_dict().values())
    g = torch.Generator().manual_seed(d)
    init = {"W_enc": torch.randn(d, F, generator=g) / d ** 0.5, "W_dec": torch.randn(F, d, generator=g),
            "b_enc": 0.01 * torch.randn(F, generator=g), "b_dec": 0.1 * torch.randn(d, generator=g)}
    init = {n: v.bfloat16() for n, v in init.items()}
    with torch.no_grad():
        wt, wd, be, bd = sae._canonical_params()
        wt.copy_(init["W_enc"].t()); wd.copy_(init["W_dec"]); be.copy_(init["b_enc"]); bd.copy_(init["b_dec"])
    p = {n: v.double() for n, v in init.items()}
    state = new_adam_state(p)
    act_freq, since_fired, n_frac, opt, sched = trainer.initialize_training_variables()
    data = (torch.randn(2 * rows, d, generator=g) * 2.0 + torch.randn(d, generator=g)).bfloat16().float()
    for t in range(2):
        xb = data[t * rows:(t + 1) * rows]
        ref = sae_train_step(p, state, xb.double(), k, lr, t + 1)
        _, mse, _, _, act_freq, since_fired, n_frac = trainer.train_step(sae, opt, sched, act_freq, since_fired, n_frac, xb.cuda().unsqueeze(1),
                                                                         t, t * rows)
        assert abs(mse.item() - float(ref["mse"])) <= 1e-4 * float(ref["mse"]), (t, mse.item(), float(ref["mse"]))
        eng = sae.step_engine()
        assert eng.W_dec.dtype == torch.float32 and eng.m_dec.dtype == torch.float32
        masters = {"W_enc": eng.W_encT.t(), "W_dec": eng.W_dec, "b_enc": eng.b_enc, "b_dec": eng.b_dec}
        want = dict(p, W_dec=p["W_dec"] / p["W_dec"].norm(dim=1, keepdim=True))     # the oracle renormalises at its next step
        sd = sae.state_dict()
        for n, m in masters.items():
            at = f"step {t + 1} {n}"
            assert rel_err(m, want[n]) <= 1e-4, f"{at}: master {rel_err(m, want[n]):.2e} from the float64 oracle"
            assert sd[n].dtype == torch.bfloat16 and torch.equal(sd[n], m.to(torch.bfloat16)), f"{at}: export is not the rounded master"
            scale = float(want[n].abs().max())
            err = float((sd[n].cpu().double() - want[n]).abs().max())
            assert err <= (2.0 ** -8 + 1e-4) * scale, f"{at}: bf16 parameter {err:.3e} from the oracle (one rounding = {2.0 ** -8 * scale:.3e})"


# ------------------------------------------------------------------------------------------------ end to end on MLP neurons
def test_wide_sae_on_mlp_neurons():
    """blocks.1.mlp.hook_post of a two-layer ViT with d_mlp 2048 through VisionActivationsStore, then three TopK steps through
    VisionSAETrainer.train_step on those activations against the oracle."""
    from torch.utils.data import TensorDataset
    from oracle.vit_oracle import recipe_state_dict, state_dict_shapes, vit_forward_with_cache
    from vit_prisma.configs.HookedViTConfig import HookedViTConfig
    from vit_prisma.models.base_vit import HookedViT
    from vit_prisma.sae.train_sae import VisionSAETrainer
    from vit_prisma.sae.training.activations_store import VisionActivationsStore
    gold = load_golden("vit_tiny_a_fp32.pt")
    cfg = dict(gold["cfg"], n_layers=2, d_mlp=2048)
    sd = recipe_state_dict(state_dict_shapes(cfg), 31)
    with contextlib.redirect_stdout(io.StringIO()):
        model = HookedViT(HookedViTConfig(**cfg))
    model.load_state_dict(sd)
    model = model.to("cuda").eval()
    batch = 8
    imgs = torch.randn(batch, 3, cfg["image_size"], cfg["image_size"], generator=torch.Generator().manual_seed(3))
    _, ref_cache = vit_forward_with_cache(sd, cfg, imgs)
    ref_acts = ref_cache["blocks.1.mlp.hook_post"]
    T, d = ref_acts.shape[1], ref_acts.shape[2]
    assert d == 2048
    F, k, rows = 4096, 8, batch * T
    scfg = _cfg(d_in=d, expansion_factor=F // d, activation_fn_kwargs={"k": k}, _dtype="float32", hook_point_layer=1,
                layer_subtype="mlp.hook_post", context_size=T, store_batch_size=batch, train_batch_size=rows, lr=1e-3,
                lr_warm_up_steps=1, lr_scheduler_name="constant", image_size=cfg["image_size"], checkpoint_path="/tmp/prisma_b200_unused",
                b_dec_init_method="zeros", verbose=False, num_workers=0)
    store = VisionActivationsStore(scfg, model, TensorDataset(imgs, torch.zeros(batch, dtype=torch.long)), create_dataloader=False)
    acts = store.get_activations(imgs.cuda())
    assert tuple(acts.shape) == (batch, T, 1, d)
    assert_close(acts[:, :, 0].cpu(), ref_acts, 1e-4, "store.get_activations on mlp.hook_post")

    with contextlib.redirect_stdout(io.StringIO()):
        trainer = VisionSAETrainer(scfg, model=None, dataset=None, activations_store=object())
    g = torch.Generator().manual_seed(12)
    p = {"W_enc": torch.randn(d, F, generator=g) / d ** 0.5, "W_dec": torch.randn(F, d, generator=g), "b_enc": 0.01 * torch.randn(F, generator=g),
         "b_dec": torch.zeros(d)}
    p["W_dec"] /= p["W_dec"].norm(dim=1, keepdim=True)
    sae = trainer.sparse_coder
    with torch.no_grad():
        wt, wd, be, bd = sae._canonical_params()
        wt.copy_(p["W_enc"].t()); wd.copy_(p["W_dec"]); be.copy_(p["b_enc"]); bd.copy_(p["b_dec"])
    act_freq, since_fired, n_frac, opt, sched = trainer.initialize_training_variables()
    state = new_adam_state(p)
    xb = acts[:, :, 0].reshape(rows, d)
    for t in range(3):
        ref = sae_train_step(p, state, xb.cpu(), k, 1e-3, t + 1)
        _, mse, _, _, act_freq, since_fired, n_frac = trainer.train_step(sae, opt, sched, act_freq, since_fired, n_frac, xb.unsqueeze(1), t, t * rows)
        assert abs(mse.item() - float(ref["mse"])) <= 1e-4 * float(ref["mse"]), (t, mse.item(), float(ref["mse"]))
    assert rel_err(sae.W_dec.data.cpu(), p["W_dec"] / p["W_dec"].norm(dim=1, keepdim=True)) <= 1e-4
    assert rel_err(sae.W_enc.data.cpu(), p["W_enc"]) <= 1e-4


# ------------------------------------------------------------------------------------------------ refusals
def _refused_untouched(fn, t, match):
    """fn() raises PrismaB200Error matching ``match`` and leaves ``t`` bitwise as it was."""
    from vit_prisma.b200 import _lib as L
    before = t.clone()
    with pytest.raises(L.PrismaB200Error, match=match):
        fn()
    torch.cuda.synchronize()
    assert torch.equal(t.view(torch.int32), before.view(torch.int32)), "a refused call wrote its operand"


def test_d_in_beyond_8192_is_refused_before_any_launch():
    from vit_prisma.b200 import _lib as L
    from vit_prisma.b200.sae_engine import SaeStepEngine, sae_prep, unit_norm_rows_
    d, F = 8196, 256
    W_enc, W_dec, b_enc, b_dec, xs = _init(d, F, d, 64, 1)
    for route in (L.GEMM_AUTO, L.GEMM_TC):                       # fused and dense encoders
        with pytest.raises(L.PrismaB200Error, match=r"d_in=8196 unsupported .*d <= 8192"):
            SaeStepEngine(W_enc.t().contiguous().cuda(), W_dec.cuda(), b_enc.cuda(), b_dec.cuda(), k=K, gemm_impl=route)
    p, _, _, _ = dense_steps._init("relu", d, F, 64, 1, d, 0)
    with pytest.raises(L.PrismaB200Error, match=r"d_in=8196 unsupported .*d <= 8192"):
        dense_steps._engine("relu", p, "layer_norm", L.GEMM_AUTO)
    W = W_dec.cuda()
    _refused_untouched(lambda: unit_norm_rows_(W), W, r"d_in=8196 unsupported .*d <= 8192")
    x = xs[0].cuda()
    _refused_untouched(lambda: sae_prep(x, b_dec.cuda(), "layer_norm"), x, r"d_in=8196 unsupported .*d <= 8192")


def test_d_in_not_a_multiple_of_4_past_1536_is_refused_before_any_launch():
    from vit_prisma.b200.sae_engine import sae_prep, unit_norm_rows_
    d = 2050
    g = torch.Generator().manual_seed(d)
    W = torch.randn(256, d, generator=g).cuda()
    _refused_untouched(lambda: unit_norm_rows_(W), W, r"d_in=2050 unsupported \(needs d % 4 == 0 and d <= 8192\)")
    x = torch.randn(64, d, generator=g).cuda()
    _refused_untouched(lambda: sae_prep(x, torch.zeros(d, device="cuda"), "none"), x,
                       r"d_in=2050 unsupported \(needs d % 4 == 0 and d <= 8192\)")


def test_data_parallel_engine_refuses_wide_d_in_at_construction():
    from vit_prisma.b200 import _lib as L
    from vit_prisma.b200.p2p import P2PGroup, SaeDPEngine
    d, F = 2048, 256
    W_enc, W_dec, b_enc, b_dec, _ = _init(d, F, 5, 64, 1)
    group = P2PGroup(0, 1, torch.device("cuda"), exchange=lambda mine: [mine])
    with pytest.raises(L.PrismaB200Error, match="1536"):
        SaeDPEngine(group, W_enc.t().contiguous().cuda(), W_dec.cuda(), b_enc.cuda(), b_dec.cuda(), k=K)
    assert not group.local, "peer buffers allocated before the refusal"
