"""Video (tubelet) HookedViTs on the GPU: both routes against fixtures made by the unmodified reference and against the CPU
checker (tests/video_oracle.py), the split attention stages past 608 tokens, a ViViT-B-sized clip, host staging and the SAE
path.  Bars are those of test_vit_gpu.py (DESIGN section 4)."""
import contextlib
import io

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle.sae_oracle import new_adam_state, sae_train_step  # noqa: E402
from oracle.vit_oracle import digest  # noqa: E402
from tests.test_vit_gpu import TOL, _bar  # noqa: E402
from tests.util import assert_close, load_golden, rel_err  # noqa: E402
from tests.video_oracle import video_forward_with_cache, video_recipe_state_dict, video_state_dict_shapes, videos  # noqa: E402

DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16}
STOP_FILTER = ["blocks.0.hook_resid_post", "blocks.1.ln1.hook_normalized"]
VIVIT_B = dict(n_layers=12, d_model=768, d_head=64, n_heads=12, d_mlp=3072, patch_size=16, image_size=224, n_channels=3,
               n_classes=400, eps=1e-6, activation_name="gelu", normalization_type="LN", use_cls_token=True, layer_norm_pre=False,
               normalize_output=False, return_type="pre_logits", classification_type="cls", is_video_transformer=True,
               video_tubelet_depth=2, video_num_frames=16)


def _model(cfg, dtype, seed=1234, device="cuda"):
    from vit_prisma.configs.HookedViTConfig import HookedViTConfig
    from vit_prisma.models.base_vit import HookedViT
    with contextlib.redirect_stdout(io.StringIO()):
        model = HookedViT(HookedViTConfig(**{k: v for k, v in cfg.items() if k != "dtype"}, dtype=dtype))
    shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    model.load_state_dict(video_recipe_state_dict(shapes, seed))
    return model.to(device, dtype).eval(), shapes


@pytest.mark.parametrize("dname", ["fp32", "bf16"])
@pytest.mark.parametrize("route", ["fused", "hooked"])
def test_tiny_video_matches_reference_golden(dname, route, monkeypatch):
    gold = load_golden(f"vit_video_c_{dname}.pt")
    dtype = DTYPES[dname]
    model, shapes = _model(gold["cfg"], dtype)
    assert shapes == gold["shapes"] == video_state_dict_shapes(gold["cfg"])
    if route == "hooked":
        monkeypatch.setenv("PRISMA_B200_ROUTE", "hooked")
    x = videos(gold["batch"], gold["cfg"], gold["images_seed"]).to("cuda", dtype)
    out, cache = model.run_with_cache(x)
    assert model.last_route.startswith(route), model.last_route
    assert list(cache.keys()) == gold["keys"], "cache key order differs from the reference"
    for k in gold["keys"]:
        assert_close(cache[k].cpu(), gold["cache"][k], _bar(k, dname), f"{route}:{k}")
    assert_close(out.cpu(), gold["out"], TOL[dname], "model output")
    # aliases of the reference cache: one tensor behind hook_ln_pre / ln_pre.hook_normalized (fp32) / blocks.0.hook_resid_pre
    assert cache["blocks.0.hook_resid_pre"].data_ptr() == cache["hook_ln_pre"].data_ptr()
    assert cache["blocks.0.hook_resid_post"].data_ptr() == cache["blocks.1.hook_resid_pre"].data_ptr()
    assert rel_err(model(x).cpu().float(), gold["out"].float()) <= TOL[dname]
    stop_out, stop_cache = model.run_with_cache(x, names_filter=STOP_FILTER, stop_at_layer=1)
    assert model.last_route.startswith(route)
    assert list(stop_cache.keys()) == gold["stop_keys"]
    assert_close(stop_out.cpu(), gold["stop_out"], TOL[dname], "stop_at_layer output")
    assert_close(stop_cache["blocks.0.hook_resid_post"].cpu(), gold["cache"]["blocks.0.hook_resid_post"], TOL[dname], "filtered key")


def test_tiny_video_other_frame_counts():
    """Frames past the last whole tubelet are never read (the fixture's 7th frame: 6 frames give the same output); a clip with
    another number of tubelets is declined by the fused route and fails at the position add on the hooked route, as in the
    reference."""
    gold = load_golden("vit_video_c_fp32.pt")
    model, _ = _model(gold["cfg"], torch.float32)
    x6 = videos(gold["batch"], gold["cfg"], gold["images_seed"])[:, :, :6].contiguous().cuda()
    out = model(x6)
    assert model.last_route == "fused"
    assert_close(out.cpu(), gold["out"], 1e-4, "6-frame clip")
    with pytest.raises(RuntimeError):
        model(videos(1, gold["cfg"], n_frames=9).cuda())
    assert model.last_route.startswith("hooked: number of tubelets")


@pytest.mark.parametrize("route", ["fused", "hooked"])
def test_641_tokens_match_reference_golden(route, monkeypatch):
    """d_head 64 at T = 641: the hooked route runs past the 608 tokens of the FFMA attention kernel."""
    gold = load_golden("vit_video_d_fp32.pt")
    model, shapes = _model(gold["cfg"], torch.float32)
    assert shapes == gold["shapes"]
    if route == "hooked":
        monkeypatch.setenv("PRISMA_B200_ROUTE", "hooked")
    out, cache = model.run_with_cache(videos(gold["batch"], gold["cfg"], gold["images_seed"]).cuda())
    assert model.last_route.startswith(route)
    assert list(cache.keys()) == gold["keys"]
    assert cache["blocks.0.attn.hook_pattern"].shape == (2, 2, 641, 641)
    for k, dg in gold["digests"].items():
        mine = digest(cache[k].cpu())
        assert mine["shape"] == dg["shape"] and mine["dtype"] == dg["dtype"], k
        e = (mine["samples"] - dg["samples"]).abs().max().item() / max(dg["max_abs"], 1e-30)
        es = abs(mine["sum"] - dg["sum"]) / max(dg["abs_sum"], 1e-30)
        assert e <= 1e-4 and es <= 1e-4, f"{route}:{k}: sample err {e:.2e}, sum err {es:.2e}"
    assert_close(cache["blocks.1.hook_resid_post"].cpu(), gold["resid_post_1"], 1e-4, "blocks.1.hook_resid_post")
    assert_close(out.cpu(), gold["out"], 1e-4, "model output")


@pytest.mark.parametrize("T", [609, 641, 1569])
@pytest.mark.parametrize("dname", ["fp32", "bf16"])
def test_split_stages_past_608_tokens_equal_fused_kernel(T, dname):
    """pb_attn_scores equals the scores spill of pb_attention bit for bit; pb_attn_pv fed pb_attention's own pattern spill
    equals its z bit for bit; both are within the bars of a float64 computation from the same operands."""
    from vit_prisma.b200 import ops
    dtype = DTYPES[dname]
    g = torch.Generator().manual_seed(T)
    B, H, dh = 2, 3, 64
    q, k, v = (torch.randn(B, T, H, dh, generator=g).to("cuda", dtype) for _ in range(3))
    scale = dh ** 0.5
    scores, pattern, z = ops.attention(q, k, v, scale)
    s_split = ops.attn_scores(q, k, scale)
    z_split = ops.attn_pv(pattern, v)
    torch.cuda.synchronize()
    assert torch.equal(s_split, scores), f"scores differ from the fused kernel's spill at T={T}"
    assert torch.equal(z_split, z), f"z differs from the fused kernel's at T={T}"
    q64, k64, v64 = (t.cpu().double() for t in (q, k, v))
    s64 = torch.einsum("bqhe,bkhe->bhqk", q64, k64) / scale
    z64 = torch.einsum("bkhe,bhqk->bqhe", v64, pattern.cpu().double())
    bar = 1e-4 if dname == "fp32" else 1e-2           # bf16: the outputs are rounded to bf16 (2^-9 relative)
    assert rel_err(s_split.cpu().double(), s64) <= bar
    assert rel_err(z_split.cpu().double(), z64) <= bar
    p64 = torch.softmax(s64, dim=-1)
    assert rel_err(pattern.cpu().double(), p64) <= (1e-4 if dname == "fp32" else 5e-2)


def test_split_stages_past_608_tokens_need_d_head_64():
    from vit_prisma.b200 import ops
    from vit_prisma.b200._lib import PrismaB200Error
    q = torch.randn(1, 641, 2, 32, device="cuda")
    with pytest.raises(PrismaB200Error, match="T=641 with d_head=32"):
        ops.attn_scores(q, q, 32 ** 0.5)
    with pytest.raises(PrismaB200Error, match="T=641 with d_head=32"):
        ops.attn_pv(torch.zeros(1, 2, 641, 641, device="cuda"), q)


@pytest.mark.parametrize("dname", ["fp32", "bf16"])
def test_vivit_b_size_two_blocks_match_oracle(dname, monkeypatch):
    """ViViT-B/16x2 geometry (224 px, 16 frames -> T = 1569, d 768, 12 heads), batch 2, the first two blocks on both routes."""
    dtype = DTYPES[dname]
    model, shapes = _model(VIVIT_B, dtype, seed=5)
    x = videos(2, VIVIT_B, seed=1)
    names = ["hook_embed", "blocks.0.hook_resid_post", "blocks.1.attn.hook_z", "blocks.1.hook_resid_post"]
    sd = {k: v for k, v in video_recipe_state_dict(shapes, 5, dtype).items() if not k.startswith("blocks.") or k.split(".")[1] in ("0", "1")}
    with torch.no_grad():
        ref_out, ref_cache = video_forward_with_cache(sd, dict(VIVIT_B, dtype=dtype), x.to(dtype), names_filter=lambda n: n in names,
                                                      stop_at_layer=2)
    assert ref_out.shape == (2, 1569, 768)
    for route in ("fused", "hooked"):
        if route == "hooked":
            monkeypatch.setenv("PRISMA_B200_ROUTE", "hooked")
        out, cache = model.run_with_cache(x.to("cuda", dtype), names_filter=names, stop_at_layer=2)
        assert model.last_route.startswith(route)
        assert list(cache.keys()) == list(ref_cache.keys())
        for k, ref in ref_cache.items():
            assert_close(cache[k].cpu(), ref, _bar(k, dname), f"{route}:{k}")
        assert_close(out.cpu(), ref_out, _bar("hook_resid_post", dname), f"{route}: output")
        del out, cache


def test_host_resident_video_model_returns_host_tensors():
    """A model left on the host (the reference's default device="cpu") is staged on the GPU for the call."""
    gold = load_golden("vit_video_c_fp32.pt")
    model, _ = _model(gold["cfg"], torch.float32, device="cpu")
    x = videos(gold["batch"], gold["cfg"], gold["images_seed"])
    out, cache = model.run_with_cache(x)
    assert out.device.type == "cpu" and all(v.device.type == "cpu" for v in cache.values())
    assert list(cache.keys()) == gold["keys"]
    for k in gold["keys"]:
        assert_close(cache[k], gold["cache"][k], 1e-4, k)
    assert_close(out, gold["out"], 1e-4, "model output")
    assert not model.cls_token.is_cuda


def test_sae_on_video_activations():
    """VisionActivationsStore.get_activations on fixture c's clips gives the cached hook values; TopK SAE steps through
    VisionSAETrainer.train_step on those token activations follow the oracle."""
    from torch.utils.data import TensorDataset
    from vit_prisma.sae.config import VisionModelSAERunnerConfig
    from vit_prisma.sae.train_sae import VisionSAETrainer
    from vit_prisma.sae.training.activations_store import VisionActivationsStore
    gold = load_golden("vit_video_c_fp32.pt")
    model, _ = _model(gold["cfg"], torch.float32)
    clips = videos(gold["batch"], gold["cfg"], gold["images_seed"])
    d, T, F, k = 32, 49, 256, 8
    rows = gold["batch"] * T
    with contextlib.redirect_stdout(io.StringIO()):
        scfg = VisionModelSAERunnerConfig(d_in=d, expansion_factor=F // d, activation_fn_str="topk", activation_fn_kwargs={"k": k},
                                          _device="cuda", _dtype="float32", hook_point_layer=1, layer_subtype="hook_resid_post",
                                          context_size=T, store_batch_size=gold["batch"], train_batch_size=rows, lr=1e-3,
                                          lr_warm_up_steps=1, lr_scheduler_name="constant", n_checkpoints=0, log_to_wandb=False,
                                          image_size=32, checkpoint_path="/tmp/prisma_b200_unused", b_dec_init_method="zeros",
                                          verbose=False, num_workers=0)
    store = VisionActivationsStore(scfg, model, TensorDataset(clips, torch.zeros(gold["batch"], dtype=torch.long)), create_dataloader=False)
    acts = store.get_activations(clips.cuda())
    assert tuple(acts.shape) == (gold["batch"], T, 1, d)
    assert_close(acts[:, :, 0].cpu(), gold["cache"]["blocks.1.hook_resid_post"], 1e-4, "store.get_activations")

    with contextlib.redirect_stdout(io.StringIO()):
        trainer = VisionSAETrainer(scfg, model=None, dataset=None, activations_store=object())
    g = torch.Generator().manual_seed(11)
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
