"""HookedTextTransformer on the GPU: both routes against the reference-made fixtures and the CPU checker, the causal
attention kernels alone against float64, and the route behaviour (hooks, filters, host-resident models, id checks)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle.vit_oracle import digest  # noqa: E402
from tests.text_oracle import (CLIP_B32_TEXT, text_forward_with_cache, text_recipe_state_dict,  # noqa: E402
                               text_state_dict_shapes, token_batch)
from tests.test_vit_gpu import TOL, _bar  # noqa: E402
from tests.util import assert_close, load_golden, rel_err  # noqa: E402

DT = {"fp32": torch.float32, "bf16": torch.bfloat16}


def _model(cfg, dtype, causal=True, device="cuda"):
    from vit_prisma.configs.HookedTextTransformerConfig import HookedTextTransformerConfig
    from vit_prisma.models.base_text_transformer import HookedTextTransformer
    model = HookedTextTransformer(HookedTextTransformerConfig(**cfg, dtype=dtype), no_causal_mask=not causal).to(dtype)
    sd = text_recipe_state_dict(text_state_dict_shapes(cfg), 1234, dtype)
    model.load_state_dict(sd)
    return model.to(device).eval(), sd


def _finite(t):
    return torch.where(t.isinf(), torch.zeros_like(t), t)


def _check_cache(model, cache, ref_keys, ref_get, dname, route, T):
    assert list(cache.keys()) == ref_keys, "cache key order differs from the reference"
    upper = torch.ones(T, T, dtype=torch.bool, device="cuda").triu(1)
    for k in ref_keys:
        got, ref = cache[k], ref_get(k)
        if k.endswith("hook_attn_scores"):       # -inf positions exactly, the finite entries within the bar
            assert torch.equal(got.isinf().cpu(), ref.isinf()), f"{route}:{k}"
            got, ref = _finite(got), _finite(ref)
        if k.endswith("hook_pattern") and model.attn_mask is not None:
            assert bool((got[..., upper] == 0).all()), f"{route}:{k} is not exactly 0 above the diagonal"
        assert_close(got.cpu(), ref, _bar(k, dname), f"{route}:{k}")
    assert cache["hook_pos_embed"].untyped_storage().data_ptr() == model.pos_embed.untyped_storage().data_ptr()
    for l in range(1, model.cfg.n_layers):
        assert cache[f"blocks.{l}.hook_resid_pre"].data_ptr() == cache[f"blocks.{l - 1}.hook_resid_post"].data_ptr()


@pytest.mark.parametrize("name", ["text_e_fp32", "text_e_bf16", "text_h_fp32"])
@pytest.mark.parametrize("route", ["fused", "hooked"])
def test_text_matches_reference_golden(name, route, monkeypatch):
    gold = load_golden(name + ".pt")
    dname = gold["dtype"]
    model, _ = _model(gold["cfg"], DT[dname], gold["causal"])
    if route == "hooked":
        monkeypatch.setenv("PRISMA_B200_ROUTE", "hooked")
    ids = token_batch(gold["batch"], gold["n_tokens"], gold["cfg"]["vocab_size"], gold["ids_seed"]).cuda()
    out, cache = model.run_with_cache(ids)
    assert model.last_route.startswith(route), model.last_route
    _check_cache(model, cache, gold["keys"], lambda k: gold["cache"][k], dname, route, gold["n_tokens"])
    assert_close(out.cpu(), gold["out"], TOL[dname], "model output")
    assert rel_err(model(ids).cpu().float(), gold["out"].float()) <= TOL[dname]


@pytest.mark.parametrize("name", ["text_f", "text_g"])
@pytest.mark.parametrize("dname", ["fp32", "bf16"])
@pytest.mark.parametrize("route", ["fused", "hooked"])
def test_text_d_head_64_matches_reference(name, dname, route, monkeypatch):
    """fp32 against the reference's digests; bf16 against the checker run in bf16 (every key in full)."""
    gold = load_golden(name + "_fp32.pt")
    cfg, T = gold["cfg"], gold["n_tokens"]
    model, sd = _model(cfg, DT[dname])
    if route == "hooked":
        monkeypatch.setenv("PRISMA_B200_ROUTE", "hooked")
    ids = token_batch(gold["batch"], T, cfg["vocab_size"], gold["ids_seed"])
    out, cache = model.run_with_cache(ids.cuda())
    assert model.last_route.startswith(route), model.last_route
    if dname == "bf16":
        ref_out, ref = text_forward_with_cache(sd, dict(cfg, dtype=torch.bfloat16), ids)
        _check_cache(model, cache, list(ref), lambda k: ref[k], dname, route, T)
        assert_close(out.cpu(), ref_out, TOL[dname], "model output")
        return
    assert list(cache.keys()) == gold["keys"]
    upper = torch.ones(T, T, dtype=torch.bool).triu(1)
    for k, dg in gold["digests"].items():
        v = cache[k].cpu()
        if k.endswith("hook_attn_scores"):
            assert torch.equal(v.isinf(), gold["inf_masks"][k].expand_as(v)), k
            v = _finite(v)
        if k.endswith("hook_pattern"):
            assert bool((v[..., upper] == 0).all()), k
        mine = digest(v)
        assert mine["shape"] == dg["shape"] and mine["dtype"] == dg["dtype"], k
        assert (mine["samples"] - dg["samples"]).abs().max().item() / max(dg["max_abs"], 1e-30) <= TOL["fp32"], k
    last = f"blocks.{cfg['n_layers'] - 1}.hook_resid_post"
    assert_close(cache[last].cpu(), gold["last_resid_post"], TOL["fp32"], last)
    assert_close(out.cpu(), gold["out"], TOL["fp32"], "model output")
    assert cache["blocks.1.hook_resid_pre"].data_ptr() == cache["blocks.0.hook_resid_post"].data_ptr()
    assert cache["hook_pos_embed"].untyped_storage().data_ptr() == model.pos_embed.untyped_storage().data_ptr()


def _masked_attention64(q, k, v, scale):
    q, k, v = q.double(), k.double(), v.double()
    T = q.shape[1]
    s = torch.einsum("bqhe,bkhe->bhqk", q, k) / scale
    s = s + torch.full((T, T), float("-inf"), dtype=torch.float64, device=q.device).triu(1)
    p = torch.softmax(s, -1)
    return s, p, torch.einsum("bhqk,bkhe->bqhe", p, v)


@pytest.mark.parametrize("T,dh", [(t, 64) for t in (1, 16, 64, 77, 128, 129, 200, 320)] + [(77, 16), (50, 32), (200, 32)])
@pytest.mark.parametrize("dname", ["fp32", "bf16"])
def test_causal_attention_kernel_matches_float64(T, dh, dname):
    from vit_prisma.b200 import ops
    g = torch.Generator().manual_seed(T * 7 + dh)
    B, H = 3, 2
    q, k, v = (torch.randn(B, T, H, dh, generator=g).to("cuda", DT[dname]) for _ in range(3))
    scale = math.sqrt(dh)
    s64, p64, z64 = _masked_attention64(q, k, v, scale)
    scores, pattern, z = ops.attention(q, k, v, scale, causal=True)
    _, _, z_nospill = ops.attention(q, k, v, scale, want_scores=False, want_pattern=False, causal=True)
    assert torch.equal(z, z_nospill), "z depends on whether the spills are requested"
    upper = torch.ones(T, T, dtype=torch.bool, device="cuda").triu(1)
    assert bool(scores[..., upper].isneginf().all()) and bool(scores[..., ~upper].isfinite().all())
    assert bool((pattern[..., upper] == 0).all())
    tol = 1e-4 if dname == "fp32" else 2e-2
    assert rel_err(_finite(scores), _finite(s64)) <= tol
    assert rel_err(pattern, p64) <= tol
    assert rel_err(z, z64) <= tol
    if T > 1:   # the unmasked kernels are untouched: causal=False still attends to every key
        _, p_full, _ = ops.attention(q, k, v, scale, causal=False)
        assert bool((p_full[..., upper] > 0).any())


@pytest.mark.parametrize("dname", ["fp32", "bf16"])
def test_fused_and_hooked_agree_at_clip_b32_text_width(dname, monkeypatch):
    cfg = dict(CLIP_B32_TEXT, n_layers=2)
    model, _ = _model(cfg, DT[dname])
    ids = token_batch(64, 77, cfg["vocab_size"], seed=3).cuda()
    out_f, cache_f = model.run_with_cache(ids)
    assert model.last_route == "fused"
    monkeypatch.setenv("PRISMA_B200_ROUTE", "hooked")
    out_h, cache_h = model.run_with_cache(ids)
    assert model.last_route.startswith("hooked")
    assert list(cache_f.keys()) == list(cache_h.keys())
    for key in cache_f:
        a, b = cache_f[key], cache_h[key]
        if key.endswith("hook_attn_scores"):
            assert torch.equal(a.isinf(), b.isinf()), key
            a, b = _finite(a), _finite(b)
        assert rel_err(a, b) <= 2 * _bar(key, dname), key
    assert rel_err(out_f, out_h) <= 2 * TOL[dname]


def test_routes_hooks_filters_and_ids():
    gold = load_golden("text_e_fp32.pt")
    cfg = gold["cfg"]
    model, sd = _model(cfg, torch.float32)
    ids_cpu = token_batch(3, 12, cfg["vocab_size"], 0)
    ids = ids_cpu.cuda()
    ref_out, _ = text_forward_with_cache(sd, cfg, ids_cpu)

    # a hook that edits hook_pattern takes the hooked route and changes the output as the checker predicts
    edit = {"blocks.0.attn.hook_pattern": lambda p: p * 0.5}
    out = model.run_with_hooks(ids, fwd_hooks=[("blocks.0.attn.hook_pattern", lambda t, hook: t * 0.5)])
    assert model.last_route.startswith("hooked")
    want, _ = text_forward_with_cache(sd, cfg, ids_cpu, hooks=edit)
    assert rel_err(out.cpu(), want) <= 1e-4 and rel_err(want, ref_out) > 1e-2

    # names_filter of one hook_resid_post
    out, cache = model.run_with_cache(ids, names_filter="blocks.0.hook_resid_post")
    assert model.last_route == "fused" and list(cache.keys()) == ["blocks.0.hook_resid_post"]
    assert rel_err(out.cpu(), ref_out) <= 1e-4
    assert rel_err(cache["blocks.0.hook_resid_post"].cpu(), gold["cache"]["blocks.0.hook_resid_post"]) <= 1e-4

    # remove_batch_dim and device
    out1, cache1 = model.run_with_cache(ids[:1], remove_batch_dim=True, device="cpu")
    assert cache1["blocks.1.hook_resid_post"].shape == (12, cfg["d_model"]) and cache1["hook_embed"].device.type == "cpu"
    assert rel_err(cache1["blocks.1.hook_resid_post"], gold["cache"]["blocks.1.hook_resid_post"][0]) <= 1e-4

    # int32 ids give the same result as int64
    assert torch.equal(model(ids.to(torch.int32)), model(ids))

    # out-of-range ids raise IndexError on both routes, before any launch
    for bad in (-1, cfg["vocab_size"]):
        x = ids.clone()
        x[1, 3] = bad
        with pytest.raises(IndexError):
            model(x)
        with pytest.raises(IndexError):
            model.run_with_hooks(x, fwd_hooks=[("hook_embed", lambda t, hook: t)])

    # a shorter input under the causal mask raises RuntimeError, as the reference does
    with pytest.raises(RuntimeError):
        model(ids[:, :9])


def test_host_resident_text_model_returns_host_tensors():
    gold = load_golden("text_e_fp32.pt")
    model, _ = _model(gold["cfg"], torch.float32, device="cpu")
    ids = token_batch(3, 12, gold["cfg"]["vocab_size"], 0)
    out, cache = model.run_with_cache(ids)
    assert out.device.type == "cpu" and cache["blocks.1.hook_resid_post"].device.type == "cpu"
    assert_close(out, gold["out"], TOL["fp32"], "host-resident output")
    assert rel_err(model(ids), gold["out"]) <= TOL["fp32"]
