"""Pin the text checker (tests/text_oracle.py) to fixtures made by the unmodified reference (tests/golden/make_golden_text.py),
and check the host side of HookedTextTransformer on CPU: parameter layout, hook names, constructor errors, the C ABI.

CPU-only: the GPU routes are then held to these fixtures and to the checker in test_text_gpu.py."""
import ctypes

import pytest
import torch

from oracle.vit_oracle import digest
from tests.text_oracle import text_forward_with_cache, text_recipe_state_dict, text_state_dict_shapes, token_batch
from tests.util import assert_close, load_golden

TOL = {"fp32": 2e-5, "bf16": 1.6e-2}
FULL = ["text_e_fp32.pt", "text_e_bf16.pt", "text_h_fp32.pt"]
DIGESTS = ["text_f_fp32.pt", "text_g_fp32.pt"]


def _run(gold):
    cfg = dict(gold["cfg"])
    dtype = torch.float32 if gold["dtype"] == "fp32" else torch.bfloat16
    sd = text_recipe_state_dict(gold["shapes"], gold["weights_seed"], dtype)
    ids = token_batch(gold["batch"], gold["n_tokens"], cfg["vocab_size"], gold["ids_seed"])
    return text_forward_with_cache(sd, dict(cfg, dtype=dtype), ids, causal=gold["causal"])


@pytest.mark.parametrize("name", FULL)
def test_text_oracle_matches_reference_every_key(name):
    gold = load_golden(name)
    assert text_state_dict_shapes(gold["cfg"]) == gold["shapes"], "state-dict layout drifted from the reference"
    out, cache = _run(gold)
    assert list(cache.keys()) == gold["keys"], "cache key order differs from the reference"
    for k in gold["keys"]:
        got, ref = cache[k], gold["cache"][k]
        if k.endswith("hook_attn_scores"):       # -inf positions exactly, the finite entries within the bar
            assert torch.equal(got.isinf(), ref.isinf()), k
            got, ref = torch.where(got.isinf(), torch.zeros_like(got), got), torch.where(ref.isinf(), torch.zeros_like(ref), ref)
        assert_close(got, ref, TOL[gold["dtype"]], k)
    assert_close(out, gold["out"], TOL[gold["dtype"]], "model output")


@pytest.mark.parametrize("name", DIGESTS)
def test_text_oracle_matches_reference_digests(name):
    gold = load_golden(name)
    assert text_state_dict_shapes(gold["cfg"]) == gold["shapes"]
    out, cache = _run(gold)
    assert list(cache.keys()) == gold["keys"]
    for k, dg in gold["digests"].items():
        v = cache[k]
        if k.endswith("hook_attn_scores"):
            inf = v.isinf()
            assert torch.equal(inf, gold["inf_masks"][k].expand_as(inf)), k
            v = torch.where(inf, torch.zeros_like(v), v)
        mine = digest(v)
        assert mine["shape"] == dg["shape"] and mine["dtype"] == dg["dtype"], k
        assert (mine["samples"] - dg["samples"]).abs().max().item() / max(dg["max_abs"], 1e-30) < 2e-5, k
        assert abs(mine["sum"] - dg["sum"]) <= 2e-5 * max(dg["abs_sum"], 1e-30), k
    last = f"blocks.{gold['cfg']['n_layers'] - 1}.hook_resid_post"
    assert_close(cache[last], gold["last_resid_post"], 2e-5, last)
    assert_close(out, gold["out"], 2e-5, "model output")


def test_token_batches_place_end_of_text_at_the_edges_and_tie():
    ids = token_batch(4, 12, 50, 0)
    assert ids.argmax(-1).tolist()[:3] == [0, 11, 2]
    assert int((ids[2] == 49).sum()) == 2


def test_oracle_raises_on_a_short_input_under_the_causal_mask():
    gold = load_golden("text_e_fp32.pt")
    sd = text_recipe_state_dict(gold["shapes"], gold["weights_seed"])
    with pytest.raises(RuntimeError):
        text_forward_with_cache(sd, dict(gold["cfg"]), token_batch(3, 9, gold["cfg"]["vocab_size"]), causal=True)


@pytest.mark.parametrize("name", FULL + DIGESTS)
def test_model_parameters_and_hook_names_equal_the_reference(name):
    from vit_prisma.configs.HookedTextTransformerConfig import HookedTextTransformerConfig
    from vit_prisma.models.base_text_transformer import HookedTextTransformer
    gold = load_golden(name)
    dtype = torch.float32 if gold["dtype"] == "fp32" else torch.bfloat16
    model = HookedTextTransformer(HookedTextTransformerConfig(**gold["cfg"], dtype=dtype), no_causal_mask=not gold["causal"]).to(dtype)
    assert {k: tuple(v.shape) for k, v in model.state_dict().items()} == gold["shapes"]
    assert list(model.hook_dict) == gold["hook_names"]
    assert model.cfg.n_tokens == gold["cfg"]["context_length"]
    model.load_state_dict(text_recipe_state_dict(gold["shapes"], gold["weights_seed"], dtype))
    if gold["causal"]:
        mask = model.attn_mask
        assert mask.dtype == dtype and mask.shape == (model.context_length,) * 2
        assert torch.equal(mask.isinf(), torch.ones_like(mask, dtype=torch.bool).triu(1))
    else:
        assert model.attn_mask is None


def test_constructor_errors_follow_the_reference():
    from vit_prisma.configs.HookedTextTransformerConfig import HookedTextTransformerConfig
    from vit_prisma.models.base_text_transformer import HookedTextTransformer
    cfg = dict(load_golden("text_e_fp32.pt")["cfg"])
    for norm in ("LNPre", None):
        with pytest.raises(ValueError):
            HookedTextTransformer(HookedTextTransformerConfig(**dict(cfg, normalization_type=norm)))
    with pytest.raises(ValueError):
        HookedTextTransformer("openai/clip-vit-base-patch32")
    m = HookedTextTransformer(HookedTextTransformerConfig(**cfg), cls_token=True)     # constructs; every forward raises
    assert m.num_pos == cfg["context_length"] + 1 and m.attn_mask.shape == (m.num_pos, m.num_pos)
    with pytest.raises(RuntimeError):
        m(torch.zeros(1, cfg["context_length"], dtype=torch.int64))


def test_token_id_check_raises_index_error_before_any_launch():
    from vit_prisma.models.base_text_transformer import check_token_ids
    assert check_token_ids(torch.tensor([[0, 49]], dtype=torch.int32), 50).dtype == torch.int64
    for bad in (-1, 50):
        with pytest.raises(IndexError):
            check_token_ids(torch.tensor([[0, bad]]), 50)


def test_text_forward_abi_matches_the_compiled_library():
    from vit_prisma.b200 import _lib as L
    lib = ctypes.CDLL(str(L.LIB_PATH))
    lib.pb_abi_sizeof.restype = ctypes.c_int
    assert lib.pb_abi_sizeof(L.ABI_TEXT_FORWARD) == ctypes.sizeof(L.PbTextForward)
    assert lib.pb_abi_sizeof(2) == ctypes.sizeof(L.PbAttention)
    assert L.PbAttention.causal.offset == ctypes.sizeof(L.PbAttention) - 8   # appended: zeroed descriptors stay unmasked
