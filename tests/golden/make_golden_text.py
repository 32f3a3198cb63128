"""Generate the text-tower golden fixtures by running the UNMODIFIED reference HookedTextTransformer on CPU.

    python tests/golden/make_golden_text.py

Like make_golden.py this needs the reference sources and runs only where they are; the fixtures it writes are committed.
Weights come from tests/text_oracle.text_recipe_state_dict and the ids from tests/text_oracle.token_batch (seeded), which puts
the end-of-text id at position 0, at T-1, and twice in one row.

  text_e_{fp32,bf16}.pt  tiny causal model: context 12, 2 layers, 2 heads of 16 (the FFMA attention kernel), batch 3.
                         Every cache key in full, the output and the key order.
  text_f_fp32.pt         d_head 64 at context 77 (the short tensor-core kernel), batch 3.
  text_g_fp32.pt         d_head 64 at context 200 (the long kernel, chunks above the diagonal skipped), batch 3.
                         f and g keep per-key digests (scores with -inf replaced by 0), the -inf pattern of each
                         hook_attn_scores as one [T, T] mask (asserted identical over batch and heads), the full output and
                         the full last hook_resid_post.
  text_h_fp32.pt         a no_causal_mask model of context 12 fed 9 positions.  Every key in full.

Each file also records the hook names and the parameter shapes, and every file stays under 700 KB.
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
import _ref_shims  # noqa: E402

_ref_shims.install()

from oracle.vit_oracle import digest  # noqa: E402
from tests.text_oracle import text_recipe_state_dict, token_batch  # noqa: E402

_BASE = dict(eps=1e-5, activation_name="quick_gelu", normalization_type="LN", normalize_output=True, return_type="class_logits")
TEXT_E = dict(_BASE, n_layers=2, d_model=32, d_head=16, n_heads=2, d_mlp=64, context_length=12, vocab_size=50, n_classes=24)
TEXT_F = dict(_BASE, n_layers=2, d_model=128, d_head=64, n_heads=2, d_mlp=256, context_length=77, vocab_size=300, n_classes=64)
TEXT_G = dict(_BASE, n_layers=2, d_model=128, d_head=64, n_heads=2, d_mlp=256, context_length=200, vocab_size=300, n_classes=64)
TEXT_H = dict(TEXT_E)


def ref_model(cfg: dict, dtype=torch.float32, no_causal_mask=False):
    from vit_prisma.configs.HookedTextTransformerConfig import HookedTextTransformerConfig
    from vit_prisma.models.base_text_transformer import HookedTextTransformer
    model = HookedTextTransformer(HookedTextTransformerConfig(**cfg, dtype=dtype), no_causal_mask=no_causal_mask).to(dtype)
    shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    model.load_state_dict(text_recipe_state_dict(shapes, seed=1234, dtype=dtype))
    model.eval()
    return model, shapes


def _meta(model, cfg, dname, shapes, batch, n_tokens, causal):
    return {"cfg": cfg, "dtype": dname, "shapes": shapes, "hook_names": list(model.hook_dict), "weights_seed": 1234,
            "ids_seed": 0, "batch": batch, "n_tokens": n_tokens, "causal": causal}


def make_text():
    for dtype, dname in ((torch.float32, "fp32"), (torch.bfloat16, "bf16")):
        model, shapes = ref_model(TEXT_E, dtype)
        ids = token_batch(3, 12, TEXT_E["vocab_size"], seed=0)
        with torch.no_grad():
            out, cache = model.run_with_cache(ids, return_cache_object=False)
        assert cache["hook_pos_embed"].shape == (12, TEXT_E["d_model"])
        path = os.path.join(HERE, f"text_e_{dname}.pt")
        torch.save(dict(_meta(model, TEXT_E, dname, shapes, 3, 12, True), keys=list(cache.keys()),
                        cache={k: v.clone() for k, v in cache.items()}, out=out.clone()), path)
        print("wrote", path, len(cache), "keys", os.path.getsize(path), "bytes")

    for name, cfg, batch in (("f", TEXT_F, 3), ("g", TEXT_G, 3)):
        model, shapes = ref_model(cfg)
        T = cfg["context_length"]
        ids = token_batch(batch, T, cfg["vocab_size"], seed=0)
        with torch.no_grad():
            out, cache = model.run_with_cache(ids, return_cache_object=False)
        digests, inf_masks = {}, {}
        for k, v in cache.items():
            if k.endswith("hook_attn_scores"):
                inf = v.isinf()
                assert bool((inf == inf[:1, :1]).all()), "the -inf pattern differs between batch rows or heads"
                inf_masks[k] = inf[0, 0].clone()
                v = torch.where(inf, torch.zeros_like(v), v)
            digests[k] = digest(v)
        last = f"blocks.{cfg['n_layers'] - 1}.hook_resid_post"
        path = os.path.join(HERE, f"text_{name}_fp32.pt")
        torch.save(dict(_meta(model, cfg, "fp32", shapes, batch, T, True), keys=list(cache.keys()), digests=digests,
                        inf_masks=inf_masks, out=out.clone(), last_resid_post=cache[last].clone()), path)
        print("wrote", path, len(cache), "keys", os.path.getsize(path), "bytes")

    model, shapes = ref_model(TEXT_H, no_causal_mask=True)
    ids = token_batch(3, 9, TEXT_H["vocab_size"], seed=0)
    with torch.no_grad():
        out, cache = model.run_with_cache(ids, return_cache_object=False)
    assert cache["hook_pos_embed"].shape == (9, TEXT_H["d_model"])
    path = os.path.join(HERE, "text_h_fp32.pt")
    torch.save(dict(_meta(model, TEXT_H, "fp32", shapes, 3, 9, False), keys=list(cache.keys()),
                    cache={k: v.clone() for k, v in cache.items()}, out=out.clone()), path)
    print("wrote", path, len(cache), "keys", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    make_text()
