"""GPU probe: a CLIP-B/32 text tower (12 layers, d 512, 8 heads of 64, d_mlp 2048, context 77, vocab 49408, projection 512,
normalize_output) on synthetic seeded weights, 1024 prompts per call.

    python tools/text_probe.py [--dtypes fp32,bf16] [--batch 1024] [--iters 5] [--json out.json]

Times, with CUDA events, per dtype:
  * the fused forward (``model(ids)``, causal attention on the tensor cores);
  * ``run_with_cache`` with ``names_filter`` on one ``hook_resid_post``;
  * one forward on the hooked route (``PRISMA_B200_ROUTE=hooked``: every scores / pattern tensor materialised);
  * the fused attention kernel alone, causal vs unmasked, at T = 77 (whole-row kernel) and T = 248 (long kernel, where the
    causal instance skips the key chunks above each 64-row query slab).
Prompts/s of the fused forward is also given as a share of the bf16 dense peak, from the FLOPs the shapes imply (below).
Not a bench value.  The card name and power limit are read with a read-only ``nvidia-smi --query-gpu`` and printed.
"""
import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "vit-prisma_b200"))
import torch  # noqa: E402

from tests.text_oracle import CLIP_B32_TEXT, text_recipe_state_dict, text_state_dict_shapes, token_batch  # noqa: E402
from vit_prisma.b200 import ops  # noqa: E402

BF16_DENSE_PEAK = 989e12     # H100 SXM data sheet, dense BF16, 700 W


def flops_per_prompt(cfg) -> dict:
    """2 * M * N * K per GEMM per token; attention counted unmasked (QK^T and PV, 2 * T * T * dh each per head)."""
    T, d, dm, L, H, dh = cfg["context_length"], cfg["d_model"], cfg["d_mlp"], cfg["n_layers"], cfg["n_heads"], cfg["d_head"]
    gemm = L * T * 2 * (3 * d * H * dh + H * dh * d + 2 * d * dm)          # QKV, O, MLP in, MLP out
    attn = L * H * 2 * (2 * T * T * dh)
    head = 2 * d * cfg["n_classes"]
    return {"gemm": gemm, "attention": attn, "head": head, "total": gemm + attn + head}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=False)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi unavailable)"


def timed(fn, iters, warmup=1):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1e3 / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dtypes", default="fp32,bf16")
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("text_probe: no CUDA device -- this probe measures the GPU and has no CPU mode")
    from vit_prisma.configs.HookedTextTransformerConfig import HookedTextTransformerConfig
    from vit_prisma.models.base_text_transformer import HookedTextTransformer

    cfg = CLIP_B32_TEXT
    fl = flops_per_prompt(cfg)
    res = {"card": card(), "batch": a.batch, "flops_per_prompt": fl, "dtypes": {}}
    print(f"card: {res['card']}")
    print(f"FLOPs per prompt: {fl['total'] / 1e9:.3f} G = {fl['gemm'] / 1e9:.3f} G GEMM + {fl['attention'] / 1e9:.4f} G attention "
          f"+ {fl['head'] / 1e6:.2f} M head")
    ids = token_batch(a.batch, cfg["context_length"], cfg["vocab_size"], seed=0).cuda()
    for dname in a.dtypes.split(","):
        dt = {"fp32": torch.float32, "bf16": torch.bfloat16}[dname]
        model = HookedTextTransformer(HookedTextTransformerConfig(**cfg, dtype=dt)).to(dt)
        model.load_state_dict(text_recipe_state_dict(text_state_dict_shapes(cfg), 1234, dt))
        model = model.cuda().eval()
        r = {}
        with torch.no_grad():
            t = timed(lambda: model(ids), a.iters)
            assert model.last_route == "fused"
            r["fused_prompts_s"] = a.batch / t
            r["fused_share_of_bf16_peak"] = fl["total"] * a.batch / t / BF16_DENSE_PEAK
            t = timed(lambda: model.run_with_cache(ids, names_filter="blocks.6.hook_resid_post"), a.iters)
            r["cache_one_resid_prompts_s"] = a.batch / t
            os.environ["PRISMA_B200_ROUTE"] = "hooked"
            try:
                t = timed(lambda: model(ids), 1)
            finally:
                del os.environ["PRISMA_B200_ROUTE"]
            r["hooked_prompts_s"] = a.batch / t
        B, H, dh = 64, cfg["n_heads"], cfg["d_head"]
        for T in (77, 248):
            q, k, v = (torch.randn(B, T, H, dh, device="cuda").to(dt) for _ in range(3))
            for causal in (False, True):
                t = timed(lambda: ops.attention(q, k, v, math.sqrt(dh), want_scores=False, want_pattern=False, causal=causal),
                          20 * a.iters, warmup=3)
                r[f"attn_T{T}_{'causal' if causal else 'full'}_us"] = t * 1e6
        res["dtypes"][dname] = r
        print(f"[{dname}] fused {r['fused_prompts_s']:.0f} prompts/s ({100 * r['fused_share_of_bf16_peak']:.1f} % of the bf16 dense "
              f"peak), run_with_cache(1 resid) {r['cache_one_resid_prompts_s']:.0f} prompts/s, hooked {r['hooked_prompts_s']:.0f} "
              f"prompts/s")
        print(f"[{dname}] attention B={B} H={H}: T=77 full {r['attn_T77_full_us']:.1f} us / causal {r['attn_T77_causal_us']:.1f} us; "
              f"T=248 full {r['attn_T248_full_us']:.1f} us / causal {r['attn_T248_causal_us']:.1f} us")
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
