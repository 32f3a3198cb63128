"""GPU probe: a video ViT at the ViViT-B/16x2 geometry (224 px, 16 frames in tubelets of 2 -> T = 1569 tokens, d 768, 12 layers).

    python tools/video_probe.py [--dtypes fp32,bf16] [--batch 4] [--iters 5] [--json out.json]

Times, with CUDA events, per dtype:
  * the fused forward (``model(x)``);
  * ``run_with_cache`` with ``names_filter`` on a residual-stream hook (what the activation store issues);
  * one forward on the hooked route (``PRISMA_B200_ROUTE=hooked``: every scores / pattern tensor materialised);
  * the kernels new to video: tubelet im2col, and the long attention kernel fused and as its two split stages,
    each against the bytes and FLOPs its shapes imply.
Synthetic seeded weights (vit_prisma.b200.synthetic, conv weight scaled by its fan-in); not a bench value.  The card name and
power limit are read with a read-only ``nvidia-smi --query-gpu`` and printed with the numbers.
"""
import argparse
import contextlib
import io
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "vit-prisma_b200"))
import torch  # noqa: E402

from vit_prisma.b200 import ops  # noqa: E402
from vit_prisma.b200.synthetic import recipe_state_dict  # noqa: E402

VIVIT_B = dict(n_layers=12, d_model=768, d_head=64, n_heads=12, d_mlp=3072, patch_size=16, image_size=224, n_channels=3,
               n_classes=400, eps=1e-6, activation_name="gelu", normalization_type="LN", use_cls_token=True, layer_norm_pre=False,
               normalize_output=False, return_type="pre_logits", classification_type="cls", is_video_transformer=True,
               video_tubelet_depth=2, video_num_frames=16)


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
    return e0.elapsed_time(e1) / iters             # ms


def model_for(dtype):
    from vit_prisma.configs.HookedViTConfig import HookedViTConfig
    from vit_prisma.models.base_vit import HookedViT
    with contextlib.redirect_stdout(io.StringIO()):
        model = HookedViT(HookedViTConfig(**VIVIT_B, dtype=dtype))
    shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    sd = recipe_state_dict(shapes, 1234)
    sd["embed.proj.weight"] /= math.sqrt(VIVIT_B["patch_size"])     # fan-in C*D*P*P
    model.load_state_dict(sd)
    return model.to("cuda", dtype).eval()


def probe(dtype, B, iters):
    es = torch.empty((), dtype=dtype).element_size()
    cfg = VIVIT_B
    T, H, dh, L = 1569, cfg["n_heads"], cfg["d_head"], cfg["n_layers"]
    model = model_for(dtype)
    assert model.cfg.n_tokens == T
    x = torch.randn(B, 3, cfg["video_num_frames"], 224, 224, generator=torch.Generator().manual_seed(0)).to("cuda", dtype)
    r = {"dtype": str(dtype).replace("torch.", ""), "batch": B, "tokens_per_clip": T}
    with torch.no_grad():
        ms = timed(lambda: model(x), iters)
        assert model.last_route == "fused", model.last_route
        r["fused_forward_ms"] = ms
        name = f"blocks.{L - 1}.hook_resid_post"
        r["run_with_cache_resid_ms"] = timed(lambda: model.run_with_cache(x, names_filter=[name], stop_at_layer=L), iters)
        os.environ["PRISMA_B200_ROUTE"] = "hooked"
        try:
            r["hooked_forward_ms"] = timed(lambda: model(x), 1)
            assert model.last_route.startswith("hooked")
        finally:
            del os.environ["PRISMA_B200_ROUTE"]
    for k in ("fused_forward", "run_with_cache_resid", "hooked_forward"):
        r[k + "_clips_per_s"] = B / (r[k + "_ms"] * 1e-3)
        r[k + "_tokens_per_s"] = B * T / (r[k + "_ms"] * 1e-3)

    # kernels, each against the bytes / FLOPs its shapes imply
    kern = {}
    n_patch = B * (T - 1) * 3 * 2 * 16 * 16
    kern["im2col_tubelets"] = (timed(lambda: ops.im2col_tubelets(x, 16, 2), 20), 2 * n_patch * es, 0)
    q, k, v = (torch.randn(B, T, H, dh, device="cuda").to(dtype) for _ in range(3))
    qkvz = 4 * B * T * H * dh * es
    tt = B * H * T * T
    flops = 4 * tt * dh                                           # QK^T + PV (the kernel computes QK^T twice: 6 * tt * dh issued)
    kern["attention_fused_no_spill"] = (timed(lambda: ops.attention(q, k, v, 8.0, False, False), 10), qkvz, flops)
    kern["attention_fused_spill"] = (timed(lambda: ops.attention(q, k, v, 8.0), 5), qkvz + 2 * tt * es, flops)
    _, pattern, _ = ops.attention(q, k, v, 8.0)
    kern["attn_scores_split"] = (timed(lambda: ops.attn_scores(q, k, 8.0), 5), (2 * B * T * H * dh + tt) * es, 2 * tt * dh)
    kern["attn_pv_split"] = (timed(lambda: ops.attn_pv(pattern, v), 5), (tt + 2 * B * T * H * dh) * es, 2 * tt * dh)
    r["kernels"] = {n: {"ms": ms, "bytes": b, "GB_per_s": b / (ms * 1e-3) / 1e9, "flops": f, "TFLOP_per_s": f / (ms * 1e-3) / 1e12}
                    for n, (ms, b, f) in kern.items()}
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dtypes", default="fp32,bf16")
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    gpu = card()
    print(f"card: {gpu}")
    out = {"card": gpu, "results": []}
    for dn in a.dtypes.split(","):
        r = probe({"fp32": torch.float32, "bf16": torch.bfloat16}[dn], a.batch, a.iters)
        out["results"].append(r)
        print(f"[{dn}] ViViT-B/16x2 B={a.batch} T={r['tokens_per_clip']}:")
        for k in ("fused_forward", "run_with_cache_resid", "hooked_forward"):
            print(f"  {k:22s} {r[k + '_ms']:9.2f} ms  {r[k + '_clips_per_s']:8.2f} clips/s  {r[k + '_tokens_per_s'] / 1e3:9.1f} k tokens/s")
        for n, kr in r["kernels"].items():
            print(f"  {n:26s} {kr['ms']:8.3f} ms  {kr['GB_per_s']:7.0f} GB/s  {kr['TFLOP_per_s']:6.1f} TFLOP/s (algorithmic)")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
