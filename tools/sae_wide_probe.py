"""GPU probe: per-stage time of one TopK SAE training step (4096 tokens, k 32, fp32) on the narrow row kernels (d_in 1536) and on
the wide ones (d_in 1664, bigG's residual stream; d_in 3072, CLIP B's MLP neurons), with the achieved bytes/s of every stage that
has a byte count, against the H100 SXM's 3.35 TB/s.  Prints the card and its power limit first.  Not a bench value."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "vit-prisma_b200"))
import torch  # noqa: E402

from vit_prisma.b200.sae_engine import SaeStepEngine, unit_norm_rows_  # noqa: E402

HBM = 3.35e12
SHAPES = ((1536, 24576), (1664, 26624), (3072, 24576))
ROWS, K = 4096, 32


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def main():
    dev = torch.device("cuda", 0)
    print(f"card: {card()}", flush=True)
    for d, F in SHAPES:
        g = torch.Generator(device=dev).manual_seed(d)
        W_dec = torch.randn(F, d, device=dev, generator=g)
        W_encT = (torch.randn(F, d, device=dev, generator=g) / d ** 0.5).contiguous()
        b_enc, b_dec = torch.zeros(F, device=dev), torch.zeros(d, device=dev)
        eng = SaeStepEngine(W_encT, W_dec, b_enc, b_dec, k=K)
        unit_norm_rows_(eng.W_dec)
        eng.refresh_lo()
        x = torch.randn(ROWS, d, device=dev, generator=g) * 2.0 + 1.0
        sf, af = torch.zeros(F, device=dev), torch.zeros(F, device=dev)
        for _ in range(3):
            eng.train_step(x, 1e-4, sf, af)
        stages = eng.time_stages(x, 1e-4, sf, af, reps=10)
        print(f"d_in {d}, d_sae {F}, {ROWS} tokens, k {K}, encoder {eng.encoder}:", flush=True)
        for name, info in stages.items():
            rate = ""
            if "bytes" in info:
                bps = info["bytes"] / (info["ms"] * 1e-3)
                rate = f"  {bps / 1e12:5.2f} TB/s ({bps / HBM:4.0%} of 3.35 TB/s)"
            print(f"  {info['ms']:8.3f} ms  {name}{rate}", flush=True)
        del eng
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
