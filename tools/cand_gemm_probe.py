"""GPU probe: the fused SAE encoder's candidate GEMM (phase 1 of pb_sae_encode_topk_fused) alone at the bench shape, next to a
plain L2-resident read bandwidth (for kernel tuning; not a bench value).

    python tools/cand_gemm_probe.py [--operands tf32,f16] [--reps 200] [--rounds 3]

Per operand type: ms per call (CUDA events over ``reps`` warm replays), TFLOP/s, and the L2 -> SM operand traffic of the
128 x 256 tiles (every tile streams its A slab [128, d] and B slab [256, d]) over that time.  With several operand types the
calls alternate, ``rounds`` times, in one process.  The read figure comes from a 16-byte-load kernel over a 24 MB buffer (fits
the 50 MB L2), compiled with nvcc into a temporary directory."""
import argparse
import ctypes as C
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "vit-prisma_b200"))
import torch  # noqa: E402

READ_KERNEL = r"""
extern "C" __global__ void k_read(const float4* __restrict__ p, long long n, float* __restrict__ sink) {
  float acc = 0.f;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float4 v = __ldcg(p + i);
    acc += v.x + v.y + v.z + v.w;
  }
  if (acc == 1234.5f) sink[0] = acc;     // keeps the loads alive; never true for the buffer below
}
extern "C" int read_bw(const void* p, long long bytes, int reps, float* sink, int sms, float* ms) {
  cudaEvent_t a, b;
  cudaEventCreate(&a); cudaEventCreate(&b);
  const long long n = bytes / 16;
  for (int i = 0; i < 3; ++i) k_read<<<sms * 8, 512>>>((const float4*)p, n, sink);
  cudaEventRecord(a);
  for (int i = 0; i < reps; ++i) k_read<<<sms * 8, 512>>>((const float4*)p, n, sink);
  cudaEventRecord(b);
  cudaEventSynchronize(b);
  cudaEventElapsedTime(ms, a, b);
  cudaEventDestroy(a); cudaEventDestroy(b);
  return (int)cudaGetLastError();
}
"""


def l2_read_tbs(reps: int) -> float:
    tmp = tempfile.mkdtemp(prefix="cand_probe_")
    src, so = os.path.join(tmp, "read.cu"), os.path.join(tmp, "read.so")
    with open(src, "w") as f:
        f.write(READ_KERNEL)
    nvcc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    subprocess.check_call([nvcc, "-O3", "-shared", "-Xcompiler", "-fPIC", "-gencode", "arch=compute_90a,code=sm_90a", src, "-o", so])
    lib = C.CDLL(so)
    lib.read_bw.argtypes = [C.c_void_p, C.c_longlong, C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_float)]
    buf = torch.rand(24 << 20 >> 2, device="cuda")
    sink = torch.zeros(1, device="cuda")
    ms = C.c_float(0)
    torch.cuda.synchronize()
    rc = lib.read_bw(buf.data_ptr(), buf.numel() * 4, reps, sink.data_ptr(), torch.cuda.get_device_properties(0).multi_processor_count,
                     C.byref(ms))
    assert rc == 0, f"read kernel failed: cudaError {rc}"
    return buf.numel() * 4 * reps / (ms.value * 1e-3) / 1e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--operands", default="tf32,f16")
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--d", type=int, default=768)
    ap.add_argument("--F", type=int, default=24576)
    ap.add_argument("--rows", type=int, default=4096)
    args = ap.parse_args()
    from vit_prisma.b200 import _lib as L
    from vit_prisma.b200.ops import _stream
    from vit_prisma.b200.sae_engine import SaeStepEngine

    d, F, rows, k = args.d, args.F, args.rows, 32
    g = torch.Generator().manual_seed(0)
    W = (torch.randn(F, d, generator=g) / d ** 0.5).cuda()
    W_dec = torch.randn(F, d, generator=g)
    W_dec = (W_dec / W_dec.norm(dim=1, keepdim=True)).cuda()
    x = (torch.randn(rows, d, generator=g) * 2.0 + torch.randn(d, generator=g)).cuda()
    engines = {}
    for op in args.operands.split(","):
        eng = SaeStepEngine(W.clone(), W_dec.clone(), torch.zeros(F, device="cuda"), torch.zeros(d, device="cuda"), k=k,
                            encoder="fused" if op == "tf32" else "auto")
        got = getattr(eng, "cand_operands", "tf32")
        if got != op:
            print(f"{op}: not available in this build (engine took {got}); skipped", flush=True)
            continue
        eng.encode_topk(x)                                  # prep (sae_in and its operand copy) + one full encode
        engines[op] = eng
    lib, st = L.get_lib(), _stream()
    flops = 2.0 * rows * d * F
    tiles_m, tiles_n = -(-rows // 128), -(-F // 256)
    for r in range(args.rounds):
        for op, eng in engines.items():
            es = 2 if op == "f16" else 4
            desc = eng._enc_desc(rows, 1)
            fn = lambda: L.check(lib.pb_sae_encode_topk_fused(C.byref(desc), st), "pb_sae_encode_topk_fused")  # noqa: E731
            for _ in range(5):
                fn()
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.reps):
                fn()
            b.record()
            torch.cuda.synchronize()
            ms = a.elapsed_time(b) / args.reps
            l2_bytes = tiles_m * tiles_n * (128 + 256) * d * es
            print(f"round {r} {op:4s} candidate GEMM d={d} F={F} rows={rows}: {ms:.4f} ms  {flops / ms / 1e9:7.1f} TFLOP/s  "
                  f"L2->SM operands {l2_bytes / 1e9:.3f} GB = {l2_bytes / (ms * 1e-3) / 1e12:.2f} TB/s", flush=True)
    print(f"L2-resident read (24 MB buffer, 16-byte loads): {l2_read_tbs(args.reps):.2f} TB/s", flush=True)


if __name__ == "__main__":
    main()
