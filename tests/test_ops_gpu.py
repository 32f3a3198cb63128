"""Per-op parity of the C-ABI kernels against plain PyTorch fp32 on the same seeded inputs (GPU only)."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from tests.util import rel_err  # noqa: E402


def _ops():
    from vit_prisma.b200 import ops
    return ops


def _L():
    from vit_prisma.b200 import _lib
    return _lib


def _rand(*shape, seed=0, dtype=torch.float32, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype)


# ------------------------------------------------------------------ GEMM
@pytest.mark.parametrize("M,N,K", [(7, 5, 3), (130, 72, 40), (257, 768, 768), (100, 33, 130), (1, 10, 8)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_gemm_simt_epilogues(M, N, K, dtype):
    ops, L = _ops(), _L()
    a, w, b, r = _rand(M, K, seed=1, dtype=dtype), _rand(N, K, seed=2, dtype=dtype, scale=K ** -0.5), _rand(N, seed=3, dtype=dtype), _rand(M, N, seed=4, dtype=dtype)
    ref = a.float() @ w.float().t() + b.float()
    tol = 2e-6 if dtype == torch.float32 else 1e-2
    pre, post = ops.gemm(a.cuda(), w.cuda(), b.cuda(), act="gelu", want_post=True, impl=L.GEMM_SIMT)
    assert rel_err(pre.float(), ref) < tol
    assert rel_err(post.float(), F.gelu(ref)) < tol
    pre, post = ops.gemm(a.cuda(), w.cuda(), b.cuda(), residual=r.cuda(), impl=L.GEMM_SIMT)
    assert rel_err(post.float(), ref + r.float()) < tol


def test_gemm_simt_strided_views():
    """Per-head slices of [B,T,H,d] as A and as output (split-qkv hooked path)."""
    ops, L = _ops(), _L()
    B, T, H, d, dh = 2, 5, 3, 16, 8
    x = _rand(B, T, H, d, seed=5).cuda()
    w = _rand(H * dh, d, seed=6).cuda()
    out = torch.zeros(B, T, H, dh, device="cuda")
    for h in range(H):
        ops.gemm(x[:, :, h, :], w[h * dh:(h + 1) * dh], None, out0=out[:, :, h, :], impl=L.GEMM_SIMT)
    ref = torch.einsum("bthd,hed->bthe", x.cpu(), w.cpu().view(H, dh, d))
    assert rel_err(out, ref) < 2e-6


TC_SHAPES = [(128, 128, 64), (256, 128, 128), (300, 256, 192), (1000, 768, 768), (512, 2304, 768), (200, 768, 3072), (128, 512, 768),
             (260, 384, 128), (5000, 3072, 768), (70, 64, 64)]


@pytest.mark.parametrize("M,N,K", TC_SHAPES)
def test_gemm_tc_bf16_matches_simt(M, N, K):
    ops, L = _ops(), _L()
    dt = torch.bfloat16
    a, w, b = _rand(M, K, seed=1, dtype=dt).cuda(), _rand(N, K, seed=2, dtype=dt, scale=K ** -0.5).cuda(), _rand(N, seed=3, dtype=dt).cuda()
    pre_s, post_s = ops.gemm(a, w, b, act="gelu", want_post=True, impl=L.GEMM_SIMT)
    pre_t, post_t = ops.gemm(a, w, b, act="gelu", want_post=True, impl=L.GEMM_TC)
    torch.cuda.synchronize()
    ref = a.float().cpu() @ w.float().cpu().t() + b.float().cpu()
    assert rel_err(pre_t.float(), ref) < 1e-2, "wgmma bf16 vs fp32 reference"
    assert rel_err(pre_t.float(), pre_s.float()) < 8e-3, "wgmma bf16 vs FFMA on the same bf16 inputs"
    assert rel_err(post_t.float(), post_s.float()) < 8e-3


@pytest.mark.parametrize("M,N,K", TC_SHAPES)
def test_gemm_tc_3xtf32_matches_fp32(M, N, K):
    ops, L = _ops(), _L()
    a, w, b, r = _rand(M, K, seed=1).cuda(), _rand(N, K, seed=2, scale=K ** -0.5).cuda(), _rand(N, seed=3).cuda(), _rand(M, N, seed=4).cuda()
    a_lo, w_lo = ops.split_tf32(a), ops.split_tf32(w)
    pre_t, post_t = ops.gemm(a, w, b, residual=r, a_lo=a_lo, w_lo=w_lo, impl=L.GEMM_TC)
    torch.cuda.synchronize()
    ref = (a.double().cpu() @ w.double().cpu().t() + b.double().cpu()).float()
    e = rel_err(pre_t, ref)
    assert e < 3e-5, f"3xTF32 rel err {e:.2e} (single-pass TF32 would be ~1e-3; fp32 accumulation noise grows with sqrt(K))"
    assert rel_err(post_t, ref + r.cpu()) < 3e-5


def test_gemm_tc_3xtf32_m_fast_raster():
    """Dictionary-sized B (> 24 MB with its lo plane) flips the persistent kernel to the m-fastest tile walk (SAE encoder shape)."""
    ops, L = _ops(), _L()
    M, N, K = 520, 24576, 768
    a, w, b = _rand(M, K, seed=1).cuda(), _rand(N, K, seed=2, scale=K ** -0.5).cuda(), _rand(N, seed=3).cuda()
    pre_t, _ = ops.gemm(a, w, b, a_lo=ops.split_tf32(a), w_lo=ops.split_tf32(w), impl=L.GEMM_TC)
    ref = torch.addmm(b.double(), a.double(), w.double().t()).float()
    assert rel_err(pre_t, ref) < 3e-5


def test_gemm_split_outputs_qkv():
    ops, L = _ops(), _L()
    import ctypes as C
    M, d, HD = 150, 64, 48
    a, w, b = _rand(M, d, seed=1).cuda(), _rand(3 * HD, d, seed=2).cuda(), _rand(3 * HD, seed=3).cuda()
    outs = [torch.empty(M, HD, device="cuda") for _ in range(3)]
    g = L.PbGemm()
    g.M, g.N, g.K, g.dtype, g.impl = M, 3 * HD, d, L.PB_F32, L.GEMM_SIMT
    g.A, g.lda, g.B, g.ldb, g.bias = a.data_ptr(), d, w.data_ptr(), d, b.data_ptr()
    g.n_split, g.split_n, g.ld0 = 3, HD, HD
    for i in range(3):
        g.out_split[i] = outs[i].data_ptr()
    ops.gemm_raw(g)
    ref = a.cpu() @ w.cpu().t() + b.cpu()
    for i in range(3):
        assert rel_err(outs[i], ref[:, i * HD:(i + 1) * HD]) < 2e-6


# ------------------------------------------------------------- LayerNorm
@pytest.mark.parametrize("rows,cols", [(10, 8), (50, 768), (33, 1024), (7, 3072), (5, 30)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_layernorm(rows, cols, dtype):
    ops = _ops()
    x, w, b = _rand(rows, cols, seed=1, dtype=dtype, scale=3.0), (1 + 0.1 * _rand(cols, seed=2)).to(dtype), _rand(cols, seed=3, dtype=dtype)
    xf = x.float()
    xc = xf - xf.mean(-1, keepdim=True)
    scale_ref = (xc.pow(2).mean(-1, keepdim=True) + 1e-5).sqrt()
    norm_ref = xc / scale_ref * w + b     # fp32 (type promotion), as hooked in the reference
    scale, normalized, out = ops.layernorm(x.cuda(), w.cuda(), b.cuda(), 1e-5, dtype)
    assert rel_err(scale, scale_ref) < 1e-6
    assert normalized.dtype == torch.float32 and rel_err(normalized, norm_ref) < 2e-6
    assert out.dtype == dtype and rel_err(out.float(), norm_ref.to(dtype).float()) < (2e-6 if dtype == torch.float32 else 8e-3)
    # LayerNormPre (no affine) and an externally supplied scale
    _, n2, _ = ops.layernorm(x.cuda(), None, None, 1e-5, dtype)
    assert rel_err(n2, xc / scale_ref) < 2e-6
    _, n3, _ = ops.layernorm(x.cuda(), w.cuda(), b.cuda(), 1e-5, dtype, scale_in=torch.full((rows, 1), 2.0, device="cuda"))
    assert rel_err(n3, xc / 2.0 * w + b) < 2e-6


# -------------------------------------------------------------- attention
def _offset_by_one(t):
    """The same values in a contiguous view one element into its storage: not 16-byte aligned."""
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    buf[1:] = t.reshape(-1)
    return buf[1:].view(t.shape)


# d_head 64: T <= 128 whole-row tensor-core kernel, T > 128 the 64-key-chunk one; unaligned q/k/v and other d_head: FFMA kernel
@pytest.mark.parametrize("B,T,H,dh,unaligned", [(2, 5, 4, 8, False), (3, 50, 12, 64, False), (1, 197, 2, 64, False), (1, 257, 2, 64, False),
                                                (2, 17, 2, 24, False), (2, 64, 3, 64, False), (2, 65, 3, 64, False), (2, 128, 3, 64, False),
                                                (2, 129, 3, 64, False), (2, 50, 3, 64, True)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_attention_fused_and_split(B, T, H, dh, unaligned, dtype):
    ops = _ops()
    q, k, v = (_rand(B, T, H, dh, seed=s, dtype=dtype) for s in (1, 2, 3))
    scale = math.sqrt(dh)
    sc_ref = (torch.einsum("bqhe,bkhe->bhqk", q.float(), k.float()) / scale).to(dtype)
    pt_ref = F.softmax(sc_ref.float(), dim=-1).to(dtype)
    z_ref = torch.einsum("bkhe,bhqk->bqhe", v.float(), pt_ref.float()).to(dtype)
    tol = 1e-5 if dtype == torch.float32 else 1.2e-2   # fp32: 3xTF32 products (d_head 64) / FFMA, fp32 accumulation
    if unaligned:
        q, k, v = (_offset_by_one(x.cuda()) for x in (q, k, v))
        assert all(x.data_ptr() % 16 for x in (q, k, v))
    else:
        q, k, v = q.cuda(), k.cuda(), v.cuda()
    sc, pt, z = ops.attention(q, k, v, scale)
    assert rel_err(sc.float(), sc_ref.float()) < tol
    assert rel_err(pt.float(), pt_ref.float()) < tol
    assert rel_err(z.float(), z_ref.float()) < tol
    # not materialising scores / pattern must not change z
    _, _, z2 = ops.attention(q, k, v, scale, want_scores=False, want_pattern=False)
    assert torch.equal(z2, z)
    # split route used by the hooked path
    sc3 = ops.attn_scores(q, k, scale)
    pt3 = ops.softmax_rows(sc3)
    z3 = ops.attn_pv(pt3, v)
    if unaligned or dh != 64:   # the fused call took the FFMA kernel too: the same scores bit for bit
        assert torch.equal(sc3, sc)
    # (d_head == 64 runs the mma.sync kernel when fused and the FFMA kernel when split: close, not bit-equal)
    assert rel_err(sc3.float(), sc.float()) < tol
    assert rel_err(pt3.float(), pt.float()) < tol and rel_err(z3.float(), z.float()) < tol


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_attention_scale_not_power_of_two(dtype):
    """d_head 64 with attn_scale 7.3: the tensor-core kernel must take its true-division branch (scores = dot / scale)."""
    ops = _ops()
    q, k, v = (_rand(2, 50, 3, 64, seed=s, dtype=dtype) for s in (4, 5, 6))
    sc_ref = (torch.einsum("bqhe,bkhe->bhqk", q.float(), k.float()).to(dtype).float() / 7.3).to(dtype)
    pt_ref = F.softmax(sc_ref.float(), dim=-1).to(dtype)
    sc, pt, _ = ops.attention(q.cuda(), k.cuda(), v.cuda(), 7.3)
    tol = 1e-5 if dtype == torch.float32 else 1.2e-2
    assert rel_err(sc.float(), sc_ref.float()) < tol and rel_err(pt.float(), pt_ref.float()) < tol


def test_softmax_nan_to_zero():
    ops = _ops()
    x = torch.zeros(2, 4, device="cuda")
    x[0, :] = float("-inf")          # all -inf row -> NaN in F.softmax -> 0 after torch.where (attention.py:149)
    y = ops.softmax_rows(x)
    assert torch.equal(y[0].cpu(), torch.zeros(4))
    assert rel_err(y[1], torch.full((4,), 0.25)) < 1e-6


# ------------------------------------------------------------ elementwise
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_elementwise(dtype):
    ops = _ops()
    a, b = _rand(3, 37, seed=1, dtype=dtype), _rand(3, 37, seed=2, dtype=dtype)
    tol = 1e-6 if dtype == torch.float32 else 8e-3
    assert rel_err(ops.add(a.cuda(), b.cuda()).float(), (a.float() + b.float())) < tol
    assert rel_err(ops.mul(a.cuda(), b.cuda()).float(), (a.float() * b.float())) < tol
    refs = {"relu": F.relu, "gelu": F.gelu, "silu": F.silu, "quick_gelu": lambda t: t * torch.sigmoid(1.702 * t),
            "gelu_new": lambda t: 0.5 * t * (1 + torch.tanh(math.sqrt(2 / math.pi) * (t + 0.044715 * t ** 3))),
            "gelu_fast": lambda t: 0.5 * t * (1 + torch.tanh(t * 0.7978845608 * (1 + 0.044715 * t * t)))}
    for name, fn in refs.items():
        assert rel_err(ops.activation(a.cuda(), name).float(), fn(a.float())) < max(tol, 2e-6), name
    assert rel_err(ops.l2_normalize_rows(a.cuda()).float(), F.normalize(a.float(), dim=-1)) < max(tol, 2e-6)
    x3 = _rand(2, 6, 8, seed=3, dtype=dtype)
    assert rel_err(ops.mean_tokens(x3.cuda()).float(), x3.float().mean(1)) < max(tol, 2e-6)


def test_im2col_matches_conv():
    ops, L = _ops(), _L()
    B, Cc, S, P, d = 2, 3, 32, 8, 16
    x, w, b = _rand(B, Cc, S, S, seed=1), _rand(d, Cc, P, P, seed=2, scale=0.1), _rand(d, seed=3)
    ref = F.conv2d(x, w, b, stride=P).flatten(2).transpose(1, 2)
    patches = ops.im2col_patches(x.cuda(), P)
    out, _ = ops.gemm(patches, w.cuda().reshape(d, -1), b.cuda(), impl=L.GEMM_SIMT)
    assert rel_err(out.view(B, -1, d), ref) < 3e-6


def test_cpu_tensor_is_refused():
    from vit_prisma.b200._lib import PrismaB200Error
    with pytest.raises(PrismaB200Error):
        _ops().add(torch.ones(4), torch.ones(4))
