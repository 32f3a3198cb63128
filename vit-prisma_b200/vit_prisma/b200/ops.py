"""One Python function per C-ABI op: tensor checks, output allocation, launch on the current stream.

PyTorch's role here is memory ownership (``torch.empty``), the stream handle and views; every
arithmetic result comes out of libprisma_b200.  All functions require CUDA tensors and raise
``PrismaB200Error`` otherwise (no CPU path).
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import torch

from . import _lib as L

_DT = {torch.float32: L.PB_F32, torch.bfloat16: L.PB_BF16}


def dtype_code(dtype: torch.dtype) -> int:
    try:
        return _DT[dtype]
    except KeyError:
        raise L.PrismaB200Error(f"unsupported dtype {dtype}: the H100 path computes in float32 or bfloat16") from None


def _need_cuda(*tensors) -> None:
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise L.PrismaB200Error(
                "prisma_b200 ops need CUDA tensors: the hot path is hand-written sm_90a CUDA and has no CPU fallback "
                f"(got a tensor on {t.device})")


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _rows2d(t: torch.Tensor):
    """View [..., K] as (tensor, rows, K, row_stride) without copying when the leading dims nest
    onto a single row stride (contiguous tensors, 2-D row slices, per-head slices [B,T,K] of [B,T,H,K])."""
    if t.stride(-1) != 1:
        t = t.contiguous()
    k = t.shape[-1]
    if t.dim() == 1:
        return t, 1, k, k
    ld = t.stride(-2)
    ok = ld >= k
    expect = ld * t.shape[-2]
    for size, stride in zip(reversed(t.shape[:-2]), reversed(t.stride()[:-2])):
        if size != 1 and stride != expect:
            ok = False
            break
        expect *= size
    if not ok:
        t = t.contiguous()
        ld = k
    return t, t.numel() // k, k, ld


def _out_ld(t: torch.Tensor, n: int) -> int:
    """Row stride of an output buffer; caller-provided strided views (e.g. one head of [B,T,H,dh]) must nest."""
    t2, _rows, k, ld = _rows2d(t)
    if t2.data_ptr() != t.data_ptr() or k != n:
        raise L.PrismaB200Error("output view must be [..., N] with unit inner stride and nesting leading dims")
    return ld


# --------------------------------------------------------------------------- GEMM
def gemm(a: torch.Tensor, w_nk: torch.Tensor, bias: Optional[torch.Tensor] = None, *,
         act: Optional[str] = None, residual: Optional[torch.Tensor] = None,
         want_pre: bool = True, want_post: bool = False,
         a_lo: Optional[torch.Tensor] = None, w_lo: Optional[torch.Tensor] = None,
         out0: Optional[torch.Tensor] = None, out1: Optional[torch.Tensor] = None,
         impl: int = L.GEMM_AUTO):
    """``pre = a @ w_nk.T + bias``; ``post = act(pre)`` or ``residual + pre``.

    a: [..., K]; w_nk: [N, K] (K-major pack). Returns (pre | None, post | None), each [..., N].
    """
    _need_cuda(a, w_nk, bias, residual)
    a2, M, K, lda = _rows2d(a)
    N = w_nk.shape[0]
    assert w_nk.shape[1] == K and w_nk.stride(1) == 1, "w_nk must be [N, K] with unit K stride"
    dt = dtype_code(a.dtype)
    out_shape = (*a.shape[:-1], N)
    g = L.PbGemm()
    g.M, g.N, g.K, g.dtype, g.act, g.impl = M, N, K, dt, L.ACT[act], impl
    g.A, g.lda, g.B, g.ldb = a2.data_ptr(), lda, w_nk.data_ptr(), w_nk.stride(0)
    if a_lo is not None and w_lo is not None:
        g.A_lo, g.B_lo = a_lo.data_ptr(), w_lo.data_ptr()
    g.bias = _ptr(bias)
    pre = post = None
    if want_pre or out0 is not None:
        pre = out0 if out0 is not None else torch.empty(out_shape, dtype=a.dtype, device=a.device)
        g.out0, g.ld0 = pre.data_ptr(), _out_ld(pre, N)
    if want_post or residual is not None or out1 is not None:
        post = out1 if out1 is not None else torch.empty(out_shape, dtype=a.dtype, device=a.device)
        g.out1, g.ld1 = post.data_ptr(), _out_ld(post, N)
    res2 = None
    if residual is not None:
        res2, rM, rN, ldr = _rows2d(residual)
        assert rM == M and rN == N
        g.residual, g.ldr = res2.data_ptr(), ldr
    L.check(L.get_lib().pb_gemm(C.byref(g), _stream()), "pb_gemm")
    return pre, post


def gemm_raw(g: "L.PbGemm") -> None:
    L.check(L.get_lib().pb_gemm(C.byref(g), _stream()), "pb_gemm")


def split_tf32(x: torch.Tensor) -> torch.Tensor:
    _need_cuda(x)
    assert x.dtype == torch.float32
    x = x.contiguous()
    lo = torch.empty_like(x)
    L.check(L.get_lib().pb_split_tf32(x.data_ptr(), lo.data_ptr(), x.numel(), _stream()), "pb_split_tf32")
    return lo


# ---------------------------------------------------------------------- LayerNorm
def layernorm_scale(x: torch.Tensor, eps: float) -> torch.Tensor:
    """Only ``sqrt(mean((x - mean)^2) + eps)`` -> fp32 [..., 1] (first half of the hooked two-step LayerNorm)."""
    _need_cuda(x)
    x = x.contiguous()
    cols = x.shape[-1]
    p = L.PbLayerNorm()
    p.rows, p.cols, p.dtype_in, p.dtype_out, p.eps = x.numel() // cols, cols, dtype_code(x.dtype), dtype_code(x.dtype), eps
    scale = torch.empty((*x.shape[:-1], 1), dtype=torch.float32, device=x.device)
    p.x, p.scale = x.data_ptr(), scale.data_ptr()
    L.check(L.get_lib().pb_layernorm(C.byref(p), _stream()), "pb_layernorm")
    return scale


def layernorm(x: torch.Tensor, w: Optional[torch.Tensor], b: Optional[torch.Tensor], eps: float,
              out_dtype: torch.dtype, want_scale: bool = True, scale_in: Optional[torch.Tensor] = None):
    """Returns (scale fp32 [...,1], hook_normalized, out).

    ``hook_normalized`` is what the reference's hook sees: the fp32 result when the model dtype is
    not fp32 (layer_norm.py:93 casts *after* the hook), else the same tensor as ``out``.
    """
    _need_cuda(x, w, b)
    x = x.contiguous()
    cols = x.shape[-1]
    rows = x.numel() // cols
    p = L.PbLayerNorm()
    p.rows, p.cols, p.dtype_in, p.dtype_out, p.eps = rows, cols, dtype_code(x.dtype), dtype_code(out_dtype), eps
    p.x, p.w, p.b = x.data_ptr(), _ptr(w), _ptr(b)
    scale = torch.empty((*x.shape[:-1], 1), dtype=torch.float32, device=x.device) if want_scale else None
    out = torch.empty(x.shape, dtype=out_dtype, device=x.device)
    p.scale, p.out = _ptr(scale), out.data_ptr()
    if scale_in is not None:
        _need_cuda(scale_in)
        scale_in = scale_in.to(torch.float32).expand(*x.shape[:-1], 1).contiguous()
        p.scale_in = scale_in.data_ptr()
    normalized = out
    if out_dtype != torch.float32:
        normalized = torch.empty(x.shape, dtype=torch.float32, device=x.device)
        p.norm_f32 = normalized.data_ptr()
    L.check(L.get_lib().pb_layernorm(C.byref(p), _stream()), "pb_layernorm")
    return scale, normalized, out


# ---------------------------------------------------------------------- attention
def _att_desc(q, k, v, attn_scale):
    B, T, H, dh = (q if q is not None else v).shape
    p = L.PbAttention()
    ref = q if q is not None else v
    p.B, p.T, p.H, p.dh, p.dtype, p.attn_scale = B, T, H, dh, dtype_code(ref.dtype), float(attn_scale)
    return p, (B, T, H, dh)


def attn_scores(q: torch.Tensor, k: torch.Tensor, attn_scale: float) -> torch.Tensor:
    _need_cuda(q, k)
    q, k = q.contiguous(), k.contiguous()
    p, (B, T, H, dh) = _att_desc(q, k, None, attn_scale)
    scores = torch.empty((B, H, T, T), dtype=q.dtype, device=q.device)
    p.q, p.k, p.scores = q.data_ptr(), k.data_ptr(), scores.data_ptr()
    L.check(L.get_lib().pb_attn_scores(C.byref(p), _stream()), "pb_attn_scores")
    return scores


def softmax_rows(x: torch.Tensor) -> torch.Tensor:
    _need_cuda(x)
    x = x.contiguous()
    y = torch.empty_like(x)
    cols = x.shape[-1]
    L.check(L.get_lib().pb_softmax_rows(x.data_ptr(), y.data_ptr(), x.numel() // cols, cols, dtype_code(x.dtype), _stream()),
            "pb_softmax_rows")
    return y


def attn_pv(pattern: torch.Tensor, v: torch.Tensor) -> torch.Tensor:
    _need_cuda(pattern, v)
    pattern, v = pattern.contiguous(), v.contiguous()
    p, (B, T, H, dh) = _att_desc(None, None, v, 1.0)
    z = torch.empty((B, T, H, dh), dtype=v.dtype, device=v.device)
    p.pattern, p.v, p.z = pattern.data_ptr(), v.data_ptr(), z.data_ptr()
    L.check(L.get_lib().pb_attn_pv(C.byref(p), _stream()), "pb_attn_pv")
    return z


def attention(q, k, v, attn_scale: float, want_scores: bool = True, want_pattern: bool = True, causal: bool = False):
    """Fused scores -> softmax -> PV; ``causal`` scores key j > query i as -inf (the text towers' additive mask)."""
    _need_cuda(q, k, v)
    q, k, v = q.contiguous(), k.contiguous(), v.contiguous()
    p, (B, T, H, dh) = _att_desc(q, k, v, attn_scale)
    p.causal = int(causal)
    scores = torch.empty((B, H, T, T), dtype=q.dtype, device=q.device) if want_scores else None
    pattern = torch.empty((B, H, T, T), dtype=q.dtype, device=q.device) if want_pattern else None
    z = torch.empty((B, T, H, dh), dtype=q.dtype, device=q.device)
    p.q, p.k, p.v = q.data_ptr(), k.data_ptr(), v.data_ptr()
    p.scores, p.pattern, p.z = _ptr(scores), _ptr(pattern), z.data_ptr()
    L.check(L.get_lib().pb_attention(C.byref(p), _stream()), "pb_attention")
    return scores, pattern, z


# -------------------------------------------------------------------- elementwise
def _binary(fn_name: str, a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    _need_cuda(a, b)
    if a.shape != b.shape:
        a, b = torch.broadcast_tensors(a, b)
    a, b = a.contiguous(), b.contiguous()
    out = torch.empty_like(a)
    fn = getattr(L.get_lib(), fn_name)
    L.check(fn(a.data_ptr(), b.data_ptr(), out.data_ptr(), a.numel(), dtype_code(a.dtype), _stream()), fn_name)
    return out


def add(a, b):
    return _binary("pb_add", a, b)


def mul(a, b):
    return _binary("pb_mul", a, b)


def activation(x: torch.Tensor, act: str) -> torch.Tensor:
    _need_cuda(x)
    x = x.contiguous()
    y = torch.empty_like(x)
    L.check(L.get_lib().pb_activation(x.data_ptr(), y.data_ptr(), x.numel(), L.ACT[act], dtype_code(x.dtype), _stream()),
            "pb_activation")
    return y


def l2_normalize_rows(x: torch.Tensor, eps: float = 1e-12) -> torch.Tensor:
    _need_cuda(x)
    x = x.contiguous()
    out = torch.empty_like(x)
    cols = x.shape[-1]
    L.check(L.get_lib().pb_l2_normalize_rows(x.data_ptr(), out.data_ptr(), x.numel() // cols, cols, eps, dtype_code(x.dtype),
                                             _stream()), "pb_l2_normalize_rows")
    return out


def mean_tokens(x: torch.Tensor) -> torch.Tensor:
    _need_cuda(x)
    x = x.contiguous()
    B, T, d = x.shape
    out = torch.empty((B, d), dtype=x.dtype, device=x.device)
    L.check(L.get_lib().pb_mean_tokens(x.data_ptr(), out.data_ptr(), B, T, d, dtype_code(x.dtype), _stream()), "pb_mean_tokens")
    return out


def im2col_patches(images: torch.Tensor, patch: int) -> torch.Tensor:
    _need_cuda(images)
    images = images.contiguous()
    B, Cc, S, S2 = images.shape
    assert S == S2, "square images only"
    g = S // patch
    out = torch.empty((B * g * g, Cc * patch * patch), dtype=images.dtype, device=images.device)
    L.check(L.get_lib().pb_im2col_patches(images.data_ptr(), out.data_ptr(), B, Cc, S, patch, dtype_code(images.dtype), _stream()),
            "pb_im2col_patches")
    return out


def im2col_tubelets(videos: torch.Tensor, patch: int, depth: int) -> torch.Tensor:
    """[B, C, F, S, S] -> [B * (F // depth) * (S // patch)^2, C * depth * patch^2], tokens ordered (t, h, w) with t slowest;
    frames past (F // depth) * depth are dropped, as ``Conv3d`` with stride ``depth`` drops them."""
    _need_cuda(videos)
    videos = videos.contiguous()
    B, Cc, F, S, S2 = videos.shape
    assert S == S2, "square frames only"
    g, nt = S // patch, F // depth
    out = torch.empty((B * nt * g * g, Cc * depth * patch * patch), dtype=videos.dtype, device=videos.device)
    L.check(L.get_lib().pb_im2col_tubelets(videos.data_ptr(), out.data_ptr(), B, Cc, F, S, patch, depth, dtype_code(videos.dtype),
                                           _stream()), "pb_im2col_tubelets")
    return out


def embed_tokens(ids: torch.Tensor, W_E: torch.Tensor, pos: torch.Tensor):
    """ids int64 [B,T] -> (hook_embed = W_E[ids], full = embed + pos[:T]), both [B,T,d] in W_E's dtype.  Ids must lie in
    [0, vocab): the kernel never reads outside W_E, and fills rows of out-of-range ids with NaN."""
    _need_cuda(ids, W_E, pos)
    assert ids.dtype == torch.int64 and ids.dim() == 2 and pos.dtype == W_E.dtype and pos.shape[0] >= ids.shape[1]
    ids, W_E, pos = ids.contiguous(), W_E.contiguous(), pos.contiguous()
    B, T = ids.shape
    vocab, d = W_E.shape
    embed = torch.empty((B, T, d), dtype=W_E.dtype, device=W_E.device)
    full = torch.empty_like(embed)
    L.check(L.get_lib().pb_embed_tokens(ids.data_ptr(), W_E.data_ptr(), pos.data_ptr(), embed.data_ptr(), full.data_ptr(), B, T, d,
                                        vocab, dtype_code(W_E.dtype), _stream()), "pb_embed_tokens")
    return embed, full


def gather_argmax_rows(ids: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    """``x[arange(B), ids.argmax(-1)]`` for ids int64 [B,T] and x [B,T,d] (first maximal index on ties)."""
    _need_cuda(ids, x)
    assert ids.dtype == torch.int64 and ids.shape == x.shape[:2]
    ids, x = ids.contiguous(), x.contiguous()
    B, T, d = x.shape
    out = torch.empty((B, d), dtype=x.dtype, device=x.device)
    L.check(L.get_lib().pb_gather_argmax_rows(ids.data_ptr(), x.data_ptr(), out.data_ptr(), B, T, d, dtype_code(x.dtype), _stream()),
            "pb_gather_argmax_rows")
    return out


def cast(x: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    _need_cuda(x)
    if x.dtype == dtype:
        return x
    x = x.contiguous()
    y = torch.empty(x.shape, dtype=dtype, device=x.device)
    L.check(L.get_lib().pb_cast(x.data_ptr(), dtype_code(x.dtype), y.data_ptr(), dtype_code(dtype), x.numel(), _stream()), "pb_cast")
    return y


def cast_into(x: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """``out[...] = x`` rounded to ``out.dtype`` (both contiguous, same element count) -- the export of fp32 master
    parameters into a reduced-precision module's storage."""
    _need_cuda(x)
    _need_cuda(out)
    assert x.is_contiguous() and out.is_contiguous() and x.numel() == out.numel(), "cast_into: contiguous tensors of equal size"
    L.check(L.get_lib().pb_cast(x.data_ptr(), dtype_code(x.dtype), out.data_ptr(), dtype_code(out.dtype), x.numel(), _stream()), "pb_cast")
    return out
