"""The fused SAE encoder's fp16 candidate GEMM (csrc/sae_fused.cu, k_enc_cand<C, __half>) and the fp16 operand copies it reads.

On one GPU with d_in % 8 == 0 and d_in >= 64, ``encoder="auto"`` runs the candidate GEMM on fp16 copies of sae_in and W_enc
(``eng.cand_operands == "f16"``): the same 11-bit significand as the tf32 read of the fp32 operands, half the bytes.  Checked here:

  * candidate keys on integer operands equal the model's bit for bit (fp16 holds them exactly);
  * the premise of the error bound: the copies round to nearest, and the tensor core multiplies fp16 subnormals exactly;
  * keys on Gaussian and worst-case-mantissa data stay within the fp16 accumulation term, ceil(d / 16) x 8 units of 2^-23;
  * a W_enc entry beyond the fp16 range is clamped (no Inf / NaN key) and its rows are still selected exactly;
  * the copy of W_enc is the fp16 rounding of W_enc after training steps and after load_state_dict, with its residual norm;
  * the fp16 and tf32 routes select the same top-k, values and counts bit for bit at the bench shape and at d_sae 49152.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle.fused_topk_model import SEG, candidate_values, encoder_norms, keys_of, ord2f

pytestmark = pytest.mark.gpu

SCALE = 2.0 ** -5
SENTINEL = 0x7FC0007F
F16_MAX = 65504.0


def f16_read(a: np.ndarray) -> np.ndarray:
    """What the fp16 candidate GEMM sees of an fp32 operand: round to nearest fp16, clamped to the finite range."""
    return np.clip(np.asarray(a, dtype=np.float32), -F16_MAX, F16_MAX).astype(np.float16).astype(np.float32)


def f16_trunc(a: np.ndarray) -> np.ndarray:
    """fp16 by truncation (13 low mantissa bits dropped, normal range only): what a truncating conversion would give."""
    return (np.asarray(a, dtype=np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def _f16_engine(x, W, b, k, c_keep=8, m_cand=None):
    """A fused-route engine on the fp16 candidate GEMM whose sae_in is x exactly (no normalisation, b_dec = 0).  Below d = 64
    (where "auto" keeps tf32) the fp16 operands are attached by hand: the kernels take any d % 8 == 0."""
    from vit_prisma.b200 import _lib as L
    from vit_prisma.b200.ops import _stream
    from vit_prisma.b200.sae_engine import SaeStepEngine
    F, d = W.shape
    W_dec = torch.zeros(F, d)
    W_dec[torch.arange(F), torch.arange(F) % d] = 1.0
    eng = SaeStepEngine(W.cuda(), W_dec.cuda(), b.cuda(), torch.zeros(d).cuda(), k=k, normalize_activations="none", c_keep=c_keep, m_cand=m_cand)
    if eng.cand_operands != "f16":
        assert d % 8 == 0 and eng.encoder == "fused"
        eng.cand_operands = "f16"
        eng.W_encT16 = torch.empty(F, d, dtype=torch.float16, device="cuda")
        eng.enc16_lo_max = torch.zeros(1, device="cuda")
        eng.refresh_lo()
    eng._ensure_rows(x.shape[0])
    eng.sae_in.copy_(x.cuda())
    L.check(L.get_lib().pb_f16_copy(eng.sae_in.data_ptr(), x.shape[0], d, eng.sae_in16.data_ptr(), None, _stream()), "pb_f16_copy")
    return eng


def _candidate_pass(eng, rows):
    from vit_prisma.b200 import _lib as L
    from vit_prisma.b200.ops import _stream
    n = rows * (eng.F // SEG) * eng.c_keep
    eng.cand = torch.full((n + 4096,), SENTINEL, dtype=torch.int32, device="cuda")
    L.check(L.get_lib().pb_sae_encode_topk_fused(C.byref(eng._enc_desc(rows, 1)), _stream()), "pb_sae_encode_topk_fused")
    got = eng.cand.cpu().numpy()
    assert np.all(got[:n] != SENTINEL), "candidate slots left unwritten"
    assert np.all(got[n:] == SENTINEL), "candidate buffer overrun"
    return got[:n].reshape(rows, eng.F // SEG, eng.c_keep)


def _int_case(rows, d, F, seed, lim=32):
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(-lim, lim + 1, (rows, d), generator=g).float() * SCALE
    W = torch.randint(-lim, lim + 1, (F, d), generator=g).float() * SCALE
    sign = torch.where(torch.rand(F, generator=g) < 0.5, -1.0, 1.0)
    b = torch.randint(1, lim + 1, (F,), generator=g).float() * sign * SCALE
    return x, W, b


def _gauss_case(rows, d, F, seed, worst_mantissa=False):
    g = torch.Generator().manual_seed(seed)
    W = torch.randn(F, d, generator=g) / math.sqrt(d)
    b = 0.01 * torch.randn(F, generator=g)
    x = torch.randn(rows, d, generator=g) * 2.0 + torch.randn(d, generator=g)
    if worst_mantissa:             # every mantissa bit fp16 drops is set: the largest residual the conversion can leave
        W = (W.view(torch.int32) | 0x1FFF).view(torch.float32)
        x = (x.view(torch.int32) | 0x1FFF).view(torch.float32)
    return x, W, b


@pytest.mark.parametrize("c_keep,rows,F,d", [
    (8, 300, 24576, 768),          # the bench shape
    (4, 127, 384, 104),            # odd segment count, a K tail of 40 that TMA zero-fills
    (6, 129, 640, 64),             # a partial second row tile
    (8, 129, 128, 768),
    (6, 300, 98304, 32),           # 768 segments, d below the "auto" threshold
])
def test_f16_candidate_keys_bit_exact_on_integer_data(c_keep, rows, F, d):
    x, W, b = _int_case(rows, d, F, seed=rows + F + d + c_keep)
    eng = _f16_engine(x, W, b, k=1, c_keep=c_keep)
    got = _candidate_pass(eng, rows)
    ref = keys_of(candidate_values(x.numpy(), W.numpy(), b.numpy(), read=f16_read), c_keep)
    bad = np.argwhere(got != ref)
    assert bad.size == 0, f"{len(bad)} keys differ from the model; first at (row, segment, slot) {tuple(bad[0])}"


def test_f16_operands_round_to_nearest_and_keep_subnormals():
    """One-hot tokens make every value a single product of two fp16 numbers, exact in fp32.  The fp32 operands have every bit
    that fp16 drops set, so rounding and truncation differ by ~2^-11 relative, far more than a key bucket (2^-16).  The second
    segment's W_enc rows are scaled into the fp16 subnormal range: a tensor core that flushed them would key them as zero."""
    rows, d, F = 64, 64, 256
    g = torch.Generator().manual_seed(7)
    W = (torch.randn(F, d, generator=g).view(torch.int32) | 0x1FFF).view(torch.float32)
    W[SEG:] *= 2.0 ** -20                                                # |w| ~ 1e-6: fp16 subnormals (below 6.1e-5)
    x = torch.diag((torch.randn(rows, generator=g).view(torch.int32) | 0x1FFF).view(torch.float32))
    b = torch.zeros(F)
    got = _candidate_pass(_f16_engine(x, W, b, k=1), rows)
    as_rn = keys_of(candidate_values(x.numpy(), W.numpy(), b.numpy(), read=f16_read), 8)
    flushed = W.numpy().copy()
    flushed[np.abs(flushed) < 2.0 ** -14] = 0.0
    as_trunc = keys_of(candidate_values(x.numpy(), W.numpy(), b.numpy(), read=f16_trunc), 8)
    as_ftz = keys_of(candidate_values(x.numpy(), flushed, b.numpy(), read=f16_read), 8)
    n_rn, n_trunc, n_ftz = int((got == as_rn).sum()), int((got == as_trunc).sum()), int((got[:, 1] == as_ftz[:, 1]).sum())
    print(f"fp16 operands: {n_rn} of {got.size} keys match round-to-nearest, {n_trunc} truncation; "
          f"subnormal segment: {n_ftz} of {got[:, 1].size} match a flush to zero")
    assert n_rn == got.size and n_trunc < got.size // 100 and n_ftz < got[:, 1].size // 100, (n_rn, n_trunc, n_ftz)


@pytest.mark.parametrize("rows,d,F,c_keep,worst", [(257, 768, 24576, 8, False), (300, 768, 4096, 8, True), (129, 104, 640, 6, True),
                                                   (300, 32, 4096, 4, True), (64, 1536, 8192, 8, True)])
def test_f16_keys_within_the_accumulation_bound(rows, d, F, c_keep, worst):
    """The tensor core accumulates the fp16 products in fp32 in an order of its own; k_cand_select allows ceil(d / 16) k16 steps
    of 8 units of 2^-23 of ||a|| max ||w|| for that (DESIGN section 4).  Every kept key must lie within it of its model value, and
    no dropped column may beat the last kept key by more."""
    x, W, b = _gauss_case(rows, d, F, seed=rows + d + F, worst_mantissa=worst)
    got = _candidate_pass(_f16_engine(x, W, b, k=1, c_keep=c_keep), rows).astype(np.int64)
    nseg = F // SEG
    assert np.all(np.diff(got, axis=2) < 0), "keys of a segment must be strictly descending"
    xn, Wn = x.numpy(), W.numpy()
    model = candidate_values(xn, Wn, b.numpy(), read=f16_read).astype(np.float64).reshape(rows, nseg, SEG)
    tol = (-(-d // 16) * 8 * 2.0 ** -23 * np.linalg.norm(xn.astype(np.float64), axis=1) * encoder_norms(Wn)[0])[:, None, None]
    lo = ord2f((got & ~127).astype(np.int32)).astype(np.float64)
    hi = ord2f((got | 127).astype(np.int32)).astype(np.float64)
    mv = np.take_along_axis(model, got & 127, axis=2)
    slack = tol + 2.0 ** -22 * np.abs(mv)
    off = np.maximum(lo - slack - mv, mv - hi - slack)
    err = np.maximum(lo - mv, mv - hi)
    print(f"d={d} worst={worst}: largest key distance from the model {err.max():.3e}, {float((err / tol).max()):.3f} of the allowance")
    assert off.max() <= 0, f"a kept key is {off.max():.3e} outside the accumulation bound at {np.unravel_index(off.argmax(), off.shape)}"
    kept = np.zeros(model.shape, dtype=bool)
    np.put_along_axis(kept, got & 127, True, axis=2)
    dropped_max = np.where(kept, -np.inf, model).max(axis=2)
    excess = dropped_max - (hi[:, :, -1] + tol[:, :, 0] + 2.0 ** -22 * np.abs(hi[:, :, -1]))
    assert excess.max() <= 0, f"a dropped column beats the last kept key by {excess.max():.3e} beyond the bound"


def test_f16_clamped_entry_still_selects_exactly():
    """A W_enc entry above 65504 is clamped in the fp16 copy: no Inf or NaN key, and the residual norm it leaves sends the rows to
    the exact path, which selects what the tf32 route selects."""
    from vit_prisma.b200.sae_engine import SaeStepEngine
    rows, d, F, k = 256, 128, 2048, 16
    x, W, b = _gauss_case(rows, d, F, seed=3)
    W[77, 5] = 1.0e5
    eng = _f16_engine(x, W, b, k=k)
    keys = _candidate_pass(eng, rows)
    assert np.isfinite(ord2f(keys & ~127)).all(), "a candidate key is not finite"
    assert eng.enc16_lo_max.item() > 3.0e4
    eng.feat_count.zero_()
    eng.encode_topk(x.cuda())                      # normalize "none", b_dec = 0: sae_in is x again
    ref = SaeStepEngine(W.cuda(), eng.W_dec.clone(), b.cuda(), torch.zeros(d).cuda(), k=k, normalize_activations="none", encoder="fused")
    assert ref.cand_operands == "tf32"
    ref.encode_topk(x.cuda())
    assert eng.fallback_rows() > 0
    assert torch.equal(eng.idx, ref.idx) and torch.equal(eng.val, ref.val) and torch.equal(eng.feat_count, ref.feat_count)


def _check_copy(eng, where):
    want = eng.W_encT.clamp(-F16_MAX, F16_MAX).half()
    assert torch.equal(eng.W_encT16.view(torch.int16), want.view(torch.int16)), f"{where}: W_encT16 is not fp16(W_encT)"
    lo = (eng.W_encT.double() - want.double()).norm(dim=1).max().item()
    got = eng.enc16_lo_max.item()
    assert abs(got - lo) <= 1e-5 * lo, f"{where}: enc16_lo_max {got} vs {lo}"


def test_f16_copy_follows_training_and_load_state_dict():
    from vit_prisma.sae.config import VisionModelSAERunnerConfig
    from vit_prisma.sae.sae import StandardSparseAutoencoder
    d, k, rows = 128, 8, 512
    cfg = VisionModelSAERunnerConfig(d_in=d, expansion_factor=16, activation_fn_str="topk", activation_fn_kwargs={"k": k}, _device="cuda",
                                     _dtype="float32", log_to_wandb=False, n_checkpoints=0, checkpoint_path="/tmp/unused")
    sae = StandardSparseAutoencoder(cfg)
    g = torch.Generator().manual_seed(1)
    x = (torch.randn(rows, d, generator=g) * 2.0 + torch.randn(d, generator=g)).cuda()
    sae(x)
    eng = sae.step_engine()
    assert eng.encoder == "fused" and eng.cand_operands == "f16"
    _check_copy(eng, "construction")
    for step in range(5):
        eng.train_step(x, lr=1e-3)
    torch.cuda.synchronize()
    _check_copy(eng, "after 5 training steps")
    state = {n: torch.randn_like(t) * 0.1 for n, t in sae.state_dict().items()}
    sae.load_state_dict(state)
    sae(x)
    assert sae.step_engine() is eng
    _check_copy(eng, "after load_state_dict")


@pytest.mark.parametrize("F", [24576, 49152])
def test_f16_and_tf32_routes_select_identically(F):
    """Same sae_in and parameters, both routes: idx, val and feat_count bit for bit (the values come from the same exact FFMA
    re-scoring either way), and the fp16 route sends no more rows to the exact path and re-scores no more candidates."""
    from vit_prisma.b200.sae_engine import SaeStepEngine
    from vit_prisma.b200.synthetic import sae_init_params
    d, k, rows = 768, 32, 4096
    p = sae_init_params(d, F, device="cuda")
    W_dec = p["W_dec"] / p["W_dec"].norm(dim=1, keepdim=True)
    g = torch.Generator().manual_seed(F)
    x = (torch.randn(rows, d, generator=g) * 2.0 + torch.randn(d, generator=g)).cuda()
    out = {}
    for encoder in ("auto", "fused"):
        eng = SaeStepEngine(p["W_encT"].clone(), W_dec.clone(), p["b_enc"].clone(), p["b_dec"].clone(), k=k, normalize_activations="layer_norm",
                            encoder=encoder)
        eng.encode_topk(x)
        out[eng.cand_operands] = (eng.idx.clone(), eng.val.clone(), eng.feat_count.clone(), eng.fallback_rows(), eng.rescored_per_row(rows))
    (i16, v16, c16, fb16, r16), (i32, v32, c32, fb32, r32) = out["f16"], out["tf32"]
    print(f"F={F}: exact-path rows fp16 {fb16} tf32 {fb32}; candidates re-scored per proven row fp16 {r16:.2f} tf32 {r32:.2f}")
    assert torch.equal(i16, i32) and torch.equal(v16, v32) and torch.equal(c16, c32)
    assert fb16 <= fb32 and r16 <= r32
