"""The fused SAE encoder (csrc/sae_fused.cu) one phase at a time, against the numpy model of oracle/fused_topk_model.py.

The end-to-end tests (test_sae_gpu.py, test_sae_fused_tiles_gpu.py, test_parity_full_gpu.py) see only the final top-k, which
a wrong candidate key rarely changes: a dropped 5th key of a segment matters only when a true winner sits there, and the
completeness proof trusts the kept lists.  Here each phase is driven alone through ``pb_sae_encode_topk_fused``'s phase mask:

  * candidate GEMM (phase 1) on integer operands, where the tensor core's result does not depend on rounding or accumulation
    order: every key of every (token, segment) must equal the model's bit for bit, every slot must be written, and nothing past
    the end of the buffer;
  * candidate GEMM on Gaussian and worst-case-mantissa operands: the kept keys are within the accumulation bound of the tf32
    product, and no dropped column beats the last kept key by more than that (the property the completeness proof uses), plus
    the premise of the bound, that the tensor core truncates its fp32 operands to tf32;
  * selection + exact path (phases 2 | 4) on keys from the model: the top-k equals a stable float64 sort bit for bit, and every
    row's proven / exact-path decision and the number of candidates re-scored equal the model's.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle.fused_topk_model import (SEG, candidate_keys_batch, candidate_values, encoder_norms, keys_of, ord2f, select_rows, tf32_round,
                                     tf32_trunc)

pytestmark = pytest.mark.gpu

SCALE = 2.0 ** -5                  # integer operands times a power of two: exact in tf32, their products and sums exact in fp32
SENTINEL = 0x7FC0007F              # the key of a positive NaN: no finite value has it
GUARD = 4096                       # sentinel slots past the end of the candidate buffer


def _int_case(rows, d, F, seed, lim=32, negative_segments=False):
    """x, W_encT integers in [-lim, lim] times SCALE, b_enc a non-zero integer times SCALE (so that no sum is a tensor-core -0).
    ``negative_segments``: every other segment's bias is shifted down by 2^17 units, so that all its values, and the keys it
    keeps, are negative (the other branch of f2ord)."""
    shift = 2 ** 12 if negative_segments else 0                         # in units of SCALE: 2^17 units of SCALE^2
    assert d * lim * lim + (shift + lim) / SCALE < 2 ** 24, "every partial sum must be an integer below 2^24 units"
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(-lim, lim + 1, (rows, d), generator=g).float() * SCALE
    W = torch.randint(-lim, lim + 1, (F, d), generator=g).float() * SCALE
    sign = torch.where(torch.rand(F, generator=g) < 0.5, -1.0, 1.0)
    b = torch.randint(1, lim + 1, (F,), generator=g).float() * sign
    b -= shift * ((torch.arange(F) // SEG) % 2)
    return x, W, b * SCALE


def _gauss_case(rows, d, F, seed, worst_mantissa=False):
    g = torch.Generator().manual_seed(seed)
    W = torch.randn(F, d, generator=g) / math.sqrt(d)
    b = 0.01 * torch.randn(F, generator=g)
    x = torch.randn(rows, d, generator=g) * 2.0 + torch.randn(d, generator=g)
    if worst_mantissa:             # every truncated mantissa bit set: the largest residual a tf32 read can leave
        W = (W.view(torch.int32) | 0x1FFF).view(torch.float32)
        x = (x.view(torch.int32) | 0x1FFF).view(torch.float32)
    return x, W, b


def _engine(x, W, b, k, c_keep=8, m_cand=None):
    """A fused-route engine whose sae_in is x exactly (no normalisation, b_dec = 0)."""
    from vit_prisma.b200.sae_engine import SaeStepEngine
    F, d = W.shape
    W_dec = torch.zeros(F, d)
    W_dec[torch.arange(F), torch.arange(F) % d] = 1.0
    eng = SaeStepEngine(W.cuda(), W_dec.cuda(), b.cuda(), torch.zeros(d).cuda(), k=k, normalize_activations="none", encoder="fused",
                        c_keep=c_keep, m_cand=m_cand)
    eng._ensure_rows(x.shape[0])
    eng.sae_in.copy_(x.cuda())
    return eng


def _phases(eng, rows, phases):
    from vit_prisma.b200 import _lib as L
    from vit_prisma.b200.ops import _stream
    L.check(L.get_lib().pb_sae_encode_topk_fused(C.byref(eng._enc_desc(rows, phases)), _stream()), "pb_sae_encode_topk_fused")
    torch.cuda.synchronize()


def _candidate_pass(eng, rows):
    """Phase 1 alone into a sentinel-filled buffer with a guard tail; returns the keys [rows, nseg, c_keep] after checking that
    every slot was written and the guard was not."""
    n = rows * (eng.F // SEG) * eng.c_keep
    eng.cand = torch.full((n + GUARD,), SENTINEL, dtype=torch.int32, device="cuda")
    _phases(eng, rows, 1)
    got = eng.cand.cpu().numpy()
    unwritten = np.flatnonzero(got[:n] == SENTINEL)
    assert unwritten.size == 0, (f"{unwritten.size} candidate slots not written, first (row, segment, slot) "
                                 f"{np.unravel_index(unwritten[0], (rows, eng.F // SEG, eng.c_keep))}")
    assert np.all(got[n:] == SENTINEL), f"{np.count_nonzero(got[n:] != SENTINEL)} guard slots past the buffer were written"
    return got[:n].reshape(rows, eng.F // SEG, eng.c_keep)


# ---------------------------------------------------------------------------------------------------------------- 1a. bit-exact
@pytest.mark.parametrize("c_keep,rows,F,d", [
    (8, 300, 24576, 768),          # the bench shape
    (4, 127, 384, 100),            # odd segment count (half-empty 256-wide tile), K tail of 4 that TMA zero-fills
    (6, 129, 640, 32),             # a partial second row tile
    (8, 1, 128, 32),               # one token, one segment
    (4, 300, 98304, 100),          # 768 segments (the selection's SPT 4 shape)
    (6, 127, 98304, 32),
    (8, 129, 128, 768),
    (6, 1, 24576, 100),
])
def test_candidate_keys_bit_exact_on_integer_data(c_keep, rows, F, d):
    x, W, b = _int_case(rows, d, F, seed=rows * 7 + F + d + c_keep, negative_segments=True)
    eng = _engine(x, W, b, k=1, c_keep=c_keep)
    got = _candidate_pass(eng, rows)
    ref = candidate_keys_batch(x.numpy(), W.numpy(), b.numpy(), c_keep)
    assert (ref < 0).any() == (F > SEG) and (ref >= 0).any(), "test premise: kept keys of both signs"
    bad = np.argwhere(got != ref)
    assert bad.size == 0, (f"{len(bad)} keys differ from the model; first at (row, segment, slot) {tuple(bad[0])}: "
                           f"got {got[tuple(bad[0])]:#x} want {ref[tuple(bad[0])]:#x}")


# ---------------------------------------------------------------------------------------------------------------- 1b. tolerance
def test_tensor_core_truncates_tf32_operands():
    """Premise of the error bound (DESIGN section 4): the tf32 wgmma reads an fp32 operand with its 13 low mantissa bits dropped.
    One-hot tokens make each value a single product, exact in fp32 (11 x 11 significant bits); with every dropped bit set,
    truncation and round-to-nearest differ by ~2^-10 relative, far more than the 2^-16 of a key bucket.  Were the hardware to
    round instead, the bound would still hold (|x - rn(x)| <= |x - trunc(x)| for every element, so the Cauchy-Schwarz term
    still covers the error), but the model's candidate values, and the tests below, would have to read the operands by rounding."""
    rows, d, F = 32, 32, 256
    g = torch.Generator().manual_seed(5)
    W = (torch.randn(F, d, generator=g).view(torch.int32) | 0x1FFF).view(torch.float32)
    x = torch.diag((torch.randn(rows, generator=g).view(torch.int32) | 0x1FFF).view(torch.float32))
    b = torch.zeros(F)
    got = _candidate_pass(_engine(x, W, b, k=1), rows)
    as_trunc = keys_of(candidate_values(x.numpy(), W.numpy(), b.numpy(), read=tf32_trunc), 8)
    as_round = keys_of(candidate_values(x.numpy(), W.numpy(), b.numpy(), read=tf32_round), 8)
    n_trunc, n_round = int((got == as_trunc).sum()), int((got == as_round).sum())
    print(f"tf32 operand read: {n_trunc} of {got.size} keys match truncation, {n_round} round-to-nearest")
    assert n_trunc == got.size and n_round < got.size // 100, (n_trunc, n_round, got.size)


@pytest.mark.parametrize("rows,d,F,c_keep,worst", [(257, 768, 24576, 8, False), (129, 100, 640, 6, True), (300, 256, 4096, 4, True),
                                                   (64, 1536, 8192, 8, True)])
def test_candidate_keys_within_the_accumulation_bound(rows, d, F, c_keep, worst):
    """General data: the tensor core accumulates in fp32 in an order of its own, so keys are checked against the bound the
    completeness proof allows for that, ceil(d / 8) 2^-21 ||a|| max ||w|| (DESIGN section 4)."""
    x, W, b = _gauss_case(rows, d, F, seed=rows + d + F, worst_mantissa=worst)
    got = _candidate_pass(_engine(x, W, b, k=1, c_keep=c_keep), rows).astype(np.int64)
    nseg = F // SEG
    assert np.all(np.diff(got, axis=2) < 0), "keys of a segment must be strictly descending"
    cols = np.sort(got & 127, axis=2)
    assert np.all(np.diff(cols, axis=2) != 0), "kept columns of a segment must be distinct"
    xn, Wn = x.numpy(), W.numpy()
    model = candidate_values(xn, Wn, b.numpy()).astype(np.float64).reshape(rows, nseg, SEG)
    w_norm = encoder_norms(Wn)[0]
    tol = (-(-d // 8) * 2.0 ** -21 * np.linalg.norm(xn.astype(np.float64), axis=1) * w_norm)[:, None, None]
    lo = ord2f((got & ~127).astype(np.int32)).astype(np.float64)
    hi = ord2f((got | 127).astype(np.int32)).astype(np.float64)
    mv = np.take_along_axis(model, got & 127, axis=2)
    slack = tol + 2.0 ** -22 * np.abs(mv)                                 # + the fp32 bias add of both sides
    off = np.maximum(lo - slack - mv, mv - hi - slack)
    assert off.max() <= 0, f"a kept key is {off.max():.3e} outside its model value's accumulation bound (row, seg, slot) {np.unravel_index(off.argmax(), off.shape)}"
    kept = np.zeros(model.shape, dtype=bool)
    np.put_along_axis(kept, got & 127, True, axis=2)
    dropped_max = np.where(kept, -np.inf, model).max(axis=2)
    excess = dropped_max - (hi[:, :, -1] + tol[:, :, 0] + 2.0 ** -22 * np.abs(hi[:, :, -1]))
    assert excess.max() <= 0, f"a dropped column beats the last kept key by {excess.max():.3e} beyond the bound at (row, seg) {np.unravel_index(excess.argmax(), excess.shape)}"


# ---------------------------------------------------------------------------------------------------------------- 1c. selection
def _boosted(rows, d, F, seed, seg, factor):
    """Integer data whose winners cluster in one segment: its kept keys are all re-scored (a saturated segment)."""
    x, W, b = _int_case(rows, d, F, seed, lim=8)
    W[seg * SEG:(seg + 1) * SEG] *= factor
    return x, W, b


def _ties(rows, d, F, seed):
    """A few winners over a constant floor: every segment's best key ties, so more than 512 keys reach the threshold."""
    x, _, _ = _int_case(rows, d, F, seed)
    W = torch.zeros(F, d)
    W[::997] = _int_case(1, d, (F + 996) // 997, seed + 1)[1]
    return x, W, torch.full((F,), SCALE)


# (data, rows, d, F, k, m_cand, c_keep, branches that must occur): nseg 1, < 32, 257..512 (SPT 2) and 769..1024 (SPT 4)
SELECT_CASES = {
    "one_segment_k1": (_int_case, 300, 32, 128, 1, 1, 8, {"proven_round1", "u_below"}),
    "one_segment_k16": (_int_case, 64, 64, 128, 16, 128, 4, {"exact_path"}),
    "3seg_k16_m128": (_int_case, 300, 100, 384, 16, 128, 6, {"saturated", "exact_path"}),
    "3seg_k4_m128": (_int_case, 300, 100, 384, 4, 128, 8, {"u_below"}),
    "20seg_k16_mk": (_int_case, 300, 64, 2560, 16, 16, 6, {"extended", "proven_round1"}),
    "192seg_k1_m128": (_int_case, 300, 64, 24576, 1, 128, 8, {"proven_round1"}),
    "320seg_k48": (lambda *a: _int_case(*a, lim=4), 300, 32, 40960, 48, 48, 8, {"proven_round1", "extended"}),
    "800seg_k16": (lambda *a: _int_case(*a, lim=4), 200, 32, 102400, 16, 16, 8, {"proven_round1", "extended"}),
    "saturated": (lambda r, d, F, s: _boosted(r, d, F, s, seg=2, factor=16), 300, 64, 1024, 16, 24, 8, {"saturated", "exact_path"}),
    "overflow_800seg_k48": (_ties, 100, 32, 102400, 48, 48, 8, {"overflow"}),
}


def _branches(r):
    out = set()
    if r["overflow"]:
        out.add("overflow")
    if not r["proven"]:
        out.add("exact_path")
    elif r["rounds"] == 1:
        out.add("proven_round1")
    else:
        out.add("extended")
    if r["proven"] and r["u_src"] == "below":
        out.add("u_below")
    if r["u_src"] == "sat":
        out.add("saturated")
    return out


@pytest.mark.parametrize("name", list(SELECT_CASES))
def test_selection_on_model_keys_matches_model_row_by_row(name):
    make, rows, d, F, k, m_cand, c_keep, expect = SELECT_CASES[name]
    x, W, b = make(rows, d, F, sum(map(ord, name)))
    xn, Wn, bn = x.numpy(), W.numpy(), b.numpy()
    keys = candidate_keys_batch(xn, Wn, bn, c_keep)
    res = select_rows(xn, Wn, bn, k, keys=keys, c_keep=c_keep, m_cand=m_cand)
    seen = set().union(*map(_branches, res))
    assert expect <= seen, f"test premise: branches {expect - seen} never taken (saw {seen})"

    eng = _engine(x, W, b, k=k, c_keep=c_keep, m_cand=m_cand)
    eng.cand.copy_(torch.from_numpy(keys.reshape(-1)))
    eng.feat_count.zero_()
    eng.idx.fill_(-1)
    eng.val.fill_(float("nan"))
    _phases(eng, rows, 2 | 4)
    idx, val = eng.idx.cpu().numpy(), eng.val.cpu().numpy()
    # integer data: the exact re-scoring is exact, so the result IS the stable float64 sort (value descending, ties -> lower index)
    exact = xn.astype(np.float64) @ Wn.astype(np.float64).T + bn.astype(np.float64)
    ref_idx = np.stack([np.lexsort((np.arange(F), -row))[:k] for row in exact])
    ref_val = np.take_along_axis(exact, ref_idx, axis=1)
    bad = np.flatnonzero((idx != ref_idx).any(axis=1) | (val != ref_val).any(axis=1))
    assert bad.size == 0, f"{bad.size} rows differ from the stable float64 sort, first {bad[0]}: {idx[bad[0]]} vs {ref_idx[bad[0]]}"
    assert np.array_equal(np.stack([r["idx"] for r in res]), ref_idx), "the model itself must select exactly"
    hist = np.bincount(ref_idx.reshape(-1), minlength=F).astype(np.float32)
    assert np.array_equal(eng.feat_count.cpu().numpy(), hist)
    # the decision of every row, and the candidates re-scored over the proven rows
    n_fb, rescored = eng.fb_count.tolist()
    gpu_fb = np.zeros(rows, dtype=bool)
    gpu_fb[eng.fb_rows[:n_fb].cpu().numpy()] = True
    model_fb = np.array([not r["proven"] for r in res])
    near = np.array([r["near"] < 1e-6 for r in res])                     # E is fp32 on the GPU, float64 in the model
    differ = np.flatnonzero(gpu_fb != model_fb)
    assert not (set(differ.tolist()) - set(np.flatnonzero(near).tolist())), f"rows {differ[:10]} decided unlike the model"
    want = sum(r["rescored"] for r in res if r["proven"])
    if near.any():
        assert abs(rescored - want) <= 128 * int(near.sum())
    else:
        assert rescored == want, (rescored, want)
    print(f"{name}: {n_fb} of {rows} rows on the exact path, {int(near.sum())} near-margin rows, branches {sorted(seen)}")
