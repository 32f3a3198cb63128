"""CPU check of the exactness argument behind the fused SAE encoder -> TopK path (DESIGN.md section 4), on the numpy model of its
decision logic (oracle/fused_topk_model.py):

  * the Cauchy-Schwarz bound really bounds |tf32 product - exact| for every feature (random and worst-case mantissas);
  * THE THEOREM: whenever the completeness proof holds, no feature outside the re-scored set reaches the k-th exact value, so the
    selection equals torch.topk of the exact pre-activations (the reference, sae/sae.py:795-808);
  * rows the proof cannot cover (saturated segments, ties) take the exact path and are right by construction;
  * on Gaussian dictionaries the proof holds for (almost) every row with k + 8 candidates -- the fast path is the common path.
The CUDA kernels are held to float64 top-k on the GPU (tests/test_sae_gpu.py); this file holds the ARGUMENT to it without a GPU."""
import numpy as np
import pytest
import torch

from oracle.fused_topk_model import (SEG, candidate_keys, candidate_keys_batch, f2ord, gather_threshold, ord2f, select_row, select_rows,
                                      tf32_trunc)


def _case(rows, d, F, seed, w_scale=None, worst_mantissa=False, offset=True):
    g = np.random.default_rng(seed)
    W = (g.standard_normal((F, d)) / np.sqrt(d)).astype(np.float32)
    if w_scale is not None:
        W = (W * w_scale[:, None]).astype(np.float32)
    b = (0.01 * g.standard_normal(F)).astype(np.float32)
    x = (g.standard_normal((rows, d)) * 2.0 + (g.standard_normal(d) if offset else 0.0)).astype(np.float32)
    if worst_mantissa:      # every low mantissa bit set: the largest truncation residual a tf32 read can have
        W = (W.view(np.uint32) | np.uint32(0x1FFF)).view(np.float32)
        x = (x.view(np.uint32) | np.uint32(0x1FFF)).view(np.float32)
    return x, W, b


def test_ordered_int_round_trip_and_monotonicity():
    v = np.array([-3.5, -1e-30, -0.0, 0.0, 1e-30, 2.25, 7e8], dtype=np.float32)
    o = f2ord(v)
    assert np.array_equal(ord2f(o), v)
    assert np.all(np.diff(o.astype(np.int64)) >= 0)
    # clearing / setting the low 7 bits brackets the value from below / above, for either sign
    lo, hi = ord2f(o & np.int32(~127)), ord2f((o & np.int32(~127)) | np.int32(127))
    assert np.all(lo <= v) and np.all(v <= hi)


@pytest.mark.parametrize("worst", [False, True])
def test_error_bound_covers_the_tf32_product(worst):
    x, W, b = _case(6, 96, 1024, seed=3, worst_mantissa=worst)
    Wd, td = W.astype(np.float64), tf32_trunc(W).astype(np.float64)
    w_norm, w_lo = np.sqrt((Wd ** 2).sum(1)).max(), np.sqrt(((Wd - td) ** 2).sum(1)).max()
    for a in x:
        ad, ta = a.astype(np.float64), tf32_trunc(a).astype(np.float64)
        err = np.abs(Wd @ ad - td @ ta).max()
        bound = np.linalg.norm(ad - ta) * w_norm + np.linalg.norm(ad) * w_lo
        assert err <= bound, (err, bound)
        if worst:
            assert err > 1e-3 * bound          # and it is not vacuous: the worst-case mantissas come within three orders of it


@pytest.mark.parametrize("rows,d,F,k,c_keep,seed", [(24, 64, 2048, 8, 8, 0), (16, 128, 4096, 32, 8, 1), (16, 96, 2048, 16, 6, 2),
                                                   (12, 64, 1024, 8, 4, 3)])
def test_proven_rows_equal_the_exact_topk(rows, d, F, k, c_keep, seed):
    x, W, b = _case(rows, d, F, seed)
    n_proven = 0
    for a in x:
        r = select_row(a, W, b, k, c_keep=c_keep)
        exact = torch.from_numpy(W.astype(np.float64) @ a.astype(np.float64) + b.astype(np.float64))
        ref = torch.topk(exact, k)
        if r["proven"]:
            n_proven += 1
            assert r["outside_max"] < r["tau_k"], "a feature outside the re-scored set reaches the k-th exact value"
        assert np.array_equal(r["idx"], ref.indices.numpy()), (r["proven"], r["idx"], ref.indices)
        assert np.all(np.diff(r["val"]) <= 0)
    if c_keep == 8:
        assert n_proven >= rows - 1, f"only {n_proven} of {rows} rows proven on a Gaussian dictionary"


def test_worst_case_mantissas_never_break_the_theorem():
    """Operands with every truncated bit set make the candidate pass as wrong as it can be: the proof may fail more often (those rows take
    the exact path) but a proven row is still exact."""
    x, W, b = _case(24, 64, 2048, seed=5, worst_mantissa=True)
    for a in x:
        r = select_row(a, W, b, 8)
        exact = W.astype(np.float64) @ a.astype(np.float64) + b.astype(np.float64)
        if r["proven"]:
            assert r["outside_max"] < r["tau_k"]
        assert np.array_equal(r["idx"], np.array(sorted(range(2048), key=lambda f: (-exact[f], f))[:8]))


def test_saturated_segments_and_ties_take_the_exact_path():
    # winners clustered in ONE 128-feature segment: its 8 kept keys are all re-scored, the 9th-best of that segment was never kept
    d, F, k = 64, 1024, 16
    scale = np.ones(F)
    scale[256:384] = 50.0
    x, W, b = _case(8, d, F, seed=7, w_scale=scale, offset=False)
    for a in x:
        r = select_row(a, W, b, k)
        exact = W.astype(np.float64) @ a.astype(np.float64) + b.astype(np.float64)
        assert not r["proven"]
        assert np.array_equal(r["idx"], np.array(sorted(range(F), key=lambda f: (-exact[f], f))[:k]))
    # an all-zero dictionary: every key ties; the proof (strict inequality) must fail and the exact path returns the lowest indices
    r = select_row(x[0], np.zeros((F, d), np.float32), np.zeros(F, np.float32), k)
    assert not r["proven"] and r["idx"].tolist() == list(range(k))


def test_kept_keys_are_the_segment_maxima():
    x, W, b = _case(1, 64, 512, seed=9)
    keys = candidate_keys(x[0], W, b, 8)
    approx = (tf32_trunc(W).astype(np.float64) @ tf32_trunc(x[0]).astype(np.float64)).astype(np.float32) + b
    for s in range(512 // SEG):
        seg = approx[s * SEG:(s + 1) * SEG]
        cols = keys[s] & 127
        assert len(set(cols.tolist())) == 8
        kept_min = seg[cols].min()
        others = np.delete(seg, cols)
        # a dropped column can only exceed a kept one inside one 128-ulp bucket (the low 7 bits were replaced by the column)
        assert np.all(f2ord(others).astype(np.int64) <= (f2ord(np.float32(kept_min)).astype(np.int64) | 127))


@pytest.mark.parametrize("nseg", [1, 3, 20, 300, 800])
def test_gather_threshold_keeps_the_quota(nseg):
    """k_cand_select gathers the keys at or above tau, the smallest of the per-warp reports: at least min(96, nseg) keys, and tau
    is one thread's best key (a segment maximum)."""
    x, W, b = _case(4, 32, nseg * SEG, seed=nseg)
    for keys in candidate_keys_batch(x, W, b, 8):
        tau = gather_threshold(keys)
        assert tau in set(keys[:, 0].tolist())
        assert (keys >= tau).sum() >= min(96, nseg)
        if nseg <= 32:                                 # every thread bids and every bid is reported: tau = the smallest maximum
            assert tau == keys[:, 0].min()


def test_u_below_and_the_early_stop_at_the_gathered_keys():
    """Three segments (24 keys): the gathered set is always smaller than 128, so the rounds stop at G, and once every gathered key
    is re-scored the bound on the rest is u_below, the best key under the threshold.  Both paths occur here, and every row is
    still the exact top-k."""
    rows, d, F, k = 64, 64, 3 * SEG, 4
    x, W, b = _case(rows, d, F, seed=11)
    keys = candidate_keys_batch(x, W, b, 8)
    res = select_rows(x, W, b, k, keys=keys, c_keep=8, m_cand=k)
    for a, kr, r in zip(x, keys, res):
        exact = W.astype(np.float64) @ a.astype(np.float64) + b.astype(np.float64)
        assert r["G"] == (kr >= r["tau"]).sum() < 128
        assert r["rescored"] <= r["G"]
        if not r["proven"]:
            assert r["rescored"] == r["G"], "an unproven row re-scores until its gathered keys run out, not until 128"
        else:
            assert r["outside_max"] < r["tau_k"]
        if r["u_src"] == "below":
            assert r["rescored"] == r["G"] and r["u_below"] == kr[kr < r["tau"]].max()
        assert np.array_equal(r["idx"], np.lexsort((np.arange(F), -exact))[:k])
    assert any(r["proven"] and r["u_src"] == "below" for r in res), "no row proven on u_below"
    assert any(r["rounds"] > 1 and r["rescored"] == r["G"] for r in res), "no row stopped early at the gathered keys"
