"""ORACLE-SIDE MODEL (test infrastructure, not product code): a numpy restatement of the DECISION LOGIC of the fused SAE
encoder -> TopK path (vit-prisma_b200/csrc/sae_fused.cu), used on the CPU to check the exactness argument of DESIGN.md section 4
independently of the CUDA implementation.

What the reference computes (sae/sae.py:568-574, 795-808): hidden_pre = sae_in @ W_enc + b_enc, then torch.topk(hidden_pre, k).
What the CUDA path does instead, and what is modelled here step by step:

  1. candidate pass (k_enc_cand): the product with both operands truncated to tf32 (low 13 mantissa bits dropped), bias added in fp32;
     per (token, 128-feature segment) the C largest values are kept as packed keys: order-preserving int of the value with its low
     7 bits replaced by the column inside the segment;
  2. selection (k_cand_select): a gather threshold tau from per-warp quotas of the per-thread best keys (gather_threshold: at
     least 96 keys of the row are >= tau); the keys >= tau sorted descending (more than 512 of them: the exact path); the first m
     are re-scored EXACTLY; tau_k = k-th largest exact value; bound on everything not re-scored:
         u = max( best key not re-scored -- the next gathered key, or once all G gathered keys are re-scored the best key
                  under tau (u_below),
                  last kept key of every segment whose C kept keys were all re-scored )
         ub = upper end of u's value bucket (low 7 bits set)
         E  = coef * (||a - trunc(a)|| max_f ||w_f|| + ||a|| max_f ||w_f - trunc(w_f)||)
              + ceil(d / 8) 2^-21 ||a|| max_f ||w_f|| + 2^-13 |tau_k|
     the row is PROVEN when ub + E < tau_k; otherwise 16 more candidates are re-scored (up to min(G, 128)), then the row goes to
     the exact path;
  3. exact path (k_topk_fallback): top-k of the exact values of the whole row.

The model computes the tf32 product with exact (float64) accumulation: the tensor core's fp32 accumulation over ceil(d / 8) k-steps is
what the ceil(d / 8) 2^-21 ||a|| max ||w|| term bounds (4 units of 2^-23 per step against magnitudes <= ||a|| max ||w||); ``coef``
(1.05) covers the norms being evaluated in fp32, and the 2^-13 |tau_k| term the rounding of the bias add and of the key bucket.  Only tests/ may import this file.
"""
from __future__ import annotations

import numpy as np

SEG = 128


def tf32_trunc(x: np.ndarray) -> np.ndarray:
    """What a tf32 wgmma tensor-core read sees of an fp32 value: the low 13 mantissa bits are ignored."""
    return (np.asarray(x, dtype=np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def tf32_round(x: np.ndarray) -> np.ndarray:
    """fp32 -> the nearest tf32 (ties to even): what a tensor core that ROUNDS its fp32 operands would read."""
    u = np.asarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    u = (u + np.uint64(0xFFF) + ((u >> np.uint64(13)) & np.uint64(1))) & np.uint64(0xFFFFE000)
    return u.astype(np.uint32).view(np.float32)


def f2ord(v: np.ndarray) -> np.ndarray:
    """Monotone map float32 -> int32 (csrc/sae_fused.cu f2ord)."""
    k = np.asarray(v, dtype=np.float32).view(np.int32)
    return k ^ ((k >> 31) & np.int32(0x7FFFFFFF))


def ord2f(k: np.ndarray) -> np.ndarray:
    k = np.asarray(k, dtype=np.int32)
    return (k ^ ((k >> 31) & np.int32(0x7FFFFFFF))).view(np.float32)


def candidate_values(x: np.ndarray, W: np.ndarray, b: np.ndarray, read=tf32_trunc) -> np.ndarray:
    """[rows, F] fp32 values of the candidate pass: the tensor core's product of the operands as ``read`` sees them (exact float64
    accumulation), rounded to fp32, plus the bias in fp32.  x [rows, d], W [F, d] feature-major, b [F]."""
    x = np.atleast_2d(np.asarray(x, dtype=np.float32))
    prod = read(x).astype(np.float64) @ read(W).astype(np.float64).T
    return prod.astype(np.float32) + np.asarray(b, dtype=np.float32)


def keys_of(values: np.ndarray, c_keep: int) -> np.ndarray:
    """[rows, F // 128, c_keep] int32 packed keys of fp32 values [rows, F]: per 128-feature segment the c_keep largest, descending."""
    rows, F = values.shape
    assert F % SEG == 0
    keys = (f2ord(values) & np.int32(~127)) | (np.arange(F, dtype=np.int32) & 127)
    keys = np.sort(keys.reshape(rows, F // SEG, SEG), axis=2)
    return np.ascontiguousarray(keys[:, :, ::-1][:, :, :c_keep])


def candidate_keys_batch(x: np.ndarray, W: np.ndarray, b: np.ndarray, c_keep: int, chunk: int = 64) -> np.ndarray:
    """[rows, F // 128, c_keep] int32: what k_enc_cand writes to its candidate buffer for the tokens x [rows, d]."""
    x = np.atleast_2d(x)
    return np.concatenate([keys_of(candidate_values(x[i:i + chunk], W, b), c_keep) for i in range(0, x.shape[0], chunk)])


def candidate_keys(a: np.ndarray, W: np.ndarray, b: np.ndarray, c_keep: int) -> np.ndarray:
    """[F // 128, c_keep] packed keys of one token (descending inside a segment).  a [d], W [F, d] feature-major, b [F]."""
    return candidate_keys_batch(np.asarray(a)[None], W, b, c_keep)[0]


def gather_threshold(keys: np.ndarray, tau_rank: int = 96) -> int:
    """k_cand_select's gather threshold for one row's keys [nseg, c_keep]: thread t of the 256 owns segments t, t + 256, ...
    and bids its best key; warp w sorts its 32 bids and reports its q_w-th largest, q_w = ceil(m_tau cnt_w / nthr) with
    cnt_w = clamp(nthr - 32 w, 0, 32) bidding threads, nthr = min(256, nseg), m_tau = min(tau_rank, nthr).  tau is the smallest
    report, so at least m_tau keys of the row are >= tau."""
    nseg = keys.shape[0]
    spt = -(-nseg // 256)
    bids = np.full(256 * spt, np.iinfo(np.int64).min, dtype=np.int64)
    bids[:nseg] = keys[:, 0]
    bids = bids.reshape(spt, 256).max(axis=0)
    nthr = min(256, nseg)
    m_tau = min(tau_rank, nthr)
    tau = None
    for w in range(8):
        cnt = max(0, min(32, nthr - 32 * w))
        q = (m_tau * cnt + nthr - 1) // nthr
        if q > 0:
            rep = int(np.sort(bids[32 * w:32 * w + 32])[::-1][q - 1])
            tau = rep if tau is None else min(tau, rep)
    return tau


def encoder_norms(W: np.ndarray):
    """(max_f ||w_f||, max_f ||w_f - trunc(w_f)||) in float64: the two norms of the error bound (enc_norm_max on the GPU)."""
    Wd = np.asarray(W, dtype=np.float64)
    return (float(np.sqrt((Wd ** 2).sum(1)).max()),
            float(np.sqrt(((Wd - tf32_trunc(W).astype(np.float64)) ** 2).sum(1)).max()))


def select_row(a: np.ndarray, W: np.ndarray, b: np.ndarray, k: int, c_keep: int = 8, m_cand: int | None = None, coef: float = 1.05,
               max_cand: int = 128, extend: int = 16, slots: int = 512, tau_rank: int = 96, keys: np.ndarray | None = None,
               exact: np.ndarray | None = None, norms=None):
    """k_cand_select for one token.  ``keys`` [nseg, c_keep] (default: candidate_keys of the token), ``exact`` [F] float64
    pre-activations and ``norms`` (encoder_norms(W)) may be passed in when many rows share them.

    Returns dict(idx, val, proven, rescored, outside_max, tau_k, E, ...): the selected features (exact values, sorted descending,
    ties -> lower index), whether the completeness proof held, how many candidates were re-scored, the largest EXACT
    pre-activation among the features that were not re-scored (for the property test), and the path the decision took:
    G (keys gathered at or above the threshold), overflow (more than ``slots``: the exact path), rounds, u_src (which bound
    decided the last round: "next" un-rescored key, "below" the best key under the threshold, "sat" a saturated segment's
    last key, None) and margin = tau_k - (ub + E) of the last round."""
    F, d = W.shape
    m_cand = k + 8 if m_cand is None else m_cand
    if exact is None:
        exact = W.astype(np.float64) @ a.astype(np.float64) + b.astype(np.float64)
    if keys is None:
        keys = candidate_keys(a, W, b, c_keep)
    keys = np.asarray(keys, dtype=np.int64)                                # [nseg, c_keep], descending per segment
    w_norm, w_lo = encoder_norms(W) if norms is None else norms
    # ---- threshold and gather (per-warp quotas), then the sort of the gathered keys: key descending, position ascending
    tau = gather_threshold(keys, tau_rank)
    flat = keys.reshape(-1)
    pos = np.flatnonzero(flat >= tau)
    below = flat[flat < tau]
    u_below = int(below.max()) if below.size else None                     # best key under the threshold
    overflow = pos.size > slots                                            # massive ties: the kernel keeps an arbitrary 512
    order = np.lexsort((pos, -flat[pos]))[:slots]
    sorted_keys, sorted_pos = flat[pos][order], pos[order]
    G = sorted_keys.size
    feat_of = (sorted_pos // c_keep) * SEG + (sorted_keys & 127)
    a32 = a.astype(np.float32)
    a_norm = float(np.sqrt(np.sum(a32.astype(np.float64) ** 2)))
    a_lo = float(np.sqrt(np.sum((a32.astype(np.float64) - tf32_trunc(a32).astype(np.float64)) ** 2)))
    last = keys[:, c_keep - 1]
    Gs = min(G, max_cand)                                                  # the rounds stop at the gathered keys or at max_cand
    m_cur = min(m_cand, Gs)
    proven, rounds, near = False, 0, np.inf
    while True:
        rounds += 1
        cand = feat_of[:m_cur]
        vals = exact[cand]
        top = np.lexsort((cand, -vals))[:k]
        tau_k = vals[top[-1]] if m_cur >= k else -np.inf
        sat = last[last >= sorted_keys[m_cur - 1]]                         # segments whose kept keys were all re-scored
        u_rest = int(sorted_keys[m_cur]) if m_cur < G else u_below
        u, u_src = u_rest, (None if u_rest is None else ("next" if m_cur < G else "below"))
        if sat.size and (u is None or int(sat.max()) > u):
            u, u_src = int(sat.max()), "sat"
        u_val = -np.inf if u is None else float(ord2f(np.int32((u & ~127) | 127)))
        E = coef * (a_lo * w_norm + a_norm * w_lo) + -(-d // 8) * 2.0 ** -21 * a_norm * w_norm + abs(tau_k) * 2.0 ** -13
        margin = tau_k - (u_val + E)
        if np.isfinite(margin):                                            # closest call, relative to the terms compared
            near = min(near, abs(margin) / (abs(tau_k) + abs(u_val) + E))
        proven = not overflow and m_cur >= k and margin > 0
        if proven or m_cur >= Gs:
            break
        m_cur = min(m_cur + extend, Gs)
    rescored = np.zeros(F, dtype=bool)
    rescored[cand] = True
    outside_max = exact[~rescored].max() if (~rescored).any() else -np.inf
    if proven:
        idx = cand[top]
    else:                                                                   # exact path
        idx = np.lexsort((np.arange(F), -exact))[:k]
    return dict(idx=idx, val=exact[idx], proven=bool(proven), rescored=int(m_cur), outside_max=float(outside_max),
                tau_k=float(tau_k), E=float(E), tau=tau, G=int(G), overflow=bool(overflow), u_below=u_below, rounds=rounds,
                u_src=u_src, u_val=u_val, margin=float(margin), near=float(near))


def select_rows(x: np.ndarray, W: np.ndarray, b: np.ndarray, k: int, keys: np.ndarray | None = None, **kw):
    """select_row for every token of x [rows, d]; ``keys`` [rows, nseg, c_keep] (default: candidate_keys_batch)."""
    c_keep = kw.get("c_keep", 8)
    if keys is None:
        keys = candidate_keys_batch(x, W, b, c_keep)
    exact = x.astype(np.float64) @ W.astype(np.float64).T + b.astype(np.float64)
    norms = encoder_norms(W)
    return [select_row(x[r], W, b, k, keys=keys[r], exact=exact[r], norms=norms, **kw) for r in range(x.shape[0])]
