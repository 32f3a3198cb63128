"""ORACLE-SIDE MODEL (test infrastructure, not product code): a numpy restatement of the DECISION LOGIC of the fused SAE
encoder -> TopK path (vit-prisma_b200/csrc/sae_fused.cu), used on the CPU to check the exactness argument of DESIGN.md section 4
independently of the CUDA implementation.

What the reference computes (sae/sae.py:568-574, 795-808): hidden_pre = sae_in @ W_enc + b_enc, then torch.topk(hidden_pre, k).
What the CUDA path does instead, and what is modelled here step by step:

  1. candidate pass (k_enc_cand): the product with both operands truncated to tf32 (low 13 mantissa bits dropped), bias added in fp32;
     per (token, 128-feature segment) the C largest values are kept as packed keys: order-preserving int of the value with its low
     7 bits replaced by the column inside the segment;
  2. selection (k_cand_select): all keys of a token sorted descending; the first m are re-scored EXACTLY; tau_k = k-th largest exact
     value; bound on everything not re-scored:
         u = max( best key not re-scored ,  last kept key of every segment whose C kept keys were all re-scored )
         ub = upper end of u's value bucket (low 7 bits set)
         E  = coef * (||a - trunc(a)|| max_f ||w_f|| + ||a|| max_f ||w_f - trunc(w_f)||)
              + ceil(d / 8) 2^-21 ||a|| max_f ||w_f|| + 2^-13 |tau_k|
     the row is PROVEN when ub + E < tau_k; otherwise 16 more candidates are re-scored (up to 128), then the row goes to the exact path;
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


def f2ord(v: np.ndarray) -> np.ndarray:
    """Monotone map float32 -> int32 (csrc/sae_fused.cu f2ord)."""
    k = np.asarray(v, dtype=np.float32).view(np.int32)
    return k ^ ((k >> 31) & np.int32(0x7FFFFFFF))


def ord2f(k: np.ndarray) -> np.ndarray:
    k = np.asarray(k, dtype=np.int32)
    return (k ^ ((k >> 31) & np.int32(0x7FFFFFFF))).view(np.float32)


def candidate_keys(a: np.ndarray, W: np.ndarray, b: np.ndarray, c_keep: int) -> np.ndarray:
    """[F // 128, c_keep] packed keys of one token (descending inside a segment).  a [d], W [F, d] feature-major, b [F]."""
    F = W.shape[0]
    assert F % SEG == 0
    approx = (tf32_trunc(W).astype(np.float64) @ tf32_trunc(a).astype(np.float64)).astype(np.float32) + b.astype(np.float32)
    keys = (f2ord(approx) & np.int32(~127)) | (np.arange(F, dtype=np.int32) & 127)
    keys = keys.reshape(F // SEG, SEG)
    return -np.sort(-keys.astype(np.int64), axis=1)[:, :c_keep]           # int64 only so that the negation cannot overflow


def select_row(a: np.ndarray, W: np.ndarray, b: np.ndarray, k: int, c_keep: int = 8, m_cand: int | None = None, coef: float = 1.05,
               max_cand: int = 128, extend: int = 16, slots: int = 512):
    """Returns dict(idx, val, proven, rescored, outside_max): the selected features (exact values, sorted descending, ties -> lower
    index), whether the completeness proof held, which features were re-scored, and -- for the property test -- the largest EXACT
    pre-activation among the features that were not re-scored."""
    F, d = W.shape
    m_cand = k + 8 if m_cand is None else m_cand
    exact = W.astype(np.float64) @ a.astype(np.float64) + b.astype(np.float64)
    keys = candidate_keys(a, W, b, c_keep)                                 # [nseg, c_keep]
    nseg = keys.shape[0]
    flat = keys.reshape(-1)
    pos = np.arange(flat.size)
    order = np.lexsort((pos, -flat))                                       # key descending, position ascending (sel_pack)
    G = min(flat.size, slots)
    sorted_keys, sorted_pos = flat[order], pos[order]
    u_below = sorted_keys[G] if flat.size > G else None                    # best key outside the sorted prefix
    feat_of = (sorted_pos // c_keep) * SEG + (sorted_keys & 127)
    a32 = a.astype(np.float32)
    a_norm = float(np.sqrt(np.sum(a32.astype(np.float64) ** 2)))
    a_lo = float(np.sqrt(np.sum((a32.astype(np.float64) - tf32_trunc(a32).astype(np.float64)) ** 2)))
    w_norm = float(np.sqrt((W.astype(np.float64) ** 2).sum(1)).max())
    w_lo = float(np.sqrt(((W.astype(np.float64) - tf32_trunc(W).astype(np.float64)) ** 2).sum(1)).max())
    Gs = min(G, max_cand)
    m_cur = min(m_cand, Gs)
    proven = False
    while True:
        cand = feat_of[:m_cur]
        vals = exact[cand]
        top = sorted(range(m_cur), key=lambda j: (-vals[j], cand[j]))[:k]
        tau_k = vals[top[-1]] if m_cur >= k else -np.inf
        key_m = sorted_keys[m_cur - 1]
        last = keys[:, c_keep - 1]
        sat = last[last >= key_m]
        u = None
        if m_cur < G:
            u = sorted_keys[m_cur]
        elif u_below is not None:
            u = u_below
        if sat.size:
            u = sat.max() if u is None else max(u, sat.max())
        u_val = -np.inf if u is None else float(ord2f(np.int32((int(u) & ~127) | 127)))
        E = coef * (a_lo * w_norm + a_norm * w_lo) + -(-a.shape[0] // 8) * 2.0 ** -21 * a_norm * w_norm + abs(tau_k) * 2.0 ** -13
        proven = m_cur >= k and (u_val + E < tau_k)
        if proven or m_cur >= Gs:
            break
        m_cur = min(m_cur + extend, Gs)
    rescored = np.zeros(F, dtype=bool)
    rescored[cand] = True
    outside_max = exact[~rescored].max() if (~rescored).any() else -np.inf
    if proven:
        idx = np.array([cand[j] for j in top])
    else:                                                                   # exact path
        idx = np.array(sorted(range(F), key=lambda f: (-exact[f], f))[:k])
    return dict(idx=idx, val=exact[idx], proven=bool(proven), rescored=int(m_cur), outside_max=float(outside_max),
                tau_k=float(tau_k), E=float(E))
