"""TopK-SAE training steps against the float64 oracle along the three axes the step kernels branch on: d_in, k and d_sae.

d_in.  The per-row kernels of the step (k_sae_prep, k_sae_decode, k_sae_grads, k_sae_grads_long, k_sae_adam_bulk /
k_sae_adam_rows) hold a d_in row as CHUNKS float4 per lane, CHUNKS in {1, 2, 4, 6, 8, 12} for d_in up to 128, 256, 512, 768,
1024, 1536 (chunks_for in csrc/sae_optim.cuh; both Adam kernels run its sae_adam_feature).  WIDTHS take every instance, full and
with idle lanes in the last chunk, on both encoder routes:

  * fused: tf32 candidate GEMM + exact re-scoring, Adam in the bulk-copy pipeline (its ring depth varies with d) or, below
    d = 64, in the rows kernel;
  * dense (GEMM_TC): 3xTF32 encoder GEMM + k_topk, Adam in the rows kernel, which also maintains the tf32 residual plane W_encT_lo.

k.  k_sae_decode reads a token's support 32 entries at a time, for the forward sum and for the dval dot products: k = 1 (one
entry, k_topk's threshold at rank 0), 31 (one partial chunk), 33 (a second chunk of one entry), 64 (two full chunks), 100 (a
partial fourth chunk) and 256 (eight chunks).  The fused encoder takes k <= 48 (m_cand = k + 8 candidates per token); at k = 49
"auto" switches to the dense encoder.  256 is the largest k pb_sae_topk takes: at d_sae 24,576 k_topk's candidate buffer then
needs 198,656 of the 204,800 bytes of shared memory it may use; k = 257 is refused.

d_sae.  pb_sae_backward's offset scan k_scan_counts<PER> runs one CTA of 1024 threads, each owning PER consecutive counts (PER =
ceil(d_sae / 1024) rounded up to a multiple of 4, instances 8, 24, 48, 64, 128); the dense route's pb_sae_topk cuts rows longer
than 24,576 features into segments and merges their winners in a second pass.  D_SAES take the upper edge of every scan
instance and the first size past it, on both routes, up to 131,072, where all 1024 runs are full and off[d_sae] is thread
1023's total; that is also the largest d_sae of the fused encoder.  131,200 is refused by train_step before any parameter
moves, and forward() at that size still matches the oracle.  A d_sae that is not a multiple of 128 takes the dense route under
"auto".  The cfg #5 dictionary (768 x 98,304) runs one step through the single-GPU engine (fp16 candidate operands) and the
one-rank data-parallel engine (tf32 operands), both against one float64 oracle step.

Consecutive steps take Adam past its first step (moments and bias correction).  A decoder bias far from the data makes a few
features fire on most tokens, so their per-feature lists take the long-list kernels (k_sae_grads_long, k_sae_norm_long) in
several 32-entry chunks.  Bars as elsewhere in the suite: 1e-4 relative (max-norm) for the loss, the gradient norm, sae_out, the
raw gradients and the parameters; TopK indices equal except rows with a near-tie; dead-feature counters exact.  What the
backward builds from the selection is checked exactly: feat_count and fired against the oracle's counts, l0, the CSC offsets
(the scan) and the CSC entry lists.

The encoder and the selection are checked first, against float64 hidden_pre.  The oracle's step then takes the engine's TopK
support, so that a near-tie row the engine legitimately resolves the other way (one such row turns sae_out 0.11 and the
gradients 5e-3 away from the oracle's) does not hide the rest of the step.  On the dense route the oracle also takes the
engine's TopK values: the 3xTF32 encoder GEMM accumulates ceil(d / 8) wgmma k-steps in fp32, and its hidden_pre was measured
(H100 80GB HBM3, 400 W) 4.6e-7 (d = 32) to 1.3e-5 (d = 1536) of max |hidden_pre| from float64 -- inside the 1e-4 bar, which is
asserted, but Adam divides every gradient element by its own magnitude, and for elements near eps that turned 1e-5-relative
gradient differences into W_dec differences of up to 1.8e-4.  The near-tie width on the dense route is twice the measured
hidden_pre error; on the fused route, whose selected values are exact fp32, it is 2e-6 of max |hidden_pre| as for cfg #3.
After every step the invariants the next step relies on are checked directly: unit-norm decoder rows, W_encT_lo ==
split_tf32(W_encT) bit for bit, and enc_norm_max (an input to the fused encoder's error bound) not below the float64 norms of W_enc.

The file runs in about 100 s on an H100 80GB HBM3 (700 W), 15 s of it the cfg #5 case, mostly its float64 oracle on the host;
that oracle alone peaks at 9.4 GB of resident host memory.
"""
import math

import numpy as np
import pytest
import torch

from oracle.fused_topk_model import tf32_trunc
from oracle.sae_oracle import new_adam_state, sae_forward, sae_grads, sae_train_step
from tests.util import rel_err

pytestmark = pytest.mark.gpu

WIDTHS = (32, 64, 100, 200, 384, 520, 768, 1000, 1024, 1536)
NORMS = ("none", "layer_norm", "constant_norm_rescale")
ROWS, K, STEPS, LR = 300, 16, 3, 1e-3
TOPK_SEG = 256 * 96                        # features per k_topk segment (pb_sae_topk)
PARAMS = ("W_encT", "W_dec", "b_enc", "b_dec")
MOMENTS = ("m_dec", "v_dec", "m_enc", "v_enc", "m_be", "v_be", "m_bd", "v_bd")


def _d_sae(d):
    return min(8192, max(128, round(4 * d / 128) * 128))


def _scan_instance(F):
    """PER of the k_scan_counts instance pb_sae_backward launches for d_sae = F (None: beyond the largest)."""
    per = ((F + 1023) // 1024 + 3) // 4 * 4
    return next((p for p in (8, 24, 48, 64, 128) if per <= p), None)


def _topk_smem(F, k):
    """Dynamic shared memory of k_topk over one unsegmented row of F features (launch_topk in csrc/sae.cu)."""
    need = -(-F // 256)
    ipt = 8 if need <= 8 else 24 if need <= 24 else 48 if need <= 48 else 96
    return 256 * 8 + max(min(ipt * k, F), k) * 8


def _init(d, F, seed, rows, steps):
    g = torch.Generator().manual_seed(seed)
    W_enc = torch.randn(d, F, generator=g) / math.sqrt(d)
    W_dec = torch.randn(F, d, generator=g)
    W_dec /= W_dec.norm(dim=1, keepdim=True)
    b_enc = 0.01 * torch.randn(F, generator=g)
    b_dec = 3.0 * torch.randn(d, generator=g)                          # far from the data: hot features
    xs = [torch.randn(rows, d, generator=g) * 2.0 + torch.randn(d, generator=g) for _ in range(steps)]
    return W_enc, W_dec, b_enc, b_dec, xs


def _engine(kind, W_enc, W_dec, b_enc, b_dec, k, norm, max_grad_norm, route):
    from vit_prisma.b200 import _lib as L
    from vit_prisma.b200.sae_engine import SaeStepEngine, unit_norm_rows_
    args = (W_enc.t().contiguous().cuda(), W_dec.clone().cuda(), b_enc.clone().cuda(), b_dec.clone().cuda())
    kw = dict(k=k, normalize_activations=norm, max_grad_norm=max_grad_norm, gemm_impl=L.GEMM_TC if route == "dense" else L.GEMM_AUTO)
    if kind == "single":
        eng = SaeStepEngine(*args, **kw)
    else:                                      # the data-parallel engine at world 1: its exchange hands a rank its own tables
        from vit_prisma.b200.p2p import P2PGroup, SaeDPEngine
        eng = SaeDPEngine(P2PGroup(0, 1, torch.device("cuda"), exchange=lambda mine: [mine]), *args, **kw)
    unit_norm_rows_(eng.W_dec)
    eng.refresh_lo()
    return eng


def _check_selection(at, eng, hp, k, dense):
    """The engine's encoder and TopK selection against float64 hidden_pre; returns (idx, val) on the host."""
    idx, val = eng.idx.cpu().long(), eng.val.cpu().double()
    if dense:
        assert rel_err(eng.hidden_pre, hp) <= 1e-4, f"{at}: hidden_pre rel err {rel_err(eng.hidden_pre, hp):.2e}"
        tie = 2.0 * float((eng.hidden_pre.cpu().double() - hp).abs().max())
    else:
        tie = 2e-6 * float(hp.abs().max())
    top = torch.topk(hp, min(k + 1, hp.shape[1]), dim=-1)
    same = (idx == top.indices[:, :k]).all(dim=1)
    near = (top.values[:, :-1] - top.values[:, 1:]).abs().min(dim=1).values < tie
    assert bool((same | near).all()), f"{at}: {(~(same | near)).sum().item()} rows select other features than the oracle"
    assert bool((hp.gather(1, idx) >= top.values[:, k - 1:k] - tie).all()), f"{at}: a selected feature is not a near-top-k one"
    assert rel_err(val, hp.gather(1, idx)) <= 1e-4, f"{at}: TopK values rel err {rel_err(val, hp.gather(1, idx)):.2e}"
    return idx, val


def _check_counts(at, eng, idx, val, F):
    """What the step builds from the selection, exactly: counts, l0, and the per-feature (CSC) entry lists."""
    rows, k = idx.shape
    counts = torch.bincount(idx.reshape(-1), minlength=F)
    pos = torch.bincount(idx[val > 0], minlength=F)
    assert torch.equal(eng.feat_count.cpu().long(), counts), f"{at}: feat_count != bincount(idx)"
    assert torch.equal(eng.fired.cpu().long(), pos), f"{at}: fired != per-feature count of positive selected values"
    l0 = np.float32(int(pos.sum())) * (np.float32(1.0) / np.float32(rows))     # pos_count * (1 / rows), fp32 as on the device
    assert eng.scalars_dict()["l0"] == float(l0), f"{at}: l0 {eng.scalars_dict()['l0']} != {float(l0)}"
    off = eng.csc_off.cpu().long()
    assert torch.equal(off, torch.cat([torch.zeros(1, dtype=torch.long), torch.cumsum(counts, 0)])), f"{at}: csc_off is not the scan"
    assert int(off[F]) == rows * k, f"{at}: csc_off[F] = {int(off[F])}, not rows * k = {rows * k}"
    ent = eng.csc_entries.cpu().long()
    assert torch.equal(torch.sort(ent).values, torch.arange(rows * k)), f"{at}: csc_entries is not a permutation of the entries"
    assert torch.equal(idx.reshape(-1)[ent], torch.repeat_interleave(torch.arange(F), counts)), f"{at}: an entry sits in another feature's list"


def _steps_match_oracle(d, F, k, route, norm, clip, rows, steps, *, seed, expect=None, engines=("single",)):
    """``steps`` training steps of every engine in ``engines`` ("single": SaeStepEngine, "dp": one-rank SaeDPEngine) from one seeded
    state, each checked against one float64 oracle step.  ``route``: "fused" (GEMM_AUTO, must take the fused encoder), "dense"
    (GEMM_TC) or "auto" (GEMM_AUTO, must take the encoder ``expect``)."""
    from vit_prisma.b200 import ops
    W_enc, W_dec, b_enc, b_dec, xs = _init(d, F, seed, rows, steps)
    p = {"W_enc": W_enc.double(), "W_dec": W_dec.double(), "b_enc": b_enc.double(), "b_dec": b_dec.double()}
    # the clipping threshold from the first step's gradient norm: active at every step (a tenth of it) or never (four times it)
    fwd = sae_forward(p, xs[0].double(), k, norm)
    gn0 = math.sqrt(sum(float((v ** 2).sum()) for v in sae_grads(p, xs[0].double(), fwd, norm).values()))
    max_grad_norm = 0.1 * gn0 if clip else 4.0 * gn0
    counts = torch.bincount(fwd["idx"].reshape(-1), minlength=F)
    assert int(counts.max()) > 64, "test premise: a feature list of more than two 32-entry chunks (k_sae_grads_long)"
    del fwd

    encoder = expect or route
    engs = {kind: _engine(kind, W_enc, W_dec, b_enc, b_dec, k, norm, max_grad_norm, route) for kind in engines}
    for kind, eng in engs.items():
        assert eng.encoder == encoder, f"test premise: {kind} engine on the {eng.encoder} encoder, not {encoder}"
    state = new_adam_state(p)
    since = {kind: torch.zeros(F, device="cuda") for kind in engs}
    freq = {kind: torch.zeros(F, device="cuda") for kind in engs}
    since_ref, freq_ref = torch.zeros(F, dtype=torch.float64), torch.zeros(F, dtype=torch.float64)
    for s, x in enumerate(xs):
        hp = sae_forward(p, x.double(), k, norm)["hidden_pre"]      # W_dec does not enter hidden_pre
        sel = {}
        for kind, eng in engs.items():
            at = f"d={d} F={F} k={k} {route} {norm} {kind} step {s + 1}"
            eng.train_step(x.cuda(), LR, since_fired=since[kind], act_freq=freq[kind], want_out=True)
            sel[kind] = _check_selection(at, eng, hp, k, encoder == "dense")
        idx, val = sel[engines[0]]
        for kind in engines[1:]:
            assert torch.equal(sel[kind][0], idx), f"step {s + 1}: the {kind} engine selects other features than the {engines[0]} engine"
        del hp
        ref = sae_train_step(p, state, x.double(), k, LR, s + 1, mode=norm, max_grad_norm=max_grad_norm, since_fired=since_ref,
                             act_freq=freq_ref, topk_idx=idx, topk_val=val if encoder == "dense" else None)
        raw, ref_dec = ref["raw_grads"], p["W_dec"] / p["W_dec"].norm(dim=1, keepdim=True)    # the oracle renormalises next step
        for kind, eng in engs.items():
            at = f"d={d} F={F} k={k} {route} {norm} {kind} step {s + 1}"
            sc = eng.scalars_dict()
            assert (ref["clip"] < 1.0) == clip and (sc["clip_coef"] < 1.0) == clip, (at, ref["clip"], sc["clip_coef"])
            errs = {"mse": abs(sc["mse"] / float(ref["mse"]) - 1), "grad_norm": abs(sc["grad_norm"] / float(ref["grad_norm"]) - 1),
                    "clip_coef": abs(sc["clip_coef"] / ref["clip"] - 1), "sae_out": rel_err(eng.sae_out, ref["fwd"]["sae_out"]),
                    "dL/dW_dec": rel_err(eng.gW_dec, raw["W_dec"]), "dL/dW_enc": rel_err(eng.gW_encT.t(), raw["W_enc"]),
                    "dL/db_enc": rel_err(eng.gb_enc, raw["b_enc"]), "dL/db_dec": rel_err(eng.gb_dec, raw["b_dec"]),
                    "W_dec": rel_err(eng.W_dec, ref_dec), "W_enc": rel_err(eng.W_encT.t(), p["W_enc"]),
                    "b_enc": rel_err(eng.b_enc, p["b_enc"]), "b_dec": rel_err(eng.b_dec, p["b_dec"])}
            bad = {n: f"{e:.2e}" for n, e in errs.items() if e > 1e-4}
            assert not bad, f"{at}: beyond 1e-4 of the float64 oracle: {bad}; all: { {n: f'{e:.1e}' for n, e in errs.items()} }"
            assert torch.equal(since[kind].cpu().double(), since_ref) and torch.equal(freq[kind].cpu().double(), freq_ref), \
                f"{at}: dead-feature counters"
            _check_counts(at, eng, *sel[kind], F)
            # invariants the next step depends on
            W_dec_now, W_encT_now = eng.W_dec.cpu().double(), eng.W_encT.cpu()
            assert (W_dec_now.norm(dim=1) - 1.0).abs().max().item() <= 1e-5, f"{at}: decoder rows not unit-norm"
            if encoder == "dense":
                assert torch.equal(eng.W_encT_lo.view(torch.int32), ops.split_tf32(eng.W_encT).view(torch.int32)), f"{at}: W_encT_lo stale"
            W64 = W_encT_now.double()
            lo64 = W64 - torch.from_numpy(tf32_trunc(W_encT_now.numpy())).double()
            want = torch.tensor([W64.norm(dim=1).max().item(), lo64.norm(dim=1).max().item()], dtype=torch.float64)
            got = eng.enc_norm_max.cpu().double()
            assert bool((got >= want * (1 - 1e-5)).all()), f"{at}: enc_norm_max {got.tolist()} below the float64 norms {want.tolist()}"
            assert bool((got <= want * (1 + 1e-5)).all()), f"{at}: enc_norm_max {got.tolist()} far above the float64 norms {want.tolist()}"
    return engs


# ------------------------------------------------------------------------------------------------ d_in
CASES = [(d, route, NORMS[(j + r) % 3], j % 2 == r) for j, d in enumerate(WIDTHS) for r, route in enumerate(("fused", "dense"))]


@pytest.mark.parametrize("d,route,norm,clip", CASES)
def test_three_steps_match_float64_oracle(d, route, norm, clip):
    _steps_match_oracle(d, _d_sae(d), K, route, norm, clip, ROWS, STEPS, seed=1000 * d + (route == "dense"))


# ------------------------------------------------------------------------------------------------ k
# (k, d_sae, route, the encoder "auto" must take)
K_AXIS = [(1, 4096, "fused", None), (31, 4096, "fused", None), (33, 4096, "fused", None), (33, 4096, "dense", None),
          (48, 4096, "fused", None), (49, 4096, "auto", "dense"), (64, 4096, "dense", None), (100, 4096, "dense", None),
          (256, 4096, "dense", None), (256, 24576, "dense", None)]


@pytest.mark.parametrize("k,F,route,expect", K_AXIS, ids=[f"k{k}-F{F}-{r}" for k, F, r, _ in K_AXIS])
def test_k_axis_steps_match_float64_oracle(k, F, route, expect):
    j = [c[:3] for c in K_AXIS].index((k, F, route))
    if F == TOPK_SEG:
        assert _topk_smem(F, k) == 198656, "test premise: k_topk's candidate buffer at its shared-memory edge"
    _steps_match_oracle(128, F, k, route, NORMS[(j + 1) % 3], j % 2 == 1, ROWS, 2, seed=10 * F + 7 * k + (route == "dense"), expect=expect)


def test_k_beyond_256_is_refused():
    from vit_prisma.b200 import _lib as L
    W_enc, W_dec, b_enc, b_dec, xs = _init(128, 4096, 257, ROWS, 1)
    eng = _engine("single", W_enc, W_dec, b_enc, b_dec, 257, "layer_norm", 1.0, "auto")
    assert eng.encoder == "dense"
    with pytest.raises(L.PrismaB200Error, match=r"k=257 > 256"):
        eng.train_step(xs[0].cuda(), LR)


# ------------------------------------------------------------------------------------------------ d_sae
# (d_sae, k_scan_counts instance, k_topk segments on the dense route)
D_SAES = [(8192, 8, 1), (8320, 24, 1), (24576, 24, 1), (24704, 48, 2), (49152, 48, 2), (49280, 64, 3), (65536, 64, 3),
          (65664, 128, 3), (98304, 128, 4), (131072, 128, 6)]
F_AXIS = [(F, per, nseg, route, 32) for F, per, nseg in D_SAES for route in ("fused", "dense")] + [(131072, 128, 6, "fused", 48)]


@pytest.mark.parametrize("F,per,nseg,route,k", F_AXIS, ids=[f"F{F}-{r}-k{k}" for F, _, _, r, k in F_AXIS])
def test_d_sae_axis_steps_match_float64_oracle(F, per, nseg, route, k):
    j = F_AXIS.index((F, per, nseg, route, k))
    assert _scan_instance(F) == per, f"test premise: d_sae {F} runs k_scan_counts<{_scan_instance(F)}>, not <{per}>"
    assert -(-F // TOPK_SEG) == nseg, f"test premise: d_sae {F} is {-(-F // TOPK_SEG)} k_topk segments, not {nseg}"
    _steps_match_oracle(64, F, k, route, NORMS[j % 3], j % 4 < 2, ROWS, 2, seed=F + 7 * k + (route == "dense"))


def test_d_sae_beyond_131072_is_refused_before_any_update():
    """The offset scan takes at most 131,072 features: train_step raises and leaves the parameters and the Adam moments as they
    were; inference, which needs no scan, still runs at that size and matches the oracle."""
    from vit_prisma.b200 import _lib as L
    d, F, k, norm = 64, 131200, 32, "layer_norm"
    assert _scan_instance(F) is None
    W_enc, W_dec, b_enc, b_dec, xs = _init(d, F, F, ROWS, 1)
    x = xs[0]
    eng = _engine("single", W_enc, W_dec, b_enc, b_dec, k, norm, 1.0, "auto")
    assert eng.encoder == "dense"
    p = {"W_enc": W_enc.double(), "W_dec": W_dec.double(), "b_enc": b_enc.double(), "b_dec": b_dec.double()}
    eng.forward(x.cuda())
    hp = sae_forward(p, x.double(), k, norm)["hidden_pre"]
    idx, val = _check_selection(f"forward d_sae={F}", eng, hp, k, True)
    ref = sae_forward(p, x.double(), k, norm, topk_idx=idx, topk_val=val)
    assert rel_err(eng.sae_out, ref["sae_out"]) <= 1e-4, f"forward d_sae={F}: sae_out rel err {rel_err(eng.sae_out, ref['sae_out']):.2e}"
    assert abs(eng.scalars_dict()["mse"] / float(ref["mse"]) - 1) <= 1e-4, (eng.scalars_dict()["mse"], float(ref["mse"]))
    before = {n: getattr(eng, n).clone() for n in PARAMS + MOMENTS}
    with pytest.raises(L.PrismaB200Error, match="131072"):
        eng.train_step(x.cuda(), LR)
    torch.cuda.synchronize()
    for n, t in before.items():
        assert torch.equal(getattr(eng, n).view(torch.int32), t.view(torch.int32)), f"{n} changed by a refused train_step"


@pytest.mark.parametrize("d,F", [(100, 300), (1000, 4000)])
def test_d_sae_not_a_multiple_of_128_takes_the_dense_route(d, F):
    _steps_match_oracle(d, F, K, "auto", NORMS[d % 3], d == 100, ROWS, 2, seed=d + F, expect="dense")


def test_cfg5_dictionary_full_width_one_step():
    """768 x 98,304, k 32: the single-GPU engine (fused, fp16 candidate operands) and the one-rank data-parallel engine (fused,
    tf32 operands) take one step from the same state; one float64 oracle step checks both."""
    engs = _steps_match_oracle(768, 98304, 32, "auto", "layer_norm", True, 256, 1, seed=98304768, expect="fused", engines=("single", "dp"))
    assert engs["single"].cand_operands == "f16" and engs["dp"].cand_operands == "tf32"
