"""Dense ReLU + L1, ReLU + ghost grads, TopK + ghost grads, Gated and Transcoder (ReLU + skip, TopK) training steps against the
float64 oracle, at every GEMM route their products can take, at the dead-feature counts where the ghost block changes shape, and
at the sizes a user trains.

Routes.  Every dense product of these steps is ``gemm32`` -> ``pb_gemm``, whose AUTO rule (csrc/gemm.cu, pb_gemm_tc_eligible in
csrc/gemm_tc.cu) picks the 3xTF32 wgmma kernel when M >= 64, N >= 64, K >= 32 and both leading dimensions are multiples of 4
floats (the residual planes are always supplied), and the exact FFMA kernel otherwise.  ``_routes`` restates that rule for each
named product; every case asserts the route mix it was chosen for, and ``test_every_product_is_seen_on_both_routes`` checks the
table as a whole.  The products whose K is the token count (gW_dec, gW_encT, gW_skip, the ghost gWd / gWe) run on transposed
operands with leading dimension ``rows``: 60 tokens sends the forward products to FFMA and the gradient products to the tensor
cores with a K tail, 61 and 302 tokens send the gradient products to FFMA, d = 48 leaves the decoder side on FFMA, d_sae = 1,030
the decoder, d = 24 everything.  (A d_in that is not a multiple of 4 is refused when any of these engines is built: pb_rownorm_max
and the per-row kernels read rows as float4.)

Dead features.  The ghost block is padded to ndp = max(32, ceil32(nd)) columns and only nd rows are scattered back: nd in
{0, 1, 31, 32, 33, 63, 64, 65, 1500} takes ndp 32, 64, 96 and 1,504 and the FFMA / tensor-core edge of the ghost dE, gWd and
gWe products (ndp = 64).  The dead set is set exactly through since_fired and dead_feature_window; dead features get b_enc = -6
(exp(h) ~ 2e-3, as in test_sae_dense_gpu), so they stay silent and the ghost term stays in the regime its bars were set for.

Selection premise.  The oracle takes the engine's support (its ReLU mask, gate and magnitude masks, or TopK indices).  That is
only legitimate where the engine's pre-activations are right: they must be within 1e-4 of float64 (max-norm), the largest
absolute error is taken as the band, and every position where the engine's mask differs from the float64 sign must lie within
twice that band of zero (for the magnitude mask, the band times max exp(r_mag)); a TopK row must select the float64 top-k unless
it has a near-tie inside the band.  This replaces the "at most 8 flipped features" rule of the mid-size tests, which would not
carry over to 4,096 x 12,288 pre-activations.

Bars.  1e-4 (max-norm) for the loss terms, sae_out and hidden_pre; 2e-4 for every raw gradient.  Ghost gradients (the dead
features' rows of dL/dW_dec and dL/dW_enc, their dL/db_enc, dL/db_dec and the gradient norm) keep the ill-conditioning bars of
test_sae_dense_gpu: 3e-3 when every product runs on FFMA, 6e-2 otherwise.  Parameters after the steps keep the mid-size bars,
1.2e-3 (3e-3 FFMA / 1e-2 tensor cores with ghost grads) of max |W_enc| = 0.28 there, i.e. 0.34, 0.84 and 2.8 learning-rate
steps absolute: Adam's m / (sqrt(v) + eps) turns a 1e-9 difference on a near-zero gradient element into a fraction of lr.  That
holds at every element whose float64 gradient (for W_dec: projected off the row) is more than 10x the gradient's error from
zero; the others may take Adam's lr * sign(g) the other way and are held to the bar plus 2 lr (measured up to 2.0 lr).  Exact: fired, since_fired and act_freq counted from the
engine's mask, l0, unit-norm decoder rows and W_encT_lo == split_tf32(W_encT).

Ghost rows outside the dead set.  The ghost blocks are added to gW_dec / gW_encT by a row scatter after the main products; the
test snapshots both arrays just before the ghost terms of the same step and requires every row outside the dead set to be
bit-equal to the snapshot, and every dead row to have received a non-zero block.  (A twin engine without ghost grads would not
give bit-equal rows: the batch-mean column sum of the prep and the TopK backward accumulate with atomics.)

Real sizes.  The trainer's default (768 x 12,288, 4,096 tokens), the ViT-L width (1,024 x 16,384) and a Transcoder TopK at
768 x 32,768 (segmented TopK), all on the tensor cores; the default dense ReLU step again on FFMA (GEMM_SIMT).

Measured on an H100 80GB HBM3 (700 W power limit), max-norm relative error against float64.  hidden_pre (K = d_in):
2.9e-6 at K = 256, 7.3e-6 at 768, 9.2e-6 at 1,024.  The decoder accumulates K = d_sae products, and its error grows about
linearly in K: sae_out 2.0e-5 at K = 2,048, 9.0e-5 at 12,288, 1.3e-4 at 16,384; mse 2.3e-5, 1.4e-4 and 1.9e-4; dL/dW_dec
2.7e-5, 1.7e-4 and 2.1e-4 (K = 4,096 tokens in the gradient products adds little: dL/dW_enc 1.1e-4 at 12,288).  The same
768 x 12,288 step on FFMA stays at mse 2.9e-7, sae_out 3.8e-6 and gradients 2.1e-6.  FINDING: past a decoder K of about 6,144
the tensor-core route misses the suite's 1e-4 / 2e-4 bars that FFMA meets.  The error grows linearly in K, as a truncating
accumulator's does: the wgmma fp32 accumulator holds the whole K chain.  The bf16 GEMM already adds each 64-wide k-slab's wgmma
result into an fp32 register total (PROMOTE in csrc/gemm_tc.cu); doing the same for 3xTF32 is the follow-up that should bring
these cases back under the bars.  Until then only the terms measured past their bar (K_SCALED: mse, aux, ghost, sae_out,
dL/dW_dec) are scaled by max(1, d_sae / 6,144), and only on a dense-activation tensor-core decoder.  The Transcoder TopK at
d_sae 32,768 keeps 1e-4 / 2e-4: its decoder input has at most k = 32 non-zeros per row, and an all-zero k-step leaves even a
truncating accumulator exact (measured mse 6.0e-6, sae_out 6.6e-6, dL/dW_dec 1.5e-5).  The positive count behind l0 is an
integer (an fp32 sum stops being exact past 2^24 positives, which every real-size ReLU / Gated case has), so l0 is checked
exactly everywhere.  Resync: every step starts from the oracle's parameters and Adam moments, so each step is checked on its own.

The file's 84 tests run in 91 s on that GPU.  The test process peaks at 11.7 GB of resident host memory, CUDA context included;
the largest oracle step, the float64 Gated step at 1,024 x 16,384 x 4,096, adds 5.0 GB of it (measured alone on the host: 1.3 GB
before the step, 6.3 GB at its peak).  The engines stay within a few GB of device memory.
"""
import json
import math

import numpy as np
import pytest
import torch

from oracle.sae_oracle import gated_train_step, new_adam_state, sae_train_step, transcoder_train_step
from tests.util import rel_err

pytestmark = pytest.mark.gpu

LR, L1, K, WINDOW = 1e-3, 2e-3, 32, 10
NORMS = ("layer_norm", "constant_norm_rescale", "none")
ENGINES = ("relu", "relu_ghost", "topk_ghost", "gated", "tc_relu_skip", "tc_topk")
TOPK_SEG = 256 * 96                        # features per k_topk segment (pb_sae_topk)
# mid-size parameter bars (fraction of max |W_enc| = 0.28 there) as absolute bars
PARAM_ABS = {"plain": 1.2e-3 * 0.28, "ghost_ffma": 3e-3 * 0.28, "ghost_tc": 1e-2 * 0.28}
# the terms measured past their bar on a dense-activation tensor-core decoder at d_sae 12,288 / 16,384 (see the docstring)
K_SCALED = ("mse", "aux", "ghost", "sae_out", "dL/dW_dec")


# ------------------------------------------------------------------------------------------------ routes
def _tc(M, N, Kd, lda, ldb):
    """pb_gemm's AUTO rule for an fp32 product with both tf32 residual planes supplied."""
    return M >= 64 and N >= 64 and Kd >= 32 and lda % 4 == 0 and ldb % 4 == 0


def _routes(kind, d, F, rows, nd, simt=False):
    """{product: "tc" | "ffma"} for the products one step of ``kind`` launches (M, N, K, lda, ldb of each)."""
    fwd = (rows, F, d, d, d)                          # encoder; d_acts = g @ W_dec^T has the same shape
    grad = (F, d, rows, rows, rows)                   # gW_dec = acts^T @ g, gW_encT = d_hid^T @ sae_in
    shapes = {"encoder": fwd}
    if kind != "topk_ghost":                          # TopK + ghost: the main gradients come from the sparse kernels
        shapes.update(decoder=(rows, d, F, F, F), d_acts=fwd, gW_dec=grad, gW_encT=grad)
    if kind == "tc_relu_skip":
        shapes.update(skip=(rows, d, d, d, d), gW_skip=(d, d, rows, rows, rows))
    if kind.endswith("ghost") and nd > 0:
        ndp = max(32, (nd + 31) // 32 * 32)
        shapes.update(ghost_dE=(rows, ndp, d, d, d), ghost_gWd=(ndp, d, rows, rows, rows), ghost_gWe=(ndp, d, rows, rows, rows))
    return {n: "ffma" if simt or not _tc(*s) else "tc" for n, s in shapes.items()}


# ------------------------------------------------------------------------------------------------ cases
def _shape_routes(fwd, dec, d_acts, grad, skip, gskip):
    return dict(encoder=fwd, decoder=dec, d_acts=d_acts, gW_dec=grad, gW_encT=grad, skip=skip, gW_skip=gskip)


T, S = "tc", "ffma"
# tag: (d, d_sae, tokens, the routes the shape is chosen for)
SHAPES = {
    "a": (256, 2048, 512, _shape_routes(T, T, T, T, T, T)),     # everything on the tensor cores
    "b": (256, 2048, 60, _shape_routes(S, S, S, T, S, T)),      # M = rows < 64 forward; K = 60 gradient products with a K tail
    "b2": (256, 2048, 61, _shape_routes(S, S, S, S, S, S)),     # + rows % 4 != 0: every product on FFMA at tensor-core-legal d, d_sae
    "c": (256, 2048, 300, _shape_routes(T, T, T, T, T, T)),     # K tail on the gradient products
    "d": (256, 2048, 302, _shape_routes(T, T, T, S, T, S)),     # leading dimension 302: gradient products on FFMA
    "e": (48, 1024, 512, _shape_routes(T, S, T, S, S, S)),      # N = d < 64: decoder side on FFMA
    "f": (100, 1000, 512, _shape_routes(T, T, T, T, T, T)),     # M and N tails, d_sae not a multiple of 128
    "g": (68, 1030, 512, _shape_routes(T, S, T, T, T, T)),      # d_sae % 4 = 2: decoder on FFMA; gradients with an N tail
    "h": (24, 512, 256, _shape_routes(S, S, S, S, S, S)),       # K = d < 32: everything on FFMA
}
ROUTE_CASES = [(tag, kind) for tag in SHAPES for kind in ENGINES]
DEAD_COUNTS = (0, 1, 31, 32, 33, 63, 64, 65, 1500)
DEAD_CASES = [(nd, kind) for nd in DEAD_COUNTS for kind in ("relu_ghost", "topk_ghost")]


def _expected_routes(tag, kind, nd):
    d, F, rows, want = SHAPES[tag]
    got = _routes(kind, d, F, rows, nd)
    exp = {n: r for n, r in want.items() if n in got}
    if "ghost_dE" in got:                      # ndp >= 64 here: the ghost products route as the encoder / the K = rows products
        exp.update(ghost_dE=want["encoder"], ghost_gWd=want["gW_encT"], ghost_gWe=want["gW_encT"])
    return got, exp


def _axis_a_dead(F):
    return len(range(3, F, 7))                 # every 7th feature dead in the axis-A ghost cases


# ------------------------------------------------------------------------------------------------ set-up
def _init(kind, d, F, rows, steps, seed, nd):
    g = torch.Generator().manual_seed(seed)
    p = {"W_enc": torch.randn(d, F, generator=g) / math.sqrt(d), "W_dec": torch.randn(F, d, generator=g)}
    if kind == "gated":
        p.update(b_gate=0.05 * torch.randn(F, generator=g), r_mag=0.1 * torch.randn(F, generator=g), b_mag=0.05 * torch.randn(F, generator=g))
    else:
        p["b_enc"] = 0.01 * torch.randn(F, generator=g)
    p["b_dec"] = 0.1 * torch.randn(d, generator=g)
    if kind.startswith("tc_"):
        p["b_dec_out"] = 0.1 * torch.randn(d, generator=g)
        if kind == "tc_relu_skip":
            p["W_skip"] = 0.3 * torch.randn(d, d, generator=g) / math.sqrt(d)
    dead = None
    if kind.endswith("ghost"):
        dead = torch.sort(torch.randperm(F, generator=g)[:nd]).values
        p["b_enc"][dead] = -6.0                # 6 sigma below zero: silent, exp(h) ~ 2e-3
    xs = [torch.randn(rows, d, generator=g) * 2.0 + torch.randn(d, generator=g) for _ in range(steps)]
    ys = None
    if kind.startswith("tc_"):
        M = torch.randn(d, d, generator=g) / math.sqrt(d)
        ys = [torch.tanh(x @ M) * 1.5 + 0.3 * torch.randn(rows, d, generator=g) + torch.randn(d, generator=g) for x in xs]
    return p, dead, xs, ys


def _engine(kind, p, norm, impl):
    from vit_prisma.b200.sae_dense import SaeDenseStepEngine
    from vit_prisma.b200.sae_engine import unit_norm_rows_
    from vit_prisma.b200.sae_gated import SaeGatedStepEngine
    from vit_prisma.b200.sae_transcoder import SaeTranscoderStepEngine
    c = lambda t: t.clone().cuda()  # noqa: E731
    WeT = p["W_enc"].t().contiguous().cuda()
    kw = dict(normalize_activations=norm, max_grad_norm=1.0, gemm_impl=impl)
    if kind == "gated":
        eng = SaeGatedStepEngine(WeT, c(p["W_dec"]), c(p["b_gate"]), c(p["r_mag"]), c(p["b_mag"]), c(p["b_dec"]), l1_coefficient=L1, **kw)
    elif kind.startswith("tc_"):
        eng = SaeTranscoderStepEngine(WeT, c(p["W_dec"]), c(p["b_enc"]), c(p["b_dec"]), c(p["b_dec_out"]),
                                      c(p["W_skip"]) if "W_skip" in p else None, k=K, activation="relu" if kind == "tc_relu_skip" else "topk",
                                      l1_coefficient=L1, **kw)
    else:
        eng = SaeDenseStepEngine(WeT, c(p["W_dec"]), c(p["b_enc"]), c(p["b_dec"]), k=K, l1_coefficient=L1, **kw)
    unit_norm_rows_(eng.W_dec)
    eng.refresh_lo()
    return eng


def _load_oracle_state(kind, eng, p, state):
    """Engine parameters and Adam moments := the oracle's: every step starts from the oracle's state."""
    eng.W_encT.copy_(p["W_enc"].t()); eng.W_dec.copy_(p["W_dec"] / p["W_dec"].norm(dim=1, keepdim=True))
    eng.b_enc.copy_(p["b_gate" if kind == "gated" else "b_enc"]); eng.b_dec.copy_(p["b_dec"])
    eng.refresh_lo()
    pairs = [("W_dec", eng.m_dec, eng.v_dec), ("b_gate" if kind == "gated" else "b_enc", eng.m_be, eng.v_be), ("b_dec", eng.m_bd, eng.v_bd)]
    if kind == "gated":
        eng.r_mag.copy_(p["r_mag"]); eng.b_mag.copy_(p["b_mag"])
        pairs += [("r_mag", eng.m_r, eng.v_r), ("b_mag", eng.m_bm, eng.v_bm)]
    if kind.startswith("tc_"):
        eng.b_dec_out.copy_(p["b_dec_out"])
        pairs.append(("b_dec_out", eng.m_bo, eng.v_bo))
        if eng.W_skip is not None:
            eng.W_skip.copy_(p["W_skip"])
            pairs.append(("W_skip", eng.m_sk, eng.v_sk))
    for name, m, v in pairs:
        m.copy_(state[name]["m"]); v.copy_(state[name]["v"])
    eng.m_enc.copy_(state["W_enc"]["m"].t()); eng.v_enc.copy_(state["W_enc"]["v"].t())


def _engine_grads(kind, eng):
    g = {"W_enc": eng.gW_encT.t(), "W_dec": eng.gW_dec, "b_dec": eng.gb_dec}
    g["b_gate" if kind == "gated" else "b_enc"] = eng.gb_enc
    if kind == "gated":
        g.update(r_mag=eng.gr_mag, b_mag=eng.gb_mag)
    if kind.startswith("tc_"):
        g["b_dec_out"] = eng.gb_dec_out
        if eng.W_skip is not None:
            g["W_skip"] = eng.gW_skip
    return g


def _engine_params(kind, eng):
    out = {"W_enc": eng.W_encT.t(), "W_dec": eng.W_dec, "b_dec": eng.b_dec}
    out["b_gate" if kind == "gated" else "b_enc"] = eng.b_gate if kind == "gated" else eng.b_enc
    if kind == "gated":
        out.update(r_mag=eng.r_mag, b_mag=eng.b_mag)
    if kind.startswith("tc_"):
        out["b_dec_out"] = eng.b_dec_out
        if eng.W_skip is not None:
            out["W_skip"] = eng.W_skip
    return out


def _spy_ghost(eng, snap):
    """Snapshots gW_dec / gW_encT just before the engine adds the ghost blocks of a step."""
    inner = eng._ghost_terms

    def wrapped(x, resid, dead_idx):
        snap["gW_dec"], snap["gW_encT"] = eng.gW_dec.clone(), eng.gW_encT.clone()
        snap["dead"] = dead_idx.clone()
        inner(x, resid, dead_idx)
    eng._ghost_terms = wrapped


def _band_check(at, what, got_pre, pre64):
    """hidden_pre (pi, on the device) within 1e-4 of float64; returns the band: the largest absolute error."""
    err = max(float((got_pre[r:r + 256].cpu().double() - pre64[r:r + 256]).abs().max()) for r in range(0, pre64.shape[0], 256))
    scale = float(pre64.abs().max())
    assert err <= 1e-4 * scale, f"{at}: {what} rel err {err / scale:.2e}"
    return err, err / scale


def _flip_check(at, what, mask, val64, band):
    diff = mask != (val64 > 0)
    if bool(diff.any()):
        worst = float(val64[diff].abs().max())
        assert worst <= 2.0 * band, f"{at}: {int(diff.sum())} {what} flips, one {worst:.2e} from zero (band {band:.2e})"
    return int(diff.sum())


def _topk_check(at, idx, pre64, band):
    top = torch.topk(pre64, K + 1, dim=-1)
    same = (torch.sort(idx, dim=1).values == torch.sort(top.indices[:, :K], dim=1).values).all(dim=1)
    near = (top.values[:, :-1] - top.values[:, 1:]).abs().min(dim=1).values < 2.0 * band
    assert bool((same | near).all()), f"{at}: {int((~(same | near)).sum())} rows select other features than float64"
    assert bool((pre64.gather(1, idx) >= top.values[:, K - 1:K] - 2.0 * band).all()), f"{at}: a selected feature is not a near-top-k one"


LOG = []


# ------------------------------------------------------------------------------------------------ the helper
def _steps_match_oracle(kind, d, F, rows, norm, steps, *, seed, nd=0, simt=False, expect=None):
    from vit_prisma.b200 import _lib as L
    from vit_prisma.b200 import ops
    from vit_prisma.b200.sae_engine import topk_support
    ghost = kind.endswith("ghost")
    routes = _routes(kind, d, F, rows, nd, simt)
    if expect is not None:
        assert routes == expect, f"test premise: routes {routes} != {expect}"
    all_ffma = all(r == "ffma" for r in routes.values())
    ghost_tol = 3e-3 if all_ffma else 6e-2
    # a dense activation on the tensor-core decoder: the terms measured to grow with K = d_sae past 6,144 get that growth (docstring)
    kscale = max(1.0, F / 6144) if routes.get("decoder") == "tc" and kind != "tc_topk" else 1.0
    tol = lambda name, bar: bar * (kscale if name in K_SCALED else 1.0)  # noqa: E731
    p32, dead, xs, ys = _init(kind, d, F, rows, steps, seed, nd)
    eng = _engine(kind, p32, norm, L.GEMM_SIMT if simt else L.GEMM_AUTO)
    p = {n: v.double() for n, v in p32.items()}
    del p32
    state = new_adam_state(p)
    sf, af = torch.zeros(F, device="cuda"), torch.zeros(F, device="cuda")
    sf_ref, af_ref = torch.zeros(F, dtype=torch.float64), torch.zeros(F, dtype=torch.float64)
    if ghost:
        sf_ref[dead] = WINDOW + 1.0                     # exactly nd features past the dead-feature window
        sf.copy_(sf_ref)
        snap = {}
        _spy_ghost(eng, snap)
    for s, x in enumerate(xs):
        at = f"{kind} d={d} F={F} rows={rows} nd={nd} {norm}{' simt' if simt else ''} step {s + 1}"
        if s > 0:
            _load_oracle_state(kind, eng, p, state)
        w0 = p["W_dec"] / p["W_dec"].norm(dim=1, keepdim=True)          # the decoder the oracle's step projects against
        xc = x.cuda()
        if ghost:
            snap.clear()
        er_max = float(p["r_mag"].exp().max()) if kind == "gated" else 0.0
        dead_mask = (sf_ref > WINDOW) if ghost else None
        # ---- engine step, and the support it chose
        if kind in ("relu", "relu_ghost"):
            eng.train_step_dense(xc, LR, sf, af, use_ghost_grads=ghost, dead_feature_window=WINDOW, want_out=True)
        elif kind == "topk_ghost":
            eng.train_step_topk_ghost(xc, LR, sf, af, WINDOW)
        elif kind == "gated":
            eng.train_step_gated(xc, LR, sf, af, want_out=True)
        else:
            eng.train_step_transcoder(xc, ys[s].cuda(), LR, sf, af, want_out=True)
        torch.cuda.synchronize()
        if ghost:
            assert "gW_dec" in snap, f"{at}: test premise: the step adds its ghost terms through SaeDenseStepEngine._ghost_terms"
        terms = eng.loss_terms(rows)
        if kind == "topk_ghost" or kind == "tc_topk":
            if kind == "topk_ghost":
                idx, val = eng.idx.long(), eng.val
            else:                                       # pb_sae_topk is deterministic: the selection the step scattered
                idx, val = topk_support(eng.hidden_pre, K)
                idx = idx.long()
                dense = torch.zeros(rows, F, device="cuda").scatter_(1, idx, torch.relu(val))
                assert torch.equal(eng.last_acts, dense), f"{at}: the step's activations are not its TopK selection"
            mask = torch.zeros(rows, F, dtype=torch.bool, device="cuda").scatter_(1, idx, val > 0).cpu()
            idx = idx.cpu()
            kw = {"topk_idx": idx}
        elif kind == "gated":
            gate = (eng.hidden_pre > 0).cpu()
            mask = (eng.last_acts > 0).cpu()            # gate AND mag_pre > 0
            assert not bool((mask & ~gate).any()), f"{at}: an active feature with a closed gate"
            kw = {"gate_mask": gate, "mag_mask": mask}
        else:
            mask = (eng.last_acts > 0).cpu()
            assert torch.equal(mask, (eng.hidden_pre > 0).cpu()), f"{at}: ReLU mask is not hidden_pre > 0"
            kw = {"relu_mask": mask}
        # ---- float64 oracle step on the engine's support
        x64 = x.double()
        if kind == "gated":
            ref = gated_train_step(p, state, x64, LR, s + 1, norm, L1, since_fired=sf_ref, act_freq=af_ref, **kw)
            pre64, out64, raw = ref["pi"], ref["sae_out"], ref["raw_grads"]
        elif kind.startswith("tc_"):
            ref = transcoder_train_step(p, state, x64, ys[s].double(), LR, s + 1, norm, "relu" if kind == "tc_relu_skip" else "topk", K, L1,
                                        since_fired=sf_ref, act_freq=af_ref, **kw)
            pre64, out64, raw = ref["hidden_pre"], ref["sae_out"], ref["raw_grads"]
        else:
            ref = sae_train_step(p, state, x64, K, LR, s + 1, mode=norm, since_fired=sf_ref, act_freq=af_ref,
                                 act="topk" if kind == "topk_ghost" else "relu", l1_coefficient=L1, use_ghost_grads=ghost,
                                 dead_feature_window=WINDOW, **kw)
            pre64, out64, raw = ref["fwd"]["hidden_pre"], ref["fwd"]["sae_out"], ref["raw_grads"]
            if ghost:
                assert ref["n_dead"] == nd and eng.last_n_dead == nd, f"{at}: dead count {ref['n_dead']} / {eng.last_n_dead}, not {nd}"
        # ---- selection premise
        band, pre_rel = _band_check(at, "hidden_pre", eng.hidden_pre, pre64)
        if "topk_idx" in kw:
            _topk_check(at, idx, pre64, band)
            flips = 0
        else:
            flips = _flip_check(at, "gate" if kind == "gated" else "ReLU", kw.get("gate_mask", mask), pre64, band)
            if kind == "gated":
                on = kw["gate_mask"]
                flips += _flip_check(at, "magnitude", mask[on], ref["mag_pre"][on], band * er_max)
        # ---- numeric bars
        errs = {"mse": abs(terms["mse"] / float(ref["mse"]) - 1), "sae_out": rel_err(eng.sae_out, out64)}
        if ref.get("l1") is not None:
            errs["l1"] = abs(terms["l1"] / float(ref["l1"]) - 1)
        if kind == "gated":
            errs["aux"] = abs(terms["aux"] / float(ref["aux"]) - 1)
        if ghost:
            errs["ghost"] = abs(terms["ghost"] / float(ref["ghost"]) - 1)
        bad = {n: e for n, e in errs.items() if e > tol(n, 1e-4)}
        got = _engine_grads(kind, eng)
        gerrs = {}
        for name, r in raw.items():
            g = got[name]
            if ghost and nd and name in ("W_dec", "W_enc", "b_enc"):
                gd = g.t() if name == "W_enc" else g                  # feature-major: [F, d]
                rd = r.t() if name == "W_enc" else r
                live = ~dead_mask
                gerrs[f"dL/d{name} live"] = e = rel_err(gd.cpu()[live], rd[live])
                if e > tol(f"dL/d{name}", 2e-4):
                    bad[f"dL/d{name} live"] = e
                e = float((gd.cpu().double()[dead_mask] - rd[dead_mask]).abs().max()) / float(rd.abs().max())
                gerrs[f"dL/d{name} dead"] = e
                if e > ghost_tol:
                    bad[f"dL/d{name} dead"] = e
            else:
                bar = ghost_tol if (ghost and nd and name == "b_dec") else tol(f"dL/d{name}", 2e-4)
                gerrs[f"dL/d{name}"] = e = rel_err(g, r)
                if e > bar:
                    bad[f"dL/d{name}"] = e
        gn_err = abs(terms["grad_norm"] / float(ref["grad_norm"]) - 1)
        if gn_err > (ghost_tol if ghost and nd else 2e-4):
            bad["grad_norm"] = gn_err
        LOG.append(dict(at=at, routes=routes, K_enc=d, K_grad=rows, hidden_pre=pre_rel, flips=flips, **errs, **gerrs, grad_norm=gn_err))
        assert not bad, f"{at}: beyond the bars: { {n: f'{e:.2e}' for n, e in bad.items()} }; all: " \
                        f"{ {n: f'{e:.1e}' for n, e in {**errs, **gerrs}.items()} }"
        # ---- exact checks
        pos = int(mask.sum())
        assert torch.equal(eng.fired.cpu(), mask.sum(0).float()), f"{at}: fired != per-feature count of the engine's mask"
        assert torch.equal(sf.cpu().double(), sf_ref) and torch.equal(af.cpu().double(), af_ref), f"{at}: dead-feature counters"
        assert eng.scalars_dict()["pos_count"] == pos, f"{at}: positive count {eng.scalars_dict()['pos_count']} != {pos}"
        want_l0 = float(np.float32(pos) * (np.float32(1.0) / np.float32(rows)))        # one rounding of the count, then * (1 / rows)
        assert terms["l0"] == want_l0, f"{at}: l0 {terms['l0']} != {want_l0}"
        assert float((eng.W_dec.double().norm(dim=1) - 1.0).abs().max()) <= 1e-5, f"{at}: decoder rows not unit-norm"
        assert torch.equal(eng.W_encT_lo.view(torch.int32), ops.split_tf32(eng.W_encT).view(torch.int32)), f"{at}: W_encT_lo stale"
        if ghost:
            dead_dev = dead_mask.cuda()
            assert torch.equal(snap["dead"].long().cpu(), torch.nonzero(dead_mask).flatten()), f"{at}: the engine's dead set"
            for name in ("gW_dec", "gW_encT"):
                now, before = getattr(eng, name), snap[name]
                assert torch.equal(now[~dead_dev].view(torch.int32), before[~dead_dev].view(torch.int32)), \
                    f"{at}: the ghost blocks changed a {name} row outside the dead set"
                if nd:
                    moved = (now[dead_dev] != before[dead_dev]).any(dim=1)
                    assert bool(moved.all()), f"{at}: {int((~moved).sum())} dead {name} rows received no ghost block"
        # ---- parameters after the step
        # an element whose gradient is within 10x the gradient's error of zero may take Adam's lr * sign(g) the other way: 2 lr
        bar = PARAM_ABS["plain" if not ghost else ("ghost_ffma" if all_ffma else "ghost_tc")]
        for name, v in _engine_params(kind, eng).items():
            r = p[name] / p[name].norm(dim=1, keepdim=True) if name == "W_dec" else p[name]   # the oracle renormalises next step
            diff = (v.cpu().double() - r).abs()
            g64, g32 = raw[name], got[name].cpu().double()
            if name == "W_dec":                                               # Adam sees the gradient projected off the row
                g64, g32 = g64 - (g64 * w0).sum(1, keepdim=True) * w0, g32 - (g32 * w0).sum(1, keepdim=True) * w0
            unsure = g64.abs() <= 10.0 * float((g32 - g64).abs().max())
            e_sure = float(diff[~unsure].max()) if bool((~unsure).any()) else 0.0
            e_all = float(diff.max())
            LOG[-1][f"{name} abs/lr"] = [e_sure / LR, e_all / LR, int(unsure.sum())]
            assert e_sure <= bar, f"{at}: {name} {e_sure:.2e} from the oracle after the step (bar {bar:.2e})"
            assert e_all <= bar + 2.0 * LR, f"{at}: {name} {e_all:.2e} from the oracle after the step at a near-zero gradient element"
        del ref, raw, got, pre64, out64, mask, kw
    print(json.dumps(LOG[-steps:]))
    return eng


# ------------------------------------------------------------------------------------------------ A. GEMM routes
@pytest.mark.parametrize("tag,kind", ROUTE_CASES, ids=[f"{tag}-{SHAPES[tag][0]}x{SHAPES[tag][1]}x{SHAPES[tag][2]}-{kind}"
                                                          + (f"-nd{_axis_a_dead(SHAPES[tag][1])}" if kind.endswith("ghost") else "")
                                                          for tag, kind in ROUTE_CASES])
def test_routes_steps_match_float64_oracle(tag, kind):
    d, F, rows, _ = SHAPES[tag]
    j = ROUTE_CASES.index((tag, kind))
    ghost = kind.endswith("ghost")
    nd = _axis_a_dead(F) if ghost else 0
    # every engine meets every mode across the shapes; ghost grads want unit-scale pre-activations (b_enc = -6 is then 6 sigma)
    norm = NORMS[(list(SHAPES).index(tag) + ENGINES.index(kind)) % (2 if ghost else 3)]
    got, exp = _expected_routes(tag, kind, nd)
    assert got == exp, f"test premise: routes {got} != {exp}"
    _steps_match_oracle(kind, d, F, rows, norm, 2, seed=1000 * j + 17, nd=nd, expect=exp)


# ------------------------------------------------------------------------------------------------ B. dead-feature count
@pytest.mark.parametrize("nd,kind", DEAD_CASES, ids=[f"256x2048x512-{kind}-nd{nd}" for nd, kind in DEAD_CASES])
def test_dead_count_steps_match_float64_oracle(nd, kind):
    got = _routes(kind, 256, 2048, 512, nd)
    ndp = max(32, (nd + 31) // 32 * 32)
    ghost_route = "tc" if ndp >= 64 else "ffma"
    assert all(got[n] == ghost_route for n in ("ghost_dE", "ghost_gWd", "ghost_gWe")) if nd else "ghost_dE" not in got
    norm = NORMS[(DEAD_COUNTS.index(nd) + (kind == "topk_ghost")) % 2]
    _steps_match_oracle(kind, 256, 2048, 512, norm, 2, seed=7 * nd + (kind == "topk_ghost"), nd=nd, expect=got)


# ------------------------------------------------------------------------------------------------ C. real sizes
REAL = [("relu", 768, 12288, 4096, 2, 0, False), ("relu_ghost", 768, 12288, 4096, 2, 1000, False), ("gated", 768, 12288, 4096, 2, 0, False),
        ("tc_relu_skip", 768, 12288, 4096, 2, 0, False), ("relu", 1024, 16384, 4096, 1, 0, False), ("gated", 1024, 16384, 4096, 1, 0, False),
        ("tc_topk", 768, 32768, 2048, 1, 0, False), ("relu", 768, 12288, 4096, 2, 0, True)]


@pytest.mark.parametrize("kind,d,F,rows,steps,nd,simt", REAL,
                         ids=[f"{d}x{F}x{rows}-{kind}" + (f"-nd{nd}" if nd else "") + ("-simt" if simt else "") for kind, d, F, rows, _, nd, simt in REAL])
def test_real_size_steps_match_float64_oracle(kind, d, F, rows, steps, nd, simt):
    got = _routes(kind, d, F, rows, nd, simt)
    assert set(got.values()) == {"ffma" if simt else "tc"}, f"test premise: {got}"
    if kind == "tc_topk":
        assert F > TOPK_SEG, "test premise: the segmented TopK"
    _steps_match_oracle(kind, d, F, rows, "layer_norm", steps, seed=d + F + rows + nd, nd=nd, simt=simt, expect=got)
    import gc
    gc.collect()


# ------------------------------------------------------------------------------------------------ the route table
def test_every_product_is_seen_on_both_routes():
    seen = {}
    for tag, kind in ROUTE_CASES:
        for n, r in _expected_routes(tag, kind, _axis_a_dead(SHAPES[tag][1]) if kind.endswith("ghost") else 0)[0].items():
            seen.setdefault(n, set()).add(r)
    for nd, kind in DEAD_CASES:
        for n, r in _routes(kind, 256, 2048, 512, nd).items():
            seen.setdefault(n, set()).add(r)
    names = ("encoder", "decoder", "d_acts", "gW_dec", "gW_encT", "skip", "gW_skip", "ghost_dE", "ghost_gWd", "ghost_gWe")
    assert set(seen) == set(names)
    assert all(seen[n] == {"tc", "ffma"} for n in names), {n: sorted(r) for n, r in seen.items()}


# ------------------------------------------------------------------------------------------------ d_in % 4 != 0
@pytest.mark.parametrize("kind", ["relu", "gated", "tc_relu_skip"])
def test_d_in_not_a_multiple_of_4_is_refused_when_the_engine_is_built(kind):
    """The per-row kernels and pb_rownorm_max read a d_in row as float4: building an engine at d_in = 66 raises before any
    kernel is launched, rather than running on a misaligned row."""
    from vit_prisma.b200 import _lib as L
    p, _, _, _ = _init(kind, 66, 1030, 64, 1, 66, 0)
    with pytest.raises(L.PrismaB200Error, match=r"pb_rownorm_max: bad arguments"):
        _engine(kind, p, "layer_norm", L.GEMM_AUTO)
