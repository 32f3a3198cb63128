"""Three TopK-SAE training steps at every d_in width the step kernels are instantiated for, against the float64 oracle.

The per-row kernels of the step (k_sae_prep, k_sae_decode, k_sae_grads, k_sae_grads_long, k_sae_adam_bulk / k_sae_adam_rows) hold
a d_in row as CHUNKS float4 per lane, CHUNKS in {1, 2, 4, 6, 8, 12} for d_in up to 128, 256, 512, 768, 1024, 1536 (chunks_for in
csrc/sae_optim.cuh; both Adam kernels run its sae_adam_feature).  The widths below take every instance, full and with idle lanes
in the last chunk, on both encoder routes:

  * fused: tf32 candidate GEMM + exact re-scoring, Adam in the bulk-copy pipeline (its ring depth varies with d) or, below
    d = 64, in the rows kernel;
  * dense (GEMM_TC): 3xTF32 encoder GEMM + k_topk, Adam in the rows kernel, which also maintains the tf32 residual plane W_encT_lo.

Three consecutive steps take Adam past its first step (moments and bias correction).  A decoder bias far from the data makes a
few features fire on most tokens, so their per-feature lists take the long-list kernels (k_sae_grads_long, k_sae_norm_long).
Bars as elsewhere in the suite: 1e-4 relative (max-norm) for the loss, the gradient norm, sae_out, the raw gradients and the
parameters; TopK indices equal except rows with a near-tie; dead-feature counters exact.

The encoder and the selection are checked first, against float64 hidden_pre.  The oracle's step then takes the engine's TopK
support, so that a near-tie row the engine legitimately resolves the other way (one such row turns sae_out 0.11 and the
gradients 5e-3 away from the oracle's) does not hide the rest of the step.  On the dense route the oracle also takes the
engine's TopK values: the 3xTF32 encoder GEMM accumulates ceil(d / 8) wgmma k-steps in fp32, and its hidden_pre was measured
(H100 80GB HBM3, 400 W) 4.6e-7 (d = 32) to 1.3e-5 (d = 1536) of max |hidden_pre| from float64 -- inside the 1e-4 bar, which is
asserted, but Adam divides every gradient element by its own magnitude, and for elements near eps that turned 1e-5-relative
gradient differences into W_dec differences of up to 1.8e-4.  The near-tie width on the dense route is twice the measured
hidden_pre error; on the fused route, whose selected values are exact fp32, it is 2e-6 of max |hidden_pre| as for cfg #3.
After every step the invariants
the next step relies on are checked directly: unit-norm decoder rows, W_encT_lo == split_tf32(W_encT) bit for bit, and
enc_norm_max (an input to the fused encoder's error bound) not below the float64 norms of W_enc.
"""
import math

import pytest
import torch

from oracle.fused_topk_model import tf32_trunc
from oracle.sae_oracle import new_adam_state, sae_forward, sae_grads, sae_train_step
from tests.util import rel_err

pytestmark = pytest.mark.gpu

WIDTHS = (32, 64, 100, 200, 384, 520, 768, 1000, 1024, 1536)
NORMS = ("none", "layer_norm", "constant_norm_rescale")
ROWS, K, STEPS, LR = 300, 16, 3, 1e-3


def _d_sae(d):
    return min(8192, max(128, round(4 * d / 128) * 128))


CASES = [(d, route, NORMS[(j + r) % 3], j % 2 == r) for j, d in enumerate(WIDTHS) for r, route in enumerate(("fused", "dense"))]


@pytest.mark.parametrize("d,route,norm,clip", CASES)
def test_three_steps_match_float64_oracle(d, route, norm, clip):
    from vit_prisma.b200 import _lib as L
    from vit_prisma.b200 import ops
    from vit_prisma.b200.sae_engine import SaeStepEngine, unit_norm_rows_
    F = _d_sae(d)
    g = torch.Generator().manual_seed(1000 * d + (route == "dense"))
    W_enc = torch.randn(d, F, generator=g) / math.sqrt(d)
    W_dec = torch.randn(F, d, generator=g)
    W_dec /= W_dec.norm(dim=1, keepdim=True)
    b_enc = 0.01 * torch.randn(F, generator=g)
    b_dec = 3.0 * torch.randn(d, generator=g)                          # far from the data: hot features
    xs = [torch.randn(ROWS, d, generator=g) * 2.0 + torch.randn(d, generator=g) for _ in range(STEPS)]

    p = {"W_enc": W_enc.double(), "W_dec": W_dec.double(), "b_enc": b_enc.double(), "b_dec": b_dec.double()}
    # the clipping threshold from the first step's gradient norm: active at every step (a tenth of it) or never (four times it)
    fwd = sae_forward(p, xs[0].double(), K, norm)
    gn0 = math.sqrt(sum(float((v ** 2).sum()) for v in sae_grads(p, xs[0].double(), fwd, norm).values()))
    max_grad_norm = 0.1 * gn0 if clip else 4.0 * gn0
    counts = torch.bincount(fwd["idx"].reshape(-1), minlength=F)
    assert int(counts.max()) > 32, "test premise: a feature with more than 32 tokens (the long-list kernels)"

    eng = SaeStepEngine(W_enc.t().contiguous().cuda(), W_dec.clone().cuda(), b_enc.clone().cuda(), b_dec.clone().cuda(), k=K,
                        normalize_activations=norm, max_grad_norm=max_grad_norm,
                        gemm_impl=L.GEMM_AUTO if route == "fused" else L.GEMM_TC)
    assert eng.encoder == route
    unit_norm_rows_(eng.W_dec)
    eng.refresh_lo()
    state = new_adam_state(p)
    since, freq = torch.zeros(F, device="cuda"), torch.zeros(F, device="cuda")
    since_ref, freq_ref = torch.zeros(F, dtype=torch.float64), torch.zeros(F, dtype=torch.float64)
    for s, x in enumerate(xs):
        at = f"d={d} {route} {norm} step {s + 1}"
        eng.train_step(x.cuda(), LR, since_fired=since, act_freq=freq, want_out=True)
        sc = eng.scalars_dict()
        idx, val = eng.idx.cpu().long(), eng.val.cpu().double()
        # the encoder and the TopK selection against float64 (W_dec does not enter hidden_pre)
        hp = sae_forward(p, x.double(), K, norm)["hidden_pre"]
        if route == "dense":
            assert rel_err(eng.hidden_pre, hp) <= 1e-4, f"{at}: hidden_pre rel err {rel_err(eng.hidden_pre, hp):.2e}"
            tie = 2.0 * float((eng.hidden_pre.cpu().double() - hp).abs().max())
        else:
            tie = 2e-6 * float(hp.abs().max())
        top = torch.topk(hp, K + 1, dim=-1)
        same = (idx == top.indices[:, :K]).all(dim=1)
        near = (top.values[:, :-1] - top.values[:, 1:]).abs().min(dim=1).values < tie
        assert bool((same | near).all()), f"{at}: {(~(same | near)).sum().item()} rows select other features than the oracle"
        assert bool((hp.gather(1, idx) >= top.values[:, K - 1:K] - tie).all()), f"{at}: a selected feature is not a near-top-k one"
        assert rel_err(val, hp.gather(1, idx)) <= 1e-4, f"{at}: TopK values rel err {rel_err(val, hp.gather(1, idx)):.2e}"
        ref = sae_train_step(p, state, x.double(), K, LR, s + 1, mode=norm, max_grad_norm=max_grad_norm, since_fired=since_ref,
                             act_freq=freq_ref, topk_idx=idx, topk_val=val if route == "dense" else None)
        assert (ref["clip"] < 1.0) == clip and (sc["clip_coef"] < 1.0) == clip, (at, ref["clip"], sc["clip_coef"])
        raw, ref_dec = ref["raw_grads"], p["W_dec"] / p["W_dec"].norm(dim=1, keepdim=True)    # the oracle renormalises next step
        errs = {"mse": abs(sc["mse"] / float(ref["mse"]) - 1), "grad_norm": abs(sc["grad_norm"] / float(ref["grad_norm"]) - 1),
                "clip_coef": abs(sc["clip_coef"] / ref["clip"] - 1), "sae_out": rel_err(eng.sae_out, ref["fwd"]["sae_out"]),
                "dL/dW_dec": rel_err(eng.gW_dec, raw["W_dec"]), "dL/dW_enc": rel_err(eng.gW_encT.t(), raw["W_enc"]),
                "dL/db_enc": rel_err(eng.gb_enc, raw["b_enc"]), "dL/db_dec": rel_err(eng.gb_dec, raw["b_dec"]),
                "W_dec": rel_err(eng.W_dec, ref_dec), "W_enc": rel_err(eng.W_encT.t(), p["W_enc"]),
                "b_enc": rel_err(eng.b_enc, p["b_enc"]), "b_dec": rel_err(eng.b_dec, p["b_dec"])}
        bad = {n: f"{e:.2e}" for n, e in errs.items() if e > 1e-4}
        assert not bad, f"{at}: beyond 1e-4 of the float64 oracle: {bad}; all: { {n: f'{e:.1e}' for n, e in errs.items()} }"
        assert torch.equal(since.cpu().double(), since_ref) and torch.equal(freq.cpu().double(), freq_ref), f"{at}: dead-feature counters"
        # invariants the next step depends on
        W_dec_now, W_encT_now = eng.W_dec.cpu().double(), eng.W_encT.cpu()
        assert (W_dec_now.norm(dim=1) - 1.0).abs().max().item() <= 1e-5, f"{at}: decoder rows not unit-norm"
        if route == "dense":
            assert torch.equal(eng.W_encT_lo.view(torch.int32), ops.split_tf32(eng.W_encT).view(torch.int32)), f"{at}: W_encT_lo stale"
        W64 = W_encT_now.double()
        lo64 = W64 - torch.from_numpy(tf32_trunc(W_encT_now.numpy())).double()
        want = torch.tensor([W64.norm(dim=1).max().item(), lo64.norm(dim=1).max().item()], dtype=torch.float64)
        got = eng.enc_norm_max.cpu().double()
        assert bool((got >= want * (1 - 1e-5)).all()), f"{at}: enc_norm_max {got.tolist()} below the float64 norms {want.tolist()}"
        assert bool((got <= want * (1 + 1e-5)).all()), f"{at}: enc_norm_max {got.tolist()} far above the float64 norms {want.tolist()}"
