"""The oracle's support overrides (``relu_mask``, ``gate_mask`` / ``mag_mask``, ``topk_idx``) are pure pass-throughs: handing a
training step the support its own default computes reproduces the default step exactly -- losses, raw gradients, updated
parameters, Adam moments and dead-feature counters bit for bit.  The GPU step tests feed the oracle an engine's support, so an
override that changed anything but the support would shift every comparison built on it."""
import math

import pytest
import torch

from oracle.sae_oracle import (GATED_PARAMS, gated_train_step, new_adam_state, normalise_in, sae_forward, sae_train_step,
                               transcoder_train_step)

D, F, ROWS, K = 24, 96, 40, 6


def _bits(t):
    return t.detach().double().view(torch.int64) if torch.is_tensor(t) else torch.tensor([t], dtype=torch.float64).view(torch.int64)


def _assert_same(a, b, what):
    if isinstance(a, dict):
        assert a.keys() == b.keys(), what
        for n in a:
            _assert_same(a[n], b[n], f"{what}.{n}")
    elif a is None or isinstance(a, (bool, int)):
        assert a == b, what
    elif torch.is_tensor(a) and a.dtype == torch.bool:
        assert torch.equal(a, b), what
    else:
        # relu(h) and h * False differ only in the sign of a zero; every value the step computes is compared bit for bit
        assert torch.equal(_bits(a + 0.0), _bits(b + 0.0)), what


def _params(g, extra=()):
    p = {"W_enc": torch.randn(D, F, generator=g, dtype=torch.float64) / math.sqrt(D),
         "W_dec": torch.randn(F, D, generator=g, dtype=torch.float64),
         "b_enc": 0.1 * torch.randn(F, generator=g, dtype=torch.float64), "b_dec": 0.1 * torch.randn(D, generator=g, dtype=torch.float64)}
    for name, shape in extra:
        p[name] = 0.1 * torch.randn(*shape, generator=g, dtype=torch.float64)
    return p


def _two_runs(step, p, masks_of):
    """Runs ``step`` twice on copies of ``p``: with its default support, and with that support handed back to it."""
    runs = []
    for masks in (None, "own"):
        q = {n: v.clone() for n, v in p.items()}
        st = new_adam_state(q)
        sf, af = torch.zeros(F, dtype=torch.float64), torch.zeros(F, dtype=torch.float64)
        sf[::5] = 10.0                                                   # dead features for the ghost term
        kw = {} if masks is None else masks_of({n: v.clone() for n, v in p.items()})
        out = step(q, st, sf, af, kw)
        runs.append((q, st, sf, af, out))
    return runs


def _compare(runs, keys):
    (q0, s0, sf0, af0, o0), (q1, s1, sf1, af1, o1) = runs
    _assert_same(q0, q1, "params")
    _assert_same(s0, s1, "adam state")
    _assert_same(sf0, sf1, "since_fired")
    _assert_same(af0, af1, "act_freq")
    for k in keys:
        _assert_same(o0[k], o1[k], k)


@pytest.mark.parametrize("act,ghost,norm", [("relu", False, "layer_norm"), ("relu", True, "none"), ("topk", True, "constant_norm_rescale"),
                                            ("topk", False, "layer_norm")])
def test_sae_step_with_its_own_support_is_unchanged(act, ghost, norm):
    g = torch.Generator().manual_seed(11)
    p = _params(g)
    x = torch.randn(ROWS, D, generator=g, dtype=torch.float64) * 2.0 + torch.randn(D, generator=g, dtype=torch.float64)

    def step(q, st, sf, af, kw):
        return sae_train_step(q, st, x, K, 1e-3, 1, mode=norm, since_fired=sf, act_freq=af, act=act, l1_coefficient=3e-3,
                              use_ghost_grads=ghost, dead_feature_window=5, **kw)

    def own(q):
        q["W_dec"] /= torch.norm(q["W_dec"], dim=1, keepdim=True)
        fwd = sae_forward(q, x, K, norm, act=act)
        return {"relu_mask": fwd["hidden_pre"] > 0} if act == "relu" else {"topk_idx": fwd["idx"]}

    runs = _two_runs(step, p, own)
    assert runs[0][4]["n_dead"] == (len(range(0, F, 5)) if ghost else 0)
    _compare(runs, ("loss", "mse", "l1", "ghost", "l0", "grad_norm", "raw_grads"))


def test_gated_step_with_its_own_masks_is_unchanged():
    g = torch.Generator().manual_seed(12)
    p = _params(g, (("r_mag", (F,)), ("b_mag", (F,))))
    p["b_gate"] = p.pop("b_enc")
    p = {n: p[n] for n in GATED_PARAMS}
    x = torch.randn(ROWS, D, generator=g, dtype=torch.float64) * 2.0 + torch.randn(D, generator=g, dtype=torch.float64)

    def step(q, st, sf, af, kw):
        return gated_train_step(q, st, x, 1e-3, 1, "layer_norm", 3e-3, since_fired=sf, act_freq=af, **kw)

    def own(q):
        q["W_dec"] /= torch.norm(q["W_dec"], dim=1, keepdim=True)
        u = (normalise_in(x, "layer_norm")[0] - q["b_dec"]) @ q["W_enc"]
        return {"gate_mask": u + q["b_gate"] > 0, "mag_mask": u * q["r_mag"].exp() + q["b_mag"] > 0}

    runs = _two_runs(step, p, own)
    assert 0 < int(runs[0][4]["active"].sum()) < ROWS * F
    _compare(runs, ("loss", "mse", "l1", "aux", "l0", "grad_norm", "raw_grads", "sae_out", "feature_acts"))


@pytest.mark.parametrize("act,skip", [("relu", True), ("topk", False)])
def test_transcoder_step_with_its_own_support_is_unchanged(act, skip):
    g = torch.Generator().manual_seed(13)
    p = _params(g, (("b_dec_out", (D,)),) + ((("W_skip", (D, D)),) if skip else ()))
    x = torch.randn(ROWS, D, generator=g, dtype=torch.float64) * 2.0 + torch.randn(D, generator=g, dtype=torch.float64)
    y = torch.tanh(x) + 0.3 * torch.randn(ROWS, D, generator=g, dtype=torch.float64)

    def step(q, st, sf, af, kw):
        return transcoder_train_step(q, st, x, y, 1e-3, 1, "layer_norm", act, K, 3e-3, since_fired=sf, act_freq=af, **kw)

    def own(q):
        q["W_dec"] /= torch.norm(q["W_dec"], dim=1, keepdim=True)
        hp = sae_forward(q, x, K, "layer_norm")["hidden_pre"]              # the transcoder's encoder is the SAE's
        return {"relu_mask": hp > 0} if act == "relu" else {"topk_idx": torch.topk(hp, K, dim=-1).indices}

    runs = _two_runs(step, p, own)
    _compare(runs, ("loss", "mse", "l1", "l0", "grad_norm", "raw_grads", "sae_out", "feature_acts"))
