"""The three SAE optimizer kernels (csrc/sae_optim.cuh's sae_adam_feature inside k_sae_adam_bulk, k_sae_adam_rows and
k_p2p_adam_allgather) update the same state bit for bit, and the peer-memory optimizer trains like the reference on ONE GPU.

A one-rank P2PGroup (handles exchanged with itself, no torch.distributed) runs the data-parallel step's reduce-scatter,
Adam / all-gather and replicated small updates on a single H100: without a process group the multicast pool is off, so the
peer-store path (and, on the dense encoder route, its W_encT_lo plane) is what runs."""
import ctypes as C

import pytest
import torch

from tests.util import load_golden, rel_err

pytestmark = pytest.mark.gpu

MOMENTS = ("m_dec", "v_dec", "m_enc", "v_enc", "m_be", "v_be", "m_bd", "v_bd")
UPDATED = ("W_dec", "W_encT", "b_enc", "b_dec") + MOMENTS + ("since_fired", "act_freq", "enc_norm_max")
LR, BETAS, EPS = 3e-4, (0.9, 0.999), 1e-8


def make_state(d: int, F: int, step: int, seed: int) -> dict:
    """Seeded parameters, gradients, moments (zero at step 1) and dead-feature counters, on the CPU."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g)  # noqa: E731
    W_dec = r(F, d)
    st = dict(W_dec=W_dec / W_dec.norm(dim=1, keepdim=True), W_encT=0.1 * r(F, d), b_enc=0.1 * r(F), b_dec=0.1 * r(d),
              gW_dec=1e-3 * r(F, d), gW_encT=1e-3 * r(F, d), gb_enc=1e-3 * r(F), gb_dec=1e-3 * r(d))
    for name in MOMENTS:
        shape = (d,) if name.endswith("bd") else (F,) if name.endswith("be") else (F, d)
        if step == 1:
            st[name] = torch.zeros(shape)
        else:
            st[name] = 1e-3 * r(*shape) if name[0] == "m" else 1e-6 * r(*shape).square()
    st["fired"] = torch.randint(0, 4, (F,), generator=g).float() * (torch.rand(F, generator=g) < 0.5).float()
    st["since_fired"] = torch.randint(0, 50, (F,), generator=g).float()
    st["act_freq"] = torch.randint(0, 1000, (F,), generator=g).float()
    return st


def run_single_gpu(st: dict, step: int, clip: float, with_lo: bool, dev) -> dict:
    """pb_sae_adam on a copy of ``st`` with the clip coefficient written into the step scalars.  Without a W_encT_lo plane it
    launches k_sae_adam_bulk (k_sae_adam_rows below d = 64), with one k_sae_adam_rows + k_sae_adam_vec."""
    from vit_prisma.b200 import _lib as L
    from vit_prisma.b200.ops import _stream
    from vit_prisma.b200.sae_engine import PbSaeStep
    t = {k: v.clone().to(dev) for k, v in st.items()}
    F, d = t["W_dec"].shape
    t["scalars"] = torch.zeros(8, device=dev)
    t["scalars"][2] = clip
    t["enc_norm_max"] = torch.zeros(2, device=dev)
    t["W_encT_lo"] = torch.full_like(t["W_encT"], float("nan")) if with_lo else None
    s = PbSaeStep()
    s.d, s.F, s.step, s.renorm_decoder = d, F, step, 1
    s.lr, s.beta1, s.beta2, s.adam_eps = LR, BETAS[0], BETAS[1], EPS
    for name in ("W_encT", "W_encT_lo", "W_dec", "b_enc", "b_dec", "gW_dec", "gW_encT", "gb_enc", "gb_dec", "fired", "scalars",
                 "since_fired", "act_freq", "enc_norm_max") + MOMENTS:
        setattr(s, name, None if t[name] is None else t[name].data_ptr())
    L.check(L.get_lib().pb_sae_adam(C.byref(s), _stream()), "pb_sae_adam")
    torch.cuda.synchronize()
    return t


def run_peer(st: dict, step: int, max_norm: float, encoder: str, dev) -> dict:
    """The data-parallel optimizer of a one-rank SaeDPEngine: gradients written into its shared buffers, then barrier ->
    reduce-scatter -> barrier -> Adam / all-gather (+ b_dec, counters) -> barrier -> encoder-norm maxima."""
    from vit_prisma.b200 import _lib as L
    from vit_prisma.b200.ops import _stream
    from vit_prisma.b200.p2p import P2PGroup, SaeDPEngine
    lib, stream = L.get_lib(), _stream()
    F, d = st["W_dec"].shape
    group = P2PGroup(0, 1, dev, exchange=lambda mine: [mine])
    eng = SaeDPEngine(group, st["W_encT"].to(dev), st["W_dec"].to(dev), st["b_enc"].to(dev), st["b_dec"].to(dev), k=8,
                      max_grad_norm=max_norm, betas=BETAS, adam_eps=EPS, encoder=encoder)
    assert eng.mc is None
    for name in ("gW_dec", "gW_encT", "gb_enc", "gb_dec", "fired") + MOMENTS:
        getattr(eng, name).copy_(st[name])
    since_fired, act_freq = st["since_fired"].to(dev), st["act_freq"].to(dev)
    eng.scalars.zero_()
    eng.step_count = step
    ps = eng._p2p_desc(1, LR, since_fired, act_freq)
    group.barrier(ps)
    L.check(lib.pb_p2p_reduce_scatter(C.byref(ps), stream), "pb_p2p_reduce_scatter")
    group.barrier(ps)
    L.check(lib.pb_p2p_adam_allgather(C.byref(ps), stream), "pb_p2p_adam_allgather")
    group.barrier(ps)
    L.check(lib.pb_p2p_wmax(C.byref(ps), eng.enc_norm_max.data_ptr(), stream), "pb_p2p_wmax")
    torch.cuda.synchronize()
    out = {name: getattr(eng, name) for name in ("W_dec", "W_encT", "b_enc", "b_dec", "W_encT_lo", "enc_norm_max", "scalars") + MOMENTS}
    out.update(since_fired=since_fired, act_freq=act_freq)
    return out


def optimizer_paths(d: int, F: int, step: int, clip_active: bool, seed: int = 0) -> dict:
    """Every optimizer path on the same inputs, per encoder route of the peer engine: {"fused" | "dense": {"peer" | "bulk" |
    "rows": {tensor name: result}}, "vec": {...}}.  The single-GPU paths take the clip coefficient the peer path computed (its
    norm is summed by atomics, so the coefficient's last bit can change from run to run); it is exactly 1 when clipping is off."""
    from vit_prisma.b200 import _lib as L
    from vit_prisma.b200.ops import _stream
    dev = torch.device("cuda")
    st = make_state(d, F, step, seed)
    out = {}
    for encoder in ("fused", "dense"):
        peer = run_peer(st, step, 1e-3 if clip_active else 0.0, encoder, dev)
        clip = peer["scalars"][2].item()
        assert (clip < 1.0) == clip_active
        out[encoder] = {"peer": peer, "bulk": run_single_gpu(st, step, clip, False, dev), "rows": run_single_gpu(st, step, clip, True, dev)}
    # b_dec through the flat-vector entry point the Gated SAE and the Transcoder use for their extra parameters
    b, m, v = st["b_dec"].to(dev), st["m_bd"].to(dev), st["v_bd"].to(dev)
    L.check(L.get_lib().pb_adam_vec(b.data_ptr(), st["gb_dec"].to(dev).data_ptr(), m.data_ptr(), v.data_ptr(), d,
                                    out["fused"]["bulk"]["scalars"].data_ptr(), LR, BETAS[0], BETAS[1], EPS, step, _stream()), "pb_adam_vec")
    torch.cuda.synchronize()
    out["vec"] = {"b_dec": b, "m_bd": m, "v_bd": v}
    return out


@pytest.mark.parametrize("clip_active", [False, True])
@pytest.mark.parametrize("step", [1, 7])
@pytest.mark.parametrize("d,F", [(32, 256), (100, 384), (768, 1024), (1536, 512)])
def test_optimizer_paths_agree_bitwise(d, F, step, clip_active):
    from vit_prisma.b200 import ops
    out = optimizer_paths(d, F, step, clip_active)
    for encoder in ("fused", "dense"):
        ref = out[encoder]["bulk"]
        for path in ("rows", "peer"):
            for name in UPDATED:
                assert torch.equal(out[encoder][path][name], ref[name]), f"{path} vs bulk ({encoder} peer engine): {name} differs"
        assert torch.equal(out[encoder]["rows"]["W_encT_lo"], ops.split_tf32(ref["W_encT"])), "rows: W_encT_lo is not split_tf32(W_encT)"
        assert ref["enc_norm_max"][0].item() > 0.0
    assert out["fused"]["peer"]["W_encT_lo"] is None
    assert torch.equal(out["dense"]["peer"]["W_encT_lo"], ops.split_tf32(out["dense"]["bulk"]["W_encT"])), "peer: W_encT_lo is not split_tf32"
    for name in ("b_dec", "m_bd", "v_bd"):
        assert torch.equal(out["vec"][name], out["fused"]["bulk"][name]), f"pb_adam_vec: {name} differs from pb_sae_adam's"


@pytest.mark.parametrize("encoder", ["fused", "dense"])
def test_one_rank_data_parallel_trainer_matches_reference(encoder):
    """tests/dp_worker.py at world 1: the golden TopK run trained through the one-rank SaeDPEngine, with the same bars."""
    from oracle.sae_oracle import lr_multiplier
    from vit_prisma.b200.p2p import P2PGroup, SaeDPEngine
    from vit_prisma.b200.sae_engine import unit_norm_rows_
    dev = torch.device("cuda")
    gold = load_golden("sae_tiny_b.pt")
    g = torch.Generator().manual_seed(gold["data_seed"])
    B, d, k, F = gold["batch"], gold["d_in"], gold["k"], gold["d_sae"]
    data = torch.randn(B * gold["n_steps"], d, generator=g) * 2.0 + torch.randn(d, generator=g)
    init = gold["init"]
    eng = SaeDPEngine(P2PGroup(0, 1, dev, exchange=lambda mine: [mine]), init["W_enc"].t().contiguous().to(dev), init["W_dec"].clone().to(dev),
                      init["b_enc"].clone().to(dev), init["b_dec"].clone().to(dev), k=k, normalize_activations=gold["norm"], max_grad_norm=1.0,
                      encoder=encoder)
    assert eng.encoder == encoder and eng.mc is None
    unit_norm_rows_(eng.W_dec)
    eng.refresh_lo()
    since_fired, act_freq = torch.zeros(F, device=dev), torch.zeros(F, device=dev)
    for s, rec in enumerate(gold["steps"]):
        x = data[s * B:(s + 1) * B].to(dev)
        eng.train_step(x, gold["lr"] * lr_multiplier(s, gold["warm_up_steps"], gold["total_steps"], gold["lr_end"]),
                       since_fired=since_fired, act_freq=act_freq)
        sc = eng.scalars_dict()
        assert abs(sc["mse"] - rec["mse"]) <= 1e-4 * abs(rec["mse"]), f"step {s}: mse {sc['mse']} vs {rec['mse']}"
        assert abs(sc["grad_norm"] - rec["grad_norm"]) <= 1e-4 * rec["grad_norm"], f"step {s}: grad_norm {sc['grad_norm']} vs {rec['grad_norm']}"
        assert torch.equal(eng.idx.cpu().long(), rec["topk_idx"]), f"step {s}: TopK indices differ"
        if "params_after" in rec:
            ref = rec["params_after"]
            ref_dec = ref["W_dec"] / ref["W_dec"].norm(dim=1, keepdim=True)
            for name, got, want in (("W_dec", eng.W_dec, ref_dec), ("W_enc", eng.W_encT.t(), ref["W_enc"]), ("b_dec", eng.b_dec, ref["b_dec"])):
                e = rel_err(got.cpu(), want)
                assert e <= 1e-4, f"step {s}: {name} rel err {e:.2e}"
    assert torch.equal(since_fired.cpu(), gold["since_fired"]) and torch.equal(act_freq.cpu(), gold["act_freq"])
