"""Pin the oracle (oracle/vit_oracle.py) to fixtures produced by the unmodified reference.

CPU-only: this is the "is the checker right" gate; the CUDA path is then checked against the oracle
and the same fixtures in test_vit_gpu.py."""
import pytest
import torch

from oracle.vit_oracle import CLIP_B32, digest, recipe_state_dict, state_dict_shapes, vit_forward_with_cache
from tests.util import assert_close, load_golden

TOL = {"fp32": 2e-5, "bf16": 1.6e-2}


def _images(batch, cfg, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(batch, cfg["n_channels"], cfg["image_size"], cfg["image_size"], generator=g)


@pytest.mark.parametrize("tag", ["a", "b", "c", "d"])
@pytest.mark.parametrize("dname", ["fp32", "bf16"])
def test_oracle_matches_reference_tiny(tag, dname):
    gold = load_golden(f"vit_tiny_{tag}_{dname}.pt")
    cfg = dict(gold["cfg"])
    dtype = torch.float32 if dname == "fp32" else torch.bfloat16
    cfg["dtype"] = dtype
    assert state_dict_shapes(cfg) == gold["shapes"], "state-dict layout drifted from the reference"
    sd = recipe_state_dict(gold["shapes"], gold["weights_seed"], dtype)
    x = _images(gold["batch"], cfg, gold["images_seed"]).to(dtype)
    out, cache = vit_forward_with_cache(sd, cfg, x)
    assert list(cache.keys()) == gold["keys"], "cache key order differs from the reference"
    for k in gold["keys"]:
        assert_close(cache[k], gold["cache"][k], TOL[dname], k)
    assert_close(out, gold["out"], TOL[dname], "model output")
    # names_filter + stop_at_layer exactly as VisionActivationsStore.get_activations uses them
    flt = ["blocks.0.hook_resid_post", "blocks.1.ln1.hook_normalized"]
    stop_out, stop_cache = vit_forward_with_cache(sd, cfg, x, names_filter=lambda n: n in flt, stop_at_layer=1)
    assert list(stop_cache.keys()) == gold["stop_keys"]
    assert_close(stop_out, gold["stop_out"], TOL[dname], "stop_at_layer output")


def test_oracle_matches_reference_clip_b32_digest():
    gold = load_golden("vit_b32_fp32_digest.pt")
    cfg = dict(gold["cfg"])
    assert cfg == CLIP_B32
    sd = recipe_state_dict(state_dict_shapes(cfg), gold["weights_seed"])
    x = _images(gold["batch"], cfg, gold["images_seed"])
    out, cache = vit_forward_with_cache(sd, cfg, x)
    assert list(cache.keys()) == gold["keys"]
    assert len(cache) == 214
    assert sum(v.numel() * v.element_size() for v in cache.values()) == gold["bytes_materialised"] == 4 * 38_980_176
    for k, dg in gold["digests"].items():
        mine = digest(cache[k])
        assert mine["shape"] == dg["shape"] and mine["dtype"] == dg["dtype"], k
        scale = max(dg["max_abs"], 1e-30)
        assert (mine["samples"] - dg["samples"]).abs().max().item() / scale < 2e-5, k
        assert abs(mine["sum"] - dg["sum"]) <= 2e-5 * max(dg["abs_sum"], 1e-30), k
    assert_close(out, gold["out"], 2e-5, "model output")


# ------------------------------------------------------------------------------------------ SAE
from oracle.sae_oracle import lr_multiplier, new_adam_state, sae_forward, sae_train_step  # noqa: E402


def _sae_data(gold):
    g = torch.Generator().manual_seed(gold["data_seed"])
    n, d = gold["batch"] * gold["n_steps"], gold["d_in"]
    return torch.randn(n, d, generator=g) * 2.0 + torch.randn(d, generator=g)


@pytest.mark.parametrize("tag", ["a", "b", "c", "d", "e", "f"])
def test_sae_oracle_matches_reference_training(tag):
    """Forward, TopK support, closed-form gradients, clipping, projection, Adam and the LR schedule of the oracle
    against torch autograd + torch.optim.Adam driving the reference's own SAE module for 6 steps.
    d: dense ReLU + L1; e: TopK + ghost grads (112-122 dead features from step 2); f: ReLU + L1 + ghost grads (77 dead)."""
    gold = load_golden(f"sae_tiny_{tag}.pt")
    data = _sae_data(gold)
    p = {k: v.clone() for k, v in gold["init"].items()}
    state = new_adam_state(p)
    since_fired, act_freq = torch.zeros(gold["d_sae"]), torch.zeros(gold["d_sae"])
    B, k = gold["batch"], gold["k"]
    for s, rec in enumerate(gold["steps"]):
        x = data[s * B:(s + 1) * B]
        lr = gold["lr"] * lr_multiplier(s, gold["warm_up_steps"], gold["total_steps"], gold["lr_end"])
        assert abs(lr - rec["lr"]) < 1e-12
        out = sae_train_step(p, state, x, k, lr, s + 1, mode=gold["norm"], since_fired=since_fired, act_freq=act_freq, act=gold["act"],
                             l1_coefficient=gold["l1_coefficient"], use_ghost_grads=gold["use_ghost_grads"],
                             dead_feature_window=gold["dead_feature_window"])
        if gold["act"] == "topk":
            assert torch.equal(out["idx"], rec["topk_idx"]), f"step {s}: TopK indices differ"
        else:
            assert torch.equal(torch.topk(out["fwd"]["hidden_pre"], 4, dim=-1).indices, rec["topk_idx"])
            assert abs(out["l1"].item() - rec["l1"]) <= 1e-5 * abs(rec["l1"])
        assert out["n_dead"] == rec["n_dead"]
        assert abs(out["ghost"].item() - rec["ghost"]) <= 2e-5 * abs(rec["ghost"]) + 1e-12
        assert abs(out["loss"].item() - rec["loss"]) <= 1e-5 * abs(rec["loss"])
        assert abs(out["mse"].item() - rec["mse"]) <= 1e-5 * abs(rec["mse"])
        assert abs(out["grad_norm"].item() - rec["grad_norm"]) <= 1e-4 * rec["grad_norm"]
        assert abs(out["l0"].item() - rec["l0"]) < 1e-6
        assert_close(out["fwd"]["sae_out"], rec["sae_out"], 1e-5, f"step {s} sae_out")
        # ghost term: d/dG [c * (G-r)^2/rcn] with c = mse / ((G-r)^2/rcn + 1e-6) divides by elements that can be ~1e-6, so fp32
        # round-off in (G - r) is amplified; the reference's own fp32 autograd and this closed form agree to ~1e-4 there
        gtol = 5e-4 if rec["n_dead"] else 2e-5
        if "raw_grads" in rec:
            for n in p:
                assert_close(out["raw_grads"][n], rec["raw_grads"][n], gtol, f"step {s} raw grad {n}")
                assert_close(out["grads"][n], rec["final_grads"][n], gtol, f"step {s} clipped+projected grad {n}")
        if "params_after" in rec:
            for n in p:
                assert_close(p[n], rec["params_after"][n], 5e-4 if gold["use_ghost_grads"] else 2e-5, f"step {s} param {n}")
    assert torch.equal(since_fired, gold["since_fired"]) and torch.equal(act_freq, gold["act_freq"])


@pytest.mark.parametrize("tag", ["g", "h"])
def test_gated_sae_oracle_matches_reference_training(tag):
    """GatedSparseAutoencoder (sae.py:648-792) for 6 steps under autograd + torch.optim.Adam vs the closed-form oracle:
    loss terms, all six parameter gradients (b_enc never enters the graph: grad None in the reference), parameters, counters."""
    from oracle.sae_oracle import GATED_PARAMS, gated_train_step
    gold = load_golden(f"sae_gated_{tag}.pt")
    g = torch.Generator().manual_seed(gold["data_seed"])
    n, d = gold["batch"] * gold["n_steps"], gold["d_in"]
    data = torch.randn(n, d, generator=g) * 2.0 + torch.randn(d, generator=g)
    p = {k: gold["init"][k].clone() for k in GATED_PARAMS}
    state = new_adam_state(p)
    since_fired, act_freq = torch.zeros(gold["d_sae"]), torch.zeros(gold["d_sae"])
    B = gold["batch"]
    for s, rec in enumerate(gold["steps"]):
        x = data[s * B:(s + 1) * B]
        lr = gold["lr"] * lr_multiplier(s, gold["warm_up_steps"], gold["total_steps"], gold["lr_end"])
        out = gated_train_step(p, state, x, lr, s + 1, gold["norm"], gold["l1_coefficient"], since_fired=since_fired, act_freq=act_freq)
        for name in ("loss", "mse", "l1", "aux"):
            assert abs(out[name].item() - rec[name]) <= 2e-5 * abs(rec[name]), (s, name, out[name].item(), rec[name])
        assert abs(out["grad_norm"].item() - rec["grad_norm"]) <= 1e-4 * rec["grad_norm"]
        assert_close(out["sae_out"], rec["sae_out"], 1e-5, f"step {s} sae_out")
        assert torch.equal(out["feature_acts"] > 0, rec["feature_acts"] > 0)
        if "raw_grads" in rec:
            assert rec["raw_grads"]["b_enc"] is None
            for name in GATED_PARAMS:
                assert_close(out["raw_grads"][name], rec["raw_grads"][name], 5e-5, f"step {s} raw grad {name}")
                assert_close(out["grads"][name], rec["final_grads"][name], 5e-5, f"step {s} clipped+projected grad {name}")
        if "params_after" in rec:
            for name in GATED_PARAMS:
                assert_close(p[name], rec["params_after"][name], 5e-5, f"step {s} param {name}")
    assert torch.equal(since_fired, gold["since_fired"]) and torch.equal(act_freq, gold["act_freq"])


def test_geometric_median_matches_reference_fixture():
    """b_dec_init_method="geometric_median" (reference sae/training/geometric_median.py:23-85; train_sae.py:245-276): our Weiszfeld
    iteration against medians computed by the unmodified reference (tests/golden/make_golden_median.py), with and without outliers."""
    from vit_prisma.sae.training.geometric_median import compute_geometric_median
    for case in load_golden("geometric_median.pt"):
        g = torch.Generator().manual_seed(case["seed"])
        n, d = case["n"], case["d"]
        pts = torch.randn(n, d, generator=g) * 2.0 + torch.randn(d, generator=g)
        if case["outliers"]:
            pts[:case["outliers"]] += 25.0 * torch.randn(case["outliers"], d, generator=g)
        out = compute_geometric_median(pts, maxiter=case["maxiter"])
        assert out.termination == case["termination"]
        err = (out.median - case["median"]).abs().max().item() / case["median"].abs().max().item()
        assert err <= 1e-5, (case["seed"], err)
        if case["outliers"]:
            assert (case["median"] - case["mean"]).norm() > 0.1          # the fixture really distinguishes median from mean


def test_sae_oracle_follows_the_fp32_twin_of_the_bf16_fixture():
    """sae_bf16_v.pt (cfg #5 shape class): the reference run in fp32 from bf16-rounded initial parameters and data -- the trajectory
    the product's fp32-master step must follow -- is reproduced by the oracle; its bf16 run stays within bf16 noise of it."""
    gold = load_golden("sae_bf16_v.pt")
    p = {k: v.float().clone() for k, v in gold["init"].items()}
    state = new_adam_state(p)
    data, B, k = gold["data"].float(), gold["batch"], gold["k"]
    for s, (rec16, rec32) in enumerate(zip(gold["steps"], gold["steps_fp32"])):
        lr = gold["lr"] * lr_multiplier(s, gold["warm_up_steps"], gold["total_steps"], gold["lr_end"])
        assert abs(lr - rec32["lr"]) < 1e-12
        out = sae_train_step(p, state, data[s * B:(s + 1) * B], k, lr, s + 1, mode=gold["norm"])
        assert abs(out["mse"].item() - rec32["mse"]) <= 1e-5 * abs(rec32["mse"])
        assert abs(out["grad_norm"].item() - rec32["grad_norm"]) <= 1e-4 * rec32["grad_norm"]
        assert_close(out["fwd"]["sae_out"], rec32["sae_out"], 1e-5, f"step {s} sae_out")
        for n in p:
            assert_close(p[n], rec32["params_after"][n], 2e-5, f"step {s} param {n}")
        assert abs(rec16["mse"] - rec32["mse"]) <= 1e-2 * rec32["mse"]
        assert rec16["params_after"]["W_dec"].dtype == torch.bfloat16


@pytest.mark.parametrize("tag", ["t", "u"])
def test_transcoder_oracle_matches_reference_training(tag):
    """transcoder_{t,u}.pt: the unmodified reference Transcoder (t: ReLU + L1, layer_norm, skip matrix; u: TopK, no normalisation, no skip)
    driven by autograd + torch.optim.Adam for 5 steps on (input, target) pairs -- forward, loss terms, all gradients (closed form
    here), clipping, decoder projection, Adam and the schedule."""
    from oracle.sae_oracle import transcoder_train_step
    gold = load_golden(f"transcoder_{tag}.pt")
    g = torch.Generator().manual_seed(gold["data_seed"])
    n, d = gold["batch"] * gold["n_steps"], gold["d"]
    x_all = torch.randn(n, d, generator=g) * 2.0 + torch.randn(d, generator=g)
    M = torch.randn(d, d, generator=g) / d ** 0.5
    y_all = torch.tanh(x_all @ M) * 1.5 + 0.3 * torch.randn(n, d, generator=g) + torch.randn(d, generator=g)
    p = {k: v.clone() for k, v in gold["init"].items()}
    assert ("W_skip" in p) == gold["skip"]
    state = new_adam_state(p)
    since_fired, act_freq = torch.zeros(gold["d_sae"]), torch.zeros(gold["d_sae"])
    B = gold["batch"]
    for s, rec in enumerate(gold["steps"]):
        lr = gold["lr"] * lr_multiplier(s, gold["warm_up_steps"], gold["total_steps"], gold["lr_end"])
        assert abs(lr - rec["lr"]) < 1e-12
        out = transcoder_train_step(p, state, x_all[s * B:(s + 1) * B], y_all[s * B:(s + 1) * B], lr, s + 1, gold["norm"], gold["act"], gold["k"],
                                    gold["l1_coefficient"], since_fired=since_fired, act_freq=act_freq)
        assert abs(out["loss"].item() - rec["loss"]) <= 1e-5 * abs(rec["loss"])
        assert abs(out["mse"].item() - rec["mse"]) <= 1e-5 * abs(rec["mse"])
        assert (out["l1"] is None) == (rec["l1"] is None)
        if rec["l1"] is not None:
            assert abs(out["l1"].item() - rec["l1"]) <= 1e-5 * abs(rec["l1"])
        assert abs(out["l0"].item() - rec["l0"]) < 1e-5
        assert abs(out["grad_norm"].item() - rec["grad_norm"]) <= 1e-4 * rec["grad_norm"]
        assert_close(out["sae_out"], rec["sae_out"], 1e-5, f"step {s} sae_out")
        if "feature_acts" in rec:
            assert_close(out["feature_acts"], rec["feature_acts"], 1e-5, "feature_acts")
        if "raw_grads" in rec:
            for name in p:
                assert_close(out["raw_grads"][name], rec["raw_grads"][name], 2e-5, f"step {s} grad {name}")
        if "params_after" in rec:
            for name in p:
                assert_close(p[name], rec["params_after"][name], 2e-5, f"step {s} param {name}")
    assert torch.equal(since_fired, gold["since_fired"]) and torch.equal(act_freq, gold["act_freq"])
