"""GPU parity tests of the individual kernels, through the C ABI, against the numpy oracle and the golden vectors.

Bars: scan outputs bit-exact up to one float32 rounding (the recurrence is carried in float64 exactly like the
reference: allow 1 ulp = 1.2e-7 relative); everything fp32 within 1e-5 of max|ref| (BASELINE.json north_star).
"""
import numpy as np
import pytest

from conftest import batch_of, load_golden, rel_err
from oracle import onpolicy as O

pytestmark = pytest.mark.gpu
TOL = 1e-5


def _rand_batch(rng, lens, f64=True):
    lens = np.asarray(lens, dtype=np.int64)
    n = int(lens.sum())
    rew = rng.standard_normal(n)
    if not f64:
        rew = rew.astype(np.float32)
    values = rng.standard_normal(n).astype(np.float32)
    last_values = rng.standard_normal(len(lens)).astype(np.float32)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    done = rng.random(len(lens)) < 0.5
    return rew, values, last_values, off, done


@pytest.mark.parametrize("lens,f64", [
    ([1], True), ([1, 1, 1, 1, 1], True), ([7], True), ([8], False), ([9, 1, 30], True),
    ([2048], True), ([2047, 1], True), ([2049], False), ([5000], True),            # multi-tile carry chains
    ([1000] * 8, True), ([1000] * 8, False), ([3, 4100, 1, 1, 2050, 17], True),
    (list(range(1, 200)), True), ([1] * 3000, True), ([12345, 6789, 1], True),
])
def test_gae_scan_matches_oracle(lens, f64):
    from gpu_helpers import gae_scan
    rng = np.random.default_rng(len(lens) * 7919 + int(sum(lens)))
    rew, values, last_values, off, done = _rand_batch(rng, lens, f64)
    adv, ret, stats = gae_scan(rew, values, last_values, off, done)
    adv_ref, ret_ref = O.gae_and_returns(rew, values, last_values, off, done, 0.99, 0.97)
    np.testing.assert_allclose(ret, ret_ref, rtol=2.4e-7, atol=1e-30)
    np.testing.assert_allclose(adv, adv_ref, rtol=2.4e-7, atol=2e-6 * np.abs(adv_ref).max())
    assert rel_err(adv, adv_ref) < 2.4e-7 and rel_err(ret, ret_ref) < 2.4e-7
    assert stats[2] == len(values)
    np.testing.assert_allclose(stats[0], adv.astype(np.float64).sum(), rtol=1e-12, atol=1e-9)
    np.testing.assert_allclose(stats[1], (adv.astype(np.float64) ** 2).sum(), rtol=1e-12)


def test_gae_scan_kats():
    from gpu_helpers import gae_scan
    g = load_golden("scan_kats")
    r, v = g["kat_r"], g["kat_v"]
    for tag, done in (("done", True), ("notdone", False)):
        adv, ret, _ = gae_scan(r, v[:3], v[3:], np.asarray([0, 3]), np.asarray([done]))
        np.testing.assert_allclose(adv, g["gae_" + tag].astype(np.float32), rtol=1.2e-7)
        np.testing.assert_allclose(ret, g["ret_" + tag].astype(np.float32), rtol=1.2e-7)


def test_gae_scan_empty():
    from gpu_helpers import gae_scan
    adv, ret, stats = gae_scan(np.zeros(0), np.zeros(0, np.float32), np.zeros(0, np.float32), np.asarray([0]), np.zeros(0, bool))
    assert adv.size == 0 and ret.size == 0 and stats[2] == 0


@pytest.mark.parametrize("case", ["ppo_categorical_cfg1", "ppo_gaussian_small", "ppo_gaussian_ragged_earlystop"])
def test_scan_against_reference_golden(case):
    from gpu_helpers import gae_scan
    g = load_golden(case)
    b = batch_of(g)
    adv, ret, _ = gae_scan(b["rew"], g["values"], g["last_values"], b["ep_offsets"], b["ep_done"])
    assert rel_err(ret, g["ret"]) < 2.4e-7
    assert rel_err(adv, g["adv_raw"]) < 2.4e-7


SHAPES = [([17, 64, 64, 6], "gaussian"), ([4, 64, 64, 2], "categorical"), ([27, 64, 64, 8], "gaussian"),
          ([17, 64, 32, 6], "gaussian"),  # the reference's own benchmark recipe (run_ppo.py:28): tensor-core path, padded
          ([9, 33, 20, 3], "categorical"), ([17, 24, 64, 6], "gaussian"),  # odd hidden widths, zero-padded to 64
          ([3, 16, 5], "categorical"), ([11, 64, 64, 64, 3], "gaussian")]  # 2 / 4 layers: fp32 kernel


def _net(rng, sizes):
    return [(rng.standard_normal((o, i)).astype(np.float32) / np.sqrt(i), 0.1 * rng.standard_normal(o).astype(np.float32))
            for i, o in zip(sizes[:-1], sizes[1:])]


@pytest.mark.parametrize("sizes,dist", SHAPES)
@pytest.mark.parametrize("n", [1, 63, 64, 65, 1000, 20011])
def test_eval_logp_and_value(sizes, dist, n):
    from gpu_helpers import loss_grad
    rng = np.random.default_rng(n + sizes[0])
    layers = _net(rng, sizes)
    obs = rng.standard_normal((n, sizes[0])).astype(np.float32)
    A = sizes[-1]
    log_std = (-0.5 + 0.1 * rng.standard_normal(A)).astype(np.float32) if dist == "gaussian" else None
    act = rng.standard_normal((n, A)).astype(np.float32) if dist == "gaussian" else rng.integers(0, A, n).astype(np.float32)
    r = loss_grad(sizes, O.flatten_layers(layers), obs, "eval", dist, act=act, log_std=log_std)
    d = O.Dist(dist, O.mlp_forward(layers, obs)[0], log_std)
    assert rel_err(r["rows"], d.log_prob(act)) < TOL
    np.testing.assert_allclose(r["scalars"][2], d.entropy().astype(np.float64).sum(), rtol=1e-5)
    np.testing.assert_allclose(r["scalars"][3], d.log_prob(act).astype(np.float64).sum(), rtol=1e-5)
    assert r["scalars"][5] == n
    # value head
    vs = sizes[:-1] + [1]
    vl = _net(rng, vs)
    rv = loss_grad(vs, O.flatten_layers(vl), obs, "eval", "none")
    assert rel_err(rv["rows"], O.mlp_forward(vl, obs)[0][:, 0]) < TOL


@pytest.mark.parametrize("sizes,dist", SHAPES)
@pytest.mark.parametrize("loss", ["ppo_clip", "vpg", "trpo_surrogate"])
@pytest.mark.parametrize("n", [50, 4097])
def test_policy_loss_grad(sizes, dist, loss, n):
    from gpu_helpers import loss_grad
    rng = np.random.default_rng(n * 3 + sizes[-1])
    layers = _net(rng, sizes)
    obs = rng.standard_normal((n, sizes[0])).astype(np.float32)
    A = sizes[-1]
    log_std = np.full(A, -0.5, np.float32) if dist == "gaussian" else None
    mean = O.mlp_forward(layers, obs)[0]
    act = (mean + np.exp(-0.5) * rng.standard_normal((n, A))).astype(np.float32) if dist == "gaussian" \
        else rng.integers(0, A, n).astype(np.float32)
    adv_raw = (3.0 * rng.standard_normal(n) + 1.0).astype(np.float32)
    a64 = adv_raw.astype(np.float64)
    stats = np.asarray([a64.sum(), (a64 ** 2).sum(), n])
    # old log-probs from a perturbed network so that ratios spread around 1 and the clip is exercised both ways
    old_layers = [(w + 0.05 * rng.standard_normal(w.shape).astype(np.float32), b) for w, b in layers]
    old_logp = O.Dist(dist, O.mlp_forward(old_layers, obs)[0], log_std).log_prob(act)
    r = loss_grad(sizes, O.flatten_layers(layers), obs, loss, dist, act=act, log_std=log_std, adv_raw=adv_raw,
                  adv_stats=stats, old_logp=old_logp)
    ref = O.policy_loss_and_grad(layers, dist, log_std, obs, act, O.normalize(adv_raw), old_logp,
                                 {"ppo_clip": "ppo", "vpg": "vpg", "trpo_surrogate": "trpo"}[loss], 0.2)
    assert rel_err(r["grad"], ref["grad"]) < TOL
    assert abs(r["scalars"][0] / n - ref["loss"]) < 1e-5 * max(1.0, abs(ref["loss"]))
    assert abs(r["scalars"][1] / n - ref["kl"]) < 1e-5
    if loss == "ppo_clip":
        ratio = np.exp(ref["logp"] - old_logp)
        assert (ratio > 1.2).any() and (ratio < 0.8).any()  # the test really clips


@pytest.mark.parametrize("sizes", [[17, 64, 64, 1], [4, 64, 64, 1], [27, 64, 32, 1], [5, 8, 1]])
@pytest.mark.parametrize("n", [1, 777, 9000])
def test_value_loss_grad(sizes, n):
    from gpu_helpers import loss_grad
    rng = np.random.default_rng(n + 11)
    layers = _net(rng, sizes)
    obs = rng.standard_normal((n, sizes[0])).astype(np.float32)
    ret = (5 * rng.standard_normal(n)).astype(np.float32)
    r = loss_grad(sizes, O.flatten_layers(layers), obs, "mse", "none", target=ret)
    ref = O.value_loss_and_grad(layers, obs, ret)
    assert rel_err(r["grad"], ref["grad"]) < TOL
    assert abs(r["scalars"][0] / n - ref["loss"]) < 1e-5 * ref["loss"]


def test_relu_hidden_activation():
    from gpu_helpers import loss_grad
    rng = np.random.default_rng(5)
    sizes = [14, 64, 64, 1]
    layers = _net(rng, sizes)
    obs = rng.standard_normal((500, 14)).astype(np.float32)
    ret = rng.standard_normal(500).astype(np.float32)
    r = loss_grad(sizes, O.flatten_layers(layers), obs, "mse", "none", target=ret, hidden_act="relu")
    ref = O.value_loss_and_grad(layers, obs, ret, hidden_act="relu")
    assert rel_err(r["grad"], ref["grad"]) < TOL


def test_gradients_against_reference_golden():
    from gpu_helpers import loss_grad
    for case in ["ppo_categorical_cfg1", "ppo_gaussian_small", "ppo_gaussian_ragged_earlystop"]:
        g = load_golden(case)
        b = batch_of(g)
        dist = "gaussian" if "log_std" in g else "categorical"
        ps, vs = [int(x) for x in g["policy_sizes"]], [int(x) for x in g["value_sizes"]]
        a64 = g["adv_raw"].astype(np.float64)
        stats = np.asarray([a64.sum(), (a64 ** 2).sum(), a64.size])
        r = loss_grad(ps, g["policy_flat0"], b["obs"], "ppo_clip", dist, act=b["act"], log_std=g.get("log_std"),
                      adv_raw=g["adv_raw"], adv_stats=stats, old_logp=g["old_logp"])
        assert rel_err(r["grad"], g["grad0"]) < TOL, case
        rv = loss_grad(vs, g["value_flat0"], b["obs"], "mse", "none", target=g["ret"])
        assert rel_err(rv["grad"], g["vgrad0"]) < TOL, case
        re = loss_grad(vs, g["value_flat0"], b["obs"], "eval", "none")
        assert rel_err(re["rows"], g["values"]) < TOL, case


def test_adam_step_matches_oracle_and_golden():
    from gpu_helpers import adam_step
    rng = np.random.default_rng(0)
    n = 5702
    p0 = rng.standard_normal(n).astype(np.float32)
    st = O.AdamState(n, 3e-4)
    p_ref = p0.copy()
    p_gpu, m, v = p0.copy(), np.zeros(n, np.float32), np.zeros(n, np.float32)
    for step in range(1, 6):
        grad = (rng.standard_normal(n) * 10.0 ** rng.integers(-6, 1, n)).astype(np.float32)
        p_ref = st.apply(p_ref, grad)
        p_gpu, m, v = adam_step(p_gpu, grad, m, v, step, 3e-4)
        assert rel_err(p_gpu, p_ref) < 1e-6
        assert rel_err(m, st.m) < 1e-6 and rel_err(v, st.v) < 1e-6
    g = load_golden("ppo_gaussian_small")
    p1, _, _ = adam_step(g["policy_flat0"], g["grad0"], np.zeros(n, np.float32), np.zeros(n, np.float32), 1, 3e-4)
    assert rel_err(p1, g["policy_flat1"]) < 1e-6


# ---- fp16 x 2 tensor-core kernel (mlp_tc2): range handling ----------------------------------------------------------
def _fallbacks():
    from rl_replicas_b200 import _lib
    return int(_lib.load().b200rl_tc_fallback_count())


@pytest.mark.parametrize("obs_scale,w_scale,ret_scale", [(1.0, 1.0, 5.0), (1e3, 1e-3, 5.0), (1e-4, 1e4, 5.0),
                                                        (1e-4, 1.0, 5.0), (1.0, 1.0, 3e4), (1.0, 1.0, 1e-3)])
def test_tc2_scaled_operands_stay_on_the_fp16_path(obs_scale, w_scale, ret_scale):
    """Power-of-two pre-scales keep small / large observations, weights and targets inside fp16's normal range: the
    fast kernel's result stands (no wide-range re-run) and still meets the 1e-5 bar."""
    from gpu_helpers import loss_grad
    rng = np.random.default_rng(5)
    n, sizes = 3000, [17, 64, 64, 1]
    layers = _net(rng, sizes)
    layers[0] = ((layers[0][0] * w_scale).astype(np.float32), layers[0][1])  # first layer absorbs the obs scale
    obs = (obs_scale * rng.standard_normal((n, sizes[0]))).astype(np.float32)
    ret = (ret_scale * rng.standard_normal(n)).astype(np.float32)
    before = _fallbacks()
    r = loss_grad(sizes, O.flatten_layers(layers), obs, "mse", "none", target=ret)
    assert _fallbacks() == before
    ref = O.value_loss_and_grad(layers, obs, ret)
    assert rel_err(r["grad"], ref["grad"]) < TOL
    assert abs(r["scalars"][0] / n - ref["loss"]) < 1e-5 * ref["loss"]


def test_tc2_out_of_range_launch_is_redone_by_the_wide_range_kernel():
    """One observation of 1e30 cannot be represented after scaling (the rest of the batch underflows next to it is
    fine, but a gradient outlier 1e12 times the typical one is not): the status slot fires and the fp32 kernel queued
    behind recomputes the launch -- results still match the oracle."""
    from gpu_helpers import loss_grad
    rng = np.random.default_rng(6)
    n, sizes = 2000, [17, 64, 64, 6]
    layers = _net(rng, sizes)
    obs = rng.standard_normal((n, sizes[0])).astype(np.float32)
    log_std = np.full(6, -0.5, np.float32)
    act = (O.mlp_forward(layers, obs)[0] + np.exp(-0.5) * rng.standard_normal((n, 6))).astype(np.float32)
    adv_raw = rng.standard_normal(n).astype(np.float32)
    adv_raw[7] = 1e12  # un-normalised advantages (adv_stats=None): one gradient row 1e12 times the others
    before = _fallbacks()
    r = loss_grad(sizes, O.flatten_layers(layers), obs, "vpg", "gaussian", act=act, log_std=log_std, adv_raw=adv_raw)
    assert _fallbacks() == before + 1
    ref = O.policy_loss_and_grad(layers, "gaussian", log_std, obs, act, adv_raw, None, "vpg", 0.2)
    assert rel_err(r["grad"], ref["grad"]) < TOL


def test_tc2_nan_input_is_reported_not_hidden():
    from gpu_helpers import loss_grad
    rng = np.random.default_rng(8)
    n, sizes = 500, [17, 64, 64, 1]
    layers = _net(rng, sizes)
    obs = rng.standard_normal((n, sizes[0])).astype(np.float32)
    obs[3, 2] = np.nan
    r = loss_grad(sizes, O.flatten_layers(layers), obs, "eval", "none")
    assert np.isnan(r["rows"][3]) and np.isfinite(np.delete(r["rows"], 3)).all()


@pytest.mark.parametrize("outlier", [None, 1e6], ids=["in_range", "obs_row_1e6"])
@pytest.mark.parametrize("sizes", [[17, 64, 32, 6], [9, 33, 20, 3]])
def test_padded_hidden_widths_on_the_wide_range_kernel(sizes, outlier):
    """Hidden layers narrower than 64 are zero-padded inside the fp16 kernel; with one observation row of 1e6 in every
    feature (every other row then sits below the precision guard) the launch is redone by the fp32 kernel, which takes
    the same shapes."""
    from gpu_helpers import loss_grad
    rng = np.random.default_rng(21)
    n = 3001
    vs = sizes[:-1] + [1]
    layers = _net(rng, vs)
    obs = rng.standard_normal((n, vs[0])).astype(np.float32)
    if outlier is not None:
        obs[11] = np.float32(outlier)
    ret = (5 * rng.standard_normal(n)).astype(np.float32)
    before = _fallbacks()
    r = loss_grad(vs, O.flatten_layers(layers), obs, "mse", "none", target=ret)
    assert _fallbacks() == before + (outlier is not None)
    ref = O.value_loss_and_grad(layers, obs, ret)
    assert rel_err(r["grad"], ref["grad"]) < TOL


def test_tc2_mixed_feature_magnitudes_and_row_outlier():
    """Per-feature observation scales: features spanning 1e-3 .. 1e3 keep full precision on the fp16 path; a single row
    1e6 times larger than the rest would silently cost every other row its l-splits -- the precision guard sends that
    launch to the wide-range kernel instead."""
    from gpu_helpers import loss_grad
    rng = np.random.default_rng(12)
    n, sizes = 6000, [17, 64, 64, 1]
    feat = (10.0 ** rng.uniform(-3, 3, 17)).astype(np.float32)
    layers = _net(rng, sizes)
    layers[0] = ((layers[0][0] / feat[None, :]).astype(np.float32), layers[0][1])
    obs = (rng.standard_normal((n, 17)) * feat[None, :]).astype(np.float32)
    ret = (5 * rng.standard_normal(n)).astype(np.float32)
    before = _fallbacks()
    r = loss_grad(sizes, O.flatten_layers(layers), obs, "mse", "none", target=ret)
    assert _fallbacks() == before
    ref = O.value_loss_and_grad(layers, obs, ret)
    assert rel_err(r["grad"], ref["grad"]) < TOL
    obs2 = obs.copy()
    obs2[11] *= 1e6
    r2 = loss_grad(sizes, O.flatten_layers(layers), obs2, "mse", "none", target=ret)
    assert _fallbacks() == before + 1
    ref2 = O.value_loss_and_grad(layers, obs2, ret)
    assert rel_err(r2["grad"], ref2["grad"]) < TOL


def test_absmax_helpers():
    """b200rl_absmax / b200rl_absmax_cols: the range hints of the fp16 kernels (a NaN makes the result +inf, which the
    kernels turn into a wide-range re-run)."""
    import ctypes as C
    import torch
    from rl_replicas_b200 import _lib
    lib = _lib.load()
    rng = np.random.default_rng(0)
    x = (rng.standard_normal((5000, 17)) * 10.0 ** rng.uniform(-3, 3, 17)).astype(np.float32)
    d = torch.from_numpy(x).cuda()
    out = torch.full((32,), -1.0, device="cuda")
    st = int(torch.cuda.current_stream().cuda_stream)
    _lib.check(lib.b200rl_absmax_cols(C.c_void_p(d.data_ptr()), 5000, 17, C.c_void_p(out.data_ptr()), st), "absmax_cols")
    np.testing.assert_array_equal(out[:17].cpu().numpy(), np.abs(x).max(axis=0))
    one = torch.zeros(1, device="cuda")
    _lib.check(lib.b200rl_absmax(C.c_void_p(d.data_ptr()), x.size, C.c_void_p(one.data_ptr()), st), "absmax")
    assert float(one.item()) == float(np.abs(x).max())
    x[123, 4] = np.nan
    d = torch.from_numpy(x).cuda()
    _lib.check(lib.b200rl_absmax_cols(C.c_void_p(d.data_ptr()), 5000, 17, C.c_void_p(out.data_ptr()), st), "absmax_cols")
    got = out[:17].cpu().numpy()
    assert np.isinf(got[4]) and np.isfinite(np.delete(got, 4)).all()


@pytest.mark.parametrize("loss", ["eval", "mse"])
def test_empty_launch_contributes_zeros(loss):
    """n_rows = 0 (an empty data-parallel shard): every partial row and scalar is zero, nothing is read."""
    from gpu_helpers import loss_grad
    rng = np.random.default_rng(3)
    sizes = [17, 64, 64, 1]
    layers = _net(rng, sizes)
    obs = np.zeros((0, 17), np.float32)
    r = loss_grad(sizes, O.flatten_layers(layers), obs, loss, "none", target=np.zeros(0, np.float32) if loss == "mse" else None)
    assert not r["scalars"].any()
    if loss == "mse":
        assert not r["grad"].any()


# ---- forward-only launches with raw outputs / the true KL (TRPO: old policy's outputs, line-search evaluations) -----
@pytest.mark.parametrize("sizes,dist", [([27, 64, 64, 8], "gaussian"), ([17, 64, 64, 6], "gaussian"),
                                        ([4, 64, 64, 2], "categorical"), ([8, 64, 64, 15], "categorical"),
                                        ([11, 64, 64, 64, 3], "gaussian")])  # last: 4 layers, fp32 kernel
@pytest.mark.parametrize("n", [1, 129, 1000, 40000])
@pytest.mark.parametrize("no_tc", [False, True])
def test_forward_outputs_and_true_kl(sizes, dist, n, no_tc):
    """trpo.py:158-175: out_full = the network's raw outputs, scalar 6 = sum KL(old || new), scalar 0 = the surrogate
    loss of the forward-only launch.  Tensor-core variant and fp32 kernel against the oracle."""
    from gpu_helpers import forward_outputs
    rng = np.random.default_rng(n + 31 * sizes[-1] + int(no_tc))
    layers = _net(rng, sizes)
    old_layers = [(w + 0.03 * rng.standard_normal(w.shape).astype(np.float32), b) for w, b in layers]
    obs = rng.standard_normal((n, sizes[0])).astype(np.float32)
    A = sizes[-1]
    log_std = (-0.5 + 0.1 * rng.standard_normal(A)).astype(np.float32) if dist == "gaussian" else None
    out_old = O.mlp_forward(old_layers, obs)[0]
    act = (out_old + np.exp(-0.5) * rng.standard_normal((n, A))).astype(np.float32) if dist == "gaussian" \
        else rng.integers(0, A, n).astype(np.float32)
    adv = rng.standard_normal(n).astype(np.float32)
    old_logp = O.Dist(dist, out_old, log_std).log_prob(act)
    before = _fallbacks()
    r = forward_outputs(sizes, O.flatten_layers(layers), obs, dist, act, log_std=log_std, old_out=out_old, adv_raw=adv,
                        old_logp=old_logp, loss="trpo_surrogate", no_tc=no_tc)
    assert _fallbacks() == before
    out_new = O.mlp_forward(layers, obs)[0]
    assert rel_err(r["out"], out_new) < TOL
    logp = O.Dist(dist, out_new, log_std).log_prob(act)
    assert rel_err(r["rows"], logp) < TOL
    kl = O.dist_kl(dist, out_old, out_new, log_std).astype(np.float64).sum()
    # per-row KL is a sum of terms that cancel to ~1e-3 of their size: 5e-7 absolute per row is float32 rounding
    np.testing.assert_allclose(r["scalars"][6], kl, rtol=2e-5, atol=5e-7 * n)
    loss = -(np.exp(logp - old_logp).astype(np.float64) * adv).sum()
    np.testing.assert_allclose(r["scalars"][0], loss, rtol=1e-5, atol=1e-5 * np.abs(adv).sum())
    assert r["scalars"][5] == n
    # plain evaluation with out_full only (the old policy's pass)
    r2 = forward_outputs(sizes, O.flatten_layers(old_layers), obs, dist, act, log_std=log_std, no_tc=no_tc)
    assert rel_err(r2["out"], out_old) < TOL and rel_err(r2["rows"], old_logp) < TOL
    assert r2["scalars"][6] == 0.0
