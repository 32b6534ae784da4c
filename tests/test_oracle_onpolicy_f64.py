"""CPU: the float64 on-policy reference (oracle/onpolicy_f64.py) against the float32 numpy oracle (oracle/onpolicy.py)
for every loss and both distributions, and its Fisher-vector product (double backprop) against an explicitly formed
J^T M J v."""
import numpy as np
import pytest

from conftest import rel_err
from oracle import onpolicy as O
from oracle import onpolicy_f64 as R

TOL = 1e-5


def _problem(sizes, dist, n, seed, hidden="tanh"):
    rng = np.random.default_rng(seed)
    layers = [(rng.standard_normal((o, i)).astype(np.float32) / np.float32(np.sqrt(i)),
               0.1 * rng.standard_normal(o).astype(np.float32)) for i, o in zip(sizes[:-1], sizes[1:])]
    obs = rng.standard_normal((n, sizes[0])).astype(np.float32)
    A = sizes[-1]
    log_std = np.linspace(-0.8, -0.2, A).astype(np.float32) if dist == "gaussian" else None
    mean = O.mlp_forward(layers, obs, hidden)[0]
    act = (mean + 0.6 * rng.standard_normal((n, A))).astype(np.float32) if dist == "gaussian" \
        else rng.integers(0, A, n).astype(np.float32)
    adv_raw = (2.0 * rng.standard_normal(n) + 0.5).astype(np.float32)
    a64 = adv_raw.astype(np.float64)
    stats = np.asarray([a64.sum(), (a64 ** 2).sum(), n])
    # old log-probs spread so that ratios fall past both clip bounds; none within 1e-4 of a bound
    logp = O.Dist(dist, mean, log_std).log_prob(act)
    old_logp = (logp + 0.3 * rng.standard_normal(n)).astype(np.float32)
    near = R.clip_margin(np.exp(logp.astype(np.float64) - old_logp)) < 1e-4
    old_logp[near] += np.float32(1e-3)
    return layers, obs, act, log_std, adv_raw, stats, old_logp


@pytest.mark.parametrize("hidden", ["tanh", "relu"])
@pytest.mark.parametrize("loss", ["ppo_clip", "vpg", "trpo_surrogate"])
@pytest.mark.parametrize("sizes,dist", [([5, 16, 12, 3], "gaussian"), ([4, 10, 7, 5], "categorical"),
                                        ([6, 9, 2], "gaussian"), ([3, 8, 8, 8, 4], "categorical")])
def test_policy_losses_match_the_float32_oracle(sizes, dist, loss, hidden):
    layers, obs, act, log_std, adv_raw, stats, old_logp = _problem(sizes, dist, 300, len(sizes) + sizes[-1], hidden)
    flat = O.flatten_layers(layers)
    got = R.policy_loss(flat, sizes, obs, act, dist, loss, log_std=log_std, adv_raw=adv_raw, adv_stats=stats,
                        old_logp=old_logp, hidden=hidden)
    if "ratio" in got:  # rows within rounding of a clip bound are clipped by whichever side the rounding lands on
        assert R.clip_margin(got["ratio"]).min() > 1e-5
    if hidden == "relu":
        assert got["margin"].min() > 1e-6
    want = O.policy_loss_and_grad(layers, dist, log_std, obs, act, O.normalize(adv_raw), old_logp,
                                  {"ppo_clip": "ppo", "vpg": "vpg", "trpo_surrogate": "trpo"}[loss], 0.2, hidden,
                                  acc=np.float64)
    assert rel_err(got["grad"], want["grad"]) < TOL
    assert rel_err(R.split(got["grad"], sizes)["W0"], got["grads"]["W0"]) == 0
    assert abs(got["loss_sum"] / 300 - want["loss"]) < TOL * max(1.0, abs(want["loss"]))
    assert abs(got["kl_sum"] / 300 - want["kl"]) < TOL
    assert rel_err(got["logp"], want["logp"]) < TOL
    assert abs(got["entropy_sum"] - want["entropy"].astype(np.float64).sum()) < TOL * abs(got["entropy_sum"])
    if dist == "gaussian":
        assert rel_err(got["grad_log_std"], want["grad_log_std"]) < TOL
    if loss == "ppo_clip":
        assert (got["ratio"] > 1.2).any() and (got["ratio"] < 0.8).any()  # the clip binds on both sides


@pytest.mark.parametrize("sizes,dist", [([5, 16, 12, 3], "gaussian"), ([4, 10, 7, 5], "categorical")])
def test_evaluation_sums(sizes, dist):
    layers, obs, act, log_std, _, _, _ = _problem(sizes, dist, 200, 3)
    got = R.policy_loss(O.flatten_layers(layers), sizes, obs, act, dist, "eval", log_std=log_std)
    d = O.Dist(dist, O.mlp_forward(layers, obs)[0], log_std)
    lp = d.log_prob(act).astype(np.float64)
    assert rel_err(got["logp"], lp) < TOL
    np.testing.assert_allclose(got["logp_sum"], lp.sum(), rtol=TOL)
    np.testing.assert_allclose(got["logp2_sum"], (lp ** 2).sum(), rtol=TOL)
    np.testing.assert_allclose(got["entropy_sum"], d.entropy().astype(np.float64).sum(), rtol=TOL)
    assert got["loss_sum"] == 0.0 and "grad" not in got


@pytest.mark.parametrize("hidden", ["tanh", "relu"])
def test_value_loss_matches_the_float32_oracle(hidden):
    sizes = [7, 20, 13, 1]
    layers, obs, _, _, _, _, _ = _problem(sizes, "gaussian", 250, 9, hidden)
    ret = (3.0 * np.random.default_rng(1).standard_normal(250)).astype(np.float32)
    got = R.value_loss(O.flatten_layers(layers), sizes, obs, ret, hidden)
    want = O.value_loss_and_grad(layers, obs, ret, hidden, acc=np.float64)
    assert rel_err(got["grad"], want["grad"]) < TOL
    assert abs(got["loss_sum"] / 250 - want["loss"]) < TOL * want["loss"]
    assert rel_err(got["values"], want["values"]) < TOL
    assert rel_err(R.values(O.flatten_layers(layers), sizes, obs, hidden), want["values"]) < TOL


@pytest.mark.parametrize("dist", ["gaussian", "categorical"])
def test_forward_kl_matches_the_float32_oracle(dist):
    sizes = [5, 16, 12, 4]
    layers, obs, act, log_std, _, _, _ = _problem(sizes, dist, 150, 4)
    old = [(w + 0.03, b) for w, b in layers]
    out_old = O.mlp_forward(old, obs)[0]
    got = R.forward_kl(O.flatten_layers(layers), sizes, obs, dist, out_old, log_std)
    out_new = O.mlp_forward(layers, obs)[0]
    assert rel_err(got["out"], out_new) < TOL
    assert rel_err(got["kl"], O.dist_kl(dist, out_old, out_new, log_std)) < 1e-4  # float32 KL: terms cancel to ~1e-2
    same = R.forward_kl(O.flatten_layers(old), sizes, obs, dist, out_old, log_std)
    assert np.abs(same["kl"]).max() < 1e-12


@pytest.mark.parametrize("dist", ["gaussian", "categorical"])
def test_fvp_matches_the_float32_oracle(dist):
    sizes = [5, 16, 12, 4]
    layers, obs, _, log_std, _, _, _ = _problem(sizes, dist, 200, 6)
    v = np.random.default_rng(2).standard_normal(O.flatten_layers(layers).size).astype(np.float32)
    got = R.fvp(O.flatten_layers(layers), sizes, obs, dist, v, log_std)
    want = O.fisher_vector_product(layers, dist, log_std, obs, v, damping=0.0)
    assert rel_err(got["fvp"], want) < TOL


@pytest.mark.parametrize("hidden", ["tanh", "relu"])
@pytest.mark.parametrize("dist", ["gaussian", "categorical"])
def test_fvp_against_explicit_jacobian(dist, hidden):
    """Double backprop of the mean KL against (1/N) sum J^T M J v with J formed column by column: agreement to float64
    rounding."""
    sizes = [3, 5, 4, 3]
    layers, obs, _, log_std, _, _, _ = _problem(sizes, dist, 7, 8, hidden)
    flat = O.flatten_layers(layers)
    v = np.random.default_rng(3).standard_normal(flat.size)
    got = R.fvp(flat, sizes, obs, dist, v, log_std, hidden)["fvp"]
    want = R.fvp_explicit(flat, sizes, obs, dist, v, log_std, hidden)
    assert rel_err(got, want) < 1e-12
    assert np.abs(want).max() > 1e-3


def test_ppo_clip_follows_torch_tie_and_boundary_rules():
    """Inside the clip range the two arguments of torch.min are equal and it splits the gradient between them, which
    sum to the whole; past the upper bound with A > 0 the clamped term wins and passes nothing; below the lower bound
    with A > 0 the unclipped term wins."""
    import torch
    sizes = [2, 3, 1]
    flat = np.zeros(13, np.float32)
    flat[-1] = 0.25  # b1: the mean of every row
    obs = np.zeros((3, 2), np.float32)
    act = np.zeros((3, 1), np.float32)
    log_std = np.zeros(1, np.float32)
    lp = float(torch.distributions.Normal(torch.tensor(0.25, dtype=torch.float64), 1.0).log_prob(torch.tensor(0.0, dtype=torch.float64)))
    # ratio 1.1 (inside), 1.5 (past the upper bound) and 0.5 (past the lower bound), all with A > 0
    old = np.asarray([lp - np.log(1.1), lp - np.log(1.5), lp - np.log(0.5)])
    r = R.policy_loss(flat, sizes, obs, act, "gaussian", "ppo_clip", log_std=log_std, adv_raw=np.ones(3),
                      old_logp=old)
    np.testing.assert_allclose(r["ratio"], [1.1, 1.5, 0.5], rtol=1e-12)
    # d loss / d b1 = -(1/N) sum_i pass_i r_i A_i dlogp/dmu with dlogp/dmu = (a - mu) / var = -0.25
    np.testing.assert_allclose(r["grads"]["b1"], [-(1.1 + 0.5) * -0.25 / 3], rtol=1e-12)


@pytest.mark.parametrize("loss", ["ppo_clip", "vpg"])
def test_gradient_scales_bound_the_gradients(loss):
    """The per-entry scale (sum over rows of |contribution|) is at least |gradient|, and equals it for one row."""
    sizes = [5, 16, 12, 3]
    layers, obs, act, log_std, adv_raw, stats, old_logp = _problem(sizes, "gaussian", 120, 12)
    flat = O.flatten_layers(layers)
    r = R.policy_loss(flat, sizes, obs, act, "gaussian", loss, log_std, adv_raw, stats, old_logp)
    for k, g in r["grads"].items():
        assert (r["scales"][k] >= np.abs(g) * (1 - 1e-12)).all(), k
    assert (r["scale_log_std"] >= np.abs(r["grad_log_std"]) * (1 - 1e-12)).all()
    assert max(np.max(r["scales"][k] / np.abs(r["grads"][k]).max()) for k in r["grads"]) > 1.5  # rows do cancel
    one = R.policy_loss(flat, sizes, obs[:1], act[:1], "gaussian", loss, log_std, adv_raw[:1], None, old_logp[:1])
    for k, g in one["grads"].items():
        np.testing.assert_allclose(one["scales"][k], np.abs(g), rtol=1e-12, atol=1e-300)
    np.testing.assert_allclose(one["scale_log_std"], np.abs(one["grad_log_std"]), rtol=1e-12)
    v = R.value_loss(O.flatten_layers([(w[:1], b[:1]) if i == len(layers) - 1 else (w, b)
                                       for i, (w, b) in enumerate(layers)]), sizes[:-1] + [1], obs[:1], np.ones(1))
    for k, g in v["grads"].items():
        np.testing.assert_allclose(v["scales"][k], np.abs(g), rtol=1e-12, atol=1e-300)


@pytest.mark.parametrize("f64", [True, False])
def test_gae_scan_reference_rounds_to_the_float32_oracle(f64):
    """The unrounded float64 scan reference, cast to float32, is the float32 oracle bit for bit, on ragged episodes
    (lengths 1 and 2 among them) with nonzero values, done and not-done episodes, and float64 or float32 rewards."""
    rng = np.random.default_rng(11)
    lens = np.concatenate([[1, 2, 1], rng.integers(1, 90, 300), [2]])
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    n, e = int(off[-1]), lens.size
    rew = rng.standard_normal(n) if f64 else rng.standard_normal(n).astype(np.float32)
    values = rng.standard_normal(n).astype(np.float32)
    last_values = rng.standard_normal(e).astype(np.float32)
    done = rng.random(e) < 0.5
    for gamma, lam in ((0.99, 0.97), (1.0, 1.0), (0.0, 0.5), (0.9, 0.0)):
        adv64, ret64, s_adv, s_ret = R.gae_scan(rew, values, last_values, off, done, gamma, lam)
        adv, ret = O.gae_and_returns(rew, values, last_values, off, done, gamma, lam)
        np.testing.assert_array_equal(adv64.astype(np.float32), adv)
        np.testing.assert_array_equal(ret64.astype(np.float32), ret)
        assert np.all(s_adv >= np.abs(adv64)) and np.all(s_ret >= np.abs(ret64))
