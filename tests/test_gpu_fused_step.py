"""The fused policy + value step kernel (csrc/mlp_tc3.cu: one pass over the batch per PPO iteration, observations
packed once per update and brought in by bulk copies) against the numpy oracle, against the two-loop path it replaces
(B200RL_FUSED_STEP=0), and through its corner cases: early stop (host polling hands the remaining value steps to the
value kernel), loops of different length, narrow / wide networks, categorical policies, range trips (redo)."""
import os

import numpy as np
import pytest

from conftest import rel_err
from oracle import onpolicy as O
from test_gpu_ppo import build, flat

pytestmark = pytest.mark.gpu


def _layers(rng, sizes, bias=0.0):
    return [(rng.standard_normal((o, i)).astype(np.float32) / np.sqrt(i),
             (bias * rng.standard_normal(o)).astype(np.float32)) for i, o in zip(sizes[:-1], sizes[1:])]


def _run(ps, vs, dist, pl, vl, log_std, b, fused=True, **hp):
    old = os.environ.get("B200RL_FUSED_STEP")
    os.environ["B200RL_FUSED_STEP"] = "1" if fused else "0"
    try:
        ppo = build(ps, vs, dist, O.flatten_layers(pl), O.flatten_layers(vl), log_std, **hp)
        ppo.train_packed(b)
    finally:
        if old is None:
            del os.environ["B200RL_FUSED_STEP"]
        else:
            os.environ["B200RL_FUSED_STEP"] = old
    return ppo


@pytest.mark.parametrize("ps,vs,dist,n_envs,horizon", [
    ([17, 64, 64, 6], [17, 64, 64, 1], "gaussian", 16, 100),
    ([17, 64, 64, 6], [17, 64, 64, 1], "gaussian", 67, 333),      # ragged tile count, tail tile
    ([4, 64, 64, 2], [4, 64, 64, 1], "categorical", 40, 100),
    ([31, 64, 32, 15], [31, 48, 64, 1], "gaussian", 20, 150),     # widest observation, narrow / uneven hidden layers
    ([11, 33, 20, 3], [11, 20, 33, 1], "categorical", 9, 77),
    ([1, 64, 64, 1], [1, 64, 64, 1], "gaussian", 3, 50),          # fewer rows than one tile
])
def test_fused_step_matches_oracle_and_two_loop_path(ps, vs, dist, n_envs, horizon):
    from rl_replicas_b200 import synthetic
    rng = np.random.default_rng(ps[0] + n_envs)
    pl, vl = _layers(rng, ps, 0.1), _layers(rng, vs, 0.1)
    discrete = dist == "categorical"
    log_std = None if discrete else np.linspace(-0.7, -0.2, ps[-1]).astype(np.float32)
    b = synthetic.fixed_batch(n_envs, horizon, ps[0], ps[-1], discrete=discrete, seed=5, frac_not_done=0.3,
                              mean_fn=None if discrete else (lambda o: O.mlp_forward(pl, o)[0]))
    hp = dict(num_policy_gradients=5, num_value_gradients=5, max_kl_divergence=float("inf"))
    f = _run(ps, vs, dist, pl, vl, log_std, b, fused=True, **hp)
    assert f.last_update_stats.fused == 1
    assert f.last_update_stats.policy_steps_applied == 5 and f.last_update_stats.value_steps_applied == 5
    two = _run(ps, vs, dist, pl, vl, log_std, b, fused=False, **hp)
    assert two.last_update_stats.fused == 0
    n_p, n_v = O.flatten_layers(pl).size, O.flatten_layers(vl).size
    out = O.ppo_train(b, pl, vl, dist, log_std, O.AdamState(n_p, 3e-4), O.AdamState(n_v, 1e-3), max_kl=float("inf"),
                      n_policy=5, n_value=5)
    for name, ppo in (("fused", f), ("two-loop", two)):
        assert rel_err(flat(ppo.policy.network), out["policy_flat"]) < 1e-5, name
        assert rel_err(flat(ppo.value_function.network), out["value_flat"]) < 1e-5, name
    st = f.last_update_stats
    assert abs(st.kl_divergence - out["kl"]) < 1e-4 * abs(out["kl"]) + 1e-8
    assert abs(st.value_loss_mean - out["value_loss_mean"]) < 1e-5 * out["value_loss_mean"]
    assert abs(st.policy_loss_before - out["loss_before"]) < 1e-6
    assert abs(st.entropy_before - out["entropy_before"]) < 1e-5 * abs(out["entropy_before"]) + 1e-6
    hist_f, hist_t = f._engine.scalar_history(), two._engine.scalar_history()
    assert hist_f.shape == hist_t.shape
    n = b["obs"].shape[0]
    assert np.max(np.abs(hist_f[1:6, 1] - hist_t[1:6, 1])) / n < 1e-6  # KL after every policy step
    assert np.max(np.abs(hist_f[6:11, 0] - hist_t[6:11, 0]) / hist_t[6:11, 0]) < 1e-5  # value losses


@pytest.mark.parametrize("K,Kv", [(3, 9), (9, 3), (1, 1), (12, 12)])
def test_fused_step_with_loops_of_different_length(K, Kv):
    from rl_replicas_b200 import synthetic
    rng = np.random.default_rng(K * 17 + Kv)
    ps, vs = [17, 64, 64, 6], [17, 64, 64, 1]
    pl, vl = _layers(rng, ps), _layers(rng, vs)
    log_std = np.full(6, -0.5, np.float32)
    b = synthetic.fixed_batch(24, 120, 17, 6, seed=2, frac_not_done=0.2, mean_fn=lambda o: O.mlp_forward(pl, o)[0])
    f = _run(ps, vs, "gaussian", pl, vl, log_std, b, num_policy_gradients=K, num_value_gradients=Kv,
             max_kl_divergence=float("inf"))
    st = f.last_update_stats
    assert st.fused == 1 and st.policy_steps_applied == K and st.value_steps_applied == Kv
    out = O.ppo_train(b, pl, vl, "gaussian", log_std, O.AdamState(5702, 3e-4), O.AdamState(5377, 1e-3),
                      max_kl=float("inf"), n_policy=K, n_value=Kv)
    assert rel_err(flat(f.policy.network), out["policy_flat"]) < 1e-5
    assert rel_err(flat(f.value_function.network), out["value_flat"]) < 1e-5
    assert abs(st.kl_divergence - out["kl"]) < 1e-4 * abs(out["kl"]) + 1e-8
    assert abs(st.value_loss_mean - out["value_loss_mean"]) < 1e-5 * out["value_loss_mean"]


@pytest.mark.parametrize("max_kl", [2e-4, 2e-3])
def test_fused_step_early_stop_hands_over_to_the_value_kernel(max_kl):
    """The KL limit trips after a few policy steps: the stop is a device-side decision (the fused kernel then runs its
    value chain only), the host notices at its next poll and finishes the value loop on the value kernel.  Same stop
    iteration and same networks as the oracle and as the two-loop path."""
    from rl_replicas_b200 import synthetic
    rng = np.random.default_rng(11)
    ps, vs = [17, 64, 64, 6], [17, 64, 64, 1]
    pl, vl = _layers(rng, ps), _layers(rng, vs)
    log_std = np.full(6, -0.5, np.float32)
    b = synthetic.fixed_batch(32, 200, 17, 6, seed=3, frac_not_done=0.25, mean_fn=lambda o: O.mlp_forward(pl, o)[0])
    hp = dict(num_policy_gradients=30, num_value_gradients=30, max_kl_divergence=max_kl)
    out = O.ppo_train(b, pl, vl, "gaussian", log_std, O.AdamState(5702, 3e-4), O.AdamState(5377, 1e-3), max_kl=max_kl,
                      n_policy=30, n_value=30)
    assert 1 <= out["policy_steps"] < 30, "the case is meant to stop early"
    f = _run(ps, vs, "gaussian", pl, vl, log_std, b, fused=True, **hp)
    two = _run(ps, vs, "gaussian", pl, vl, log_std, b, fused=False, **hp)
    for name, ppo in (("fused", f), ("two-loop", two)):
        st = ppo.last_update_stats
        # the reference counts the step whose KL tripped as taken (ppo.py:176-181); `applied` counts Adam updates
        assert st.policy_steps_applied == out["policy_steps"], name
        assert st.value_steps_applied == 30, name
        assert rel_err(flat(ppo.policy.network), out["policy_flat"]) < 1e-5, name
        assert rel_err(flat(ppo.value_function.network), out["value_flat"]) < 2e-5, name
        assert abs(st.kl_divergence - out["kl"]) < 1e-4 * abs(out["kl"]) + 1e-8, name
    assert f.last_update_stats.fused == 1


def test_fused_step_range_trip_is_redone_on_the_wide_range_path():
    """One transition 1e6 times larger than the rest: every other row would lose its l-splits in the packed
    observations.  pack_obs raises the flag, the engine restores its snapshot and redoes the update on the two-loop
    path (whose own guards route the launches to the wide-range kernels): same result as never having tried."""
    from rl_replicas_b200 import synthetic
    rng = np.random.default_rng(4)
    ps, vs = [17, 64, 64, 6], [17, 64, 64, 1]
    pl, vl = _layers(rng, ps), _layers(rng, vs)
    log_std = np.full(6, -0.5, np.float32)
    b = synthetic.fixed_batch(10, 100, 17, 6, seed=8, mean_fn=lambda o: O.mlp_forward(pl, o)[0])
    b["obs"][37] *= 1e6
    hp = dict(num_policy_gradients=3, num_value_gradients=3, max_kl_divergence=float("inf"))
    f = _run(ps, vs, "gaussian", pl, vl, log_std, b, fused=True, **hp)
    two = _run(ps, vs, "gaussian", pl, vl, log_std, b, fused=False, **hp)
    assert f.last_update_stats.fused == 0  # the fused attempt was abandoned
    np.testing.assert_array_equal(flat(f.policy.network), flat(two.policy.network))
    np.testing.assert_array_equal(flat(f.value_function.network), flat(two.value_function.network))
    out = O.ppo_train(b, pl, vl, "gaussian", log_std, O.AdamState(5702, 3e-4), O.AdamState(5377, 1e-3),
                      max_kl=float("inf"), n_policy=3, n_value=3)
    assert rel_err(flat(f.value_function.network), out["value_flat"]) < 1e-5
    # a second, clean update on the same learner goes through the fused kernel again
    b2 = synthetic.fixed_batch(10, 100, 17, 6, seed=9, mean_fn=lambda o: O.mlp_forward(pl, o)[0])
    f.train_packed(b2)
    assert f.last_update_stats.fused == 1


def _assert_bit_reproducible(n_envs, horizon):
    """Two PPO updates of 4 + 4 fused iterations on the same learner state and batch leave identical networks."""
    from rl_replicas_b200 import synthetic
    rng = np.random.default_rng(6)
    ps, vs = [17, 64, 64, 6], [17, 64, 64, 1]
    pl, vl = _layers(rng, ps), _layers(rng, vs)
    log_std = np.full(6, -0.5, np.float32)
    b = synthetic.fixed_batch(n_envs, horizon, 17, 6, seed=1, mean_fn=lambda o: O.mlp_forward(pl, o)[0])
    hp = dict(num_policy_gradients=4, num_value_gradients=4, max_kl_divergence=float("inf"))
    runs = [_run(ps, vs, "gaussian", pl, vl, log_std, b, **hp) for _ in range(2)]
    assert all(r.last_update_stats.fused == 1 for r in runs)
    np.testing.assert_array_equal(flat(runs[0].policy.network), flat(runs[1].policy.network))
    np.testing.assert_array_equal(flat(runs[0].value_function.network), flat(runs[1].value_function.network))


def test_fused_step_is_bit_reproducible():
    _assert_bit_reproducible(300, 100)


def test_fused_step_is_bit_reproducible_at_nine_tiles_per_cta():
    """Nine full 128-row tiles on every CTA (the grid is one CTA per SM): both observation buffers, the b3 class sums
    and the mbarrier phases go round several times per launch."""
    import torch
    _assert_bit_reproducible(9 * torch.cuda.get_device_properties(0).multi_processor_count, 128)
