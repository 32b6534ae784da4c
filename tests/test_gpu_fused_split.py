"""The fused PPO step runs each network in CTAs of its own: with both networks, CTA 2 slot + c runs network c on the
tiles of slot `slot`, and the two CTAs of a slot write disjoint entries of the slot's partial rows.  A launch with one
network runs one CTA per slot.  Its partial rows must equal, bit for bit, that network's entries after a two-network
launch, at tile counts where the slot mapping is most likely to go wrong: one (short) tile, fewer tiles than SMs, tile
counts that leave slots with different numbers of tiles, and a short last tile."""
import numpy as np
import pytest

from oracle import onpolicy as O
from test_gpu_ppo import build

pytestmark = pytest.mark.gpu

N_SCALARS = 8


def _layers(rng, sizes):
    return [(rng.standard_normal((o, i)).astype(np.float32) / np.sqrt(i),
             (0.1 * rng.standard_normal(o)).astype(np.float32)) for i, o in zip(sizes[:-1], sizes[1:])]


@pytest.mark.parametrize("ps,vs,dist,n_envs,horizon", [
    ([17, 64, 64, 6], [17, 64, 64, 1], "gaussian", 3, 40),        # one tile, 120 rows
    ([17, 64, 64, 6], [17, 64, 64, 1], "gaussian", 16, 400),      # 50 whole tiles: fewer tiles than SMs
    ([17, 64, 64, 6], [17, 64, 64, 1], "gaussian", 61, 1000),     # 477 tiles: slots with 4 and with 3 tiles, short last
    ([4, 64, 64, 2], [4, 64, 64, 1], "categorical", 40, 100),     # 31.25 tiles
])
def test_one_network_launches_match_two_network_launch(ps, vs, dist, n_envs, horizon):
    import torch
    from rl_replicas_b200 import synthetic
    rng = np.random.default_rng(n_envs)
    pl, vl = _layers(rng, ps), _layers(rng, vs)
    discrete = dist == "categorical"
    log_std = None if discrete else np.linspace(-0.7, -0.2, ps[-1]).astype(np.float32)
    b = synthetic.fixed_batch(n_envs, horizon, ps[0], ps[-1], discrete=discrete, seed=3, frac_not_done=0.3,
                              mean_fn=None if discrete else (lambda o: O.mlp_forward(pl, o)[0]))
    ppo = build(ps, vs, dist, O.flatten_layers(pl), O.flatten_layers(vl), log_std, num_policy_gradients=2,
                num_value_gradients=2, max_kl_divergence=float("inf"))
    ppo.train_packed(b)
    assert ppo.last_update_stats.fused == 1
    e = ppo._engine
    hp = ppo._hparams(e, 0)
    for s in ("preamble", "old_logp", "pack_obs"):
        e.run_stage(s, hp)
    n_p, n_v = O.flatten_layers(pl).size, O.flatten_layers(vl).size
    rows = 2 * min(-(-n_envs * horizon // 128), torch.cuda.get_device_properties(0).multi_processor_count)

    def launch(stage):
        part, scal = e.view("fused_partials"), e.view("fused_scalar_partials")
        part.fill_(float("nan"))  # every entry the launch owns must be written
        scal.fill_(float("nan"))
        e.run_stage(stage, hp)
        torch.cuda.synchronize()
        return part.cpu().numpy().reshape(rows, n_p + n_v), scal.cpu().numpy().reshape(rows, 2 * N_SCALARS)

    both_p, both_s = launch("fused_step_kernel")
    assert not np.isnan(both_p).any() and not np.isnan(both_s).any()
    assert np.abs(both_p[:, :n_p]).max() > 0 and np.abs(both_p[:, n_p:]).max() > 0
    pol_p, pol_s = launch("fused_step_kernel_policy")
    val_p, val_s = launch("fused_step_kernel_value")
    np.testing.assert_array_equal(pol_p[:, :n_p], both_p[:, :n_p])
    np.testing.assert_array_equal(val_p[:, n_p:], both_p[:, n_p:])
    np.testing.assert_array_equal(pol_s[:, :N_SCALARS], both_s[:, :N_SCALARS])
    np.testing.assert_array_equal(val_s[:, N_SCALARS:], both_s[:, N_SCALARS:])
    # the network that does not run gets zero scalar sums; its gradient entries are left alone
    assert (pol_s[:, N_SCALARS:] == 0).all() and (val_s[:, :N_SCALARS] == 0).all()
    assert np.isnan(pol_p[:, n_p:]).all() and np.isnan(val_p[:, :n_p]).all()
