"""Pin oracle/offpolicy.py against the reference's own TD3.train / DDPG.train outputs (CPU)."""
import numpy as np
import pytest

from conftest import load_golden, rel_err
from oracle import offpolicy as OP
from oracle import onpolicy as O

O_DIM, A_DIM, H = 11, 3, 64
PS, QS = [O_DIM, H, H, A_DIM], [O_DIM + A_DIM, H, H, 1]


def setup(g, twin):
    nets = {"policy": O.unflatten_layers(g["policy_flat0"], PS), "q1": O.unflatten_layers(g["q1_flat0"], QS)}
    nets["target_policy"] = O.unflatten_layers(g["policy_flat0"], PS)
    nets["target_q1"] = O.unflatten_layers(g["q1_flat0"], QS)
    if twin:
        nets["q2"] = O.unflatten_layers(g["q2_flat0"], QS)
        nets["target_q2"] = O.unflatten_layers(g["q2_flat0"], QS)
    adams = {k: O.AdamState(g[k + "_flat0"].size, 1e-3) for k in (["policy", "q1", "q2"] if twin else ["policy", "q1"])}
    mbs = [{k: g["mb_" + k][s] for k in ("observations", "actions", "rewards", "next_observations", "dones")}
           for s in range(int(g["S"]))]
    return nets, adams, mbs


@pytest.mark.parametrize("case,twin", [("td3_small", True), ("ddpg_small", False)])
def test_offpolicy_oracle_matches_reference(case, twin):
    g = load_golden(case)
    nets, adams, mbs = setup(g, twin)
    logs = OP.offpolicy_train(nets, adams, mbs, g["noise"] if twin else None, policy_delay=2 if twin else 1, twin=twin)
    names = ["policy", "q1"] + (["q2"] if twin else [])
    for n in names:
        assert rel_err(O.flatten_layers(nets[n]), g[n + "_flat_final"]) < 1e-5, n
        assert rel_err(O.flatten_layers(nets["target_" + n]), g["target_" + n + "_flat_final"]) < 1e-5, n
    pre = "q-function_1" if twin else "q-function"
    assert abs(np.mean(logs["q1_losses"]) - g["metric:" + pre + "/average_loss"]) < 1e-5
    assert abs(np.mean(np.concatenate(logs["q1_values"])) - g["metric:" + pre + "/avarage_q-value"]) < 1e-6
    assert abs(np.mean(logs["policy_losses"]) - g["metric:policy/average_loss"]) < 1e-6
    assert len(logs["policy_losses"]) == (4 if twin else 7)


def _small_problem(seed, O_, A_, B, sizes_p, sizes_q, n_q, limit=1.0):
    rng = np.random.default_rng(seed)
    mk = lambda sz: O.flatten_layers([(rng.standard_normal((o, i)).astype(np.float32) / np.sqrt(i),
                                       0.1 * rng.standard_normal(o).astype(np.float32)) for i, o in zip(sz[:-1], sz[1:])])
    nets = {"policy": mk(sizes_p), "q1": mk(sizes_q)}
    if n_q == 2:
        nets["q2"] = mk(sizes_q)
    for k in list(nets):
        nets["target_" + k] = (nets[k] + 0.05 * rng.standard_normal(nets[k].size)).astype(np.float32)
    mb = {"observations": rng.standard_normal((B, O_)).astype(np.float32),
          "actions": rng.uniform(-limit, limit, (B, A_)).astype(np.float32),
          "rewards": rng.standard_normal(B).astype(np.float32),
          "next_observations": rng.standard_normal((B, O_)).astype(np.float32),
          "dones": (rng.random(B) < 0.2).astype(np.float32)}
    return rng, nets, mb


@pytest.mark.parametrize("twin", [True, False])
def test_float64_reference_agrees_with_the_float32_oracle_on_one_step(twin):
    """oracle/offpolicy_f64.py (torch autograd, float64, stage by stage) against oracle/offpolicy.py (numpy, float32,
    hand-written backward) on one TD3 / DDPG step at a small shape: Q-values, losses, and the gradients the float32
    oracle's Adam saw (exp_avg after one step from zero is (1 - beta1) g)."""
    from oracle import offpolicy_f64 as R
    PS_, QS_ = [5, 24, 20, 2], [7, 24, 20, 1]
    rng, nets, mb = _small_problem(3, 5, 2, 16, PS_, QS_, 2 if twin else 1, limit=0.5)
    noise = rng.standard_normal((1, 16, 2)).astype(np.float32) if twin else None
    hp = dict(gamma=0.99, noise_scale=0.4, noise_clip=0.3, action_limit=0.5)
    ref = R.td3_critic_stage(nets, mb, None if noise is None else noise[0], PS_, QS_, **hp)
    names = ["policy", "q1"] + (["q2"] if twin else [])
    layers = {k: O.unflatten_layers(v, PS_ if "policy" in k else QS_) for k, v in nets.items()}
    adams = {k: O.AdamState(nets[k].size, 1e-3) for k in names}
    logs = OP.offpolicy_train(layers, adams, [mb], noise, policy_delay=1, twin=twin, **hp)
    for i, name in enumerate(names[1:]):
        assert rel_err(logs[name + "_values"][0], ref["q_values"][i]) < 1e-5, name
        assert rel_err(logs[name + "_losses"][0], ref["losses"][i]) < 1e-5, name
        assert rel_err(adams[name].m / np.float32(0.1), ref["grads"][i]) < 1e-5, name
    assert np.isfinite(ref["margin"]).all() and (ref["margin"] > 0).all()
    pol = R.td3_policy_stage(nets["policy"], O.flatten_layers(layers["q1"]), mb["observations"], PS_, QS_)
    assert rel_err(logs["policy_losses"][0], pol["loss"]) < 1e-5
    assert rel_err(adams["policy"].m / np.float32(0.1), pol["grad"]) < 1e-5


@pytest.mark.parametrize("learn_alpha", [False, True])
def test_float64_reference_agrees_with_the_sac_oracle_on_one_step(learn_alpha):
    """oracle/offpolicy_f64.py against oracle/sac.py (float32 autograd, torch.optim.Adam) on one SAC step."""
    import torch
    from oracle import offpolicy_f64 as R
    from oracle import sac as OS
    A_, PS_, QS_, B = 2, [5, 24, 20, 4], [7, 24, 20, 1], 16
    rng, nets, mb = _small_problem(4, 5, A_, B, PS_, QS_, 2)
    nets["target_q1"], nets["target_q2"] = nets["q1"].copy(), nets["q2"].copy()  # the SAC oracle copies the critics
    noise = rng.standard_normal((1, 2, B, A_)).astype(np.float32)

    def module(flat, sizes):
        m = torch.nn.Sequential(*[x for i, o in zip(sizes[:-1], sizes[1:]) for x in (torch.nn.Linear(i, o), torch.nn.ReLU())][:-1])
        torch.nn.utils.vector_to_parameters(torch.as_tensor(flat), m.parameters())
        return m

    orc = OS.SacOracle(module(nets["policy"], PS_), module(nets["q1"], QS_), module(nets["q2"], QS_), alpha=0.3,
                       learn_alpha=learn_alpha, limit=1.5)
    logs = orc.train([mb], noise)
    alpha = float(np.exp(np.float32(np.log(0.3)))) if learn_alpha else 0.3
    ref = R.sac_critic_stage(nets, mb, noise[0, 0], alpha, PS_, QS_, action_limit=1.5)
    for i, (q, opt) in enumerate(((orc.q1, orc.q1_opt), (orc.q2, orc.q2_opt))):
        assert rel_err(logs[f"q{i + 1}_values"][0], ref["q_values"][i]) < 1e-5
        assert rel_err(logs[f"q{i + 1}_losses"][0], ref["losses"][i]) < 1e-5
        g = np.concatenate([opt.state[p]["exp_avg"].reshape(-1).numpy() for p in q.parameters()]) / np.float32(0.1)
        assert rel_err(g, ref["grads"][i]) < 1e-5
    flat = lambda m: torch.nn.utils.parameters_to_vector(m.parameters()).detach().numpy()
    pol = R.sac_policy_stage(nets["policy"], flat(orc.q1), flat(orc.q2), mb["observations"], noise[0, 1], alpha, PS_,
                             QS_, action_limit=1.5)
    g = np.concatenate([orc.pi_opt.state[p]["exp_avg"].reshape(-1).numpy() for p in orc.pi.parameters()]) / np.float32(0.1)
    assert rel_err(logs["policy_losses"][0], pol["loss"]) < 1e-5
    assert rel_err(logs["log_prob_means"][0], pol["logp_mean"]) < 1e-5
    assert rel_err(g, pol["grad"]) < 1e-5
    if learn_alpha:
        m = float(orc.alpha_opt.state[orc.log_alpha]["exp_avg"]) / np.float32(0.1)
        assert rel_err(m, pol["alpha_grad"]) < 1e-5


def test_fma_f32_rounds_once():
    """oracle/offpolicy_f64.fma_f32 against exact rational arithmetic, including float64 sums that land exactly halfway
    between two float32 values (where rounding to float64 first and then to float32 would err)."""
    from fractions import Fraction
    from oracle import offpolicy_f64 as R
    rng = np.random.default_rng(0)
    n = 3000
    a = rng.standard_normal(n).astype(np.float32)
    b = (rng.standard_normal(n) * 10.0 ** rng.integers(-6, 3, n)).astype(np.float32)
    c = rng.standard_normal(n).astype(np.float32)
    # crafted: a * b = +-(2^-24 - 2^-70), so a * b + c rounds to float64 exactly on a float32 midpoint whose
    # ties-to-even neighbour is the wrong one (below the midpoint, below in magnitude, above it); the last is plain
    u = 2.0 ** -23
    a[:4] = np.float32(1 + u)
    b[:4] = np.float32(2.0 ** -24 * (1 - u)) * np.array([1, -1, -1, 1], np.float32)
    c[:4] = np.array([1 + u, -(1 + u), 1 + 2 * u + u, 1.0], np.float32)
    got = R.fma_f32(a, b, c)

    def exact(x, y, z):
        v = Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))
        lo = np.float32(float(v))  # a neighbour; then pick the nearest float32 (ties to even) exactly
        cands = [np.nextafter(lo, np.float32(-np.inf)), lo, np.nextafter(lo, np.float32(np.inf))]
        dist = [abs(Fraction(float(cd)) - v) for cd in cands]
        best = min(dist)
        ties = [cd for cd, d in zip(cands, dist) if d == best]
        return ties[0] if len(ties) == 1 else [t for t in ties if (t.view(np.int32) & 1) == 0][0]

    want = np.array([exact(x, y, z) for x, y, z in zip(a, b, c)], dtype=np.float32)
    np.testing.assert_array_equal(got, want)
    naive = (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)
    assert (naive[:4] != want[:4]).any()  # the crafted cases do hit double rounding
