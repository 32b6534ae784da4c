"""GPU: SAC.train on the off-policy engine against the torch-autograd oracle (oracle/sac.py), bit-identical results
across its execution paths, the device-side draws, the engine's refusals, and SAC.learn end to end."""
import os
import types

import numpy as np
import pytest
import torch

from conftest import rel_err
from oracle import sac as OS
from test_sac import LEARN, RETURN_BAR, evaluation_return, make_sac

pytestmark = pytest.mark.gpu

SHAPES = {  # (obs, act, hidden, hidden activation, action limit, minibatch)
    "halfcheetah": (17, 6, 256, torch.nn.ReLU, 1.0, 256),
    "small_tanh": (5, 2, 64, torch.nn.Tanh, 2.0, 64),
}


def build(shape, seed=0, learn_alpha=False, clamp_rows=False, **kw):
    from rl_replicas_b200.algorithms import SAC
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import RandomPolicy, SquashedGaussianPolicy
    from rl_replicas_b200.q_function import QFunction
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    O, A, H, act, L, _ = SHAPES[shape]
    torch.manual_seed(seed)
    pnet = MLP([O, H, H, 2 * A], act)
    if clamp_rows:  # log_std above log_std_max = 2 on part of the batch: the clamp's zero gradient is exercised
        with torch.no_grad():
            pnet.network[-2].weight[A:] *= 8.0
            pnet.network[-2].bias[A:] = 1.9
    q1, q2 = MLP([O + A, H, H, 1], act), MLP([O + A, H, H, 1], act)
    hi = np.full(A, L, np.float32)
    env = types.SimpleNamespace(action_space=types.SimpleNamespace(high=hi, low=-hi, shape=(A,)),
                                spec=types.SimpleNamespace(id="stub"))
    algo = SAC(SquashedGaussianPolicy(pnet, torch.optim.Adam(pnet.parameters(), lr=1e-3), action_limit=L),
               RandomPolicy(None), QFunction(q1, torch.optim.Adam(q1.parameters(), lr=1e-3)),
               QFunction(q2, torch.optim.Adam(q2.parameters(), lr=1e-3)), env, None, ReplayBuffer(), None,
               learn_alpha=learn_alpha, alpha_lr=3e-3, **kw)
    algo.metrics_manager = None
    algo.current_total_steps = 0
    return algo


def fill(rb, O, A, L, n=5000, seed=1):
    from rl_replicas_b200.experience import Experience
    rng = np.random.default_rng(seed)
    e = Experience()
    obs = rng.standard_normal((n + 1, O)).astype(np.float32)
    e.observations = [[obs[i] for i in range(n)]]
    e.actions = [[a for a in rng.uniform(-L, L, (n, A)).astype(np.float32)]]
    e.rewards = [[float(x) for x in rng.standard_normal(n)]]
    e.dones = [[bool(x) for x in (rng.random(n) < 0.05)]]
    e.last_observations = [obs[n]]
    rb.add_experience(e)


def flat(m):
    return torch.nn.utils.parameters_to_vector(m.parameters()).detach().numpy()


def adam_flat(opt, key):
    ps = opt.param_groups[0]["params"]
    return np.concatenate([opt.state[p][key].reshape(-1).numpy() for p in ps]), int(float(opt.state[ps[0]]["step"]))


def oracle_for(algo):
    return OS.SacOracle(algo.policy.network, algo.q_function_1.network, algo.q_function_2.network, gamma=algo.gamma,
                        rho=algo.polyak_rho, alpha=algo.alpha, learn_alpha=algo.learn_alpha,
                        target_entropy=algo.target_entropy, alpha_lr=3e-3, limit=algo.policy.action_limit)


def compare(algo, oracle, logs, out):
    errs = {}
    for k in ("q1_values", "q2_values"):
        errs[k] = rel_err(out[k], np.stack(logs[k]))
    for k in ("q1_losses", "q2_losses", "policy_losses", "log_prob_means", "alphas"):
        errs[k] = rel_err(out[k], np.asarray(logs[k]))
    pairs = {"policy": (algo.policy, oracle.pi), "q1": (algo.q_function_1, oracle.q1), "q2": (algo.q_function_2, oracle.q2)}
    for name, (m, o) in pairs.items():
        errs[name] = rel_err(flat(m.network), flat(o))
        opt = {"policy": oracle.pi_opt, "q1": oracle.q1_opt, "q2": oracle.q2_opt}[name]
        for key in ("exp_avg", "exp_avg_sq"):
            got, step = adam_flat(m.optimizer, key)
            want, step_o = adam_flat(opt, key)
            errs[f"{name}.{key}"] = rel_err(got, want)
            assert step == step_o, (name, step, step_o)
    errs["target_q1"] = rel_err(flat(algo.target_q_function_1.network), flat(oracle.q1_targ))
    errs["target_q2"] = rel_err(flat(algo.target_q_function_2.network), flat(oracle.q2_targ))
    errs["log_alpha"] = rel_err(float(algo.log_alpha.detach()), float(oracle.log_alpha.detach()))
    if algo.learn_alpha:
        for key in ("exp_avg", "exp_avg_sq"):
            got, step = adam_flat(algo.alpha_optimizer, key)
            want, step_o = adam_flat(oracle.alpha_opt, key)
            errs[f"alpha.{key}"] = rel_err(got, want)
            assert step == step_o
    return errs


@pytest.mark.parametrize("learn_alpha", [False, True])
@pytest.mark.parametrize("shape", ["halfcheetah", "small_tanh"])
def test_train_matches_the_oracle(shape, learn_alpha):
    """Ten SAC steps through SAC.train (device replay, graph replay) against the autograd oracle with the same
    minibatches and noise.  small_tanh starts with log_std above the clamp on part of the batch."""
    O, A, H, act, L, B = SHAPES[shape]
    S = 10
    algo = build(shape, learn_alpha=learn_alpha, clamp_rows=shape == "small_tanh")
    fill(algo.replay_buffer, O, A, L)
    if shape == "small_tanh":
        with torch.no_grad():
            o = torch.as_tensor(np.stack(algo.replay_buffer.observations[:1000]))
            frac = (algo.policy.network(o)[:, A:] > 2.0).float().mean()
        assert 0.05 < float(frac) < 0.95, float(frac)
    oracle = oracle_for(algo)
    np.random.seed(7)
    torch.manual_seed(7)
    state_np, state_t = np.random.get_state(), torch.get_rng_state()
    algo.train(algo.replay_buffer, S, B)
    out = algo.last_train_output
    np.random.set_state(state_np)
    torch.set_rng_state(state_t)
    mbs = [algo.replay_buffer.sample_minibatch(B) for _ in range(S)]
    noise = torch.stack([torch.stack([torch.randn(B, A), torch.randn(B, A)]) for _ in range(S)]).numpy()
    logs = oracle.train(mbs, noise)
    assert len(out["policy_losses"]) == S
    errs = compare(algo, oracle, logs, out)
    print(f"{shape} learn_alpha={learn_alpha}:", {k: f"{v:.2e}" for k, v in errs.items()})
    # Measured on H100, halfcheetah with a learned alpha: through step 7 the policy is within 4e-6 of the oracle; in
    # step 8 unit 26 of the second hidden layer has a pre-activation 5e-9 from the ReLU kink on one row, so float
    # rounding decides whether that row's gradient passes.  That unit's Adam exp_avg_sq is 6.5e-10, so Adam turns the
    # one-row difference into an lr-sized step on its incoming weights: the policy and its moments then differ by
    # ~2e-3 of their maximum.  Everything else (losses, Q-values, log pi, alpha, critics, targets) stays below 2e-5.
    kink = {"policy", "policy.exp_avg", "policy.exp_avg_sq"} if (shape, learn_alpha) == ("halfcheetah", True) else set()
    for k, v in errs.items():
        assert v < (1e-2 if k in kink else 2e-5), (k, v, errs)
    if not learn_alpha:
        assert (out["alphas"] == np.float32(0.2)).all()


def test_host_staged_graph_replay_and_device_gather_are_bit_identical():
    """Plain launches on host-staged minibatches, the captured graph replayed across calls (the third call changes S
    and recaptures) and the device-replay gather all agree bit for bit."""
    O, A, _, _, L, _ = SHAPES["small_tanh"]
    S, B = 6, 32

    def run(device_replay, graph):
        os.environ["B200RL_OFFPOLICY_GRAPH"] = "1" if graph else "0"
        algo = build("small_tanh", learn_alpha=True)
        fill(algo.replay_buffer, O, A, L, n=3000, seed=3)
        algo.use_device_replay = device_replay
        outs = []
        for call in range(3):
            np.random.seed(10 + call)
            torch.manual_seed(10 + call)
            algo.train(algo.replay_buffer, S + (call == 2), B)
            outs.append(algo.last_train_output)
        nets = [flat(m.network) for m in (algo.policy, algo.q_function_1, algo.q_function_2, algo.target_q_function_1,
                                          algo.target_q_function_2)]
        return outs, nets + [algo.log_alpha.detach().numpy().reshape(1)]

    try:
        ref_outs, ref_nets = run(False, False)
        for dev, graph in ((True, True), (False, True), (True, False)):
            outs, nets = run(dev, graph)
            for a, b in zip(outs, ref_outs):
                assert a.keys() == b.keys()
                for k in a:
                    np.testing.assert_array_equal(a[k], b[k], err_msg=f"{k} dev={dev} graph={graph}")
            for i, (a, b) in enumerate(zip(nets, ref_nets)):
                np.testing.assert_array_equal(a, b, err_msg=f"net {i} dev={dev} graph={graph}")
    finally:
        os.environ.pop("B200RL_OFFPOLICY_GRAPH", None)


def test_device_side_draws_replay_through_the_oracle():
    O, A, _, _, L, _ = SHAPES["small_tanh"]
    S, B = 8, 64
    algo = build("small_tanh", learn_alpha=True)
    fill(algo.replay_buffer, O, A, L, n=3000, seed=4)
    algo.use_device_rng, algo.device_rng_seed = True, 77
    oracle = oracle_for(algo)
    algo.train(algo.replay_buffer, S, B)
    idx, noise = algo._engine.get_draws(S, B)
    assert idx.shape == (S, B) and noise.shape == (S, 2, B, A)
    rb = algo.replay_buffer
    mbs = [{k: rb._cols[k][idx[s]] for k in rb.COLUMNS} for s in range(S)]
    logs = oracle.train(mbs, noise)
    errs = compare(algo, oracle, logs, algo.last_train_output)
    for k, v in errs.items():
        assert v < 2e-5, (k, v, errs)
    algo.train(rb, 50, 256)
    _, big = algo._engine.get_draws(50, 256)
    assert big.shape == (50, 2, 256, A)
    assert abs(big.mean()) < 0.03 and abs(big.std() - 1.0) < 0.03 and np.abs(big).max() < 6.5
    assert abs(np.mean(big ** 3)) < 0.1 and abs(np.mean(big ** 4) - 3.0) < 0.25
    assert abs(np.corrcoef(big[:, 0].ravel(), big[:, 1].ravel())[0, 1]) < 0.02  # the two draws are independent


def test_engine_refuses_bad_sac_configurations():
    from rl_replicas_b200._lib import B200RLError
    from rl_replicas_b200.engine import OffPolicyEngine
    with pytest.raises(B200RLError, match="n_q = 2"):
        OffPolicyEngine([5, 32, 32, 4], [7, 32, 32, 1], 1, 16, 2, ("relu", "identity"), algo=OffPolicyEngine.SAC)
    with pytest.raises(B200RLError, match="mean \\| log_std"):
        OffPolicyEngine([5, 32, 32, 3], [7, 32, 32, 1], 2, 16, 2, ("relu", "identity"), algo=OffPolicyEngine.SAC)
    algo = build("small_tanh")
    e = algo._ensure_engine(2, 8)
    layout, _ = e.state_layout()
    assert [i for kind, i, _, _ in layout if kind == "params"] == [0, 1, 2, 4, 5]
    O, A = 5, 2
    z = lambda *s: np.zeros(s, np.float32)
    with pytest.raises(B200RLError, match="set_sac"):
        e.train(algo._hparams(True, 1), z(2, 8, O), z(2, 8, A), z(2, 8), z(2, 8, O), z(2, 8), z(2, 2, 8, A))
    e.set_sac(algo._sac_hparams())
    with pytest.raises(B200RLError, match="noise"):
        e.train(algo._hparams(True, 1), z(2, 8, O), z(2, 8, A), z(2, 8), z(2, 8, O), z(2, 8), None)


def test_learn_solves_the_bandit(tmp_path, capsys):
    """SAC.learn end to end on the one-step bandit of tests/test_sac.py with the seeds the oracle-driven loop used
    there: the tags are recorded, model.pt is written, and the evaluation return clears the same bar."""
    np.random.seed(0)
    algo = make_sac(learn_alpha=True)
    algo.learn(output_dir=str(tmp_path), **LEARN)
    after = evaluation_return(algo)
    printed = capsys.readouterr().out
    with capsys.disabled():
        print(f"SAC.learn on the bandit: evaluation return {after:.3f}")
    for tag in ("policy/average_loss", "policy/average_log_prob", "alpha/value", "q-function_1/average_loss",
                "q-function_2/average_loss", "q-function_1/avarage_q-value", "evaluation/average_episode_return"):
        assert f"\n{tag}: " in printed, tag
    assert os.path.exists(os.path.join(tmp_path, "model.pt"))
    assert after > RETURN_BAR
