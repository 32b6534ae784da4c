"""CPU: CQL's host side -- the float32 oracle against the float64 stage, the penalty head's closed-form gradients,
the constructor's refusals, ReplayBuffer.from_dataset, the checkpoint round trip, the group signature, and an
oracle-driven learn_offline run on a fixed bandit dataset that sets the bars for the GPU run (tests/test_gpu_cql.py)."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import cql as OC
from test_sac import A_DIM, O_DIM, RETURN_BAR, BanditEnv, OracleSAC, evaluation_return

N_DATA = 20000
OFFLINE = dict(num_epochs=4, num_train_steps=250, minibatch_size=64, num_evaluation_episodes=10, evaluation_interval=1,
               model_saving_interval=4)
GAP_MARGIN = 1.0  # mean Q on dataset actions minus mean Q on uniform actions, at least (the oracle reaches 3.1)


def bandit_dataset(n=N_DATA, seed=0, noise=0.3):
    """D4RL-style columns from a seeded noisy behaviour policy on BanditEnv: a = clip(f(obs) + N(0, 0.3^2), -1, 1)."""
    rng = np.random.default_rng(seed)
    obs = rng.uniform(-1, 1, (n, O_DIM)).astype(np.float32)
    f = 0.8 * np.tanh(obs @ BanditEnv.M.T)
    act = np.clip(f + noise * rng.standard_normal((n, A_DIM)), -1, 1).astype(np.float32)
    rew = -np.sum((act.astype(np.float64) - f) ** 2, axis=1)
    nobs = rng.uniform(-1, 1, (n, O_DIM)).astype(np.float32)
    return dict(observations=obs, actions=act, rewards=rew, next_observations=nobs, terminals=np.ones(n, bool))


def make_offline(cls_name="CQL", hidden=64, seed=0, dataset=None, **kw):
    from rl_replicas_b200 import algorithms
    from rl_replicas_b200.evaluator import Evaluator
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import SquashedGaussianPolicy
    from rl_replicas_b200.q_function import QFunction
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    torch.manual_seed(seed)
    env = BanditEnv()
    pnet = MLP([O_DIM, hidden, hidden, 2 * A_DIM], torch.nn.ReLU)
    q1, q2 = (MLP([O_DIM + A_DIM, hidden, hidden, 1], torch.nn.ReLU) for _ in range(2))
    rb = ReplayBuffer.from_dataset(bandit_dataset() if dataset is None else dataset)
    policy = SquashedGaussianPolicy(pnet, torch.optim.Adam(pnet.parameters(), lr=1e-3))
    return getattr(algorithms, cls_name)(policy, None, QFunction(q1, torch.optim.Adam(q1.parameters(), lr=1e-3)),
                                         QFunction(q2, torch.optim.Adam(q2.parameters(), lr=1e-3)), env, None, rb,
                                         Evaluator(seed=0), **kw)


def q_gap(algo, n=2000, seed=9):
    """mean over critics and dataset rows of Q(s, a_data) - mean over uniform actions of Q(s, u)."""
    d = bandit_dataset(n, seed=seed)
    o, a = torch.as_tensor(d["observations"]), torch.as_tensor(d["actions"])
    u = torch.as_tensor(np.random.default_rng(seed).uniform(-1, 1, a.shape).astype(np.float32))
    with torch.no_grad():
        qs = [q.network(torch.cat([o, x], -1)).mean().item() for q in (algo.q_function_1, algo.q_function_2)
              for x in (a, u)]
    return (qs[0] - qs[1] + qs[2] - qs[3]) / 2


class OracleCQL:
    """CQL.train with the oracle in place of the engine, on the learner's host draw order."""

    @staticmethod
    def patch(algo):
        from rl_replicas_b200.algorithms._onpolicy import describe_mlp, flat_params, write_flat
        oracle = OC.CqlOracle(algo.policy.network, algo.q_function_1.network, algo.q_function_2.network,
                              cql_weight=algo.cql_weight, cql_n_actions=algo.cql_n_actions,
                              cql_temperature=algo.cql_temperature, cql_target_action_gap=algo.cql_target_action_gap,
                              backup_entropy=algo.backup_entropy, gamma=algo.gamma, rho=algo.polyak_rho,
                              alpha=algo.alpha, learn_alpha=algo.learn_alpha, target_entropy=algo.target_entropy,
                              limit=algo.policy.action_limit)

        def train(replay_buffer, num_train_steps, minibatch_size):
            S, B = num_train_steps, minibatch_size
            idx = np.stack([replay_buffer.sample_indices(B) for _ in range(S)])
            oracle.train([replay_buffer.gather(idx[s]) for s in range(S)], algo._noise(S, B))
            for src, dst in ((oracle.pi, algo.policy.network), (oracle.q1, algo.q_function_1.network),
                             (oracle.q2, algo.q_function_2.network)):
                write_flat(describe_mlp(dst)[3], flat_params(describe_mlp(src)[3]))
        algo.train = train
        return oracle


def _random_nets(psz, qsz, seed):
    rng = np.random.default_rng(seed)
    size = lambda s: sum(s[i + 1] * (s[i] + 1) for i in range(len(s) - 1))
    mk = lambda s: rng.standard_normal(size(s)) * 0.3
    return dict(policy=mk(psz), q1=mk(qsz), q2=mk(qsz), target_q1=mk(qsz), target_q2=mk(qsz))


def _modules(nets, psz, qsz):
    from rl_replicas_b200.networks import MLP
    mods = {}
    for k, v in nets.items():
        m = MLP(psz if k == "policy" else qsz, torch.nn.ReLU)
        torch.nn.utils.vector_to_parameters(torch.as_tensor(v, dtype=torch.float32), m.parameters())
        mods[k] = m
    return mods


@pytest.mark.parametrize("T,tau,backup", [(1.0, None, False), (0.5, None, True), (2.0, 1.0, False), (1.0, -2.0, True)])
def test_float32_oracle_agrees_with_the_float64_stage(T, tau, backup):
    """One oracle step's critic gradients (Adam's first moment / 0.1), losses, gaps and Lagrange gradient against
    critic_stage_f64 on the same draws."""
    O, A, H, B, N = 4, 2, 16, 32, 5
    psz, qsz = [O, H, H, 2 * A], [O + A, H, H, 1]
    nets = _random_nets(psz, qsz, 3)
    mods = _modules(nets, psz, qsz)
    rng = np.random.default_rng(4)
    f32 = lambda x: np.asarray(x, np.float32)
    mb = dict(observations=f32(rng.standard_normal((B, O))), actions=f32(rng.uniform(-1, 1, (B, A))),
              rewards=f32(rng.standard_normal(B)), next_observations=f32(rng.standard_normal((B, O))),
              dones=rng.random(B) < 0.2)
    sac = f32(rng.standard_normal((1, 2, B, A)))
    draws = np.concatenate([rng.random((1, 1, B, N, A)), rng.standard_normal((1, 2, B, N, A))], 1).astype(np.float32)
    oracle = OC.CqlOracle(mods["policy"], mods["q1"], mods["q2"], cql_weight=3.0, cql_n_actions=N,
                          cql_temperature=T, cql_target_action_gap=tau, backup_entropy=backup)
    with torch.no_grad():
        for k in ("q1", "q2"):
            torch.nn.utils.vector_to_parameters(torch.as_tensor(nets["target_" + k], dtype=torch.float32),
                                                getattr(oracle, k + "_targ").parameters())
    logs = oracle.train([mb], (sac, draws))
    c = OC.critic_stage_f64(nets, mb, sac[0, 0], draws[0], 0.2, psz, qsz, 3.0, T, alpha_prime=1.0,
                            target_action_gap=tau, backup_entropy=backup)
    rel = lambda a, b: float(np.max(np.abs(np.asarray(a, np.float64) - b)) / max(np.max(np.abs(b)), 1e-12))
    for k, opt in ((1, oracle.q1_opt), (2, oracle.q2_opt)):
        g = torch.cat([opt.state[p]["exp_avg"].reshape(-1) for p in opt.param_groups[0]["params"]]).numpy() / 0.1
        assert rel(g, c[f"q{k}_grad"]) < 1e-4
        assert rel(logs[f"q{k}_losses"][0], c[f"q{k}_loss"]) < 1e-5
        assert rel(logs[f"cql_gap_{k}"][0], c[f"q{k}_gap"]) < 1e-4
        assert rel(logs[f"q{k}_values"][0], c[f"q{k}_values"]) < 1e-5
    if tau is not None:
        st = oracle.alpha_prime_opt.state[oracle.log_alpha_prime]
        assert rel(float(st["exp_avg"]) / 0.1, c["alpha_prime_grad"]) < 1e-4


def test_closed_form_penalty_gradients_match_autograd():
    rng = np.random.default_rng(0)
    B, n3, T, w = 16, 30, 0.7, 2.5
    qs = torch.tensor(rng.standard_normal((B, n3)), requires_grad=True)
    qd = torch.tensor(rng.standard_normal(B), requires_grad=True)
    logd = torch.tensor(rng.standard_normal((B, n3)))
    (w * OC.penalty(qs, logd, qd, T)).backward()
    gs, gd = OC.penalty_grad_closed_form(qs.detach(), logd, w, T)
    np.testing.assert_allclose(qs.grad.numpy(), gs.numpy(), rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(qd.grad.numpy(), gd.numpy(), rtol=1e-12)


def test_constructor_refusals():
    from rl_replicas_b200.critics import ContinuousQuantileQFunction
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.replay_buffer import PrioritizedReplayBuffer
    for kw, match in ((dict(cql_weight=-1.0), "cql_weight"), (dict(cql_temperature=0.0), "cql_temperature"),
                      (dict(cql_n_actions=0), "cql_n_actions"), (dict(cql_n_actions=65), "cql_n_actions"),
                      (dict(cql_n_actions=2.0), "cql_n_actions"), (dict(cql_weight=math.inf), "finite"),
                      (dict(cql_target_action_gap=math.nan), "finite")):
        with pytest.raises(ValueError, match=match):
            make_offline(**kw)
    algo = make_offline()
    qn = MLP([O_DIM + A_DIM, 8, 5], torch.nn.ReLU)
    from rl_replicas_b200.algorithms import CQL
    with pytest.raises(TypeError, match="quantile"):
        CQL(algo.policy, None, ContinuousQuantileQFunction(qn, torch.optim.Adam(qn.parameters()), n_quantiles=5),
            algo.q_function_2, algo.env, None, algo.replay_buffer, None)
    with pytest.raises(ValueError, match="PrioritizedReplayBuffer"):
        CQL(algo.policy, None, algo.q_function_1, algo.q_function_2, algo.env, None, PrioritizedReplayBuffer(), None)
    with pytest.raises(ValueError, match="learn_offline"):
        algo.learn(num_epochs=1)


def test_from_dataset_columns_dones_and_episode_ends():
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    d = bandit_dataset(10)
    d["terminals"] = np.zeros(10, bool)
    d["terminals"][3] = True
    d["timeouts"] = np.zeros(10, bool)
    d["timeouts"][6] = True
    rb = ReplayBuffer.from_dataset(d)
    assert rb.current_size == 10 and rb.buffer_size == 10
    np.testing.assert_array_equal(np.asarray(rb.observations), d["observations"])
    np.testing.assert_array_equal(np.asarray(rb.actions), d["actions"])
    np.testing.assert_array_equal(np.asarray(rb.rewards), d["rewards"])
    np.testing.assert_array_equal(np.asarray(rb.next_observations), d["next_observations"])
    np.testing.assert_array_equal(np.asarray(rb.dones), d["terminals"])
    assert [i for i, e in enumerate(rb.episode_ends) if e] == [3, 6, 9]
    np.random.seed(0)
    mb = rb.sample_minibatch(32)
    assert np.asarray(mb["observations"]).shape == (32, O_DIM)
    assert ReplayBuffer.from_dataset(d, buffer_size=50).buffer_size == 50


@pytest.mark.parametrize("change,match", [
    (lambda d: d.pop("terminals"), "lacks"),
    (lambda d: d.__setitem__("rewards", d["rewards"][:-1]), "length"),
    (lambda d: d["actions"].__setitem__((2, 0), np.nan), "non-finite"),
    (lambda d: d["observations"].__setitem__((1, 1), np.inf), "non-finite"),
])
def test_from_dataset_refusals(change, match):
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    d = bandit_dataset(10)
    change(d)
    with pytest.raises(ValueError, match=match):
        ReplayBuffer.from_dataset(d)


def test_from_dataset_refuses_a_smaller_buffer():
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    with pytest.raises(ValueError, match="smaller"):
        ReplayBuffer.from_dataset(bandit_dataset(10), buffer_size=9)


def test_save_and_load_round_trip(tmp_path):
    algo = make_offline(cql_target_action_gap=1.0)
    with torch.no_grad():
        algo.log_alpha_prime.fill_(0.7)
    algo._store_alpha_prime_state(0.7, 0.1, 0.2, 3)
    path = os.path.join(tmp_path, "model.pt")
    algo.save_model(2, path)
    other = make_offline(seed=5, cql_target_action_gap=1.0)
    assert other.load_model(path) == 2
    assert other._alpha_prime_state() == algo._alpha_prime_state()
    for a, b in ((algo.q_function_1, other.q_function_1), (algo.policy, other.policy)):
        for x, y in zip(a.network.parameters(), b.network.parameters()):
            assert torch.equal(x, y)
    assert {"log_alpha_prime", "alpha_prime_optimizer_state_dict", "log_alpha"} <= set(torch.load(path).keys())


def test_group_signature():
    from rl_replicas_b200.algorithms import LearnerGroup
    g = LearnerGroup()
    g.add(make_offline())
    g.add(make_offline(seed=1))
    for kw in (dict(cql_n_actions=4), dict(cql_weight=1.0), dict(cql_target_action_gap=1.0)):
        with pytest.raises(ValueError, match="differs"):
            g.add(make_offline(seed=2, **kw))


def _offline_run(cls_name, tmp_path, **kw):
    np.random.seed(0)
    torch.manual_seed(0)
    algo = make_offline(cls_name, **kw)
    (OracleCQL if cls_name == "CQL" else OracleSAC).patch(algo)
    algo.learn_offline(output_dir=str(tmp_path), **OFFLINE)
    return algo


def test_oracle_driven_learn_offline_is_conservative(tmp_path):
    """The bars test_gpu_cql.py's learn_offline run must clear, reached here by the oracle with the same seeds: the
    evaluation return clears the SAC tests' bar, the critics rank dataset actions above uniform ones by GAP_MARGIN, and
    by more than offline SAC's critics do on the same data."""
    cql = _offline_run("CQL", tmp_path / "cql")
    sac = _offline_run("SAC", tmp_path / "sac")
    ret, gap, gap_sac = evaluation_return(cql), q_gap(cql), q_gap(sac)
    print(f"CQL return {ret:.3f}, Q gap {gap:.3f}; offline SAC Q gap {gap_sac:.3f}")
    assert ret > RETURN_BAR
    assert gap > GAP_MARGIN
    assert gap > gap_sac
    assert os.path.exists(tmp_path / "cql" / "model.pt")
