"""CPU: D4PG's host side -- DistributionalQFunction, the D4PG constructor's refusals, the float32 oracle against the
float64 reference, the projection against Algorithm 1, the LearnerGroup signature, the checkpoint round trip, and the
oracle-driven learn() loop that sets the bar for the GPU end-to-end test (tests/test_gpu_d4pg.py)."""
import types

import numpy as np
import pytest
import torch

from oracle import c51 as OC
from oracle import d4pg as OD
from test_sac import A_DIM, O_DIM, BanditEnv

N_ATOMS, V = 51, (-4.0, 1.0)  # BanditEnv's rewards lie in [-8, 0] and are mostly above -3


def make_d4pg(hidden=64, seed=0, n_atoms=N_ATOMS, v=V, act=torch.nn.ReLU, replay_buffer=None, env=None, **kw):
    from rl_replicas_b200.algorithms import D4PG
    from rl_replicas_b200.critics import DistributionalQFunction
    from rl_replicas_b200.evaluator import Evaluator
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import DeterministicPolicy, RandomPolicy
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    from rl_replicas_b200.samplers import BatchSampler
    torch.manual_seed(seed)
    env = env or BanditEnv()
    pnet = MLP([O_DIM, hidden, hidden, A_DIM], act, torch.nn.Tanh)
    qnet = MLP([O_DIM + A_DIM, hidden, hidden, n_atoms], act)
    policy = DeterministicPolicy(pnet, torch.optim.Adam(pnet.parameters(), lr=1e-3))
    qf = DistributionalQFunction(qnet, torch.optim.Adam(qnet.parameters(), lr=1e-3), n_atoms=n_atoms, v_min=v[0],
                                 v_max=v[1])
    return D4PG(policy, RandomPolicy(env.action_space), qf, env, BatchSampler(env, seed=0),
                replay_buffer if replay_buffer is not None else ReplayBuffer(buffer_size=100000), Evaluator(seed=0),
                **kw)


def evaluation_return(algo):
    """test_sac.evaluation_return with DDPG's deterministic policy."""
    from rl_replicas_b200.evaluator import Evaluator
    returns, _ = Evaluator(seed=123).evaluate(algo.policy, BanditEnv(), 200)
    return float(np.mean(returns))


def flat(m):
    return torch.cat([p.detach().reshape(-1) for p in m.parameters()]).numpy()


def random_minibatch(B, rng, O=O_DIM, A=A_DIM, v_max=V[1]):
    rew = (rng.standard_normal(B) - 1.0).astype(np.float32)
    rew[::7] = 3.0 * v_max  # every Tz_j clamps at v_max
    return dict(observations=rng.uniform(-1, 1, (B, O)).astype(np.float32),
                actions=rng.uniform(-1, 1, (B, A)).astype(np.float32), rewards=rew,
                next_observations=rng.uniform(-1, 1, (B, O)).astype(np.float32), dones=rng.random(B) < 0.3)


def oracle_for(algo, **kw):
    q = algo.q_function
    return OD.D4pgOracle(algo.policy.network, q.network, algo.target_policy.network, algo.target_q_function.network,
                         algo.policy.optimizer, q.optimizer, n_atoms=q.n_atoms, v_min=q.v_min, v_max=q.v_max,
                         gamma=algo.gamma, rho=algo.polyak_rho, **kw)


def test_distributional_q_function_has_c51s_support_and_normalised_distributions():
    from rl_replicas_b200.critics import CategoricalQFunction, DistributionalQFunction
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.q_function import DistributionalQFunction as Reexported
    assert Reexported is DistributionalQFunction
    net = MLP([5, 16, 11], torch.nn.ReLU)
    opt = torch.optim.Adam(net.parameters())
    qf = DistributionalQFunction(net, opt, n_atoms=11, v_min=-3.0, v_max=7.0)
    c51 = CategoricalQFunction(MLP([5, 16, 11], torch.nn.ReLU), opt, n_atoms=11, v_min=-3.0, v_max=7.0)
    assert qf.support.dtype == torch.float32 and torch.equal(qf.support, c51.support)
    assert torch.equal(qf.support, torch.from_numpy(OC.support(11, -3.0, 7.0)))
    o, a = torch.randn(9, 3), torch.randn(9, 2)
    p = qf.distribution(o, a)
    assert p.shape == (9, 11)
    torch.testing.assert_close(p.sum(-1), torch.ones(9), rtol=0, atol=1e-6)
    torch.testing.assert_close(qf(o, a), (p * qf.support).sum(-1))
    for bad in (dict(n_atoms=1), dict(n_atoms=257), dict(v_min=1.0, v_max=1.0), dict(v_max=float("inf"))):
        with pytest.raises(ValueError):
            DistributionalQFunction(net, opt, **bad)


def test_constructor_refusals():
    from rl_replicas_b200.algorithms import D4PG
    from rl_replicas_b200.critics import QFunction
    from rl_replicas_b200.networks import MLP, NoisyMLP
    good = make_d4pg()
    args = lambda **o: dict(dict(policy=good.policy, exploration_policy=None, q_function=good.q_function, env=good.env,
                                 sampler=None, replay_buffer=None, evaluator=None), **o)
    discrete = types.SimpleNamespace(action_space=types.SimpleNamespace(n=3, shape=()),
                                     observation_space=types.SimpleNamespace(shape=(O_DIM,)))
    with pytest.raises(ValueError, match="continuous action space"):
        D4PG(**args(env=discrete))
    qnet = MLP([O_DIM + A_DIM, 16, 1], torch.nn.ReLU)
    with pytest.raises(ValueError, match="DistributionalQFunction"):
        D4PG(**args(q_function=QFunction(qnet, torch.optim.Adam(qnet.parameters()))))
    from rl_replicas_b200.critics import DistributionalQFunction
    with pytest.raises(ValueError, match="the critic must map"):
        D4PG(**args(q_function=DistributionalQFunction(good.q_function.network, good.q_function.optimizer, n_atoms=11)))
    wide = make_d4pg()
    wide_net = MLP([O_DIM + 1, 16, N_ATOMS], torch.nn.ReLU)
    wide.q_function.network = wide_net
    wide.q_function.optimizer = torch.optim.Adam(wide_net.parameters())
    with pytest.raises(ValueError, match="the critic must map"):
        D4PG(**args(q_function=wide.q_function))
    pnet = MLP([O_DIM, 16, A_DIM + 1], torch.nn.ReLU, torch.nn.Tanh)
    with pytest.raises(ValueError, match="the policy must map"):
        D4PG(**args(policy=type(good.policy)(pnet, torch.optim.Adam(pnet.parameters()))))
    for n in (0, 33, 1.5, True):
        with pytest.raises(ValueError, match="n_step"):
            D4PG(**args(n_step=n))
    noisy = NoisyMLP([O_DIM + A_DIM, 16, N_ATOMS], torch.nn.ReLU)
    with pytest.raises(NotImplementedError, match="noisy"):
        D4PG(**args(q_function=DistributionalQFunction(noisy, torch.optim.Adam(noisy.parameters()), n_atoms=N_ATOMS)))
    qf = good.q_function
    sgd = DistributionalQFunction(qf.network, torch.optim.SGD(qf.network.parameters(), lr=0.1), n_atoms=N_ATOMS)
    with pytest.raises(NotImplementedError, match="Adam"):
        D4PG(**args(q_function=sgd))
    # n-step windows and prioritized draws are assembled on the device: refused without the device replay
    from rl_replicas_b200.replay_buffer import PrioritizedReplayBuffer
    for algo in (make_d4pg(n_step=3), make_d4pg(replay_buffer=PrioritizedReplayBuffer(1000))):
        algo.use_device_replay = False
        with pytest.raises(ValueError, match="use_device_replay = True"):
            algo.train(algo.replay_buffer, 2, 8)


def test_projection_agrees_with_algorithm_1():
    rng = np.random.default_rng(3)
    for N, (v_min, v_max) in ((2, (-1.0, 1.0)), (51, V), (101, (-5.0, 5.0))):
        z = OC.support(N, v_min, v_max)
        p = rng.dirichlet(np.ones(N), 40)
        rew = 3.0 * rng.standard_normal(40)
        rew[::5] = z[rng.integers(0, N, 8)]  # targets on an atom
        done = rng.random(40) < 0.3
        disc = 0.99 ** rng.integers(1, 6, 40)
        m = OC.project(torch.as_tensor(p), torch.as_tensor(rew), torch.as_tensor(done, dtype=torch.float64),
                       torch.as_tensor(z, dtype=torch.float64), v_min, v_max, (v_max - v_min) / (N - 1),
                       torch.as_tensor(disc)[:, None]).numpy()
        from oracle.nstep import project_f64
        np.testing.assert_allclose(m, project_f64(p, rew, done, z, v_min, v_max, disc), rtol=0, atol=1e-12)


@pytest.mark.parametrize("weighted", [False, True])
def test_float32_oracle_agrees_with_the_float64_reference(weighted):
    """One oracle step from a fresh Adam: its exp_avg is 0.1 x the gradient.  The actor's gradient is taken through the
    oracle's own critic after its update, as the step takes it."""
    algo = make_d4pg(seed=1)
    with torch.no_grad():
        for p in algo.target_q_function.network.parameters():
            p.add_(0.05 * torch.randn_like(p))
    rng = np.random.default_rng(5)
    B = 64
    mb = random_minibatch(B, rng)
    prio = rng.uniform(0.1, 2.0, B) if weighted else None
    oracle = oracle_for(algo)
    logs = oracle.train([mb], [prio] if weighted else None, [0.6] if weighted else None)
    nets = dict(policy=flat(algo.policy.network), q1=flat(algo.q_function.network),
                target_policy=flat(algo.target_policy.network), target_q1=flat(algo.target_q_function.network))
    psz, qsz = [O_DIM, 64, 64, A_DIM], [O_DIM + A_DIM, 64, 64, N_ATOMS]
    w = OD.per_weights(prio, 0.6).astype(np.float32) if weighted else None
    ref = OD.d4pg_step_f64(nets, mb, psz, qsz, N_ATOMS, *V, gamma=algo.gamma, q_after=flat(oracle.q), weights=w)
    m_q = torch.cat([oracle.opt_q.state[p]["exp_avg"].reshape(-1) for p in oracle.q.parameters()]).numpy()
    m_pi = torch.cat([oracle.opt_pi.state[p]["exp_avg"].reshape(-1) for p in oracle.pi.parameters()]).numpy()
    for got, want, scale in ((m_q / 0.1, ref["grad_q"], ref["scale_q"]), (m_pi / 0.1, ref["grad_pi"], ref["scale_pi"])):
        assert np.max(np.abs(got - want) / np.maximum(scale, 1e-12)) < 1e-3
        assert np.linalg.norm(got - want) / np.linalg.norm(want) < 1e-5
    np.testing.assert_allclose(logs["q1_values"][0], ref["q_values"], rtol=0, atol=1e-5)
    assert abs(logs["q1_losses"][0] - ref["loss"]) < 1e-5 * abs(ref["loss"])
    assert abs(logs["policy_losses"][0] - ref["policy_loss"]) < 1e-5 * max(abs(ref["policy_loss"]), 1.0)
    np.testing.assert_allclose(logs["kl"][0], ref["kl"], rtol=0, atol=2e-5)
    assert (ref["kl"] > -1e-12).all()
    if weighted:
        np.testing.assert_allclose(logs["weights"][0], OD.per_weights(prio, 0.6))
        np.testing.assert_allclose(logs["priorities"][0], (np.maximum(logs["kl"][0].astype(np.float64), 0) + 1e-6) ** 0.6)


def _member(seed=0, **kw):
    return make_d4pg(seed=seed, **kw)


def test_group_signature():
    from rl_replicas_b200.algorithms import LearnerGroup
    from rl_replicas_b200.replay_buffer import PrioritizedReplayBuffer
    g = LearnerGroup()
    g.add(_member(0))
    g.add(_member(1))  # same shapes and settings, other weights
    for other, what in ((_member(2, n_atoms=21), "network"), (_member(2, v=(-5.0, 1.0)), "n_atoms, v_min, v_max"),
                        (_member(2, n_step=3), "n_step"),
                        (_member(2, replay_buffer=PrioritizedReplayBuffer(1000)), "prioritized replay")):
        with pytest.raises(ValueError, match=what):
            g.add(other)
    p = LearnerGroup()
    p.add(_member(0, replay_buffer=PrioritizedReplayBuffer(1000, alpha=0.6)))
    with pytest.raises(ValueError, match="prioritized replay alpha"):
        p.add(_member(1, replay_buffer=PrioritizedReplayBuffer(1000, alpha=0.5)))
    shared = PrioritizedReplayBuffer(1000, alpha=0.6)
    with pytest.raises(ValueError, match="share one PrioritizedReplayBuffer"):
        q = LearnerGroup()
        q.add(_member(0, replay_buffer=shared))
        q.add(_member(1, replay_buffer=shared))


def test_save_and_load_round_trip(tmp_path):
    algo = make_d4pg(seed=2)
    oracle = oracle_for(algo)
    oracle.train([random_minibatch(32, np.random.default_rng(1))])
    for src, dst in ((oracle.pi, algo.policy.network), (oracle.q, algo.q_function.network)):
        dst.load_state_dict(src.state_dict())
    algo.policy.optimizer.load_state_dict(oracle.opt_pi.state_dict())
    algo.q_function.optimizer.load_state_dict(oracle.opt_q.state_dict())
    algo.current_total_steps = 123
    path = str(tmp_path / "model.pt")
    algo.save_model(7, path)
    other = make_d4pg(seed=9)
    assert other.load_model(path) == 7 and other.current_total_steps == 123
    for a, b in ((algo.policy, other.policy), (algo.q_function, other.q_function)):
        np.testing.assert_array_equal(flat(a.network), flat(b.network))
        sa, sb = a.optimizer.state_dict()["state"], b.optimizer.state_dict()["state"]
        for k in sa:
            for key in ("exp_avg", "exp_avg_sq", "step"):
                assert torch.equal(sa[k][key], sb[k][key])
    np.testing.assert_array_equal(flat(algo.target_q_function.network), flat(other.target_q_function.network))


class OracleD4PG:
    """D4PG.train with the oracle in place of the engine: the same host index draws, the oracle's parameters written
    back into the learner's networks (targets included)."""

    @staticmethod
    def patch(algo):
        oracle = oracle_for(algo)

        def train(replay_buffer, num_train_steps, minibatch_size):
            S, B = num_train_steps, minibatch_size
            idx = np.stack([replay_buffer.sample_indices(B) for _ in range(S)])
            oracle.train([replay_buffer.gather(idx[s]) for s in range(S)])
            for src, dst in ((oracle.pi, algo.policy.network), (oracle.q, algo.q_function.network),
                             (oracle.pi_t, algo.target_policy.network), (oracle.q_t, algo.target_q_function.network)):
                dst.load_state_dict(src.state_dict())
        algo.train = train
        return oracle


LEARN = dict(num_epochs=40, batch_size=50, minibatch_size=64, num_start_steps=500, num_steps_before_update=500,
             num_train_steps=50, num_evaluation_episodes=10, evaluation_interval=500, model_saving_interval=500)
RETURN_BAR = -0.1  # tests/test_sac.py's bar: a uniform random policy scores about -0.85 on BanditEnv


def test_oracle_driven_learn_loop_solves_the_bandit(tmp_path):
    """The bar the GPU learn() loop must clear (tests/test_gpu_d4pg.py) is one the oracle reaches with the same seeds."""
    np.random.seed(0)
    algo = make_d4pg(polyak_rho=0.95)
    OracleD4PG.patch(algo)
    before = evaluation_return(algo)
    algo.learn(output_dir=str(tmp_path), **LEARN)
    after = evaluation_return(algo)
    print(f"oracle-driven learn: evaluation return {before:.3f} -> {after:.3f}")
    assert before < -0.3 and after > RETURN_BAR, (before, after)
