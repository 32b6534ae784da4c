"""CPU: C51's host side -- the float32 oracle (oracle/c51.py) against the float64 reference, the triangular projection
against Bellemare's Algorithm 1, CategoricalQFunction, the C51 constructor's refusals, its checkpoint round trip, the
LearnerGroup signature for C51 members, and the oracle-driven learn() loop that sets the bar for the GPU end-to-end
test (tests/test_gpu_c51.py)."""
import types

import numpy as np
import pytest
import torch

from oracle import c51 as OC
from test_dqn import DQN_KW, LEARN, N_ACT, O_DIM, RETURN_BAR, ChooseEnv, evaluation_return, flat, random_minibatch

C51_KW = dict(DQN_KW)
ATOMS = dict(n_atoms=51, v_min=-1.0, v_max=2.0)  # the choice task's returns are 0 and 1


def make_c51(hidden=64, seed=0, lr=1e-3, atoms=ATOMS, replay_buffer=None, **kw):
    from rl_replicas_b200.algorithms import C51
    from rl_replicas_b200.critics import CategoricalQFunction
    from rl_replicas_b200.evaluator import Evaluator
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import RandomPolicy
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    from rl_replicas_b200.samplers import BatchSampler
    torch.manual_seed(seed)
    env = ChooseEnv()
    net = MLP([O_DIM, hidden, hidden, N_ACT * atoms["n_atoms"]], torch.nn.ReLU)
    qf = CategoricalQFunction(net, torch.optim.Adam(net.parameters(), lr=lr), **atoms)
    return C51(qf, RandomPolicy(env.action_space), env, BatchSampler(env, seed=0),
               replay_buffer if replay_buffer is not None else ReplayBuffer(buffer_size=100000), Evaluator(seed=0), **kw)


@pytest.mark.parametrize("double_q", [False, True])
def test_float32_oracle_agrees_with_the_float64_reference(double_q):
    """One step: loss, Q(s, a) and the gradient (read from Adam's first moment) of the float32 autograd oracle within
    1e-5 of the float64 reference."""
    from rl_replicas_b200.networks import MLP
    torch.manual_seed(3)
    n, N, sizes = 5, 21, [4, 32, 32, 5 * 21]
    net, targ = MLP(sizes, torch.nn.Tanh), MLP(sizes, torch.nn.Tanh)
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    mb = random_minibatch(np.random.default_rng(0), 64, n=n, O=4)
    mb["rewards"] = mb["rewards"] * 4.0  # Tz clamps at both ends
    ref = OC.c51_step_f64(flat(net), flat(targ), mb, sizes, N, -3.0, 3.0, "tanh", 0.99, double_q)
    o = OC.C51Oracle(net, targ, opt, n_atoms=N, v_min=-3.0, v_max=3.0, gamma=0.99, target_update_interval=100,
                     double_q=double_q)
    logs = o.train([mb])
    grad = torch.cat([o.opt.state[p]["exp_avg"].reshape(-1) for p in o.q.parameters()]).numpy() / 0.1
    rel = lambda x, r: float(np.max(np.abs(np.asarray(x, np.float64) - r)) / np.max(np.abs(r)))
    assert rel(logs["q1_values"][0], ref["q_values"]) < 1e-5
    assert abs(logs["q1_losses"][0] - ref["loss"]) <= 1e-5 * abs(ref["loss"])
    assert rel(grad, ref["grad"]) < 1e-5
    assert (ref["scale"] >= np.abs(ref["grad"]) * (1 - 1e-12)).all()
    np.testing.assert_allclose(ref["m"].sum(1), 1.0, rtol=0, atol=1e-12)


def _projection_case(N, v_min, v_max, seed=0):
    """Rows that clamp at both ends (partly, then wholly), terminal rows landing exactly on atoms, and generic rows, with random p(s', a*)."""
    rng = np.random.default_rng(seed)
    z = v_min + np.arange(N) * ((v_max - v_min) / (N - 1))  # the support's formula, kept in float64
    B = 12
    rew = np.concatenate([[v_max + 5.0, v_min - 5.0, 1e3, -1e3], z[[0, N - 1, N // 2, 1]],
                          rng.uniform(v_min, v_max, B - 8)])
    done = np.zeros(B)
    done[4:8] = 1.0  # terminal: Tz = r, on an atom
    p = rng.random((B, N))
    p /= p.sum(1, keepdims=True)
    return p, rew, done, z


@pytest.mark.parametrize("N,v_min,v_max", [(51, -10.0, 10.0), (2, -1.0, 1.0), (11, 0.0, 1.0), (101, -5.0, 20.0)])
def test_triangular_projection_matches_algorithm_1(N, v_min, v_max):
    p, rew, done, z = _projection_case(N, v_min, v_max)
    want = OC.project_f64(p, rew, done, z, v_min, v_max, 0.9)
    t = lambda x: torch.as_tensor(x, dtype=torch.float64)
    got = OC.project(t(p), t(rew), t(done), t(z), v_min, v_max, (v_max - v_min) / (N - 1), 0.9).numpy()
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-12)
    np.testing.assert_allclose(got.sum(1), 1.0, rtol=0, atol=1e-12)  # mass is conserved
    # rows whose every Tz_j clamps put everything on an end atom, terminal rows on an atom exactly
    np.testing.assert_allclose(got[2, -1], 1.0, rtol=0, atol=1e-12)
    np.testing.assert_allclose(got[3, 0], 1.0, rtol=0, atol=1e-12)
    for r, k in zip(range(4, 8), (0, N - 1, N // 2, 1)):
        np.testing.assert_allclose(got[r, k], 1.0, rtol=0, atol=1e-12)


def test_projected_mass_sums_to_one_in_float32():
    p, rew, done, _ = _projection_case(51, -10.0, 10.0, seed=1)
    z = torch.from_numpy(OC.support(51, -10.0, 10.0))
    t = lambda x: torch.as_tensor(x, dtype=torch.float32)
    m = OC.project(t(p), t(rew), t(done), z, np.float32(-10.0), np.float32(10.0), np.float32(0.4), np.float32(0.99))
    np.testing.assert_allclose(m.sum(1).numpy(), 1.0, rtol=0, atol=1e-6)


def test_categorical_q_function():
    from rl_replicas_b200.critics import CategoricalQFunction
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import GreedyPolicy
    from rl_replicas_b200.q_function import CategoricalQFunction as Exported
    assert Exported is CategoricalQFunction
    torch.manual_seed(0)
    net = MLP([3, 16, 4 * 7], torch.nn.ReLU)
    qf = CategoricalQFunction(net, torch.optim.Adam(net.parameters()), n_atoms=7, v_min=-1.5, v_max=2.5)
    assert qf.support.dtype == torch.float32
    dz = 4.0 / 6
    assert qf.support.tolist() == [float(np.float32(-1.5 + i * dz)) for i in range(7)]
    wide = CategoricalQFunction(net, None, n_atoms=51, v_min=-10.0, v_max=10.0)
    np.testing.assert_array_equal(wide.support.numpy(), OC.support(51, -10.0, 10.0))
    obs = torch.randn(9, 3)
    d = qf.distribution(obs)
    assert d.shape == (9, 4, 7)
    torch.testing.assert_close(d.sum(-1), torch.ones(9, 4))
    q = qf(obs)
    assert torch.equal(q, (d * qf.support).sum(-1))
    assert (GreedyPolicy(qf).get_action_numpy(obs.numpy()) == q.argmax(-1).numpy()).all()


def test_constructor_refusals():
    from rl_replicas_b200.algorithms import C51
    from rl_replicas_b200.critics import CategoricalQFunction, DiscreteQFunction
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.replay_buffer import PrioritizedReplayBuffer
    env = ChooseEnv()
    net = MLP([O_DIM, 16, N_ACT * 11], torch.nn.ReLU)
    opt = torch.optim.Adam(net.parameters())
    qf = CategoricalQFunction(net, opt, n_atoms=11)
    with pytest.raises(ValueError, match=r"must map 2 -> 36 \(3 actions x 12 atoms logits\)"):
        C51(CategoricalQFunction(net, opt, n_atoms=12), None, env, None, None, None)
    with pytest.raises(ValueError, match="n_atoms must be 2"):
        CategoricalQFunction(net, opt, n_atoms=1)
    with pytest.raises(ValueError, match="n_atoms must be 2"):
        CategoricalQFunction(net, opt, n_atoms=257)
    with pytest.raises(ValueError, match="v_min < v_max"):
        CategoricalQFunction(net, opt, n_atoms=11, v_min=1.0, v_max=1.0)
    with pytest.raises(ValueError, match="v_min < v_max"):
        CategoricalQFunction(net, opt, n_atoms=11, v_min=0.0, v_max=float("inf"))
    cont = types.SimpleNamespace(action_space=types.SimpleNamespace(shape=(2,), high=np.ones(2)),
                                 observation_space=env.observation_space, spec=env.spec)
    with pytest.raises(ValueError, match="discrete"):
        C51(qf, None, cont, None, None, None)
    with pytest.raises(ValueError, match="CategoricalQFunction"):
        C51(DiscreteQFunction(net, opt), None, env, None, None, None)
    with pytest.raises(ValueError, match="PrioritizedReplayBuffer"):
        C51(qf, None, env, None, PrioritizedReplayBuffer(1000), None)
    algo = C51(qf, None, env, None, None, None, target_update_interval=5, double_q=True)
    assert (algo.target_update_interval, algo.double_q, algo.gamma, algo.epsilon_end) == (5, True, 0.99, 0.05)
    with pytest.raises(ValueError, match="PrioritizedReplayBuffer"):  # a buffer swapped in after construction
        algo.train(PrioritizedReplayBuffer(1000), 1, 4)


def test_save_and_load_round_trip(tmp_path):
    algo = make_c51(seed=1)
    algo.current_total_steps = 77
    algo.q_function(torch.randn(8, O_DIM)).sum().backward()
    algo.q_function.optimizer.step()
    with torch.no_grad():
        for p in algo.target_q_function.network.parameters():
            p.add_(0.5)
    path = str(tmp_path / "model.pt")
    algo.save_model(3, path)
    ckpt = torch.load(path, weights_only=True)
    assert set(ckpt) == {"epoch", "total_steps", "q_function_state_dict", "q_function_optimizer_state_dict",
                         "target_q_function_state_dict"}  # DQN's keys
    other = make_c51(seed=2)
    assert other.load_model(path) == 3 and other.current_total_steps == 77
    for a, b in ((algo.q_function.network, other.q_function.network),
                 (algo.target_q_function.network, other.target_q_function.network)):
        for (k, x), (_, y) in zip(a.state_dict().items(), b.state_dict().items()):
            assert torch.equal(x, y), k
    assert other._adam_step_count(other.q_function.optimizer, list(other.q_function.network.network)[::2]) == 1
    obs = torch.randn(5, O_DIM)
    assert torch.equal(algo.q_function(obs), other.q_function(obs))


def test_group_signature_refuses_differing_supports():
    from rl_replicas_b200.algorithms import LearnerGroup
    from test_dqn import make_dqn
    g = LearnerGroup()
    g.add(make_c51(seed=0))
    g.add(make_c51(seed=1))
    for name, atoms in (("n_atoms", dict(ATOMS, n_atoms=41)), ("v_min", dict(ATOMS, v_min=-2.0)),
                        ("v_max", dict(ATOMS, v_max=3.0))):
        with pytest.raises(ValueError, match=name if name != "n_atoms" else "network|n_atoms"):
            g.add(make_c51(seed=2, atoms=atoms))
    with pytest.raises(ValueError, match="class"):
        g.add(make_dqn(seed=2))
    with pytest.raises(ValueError, match="target_update_interval"):
        g.add(make_c51(seed=2, target_update_interval=7))


class OracleC51:
    """C51.train with the float32 oracle in place of the engine: the same host random stream for the indices, the
    oracle's networks written back into the learner's."""

    @staticmethod
    def patch(algo):
        q = algo.q_function
        oracle = OC.C51Oracle(q.network, algo.target_q_function.network, q.optimizer, n_atoms=q.n_atoms,
                              v_min=q.v_min, v_max=q.v_max, gamma=algo.gamma,
                              target_update_interval=algo.target_update_interval, double_q=algo.double_q)

        def train(replay_buffer, num_train_steps, minibatch_size):
            S, B = num_train_steps, minibatch_size
            idx = np.stack([replay_buffer.sample_indices(B) for _ in range(S)])
            oracle.train([replay_buffer.gather(idx[s]) for s in range(S)])
            algo.q_function.network.load_state_dict(oracle.q.state_dict())
            algo.target_q_function.network.load_state_dict(oracle.q_targ.state_dict())
        algo.train = train
        return oracle


def test_oracle_driven_learn_loop_solves_the_choice_task(tmp_path):
    """The bar the GPU learn() loop must clear (tests/test_gpu_c51.py) is one the oracle reaches with the same seeds."""
    np.random.seed(0)
    algo = make_c51(**C51_KW)
    OracleC51.patch(algo)
    before = evaluation_return(algo)
    algo.learn(output_dir=str(tmp_path), **LEARN)
    after = evaluation_return(algo)
    print(f"oracle-driven learn: evaluation return {before:.3f} -> {after:.3f}")
    assert before < 0.6 and after > RETURN_BAR, (before, after)
