"""CPU: DQN's host side -- the oracles (oracle/dqn.py) against each other and at the Huber / argmax edges, the epsilon
schedule and the epsilon-greedy use of NumPy's stream, the DQN constructor's refusals, its checkpoint round trip, the
LearnerGroup signature for DQN members, and the oracle-driven learn() loop that sets the bar for the GPU end-to-end test
(tests/test_gpu_dqn.py)."""
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import dqn as OD

O_DIM, N_ACT = 2, 3


class ChooseEnv:
    """One-step discrete task (gymnasium protocol): obs ~ U[-1, 1]^2; reward 1 for the action argmax(M obs), else 0;
    every episode ends after its single step.  A uniform random policy scores 1/3."""
    M = np.asarray([[1.0, 0.0], [-0.5, 0.87], [-0.5, -0.87]], np.float32)

    def __init__(self):
        self.rng = np.random.default_rng(0)
        space_rng = np.random.default_rng(1)
        self.action_space = types.SimpleNamespace(n=N_ACT, shape=(), sample=lambda: np.int64(space_rng.integers(N_ACT)))
        self.observation_space = types.SimpleNamespace(shape=(O_DIM,))
        self.spec = types.SimpleNamespace(id="ChooseEnv-v0")

    def reset(self, seed=None):
        if seed is not None:
            self.rng = np.random.default_rng(seed)
        self.obs = self.rng.uniform(-1, 1, O_DIM).astype(np.float32)
        return self.obs, {}

    def step(self, action):
        reward = float(int(action) == int(np.argmax(self.M @ self.obs)))
        obs, _ = self.reset()
        return obs, reward, True, False, {}


def make_dqn(hidden=64, seed=0, lr=1e-3, **kw):
    from rl_replicas_b200.algorithms import DQN
    from rl_replicas_b200.critics import DiscreteQFunction
    from rl_replicas_b200.evaluator import Evaluator
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import RandomPolicy
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    from rl_replicas_b200.samplers import BatchSampler
    torch.manual_seed(seed)
    env = ChooseEnv()
    net = MLP([O_DIM, hidden, hidden, N_ACT], torch.nn.ReLU)
    return DQN(DiscreteQFunction(net, torch.optim.Adam(net.parameters(), lr=lr)), RandomPolicy(env.action_space), env,
               BatchSampler(env, seed=0), ReplayBuffer(buffer_size=100000), Evaluator(seed=0), **kw)


def random_minibatch(rng, B, n=N_ACT, O=O_DIM):
    return dict(observations=rng.standard_normal((B, O)).astype(np.float32),
                actions=rng.integers(0, n, B).astype(np.float32), rewards=rng.standard_normal(B),
                next_observations=rng.standard_normal((B, O)).astype(np.float32), dones=rng.random(B) < 0.2)


def flat(m):
    return torch.nn.utils.parameters_to_vector(m.parameters()).detach().numpy().astype(np.float64)


@pytest.mark.parametrize("double_q", [False, True])
def test_float32_oracle_agrees_with_the_float64_reference(double_q):
    """One step: loss, Q(s, a) and the gradient (read from Adam's first moment) of the float32 autograd oracle within
    1e-5 of the float64 reference."""
    from rl_replicas_b200.networks import MLP
    torch.manual_seed(3)
    net, targ = MLP([4, 32, 32, 5], torch.nn.Tanh), MLP([4, 32, 32, 5], torch.nn.Tanh)
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    mb = random_minibatch(np.random.default_rng(0), 64, n=5, O=4)
    mb["rewards"] = mb["rewards"] * 3.0  # both Huber branches
    ref = OD.dqn_step_f64(flat(net), flat(targ), mb, [4, 32, 32, 5], "tanh", 0.99, double_q)
    assert (np.abs(ref["delta"]) < 1).any() and (np.abs(ref["delta"]) > 1).any()
    o = OD.DqnOracle(net, targ, opt, gamma=0.99, target_update_interval=100, double_q=double_q)
    logs = o.train([mb])
    grad = torch.cat([o.opt.state[p]["exp_avg"].reshape(-1) for p in o.q.parameters()]).numpy() / 0.1
    rel = lambda x, r: float(np.max(np.abs(np.asarray(x, np.float64) - r)) / np.max(np.abs(r)))
    assert rel(logs["q1_values"][0], ref["q_values"]) < 1e-5
    assert abs(logs["q1_losses"][0] - ref["loss"]) <= 1e-5 * abs(ref["loss"])
    assert rel(grad, ref["grad"]) < 1e-5
    assert (ref["scale"] >= np.abs(ref["grad"]) * (1 - 1e-12)).all()


def test_huber_gradient_is_exact_at_and_around_one():
    d = torch.tensor([-2.0, -1.0 - 2 ** -20, -1.0, -0.5, 0.0, 0.5, 1.0 - 2 ** -20, 1.0, 1.0 + 2 ** -20, 3.0],
                     dtype=torch.float64, requires_grad=True)
    y = torch.zeros_like(d)
    F.smooth_l1_loss(d, y, reduction="sum").backward()
    want = torch.clamp(d.detach(), -1, 1)
    assert torch.equal(d.grad, want)
    d2 = d.detach().clone().requires_grad_(True)
    OD.huber_f64(d2).sum().backward()
    assert torch.equal(d2.grad, want)
    assert torch.allclose(OD.huber_f64(d.detach()), F.smooth_l1_loss(d.detach(), y, reduction="none"), rtol=0, atol=0)
    # both branches agree at |delta| = 1
    assert float(OD.huber_f64(torch.tensor([1.0], dtype=torch.float64))) == 0.5


def test_argmax_takes_the_first_of_tied_maxima_and_nan_propagates():
    q = torch.tensor([[1.0, 3.0, 3.0, 2.0], [5.0, 5.0, 5.0, 5.0], [1.0, float("nan"), 7.0, float("nan")]])
    qt = torch.tensor([[10.0, 20.0, 30.0, 40.0]] * 3)
    assert q.argmax(1).tolist()[:2] == [1, 0]
    v = OD.td_values(qt, q, double_q=True)
    assert v[:2].tolist() == [20.0, 10.0] and float(v[2]) == 20.0  # the first NaN wins argmax
    vmax = OD.td_values(q, None, double_q=False)
    assert vmax[:2].tolist() == [3.0, 5.0] and torch.isnan(vmax[2])


def test_epsilon_schedule_and_the_numpy_stream():
    from rl_replicas_b200.policies import EpsilonGreedyPolicy, GreedyPolicy
    algo = make_dqn(epsilon_start=1.0, epsilon_end=0.1, epsilon_decay_steps=100)
    for t, want in ((0, 1.0), (50, 0.55), (100, 0.1), (10 ** 6, 0.1)):
        algo.current_total_steps = t
        assert algo.epsilon() == pytest.approx(want, abs=1e-12)
        assert algo.noised_policy.epsilon == pytest.approx(want, abs=1e-12)
    q = algo.q_function
    greedy = GreedyPolicy(q)
    obs = np.random.default_rng(5).uniform(-1, 1, (40, O_DIM)).astype(np.float32)
    with torch.no_grad():
        want_greedy = torch.argmax(q(torch.from_numpy(obs)), -1).numpy()
    assert (greedy.get_action_numpy(obs) == want_greedy).all()
    space = types.SimpleNamespace(n=N_ACT, sample=lambda: np.int64(99))  # marks the exploring actions
    pol = EpsilonGreedyPolicy(q, space, 0.3)
    np.random.seed(11)
    got = [int(pol.get_action_numpy(o)) for o in obs]
    np.random.seed(11)
    draws = np.random.random(len(obs))  # one draw per action, also for the greedy ones
    want = [99 if u < 0.3 else int(g) for u, g in zip(draws, want_greedy)]
    assert got == want
    np.random.seed(11)
    assert pol.get_action_numpy(obs).tolist() == want  # a batch draws per row, in order
    tie = GreedyPolicy(lambda o: torch.tensor([[1.0, 2.0, 2.0]]))
    assert int(tie.get_action_numpy(np.zeros((1, 2), np.float32))[0]) == 1


def test_constructor_refusals():
    from rl_replicas_b200.algorithms import DQN
    from rl_replicas_b200.critics import DiscreteQFunction
    from rl_replicas_b200.networks import MLP
    env = ChooseEnv()
    net = MLP([O_DIM, 16, N_ACT], torch.nn.ReLU)
    qf = DiscreteQFunction(net, torch.optim.Adam(net.parameters()))
    cont = types.SimpleNamespace(action_space=types.SimpleNamespace(shape=(2,), high=np.ones(2)),
                                 observation_space=env.observation_space, spec=env.spec)
    with pytest.raises(ValueError, match="discrete"):
        DQN(qf, None, cont, None, None, None)
    wide = MLP([O_DIM, 16, N_ACT + 1], torch.nn.ReLU)
    with pytest.raises(ValueError, match="one value per action"):
        DQN(DiscreteQFunction(wide, torch.optim.Adam(wide.parameters())), None, env, None, None, None)
    narrow_in = MLP([O_DIM + 1, 16, N_ACT], torch.nn.ReLU)
    with pytest.raises(ValueError, match="must map 2 -> 3"):
        DQN(DiscreteQFunction(narrow_in, torch.optim.Adam(narrow_in.parameters())), None, env, None, None, None)
    with pytest.raises(NotImplementedError, match="Adam"):
        DQN(DiscreteQFunction(net, torch.optim.SGD(net.parameters(), lr=0.1)), None, env, None, None, None)
    with pytest.raises(ValueError, match="target_update_interval"):
        DQN(qf, None, env, None, None, None, target_update_interval=0)


def test_save_and_load_round_trip(tmp_path):
    algo = make_dqn(seed=1)
    algo.current_total_steps = 1234
    o = algo.q_function.network(torch.randn(8, O_DIM)).sum()  # give the optimizer a state with a step count
    o.backward()
    algo.q_function.optimizer.step()
    with torch.no_grad():
        for p in algo.target_q_function.network.parameters():
            p.add_(0.5)
    path = str(tmp_path / "model.pt")
    algo.save_model(7, path)
    ckpt = torch.load(path, weights_only=True)
    assert set(ckpt) == {"epoch", "total_steps", "q_function_state_dict", "q_function_optimizer_state_dict",
                         "target_q_function_state_dict"}
    other = make_dqn(seed=2)
    assert other.load_model(path) == 7 and other.current_total_steps == 1234
    for a, b in ((algo.q_function.network, other.q_function.network),
                 (algo.target_q_function.network, other.target_q_function.network)):
        for (k, x), (_, y) in zip(a.state_dict().items(), b.state_dict().items()):
            assert torch.equal(x, y), k
    sa, sb = algo.q_function.optimizer.state_dict()["state"], other.q_function.optimizer.state_dict()["state"]
    for k in sa:
        for key in ("step", "exp_avg", "exp_avg_sq"):
            assert torch.equal(sa[k][key], sb[k][key])
    assert other._adam_step_count(other.q_function.optimizer, list(other.q_function.network.network)[::2]) == 1


def test_group_signature_refuses_mixes_and_differing_intervals():
    from rl_replicas_b200.algorithms import LearnerGroup
    from test_offpolicy_group import td3 as make_td3
    g = LearnerGroup()
    g.add(make_dqn(seed=0, target_update_interval=10, double_q=True))
    g.add(make_dqn(seed=1, target_update_interval=10, double_q=True))
    with pytest.raises(ValueError, match="target_update_interval"):
        g.add(make_dqn(seed=2, target_update_interval=20, double_q=True))
    with pytest.raises(ValueError, match="double_q"):
        g.add(make_dqn(seed=2, target_update_interval=10, double_q=False))
    with pytest.raises(ValueError, match="class"):
        g.add(make_td3(0))
    t = LearnerGroup()
    t.add(make_td3(0))
    with pytest.raises(ValueError, match="class"):
        t.add(make_dqn(seed=0))


class OracleDQN:
    """DQN.train with the float32 oracle in place of the engine: the same host random stream for the indices, the
    oracle's networks and Adam state written back into the learner's."""

    @staticmethod
    def patch(algo):
        oracle = OD.DqnOracle(algo.q_function.network, algo.target_q_function.network, algo.q_function.optimizer,
                              gamma=algo.gamma, target_update_interval=algo.target_update_interval,
                              double_q=algo.double_q)

        def train(replay_buffer, num_train_steps, minibatch_size):
            S, B = num_train_steps, minibatch_size
            idx = np.stack([replay_buffer.sample_indices(B) for _ in range(S)])
            oracle.train([replay_buffer.gather(idx[s]) for s in range(S)])
            algo.q_function.network.load_state_dict(oracle.q.state_dict())
            algo.target_q_function.network.load_state_dict(oracle.q_targ.state_dict())
        algo.train = train
        return oracle


LEARN = dict(num_epochs=40, batch_size=50, minibatch_size=64, num_start_steps=500, num_steps_before_update=500,
             num_train_steps=50, num_evaluation_episodes=10, evaluation_interval=500, model_saving_interval=500)
DQN_KW = dict(target_update_interval=100, double_q=True, epsilon_start=1.0, epsilon_end=0.05, epsilon_decay_steps=1500)
RETURN_BAR = 0.85  # a uniform random policy scores 1/3 on ChooseEnv


def evaluation_return(algo):
    from rl_replicas_b200.evaluator import Evaluator
    returns, _ = Evaluator(seed=123).evaluate(algo.evaluation_policy, ChooseEnv(), 400)
    return float(np.mean(returns))


def test_oracle_driven_learn_loop_solves_the_choice_task(tmp_path):
    """The bar the GPU learn() loop must clear (tests/test_gpu_dqn.py) is one the oracle reaches with the same seeds."""
    np.random.seed(0)
    algo = make_dqn(**DQN_KW)
    OracleDQN.patch(algo)
    before = evaluation_return(algo)
    algo.learn(output_dir=str(tmp_path), **LEARN)
    after = evaluation_return(algo)
    print(f"oracle-driven learn: evaluation return {before:.3f} -> {after:.3f}")
    assert before < 0.6 and after > RETURN_BAR, (before, after)
