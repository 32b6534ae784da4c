"""CPU: n-step returns for DQN / C51 -- the replay buffer's episode-end flags through appends, truncation, ring overwrites
and growth; the float32 ring walk of oracle/nstep.py against its independent float64 episode-list form; the oracles with
per-row discounts; the refusals; and the oracle-driven learn() loop on a delayed-reward task that sets the bar for the
GPU end-to-end test (tests/test_gpu_nstep.py)."""
import types

import numpy as np
import pytest
import torch

from oracle import dqn as OD
from oracle import nstep as ON

O_DIM, N_ACT = 4, 3


def nested(episodes, O=3, seed=0):
    """A nested-list Experience from [(length, last row done)]; rewards random, observations numbered by row."""
    from rl_replicas_b200.experience import Experience
    rng = np.random.default_rng(seed)
    e = Experience()
    for L, d in episodes:
        obs = rng.standard_normal((L + 1, O)).astype(np.float32)
        e.observations.append([obs[t] for t in range(L)])
        e.actions.append([np.int64(rng.integers(0, 3)) for _ in range(L)])
        e.rewards.append([float(x) for x in rng.standard_normal(L)])
        e.dones.append([False] * (L - 1) + [bool(d)])
        e.last_observations.append(obs[L])
        e.episode_lengths.append(L)
    return e


def packed(episodes, O=3, seed=0):
    from rl_replicas_b200.experience import PackedExperience
    rng = np.random.default_rng(seed)
    e = PackedExperience(sum(L for L, _ in episodes), O, 1, scalar_actions=True)
    for L, d in episodes:
        e.append_episode(rng.standard_normal((L, O)), rng.integers(0, 3, L), rng.standard_normal(L),
                         [False] * (L - 1) + [bool(d)], rng.standard_normal(O))
    return e


class Columns:
    """An object with transition_columns() only, like the column stub tools/bench_dqn.py appends."""

    def __init__(self, n, O=3, seed=0):
        rng = np.random.default_rng(seed)
        self.cols = (rng.standard_normal((n, O)).astype(np.float32), rng.integers(0, 3, n).astype(np.float32),
                     rng.standard_normal(n), rng.standard_normal((n, O)).astype(np.float32), rng.random(n) < 0.3)

    def transition_columns(self):
        return self.cols


def ends_of(episodes):
    return [t == L - 1 for L, _ in episodes for t in range(L)]


def check_views(rb, appended):
    """The five views and the flags equal the newest current_size rows of everything appended, and the newest row is
    marked."""
    flat = {k: [x for a in appended for x in a[k]] for k in ("observations", "rewards", "dones", "ends")}
    n = rb.current_size
    assert rb.episode_ends == [bool(x) for x in flat["ends"][-n:]]
    assert rb.rewards == [float(x) for x in flat["rewards"][-n:]]
    assert rb.dones == [bool(x) for x in flat["dones"][-n:]]
    np.testing.assert_array_equal(np.stack(rb.observations), np.stack(flat["observations"][-n:]))
    assert rb.episode_ends[-1]


def record(e, episodes=None):
    if hasattr(e, "transition_columns"):
        o, _, r, _, d = e.transition_columns()
        ends = ends_of(episodes) if episodes is not None else [False] * (len(r) - 1) + [True]
        return dict(observations=list(o), rewards=list(r), dones=list(d), ends=ends)
    return dict(observations=e.flattened_observations, rewards=e.flattened_rewards, dones=e.flattened_dones,
                ends=ends_of(episodes))


def test_episode_end_flags_follow_appends_truncation_wrap_and_growth():
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    rng = np.random.default_rng(7)
    # a small ring: wraps with overwrite, truncation of an append of buffer_size rows or more
    rb, appended = ReplayBuffer(buffer_size=50), []
    for k in range(40):
        eps = [(int(rng.integers(1, 9)), bool(rng.random() < 0.5)) for _ in range(int(rng.integers(1, 4)))]
        kind = k % 3
        e = nested(eps, seed=k) if kind == 0 else packed(eps, seed=k) if kind == 1 else Columns(sum(L for L, _ in eps), seed=k)
        rb.add_experience(e)
        appended.append(record(e, None if kind == 2 else eps))
        check_views(rb, appended)
    big = [(30, True), (25, False), (12, False)]  # 67 rows >= buffer_size: only the newest 50 survive
    for e in (nested(big, seed=99), packed(big, seed=98)):
        rb.add_experience(e)
        appended.append(record(e, big))
        check_views(rb, appended)
    # geometric growth (the first allocation holds 1024 rows) with the reorder of _grow
    rb, appended = ReplayBuffer(buffer_size=5000), []
    for k in range(12):
        eps = [(int(rng.integers(50, 300)), bool(rng.random() < 0.5)) for _ in range(3)]
        e = packed(eps, seed=k) if k % 2 else nested(eps, seed=k)
        rb.add_experience(e)
        appended.append(record(e, eps))
        check_views(rb, appended)
    assert rb._capacity == 5000 and rb.current_size == 5000


def ring_with_episodes(buffer_size, n_appends, seed):
    """A ReplayBuffer filled by appends of several episodes (done or cut, some shorter than any n), and the episode
    lists in append order."""
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    rng = np.random.default_rng(seed)
    rb, episodes = ReplayBuffer(buffer_size=buffer_size), []
    for k in range(n_appends):
        eps = [(int(rng.integers(1, 12)), bool(rng.random() < 0.5)) for _ in range(int(rng.integers(1, 5)))]
        e = nested(eps, seed=1000 * seed + k) if k % 2 else packed(eps, seed=1000 * seed + k)
        rb.add_experience(e)
        if hasattr(e, "transition_columns"):
            _, _, r, _, d = e.transition_columns()
            off = e.ep_offsets
            episodes += [(r[a:b], d[a:b]) for a, b in zip(off[:-1], off[1:])]
        else:
            episodes += list(zip(e.rewards, e.dones))
    return rb, episodes


@pytest.mark.parametrize("n", [1, 2, 3, 5, 32])
def test_ring_walk_agrees_with_the_episode_list_form(n):
    rb, episodes = ring_with_episodes(97, 40, seed=n)
    rb._cols["dones"][rb._physical(np.arange(0, rb.current_size, 7))] = True  # dones inside windows
    # the episode lists see the same dones
    flat_d = np.concatenate([np.asarray(d, bool) for _, d in episodes])
    total = len(flat_d)
    dropped = total - rb.current_size
    flat_d[dropped + np.arange(0, rb.current_size, 7)] = True
    o = 0
    for i, (r, d) in enumerate(episodes):
        episodes[i] = (np.asarray(r, np.float32).astype(np.float64), flat_d[o:o + len(r)])
        o += len(r)
    last64, R64, g64 = ON.episode_returns_f64(episodes, n, 0.97)
    logical = np.arange(rb.current_size)
    phys = rb.physical_rows(logical)
    last, R, g = ON.walk_f32(rb._cols["rewards"].astype(np.float32), rb._cols["dones"], rb._ends, phys, n, 0.97)
    assert rb._head > 0  # the ring has wrapped: some windows cross the physical end
    np.testing.assert_array_equal(last, rb.physical_rows(last64[dropped:] - dropped))
    np.testing.assert_allclose(R, R64[dropped:], rtol=0, atol=1e-5 * max(1.0, np.abs(R64).max()) * n)
    np.testing.assert_allclose(g, g64[dropped:], rtol=4e-7 * n, atol=0)
    if n == 1:
        np.testing.assert_array_equal(R, rb._cols["rewards"][phys].astype(np.float32))
        assert (g == np.float32(0.97)).all() and (last == phys).all()
    else:
        assert (last != phys).any() and (last == phys).any()  # some windows are cut short, some are not


def test_nstep_minibatch_and_the_oracles_with_per_row_discounts():
    from rl_replicas_b200.networks import MLP
    rb, _ = ring_with_episodes(300, 30, seed=3)
    phys = rb.physical_rows(np.random.default_rng(0).integers(0, rb.current_size, 64))
    mb = ON.nstep_minibatch(rb, phys, 1, 0.99)
    assert set(mb) == set(rb.COLUMNS) | {"discounts"}
    one = {k: v for k, v in ON.nstep_minibatch(rb, phys, 1, 0.99).items() if k != "discounts"}
    torch.manual_seed(0)
    net, targ = MLP([3, 16, 16, 3], torch.nn.Tanh), MLP([3, 16, 16, 3], torch.nn.Tanh)
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    # n = 1 with per-row discounts gamma is the one-step oracle bit for bit
    a = OD.DqnOracle(net, targ, opt, gamma=0.99, target_update_interval=2).train([one, one])
    b = ON.NStepDqnOracle(net, targ, opt, gamma=0.99, target_update_interval=2).train([mb, mb])
    for k in a:
        np.testing.assert_array_equal(np.asarray(a[k]), np.asarray(b[k]))
    # n = 4: the float32 oracle against the float64 reference with an array gamma
    mb4 = ON.nstep_minibatch(rb, phys, 4, 0.99)
    assert (mb4["discounts"] < np.float32(0.99)).any()
    flat = lambda m: torch.nn.utils.parameters_to_vector(m.parameters()).detach().numpy().astype(np.float64)
    ref = OD.dqn_step_f64(flat(net), flat(targ), mb4, [3, 16, 16, 3], "tanh",
                          torch.as_tensor(mb4["discounts"], dtype=torch.float64))
    o = ON.NStepDqnOracle(net, targ, opt, gamma=0.99, target_update_interval=100)
    logs = o.train([mb4])
    assert abs(logs["q1_losses"][0] - ref["loss"]) <= 1e-5 * abs(ref["loss"])
    # the per-row projection against Algorithm 1
    rng = np.random.default_rng(1)
    p = rng.random((64, 11))
    p /= p.sum(1, keepdims=True)
    from oracle import c51 as OC
    z = OC.support(11, -5.0, 5.0)
    tri = OC.project(torch.as_tensor(p), torch.as_tensor(mb4["rewards"], dtype=torch.float64),
                     torch.as_tensor(mb4["dones"], dtype=torch.float64), torch.as_tensor(z, dtype=torch.float64),
                     -5.0, 5.0, 1.0, mb4["discounts"].astype(np.float64)[:, None]).numpy()
    alg1 = ON.project_f64(p, mb4["rewards"], mb4["dones"], z, -5.0, 5.0, mb4["discounts"])
    np.testing.assert_allclose(tri, alg1, atol=1e-6)


# ---- refusals ---------------------------------------------------------------------------------------------------------
class DelayEnv:
    """A three-step task with a delayed reward (gymnasium protocol).  The first observation shows a cue x ~ U[-1, 1]^2;
    the first action is right when it is argmax(M x).  The next two observations carry the cue, the phase and whether
    the first action was right; the reward, 1 for a right first action and 0 otherwise, comes with the third step, which
    ends the episode.  A uniform random policy scores 1/3; one-step targets need two bootstraps to carry the reward back
    to the decision, a 3-step return none."""
    M = np.asarray([[1.0, 0.0], [-0.5, 0.87], [-0.5, -0.87]], np.float32)

    def __init__(self):
        self.rng = np.random.default_rng(0)
        space_rng = np.random.default_rng(1)
        self.action_space = types.SimpleNamespace(n=N_ACT, shape=(), sample=lambda: np.int64(space_rng.integers(N_ACT)))
        self.observation_space = types.SimpleNamespace(shape=(O_DIM,))
        self.spec = types.SimpleNamespace(id="DelayEnv-v0")

    def _obs(self):
        return np.asarray([*self.x, self.t / 2.0, self.flag], np.float32)

    def reset(self, seed=None):
        if seed is not None:
            self.rng = np.random.default_rng(seed)
        self.x, self.t, self.flag = self.rng.uniform(-1, 1, 2).astype(np.float32), 0, 0.0
        return self._obs(), {}

    def step(self, action):
        if self.t == 0:
            self.flag = 1.0 if int(action) == int(np.argmax(self.M @ self.x)) else -1.0
        self.t += 1
        if self.t < 3:
            return self._obs(), 0.0, False, False, {}
        reward = float(self.flag > 0)
        obs, _ = self.reset()
        return obs, reward, True, False, {}


def make_nstep_dqn(n_step=3, hidden=64, seed=0, lr=1e-3, algo=None, **kw):
    from rl_replicas_b200.algorithms import DQN
    from rl_replicas_b200.critics import DiscreteQFunction
    from rl_replicas_b200.evaluator import Evaluator
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import RandomPolicy
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    from rl_replicas_b200.samplers import BatchSampler
    torch.manual_seed(seed)
    env = DelayEnv()
    net = MLP([O_DIM, hidden, hidden, N_ACT], torch.nn.ReLU)
    return (algo or DQN)(DiscreteQFunction(net, torch.optim.Adam(net.parameters(), lr=lr)), RandomPolicy(env.action_space),
                         env, BatchSampler(env, seed=0), ReplayBuffer(buffer_size=100000), Evaluator(seed=0),
                         n_step=n_step, **kw)


@pytest.mark.parametrize("bad", [0, 33, 2.5, "3", True, -1])
def test_constructor_refuses_bad_n_step(bad):
    with pytest.raises(ValueError, match="n_step must be an integer from 1 to 32"):
        make_nstep_dqn(n_step=bad)


def test_train_refuses_host_replay_and_reference_style_buffers():
    algo = make_nstep_dqn(n_step=3)
    algo.replay_buffer.add_experience(nested([(5, True)], O=O_DIM))
    algo.use_device_replay = False
    with pytest.raises(ValueError, match="n_step = 3 needs use_device_replay = True"):
        algo.train(algo.replay_buffer, 2, 4)
    algo.use_device_replay = True

    class Reference:  # the reference's interface: sample_minibatch only
        def sample_minibatch(self, B):
            raise AssertionError("never drawn")
    with pytest.raises(ValueError, match="n_step = 3 needs a replay buffer with device_episode_ends"):
        algo.train(Reference(), 2, 4)


def test_group_refuses_members_whose_n_step_differs():
    from rl_replicas_b200.algorithms import LearnerGroup
    g = LearnerGroup()
    g.add(make_nstep_dqn(n_step=3, seed=0))
    g.add(make_nstep_dqn(n_step=3, seed=1))
    with pytest.raises(ValueError, match="n_step differs"):
        g.add(make_nstep_dqn(n_step=5, seed=2))


# ---- the oracle-driven learn loop ------------------------------------------------------------------------------------
class OracleNStepDQN:
    """DQN.train with the float32 n-step oracle in place of the engine: the same host random stream for the indices."""

    @staticmethod
    def patch(algo):
        oracle = ON.NStepDqnOracle(algo.q_function.network, algo.target_q_function.network, algo.q_function.optimizer,
                                   gamma=algo.gamma, target_update_interval=algo.target_update_interval,
                                   double_q=algo.double_q)

        def train(replay_buffer, num_train_steps, minibatch_size):
            S, B = num_train_steps, minibatch_size
            idx = replay_buffer.physical_rows(np.stack([replay_buffer.sample_indices(B) for _ in range(S)]))
            oracle.train([ON.nstep_minibatch(replay_buffer, idx[s], algo.n_step, algo.gamma) for s in range(S)])
            algo.q_function.network.load_state_dict(oracle.q.state_dict())
            algo.target_q_function.network.load_state_dict(oracle.q_targ.state_dict())
        algo.train = train
        return oracle


LEARN = dict(num_epochs=40, batch_size=50, minibatch_size=64, num_start_steps=500, num_steps_before_update=500,
             num_train_steps=50, num_evaluation_episodes=10, evaluation_interval=500, model_saving_interval=500)
NSTEP_KW = dict(n_step=3, target_update_interval=100, double_q=True, epsilon_start=1.0, epsilon_end=0.05,
                epsilon_decay_steps=1500)
RETURN_BAR = 0.8  # a uniform random policy scores 1/3 on DelayEnv


def evaluation_return(algo):
    from rl_replicas_b200.evaluator import Evaluator
    returns, _ = Evaluator(seed=123).evaluate(algo.evaluation_policy, DelayEnv(), 400)
    return float(np.mean(returns))


def test_oracle_driven_learn_loop_solves_the_delayed_reward_task(tmp_path):
    """The bar the GPU learn() loop must clear (tests/test_gpu_nstep.py) is one the oracle reaches with the same seeds."""
    np.random.seed(0)
    algo = make_nstep_dqn(**NSTEP_KW)
    OracleNStepDQN.patch(algo)
    before = evaluation_return(algo)
    algo.learn(output_dir=str(tmp_path), **LEARN)
    after = evaluation_return(algo)
    print(f"oracle-driven n-step learn: evaluation return {before:.3f} -> {after:.3f}")
    assert before < 0.6 and after > RETURN_BAR, (before, after)
