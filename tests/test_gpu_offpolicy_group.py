"""GPU: learner groups on the off-policy engine.  Every member of a group must produce bit for bit what it produces
alone: the engine at K = 3 on every minibatch path with the graph on and off, tile edges under the learner offset,
isolation of a NaN member, and LearnerGroup.train / LearnerGroup.learn against solo runs from the same seeds."""
import os
import random
import types

import numpy as np
import pytest
import torch
from numpy.testing import assert_array_equal

pytestmark = pytest.mark.gpu

A = 2


def engine(kind, K, psz, qsz, B, S):
    from rl_replicas_b200 import _lib
    from rl_replicas_b200.engine import OffPolicyEngine
    sac = kind.startswith("sac")
    e = OffPolicyEngine(psz, qsz, 1 if kind == "ddpg" else 2, B, S, ("relu", "identity" if sac else "tanh"),
                        ("relu", "identity"), algo=OffPolicyEngine.SAC if sac else OffPolicyEngine.TD3, n_learners=K)
    if sac:
        sp = _lib.SacHparams()
        sp.alpha, sp.learn_alpha, sp.target_entropy = 0.2, int(kind == "sac_learned"), -float(qsz[0] - psz[0])
        sp.alpha_lr, sp.alpha_beta1, sp.alpha_beta2, sp.alpha_eps = 3e-3, 0.9, 0.999, 1e-8
        sp.log_std_min, sp.log_std_max = -20.0, 2.0
        e.set_sac(sp)
    return e


def hparams(kind):
    from rl_replicas_b200._lib import OffPolicyHparams
    hp = OffPolicyHparams()
    hp.gamma, hp.polyak_rho = 0.99, 0.995
    hp.target_noise_scale, hp.target_noise_clip, hp.action_limit = 0.2, 0.5, 1.0
    hp.policy_delay, hp.use_target_noise = (2, 1) if kind == "td3" else (1, int(kind != "ddpg"))
    hp.policy_lr, hp.policy_beta1, hp.policy_beta2, hp.policy_eps = 1e-3, 0.9, 0.999, 1e-8
    hp.q1_lr, hp.q2_lr, hp.q_beta1, hp.q_beta2, hp.q_eps = 1e-3, 2e-3, 0.9, 0.999, 1e-8
    return hp


def member_state(e, rng, step, scale=0.3):
    """A random learner state: parameters, Adam moments (exp_avg_sq >= 0) and step counts ``step``."""
    layout, per = e.state_layout()
    blob = (rng.standard_normal(per) * scale).astype(np.float32)
    for kind, _, off, n in layout:
        if kind == "v":
            blob[off:off + n] = np.abs(blob[off:off + n]) * 1e-3
    return blob, [step, step, step]


def inputs(rng, kind, S, B, O, rows=None):
    """One learner's host minibatches (or, with ``rows``, physical replay rows) and noise for S steps."""
    noise = None
    if kind.startswith("sac"):
        noise = rng.standard_normal((S, 2, B, A)).astype(np.float32)
    elif kind == "td3":
        noise = rng.standard_normal((S, B, A)).astype(np.float32)
    if rows is not None:
        return rng.integers(0, rows, (S, B)), noise
    return (rng.standard_normal((S, B, O)).astype(np.float32), rng.uniform(-1, 1, (S, B, A)).astype(np.float32),
            rng.standard_normal((S, B)).astype(np.float32), rng.standard_normal((S, B, O)).astype(np.float32),
            (rng.random((S, B)) < 0.1).astype(np.float32), noise)


def replay(rng, rows, O):
    cols = (rng.standard_normal((rows, O)), rng.uniform(-1, 1, (rows, A)), rng.standard_normal(rows),
            rng.standard_normal((rows, O)), (rng.random(rows) < 0.1))
    return tuple(torch.as_tensor(np.asarray(c, np.float32), device="cuda") for c in cols), rows


def assert_same(got, want, what):
    assert set(got) == set(want), what
    for k in want:
        assert_array_equal(np.asarray(got[k]), np.asarray(want[k]), err_msg=f"{what}: {k}")


def run_group_vs_solo(kind, path, psz, qsz, B, calls, K=3, steps=(0, 7, 100), poison=None, seed=0):
    """Group of K against K solo engines fed each member's inputs; returns nothing, asserts bit identity (members in
    ``poison`` get NaN parameters and are not compared)."""
    O = psz[0]
    rng = np.random.default_rng(seed)
    maxS = max(calls)
    g = engine(kind, K, psz, qsz, B, maxS)
    solos = [engine(kind, 1, psz, qsz, B, maxS) for _ in range(K)]
    states = [member_state(g, rng, steps[z % len(steps)]) for z in range(K)]
    for z in poison or ():
        states[z][0][:] = np.nan
    g.set_state(np.concatenate([s[0] for s in states]), [s[1] for s in states])
    for e, (blob, st) in zip(solos, states):
        e.set_state(blob, st)
    if kind.startswith("sac"):
        alphas = [(float(np.log(0.1 + 0.1 * z)), 0.01 * z, 1e-4 * z, steps[z % len(steps)]) for z in range(K)]
        g.set_alpha_group(alphas)
        for e, a in zip(solos, alphas):
            e.set_alpha(*a)
    replays = [replay(rng, 300 + 200 * z, O) for z in range(K)] if path != "host" else None
    hp = hparams(kind)
    for c, S in enumerate(calls):
        if path == "host":
            ins = [inputs(rng, kind, S, B, O) for _ in range(K)]
            out = g.train(hp, *[None if ins[0][i] is None else np.stack([x[i] for x in ins]) for i in range(6)])
            solo_out = [e.train(hp, *x) for e, x in zip(solos, ins)]
        elif path == "gather":
            ins = [inputs(rng, kind, S, B, O, rows=r[1]) for r in replays]
            noise = None if ins[0][1] is None else np.stack([x[1] for x in ins])
            out = g.train_gather_group(hp, replays, np.stack([x[0] for x in ins]), noise)
            solo_out = [e.train_gather(hp, r[0], r[1], *x) for e, r, x in zip(solos, replays, ins)]
        else:
            starts = [(17 * z + c) % r[1] for z, r in enumerate(replays)]
            sizes = [r[1] - 5 * z for z, r in enumerate(replays)]
            seeds, cs = [1000 + z for z in range(K)], [c + 1] * K
            out = g.train_gather_rng_group(hp, replays, starts, sizes, S, B, seeds, cs)
            solo_out = [e.train_gather_rng(hp, r[0], r[1], a, b, S, B, sd, cc)
                        for e, r, a, b, sd, cc in zip(solos, replays, starts, sizes, seeds, cs)]
            gi, gn = g.get_draws(S, B, with_noise=kind != "ddpg")
            for z, e in enumerate(solos):
                si, sn = e.get_draws(S, B, with_noise=kind != "ddpg")
                assert_array_equal(gi[z], si)
                if sn is not None:
                    assert_array_equal(gn[z], sn)
        blob, gsteps = g.get_state()
        blob = blob.reshape(K, -1)
        galpha = g.get_alpha_group() if kind.startswith("sac") else None
        for z, e in enumerate(solos):
            if z in (poison or ()):
                continue
            assert_same({k: v[z] for k, v in out.items()}, solo_out[z], f"{kind}/{path} call {c} learner {z}")
            sblob, ssteps = e.get_state()
            assert_array_equal(blob[z], sblob, err_msg=f"{kind}/{path} call {c} learner {z}: state")
            assert gsteps[z] == ssteps
            if galpha is not None:
                assert galpha[z] == e.get_alpha()


@pytest.mark.parametrize("graph", ["1", "0"])
@pytest.mark.parametrize("path", ["host", "gather", "rng"])
@pytest.mark.parametrize("kind", ["td3", "ddpg", "sac_fixed", "sac_learned"])
def test_group_of_three_matches_solo_engines(kind, path, graph, monkeypatch):
    """K = 3 with different parameters, Adam states (steps 0, 7, 100), minibatches, noise and replay sizes: capture,
    replay, then a changed S (the graph is rebuilt)."""
    monkeypatch.setenv("B200RL_OFFPOLICY_GRAPH", graph)
    O = 5
    pout = 2 * A if kind.startswith("sac") else A
    run_group_vs_solo(kind, path, [O, 32, 32, pout], [O + A, 32, 32, 1], 16, (4, 4, 3))


def test_tile_edges_under_the_learner_offset():
    """Ragged widths 31 / 33, B = 33, a 4-layer critic at K = 2; and K = 16 at a small shape."""
    run_group_vs_solo("td3", "host", [31, 33, 31, A], [31 + A, 33, 31, 33, 1], 33, (3, 2), K=2)
    run_group_vs_solo("sac_learned", "gather", [31, 33, 31, 2 * A], [31 + A, 33, 31, 33, 1], 33, (2,), K=2)
    run_group_vs_solo("td3", "rng", [5, 16, 16, A], [5 + A, 16, 16, 1], 8, (3,), K=16, steps=(0, 3, 9, 40))


def test_a_nan_member_does_not_touch_the_others():
    run_group_vs_solo("td3", "gather", [5, 32, 32, A], [5 + A, 32, 32, 1], 16, (4, 3), poison=(1,))
    run_group_vs_solo("sac_learned", "host", [5, 32, 32, 2 * A], [5 + A, 32, 32, 1], 16, (3,), poison=(0,))


# ---- LearnerGroup against solo runs from the same seeds -------------------------------------------------------------
class PointEnv:
    """1-D point mass: obs = [x, v, target], action in [-1, 1]; reward = -|x - target|; 25-step episodes."""

    def __init__(self, seed=0):
        self.rng = np.random.default_rng(seed)
        self.action_space = types.SimpleNamespace(high=np.ones(1, np.float32), low=-np.ones(1, np.float32), shape=(1,),
                                                  sample=lambda: self.rng.uniform(-1, 1, 1).astype(np.float32))
        self.observation_space = types.SimpleNamespace(shape=(3,))
        self.spec = types.SimpleNamespace(id="GroupPoint-v0")

    def _obs(self):
        return np.asarray([self.x, self.v, self.target], dtype=np.float32)

    def reset(self, seed=None):
        if seed is not None:
            self.rng = np.random.default_rng(seed)
        self.x, self.v, self.target, self.t = 0.0, 0.0, float(self.rng.uniform(-1, 1)), 0
        return self._obs(), {}

    def step(self, action):
        a = float(np.clip(np.asarray(action).reshape(-1)[0], -1, 1))
        self.v = 0.9 * self.v + 0.1 * a
        self.x += self.v
        self.t += 1
        return self._obs(), -abs(self.x - self.target), False, self.t >= 25, {}


def build(kind, seed, fill_rows=0):
    """A learner on its own PointEnv, sampler, evaluator and replay buffer; built after seeding, like a user would."""
    from rl_replicas_b200.algorithms import DDPG, SAC, TD3
    from rl_replicas_b200.evaluator import Evaluator
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import DeterministicPolicy, RandomPolicy, SquashedGaussianPolicy
    from rl_replicas_b200.q_function import QFunction
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    from rl_replicas_b200.samplers import BatchSampler
    env = PointEnv(seed)
    opt = lambda net: torch.optim.Adam(net.parameters(), lr=1e-3)
    qs = [MLP([4, 32, 32, 1], torch.nn.ReLU) for _ in range(1 if kind == "ddpg" else 2)]
    qfs = [QFunction(q, opt(q)) for q in qs]
    rest = (env, BatchSampler(env, seed=seed, is_continuous=True), ReplayBuffer(buffer_size=5000), Evaluator(seed))
    if kind == "sac":
        pnet = MLP([3, 32, 32, 2], torch.nn.ReLU)
        algo = SAC(SquashedGaussianPolicy(pnet, opt(pnet)), RandomPolicy(env.action_space), *qfs, *rest,
                   learn_alpha=True, alpha_lr=3e-3)
    else:
        pnet = MLP([3, 32, 32, 1], torch.nn.ReLU, torch.nn.Tanh)
        cls = DDPG if kind == "ddpg" else TD3
        algo = cls(DeterministicPolicy(pnet, opt(pnet)), RandomPolicy(env.action_space), *qfs, *rest)
    if fill_rows:
        rng = np.random.default_rng(seed + 100)
        from rl_replicas_b200.experience import Experience
        e = Experience()
        obs = rng.standard_normal((fill_rows + 1, 3)).astype(np.float32)
        e.observations = [[obs[i] for i in range(fill_rows)]]
        e.actions = [[a for a in rng.uniform(-1, 1, (fill_rows, 1)).astype(np.float32)]]
        e.rewards = [[float(x) for x in rng.standard_normal(fill_rows)]]
        e.dones = [[bool(x) for x in (rng.random(fill_rows) < 0.05)]]
        e.last_observations = [obs[fill_rows]]
        algo.replay_buffer.add_experience(e)
    return algo


class Recorder:
    """A metrics manager that keeps what was recorded."""

    def __init__(self):
        self.rows = []

    def record_scalar(self, tag, value, step=None, tensorboard=False):
        self.rows.append((tag, value, step))


def modules(algo):
    names = ["policy", "q_function_1", "q_function_2", "q_function", "target_policy", "target_q_function_1",
             "target_q_function_2", "target_q_function"]
    return {n: getattr(algo, n) for n in names if hasattr(algo, n)}


def assert_same_learner(a, b, what):
    for n, m in modules(a).items():
        o = modules(b)[n]
        for (k, x), (_, y) in zip(m.network.state_dict().items(), o.network.state_dict().items()):
            assert torch.equal(x, y), f"{what}: {n}.{k}"
        if hasattr(m, "optimizer") and n in ("policy", "q_function", "q_function_1", "q_function_2"):
            assert_state_dicts(m.optimizer.state_dict(), o.optimizer.state_dict(), f"{what}: {n} optimizer")
    if hasattr(a, "log_alpha"):
        assert torch.equal(a.log_alpha.detach(), b.log_alpha.detach()), what
        assert_state_dicts(a.alpha_optimizer.state_dict(), b.alpha_optimizer.state_dict(), f"{what}: alpha optimizer")


def assert_state_dicts(x, y, what):
    if isinstance(x, dict):
        assert set(x) == set(y), what
        for k in x:
            assert_state_dicts(x[k], y[k], f"{what}.{k}")
    elif isinstance(x, (list, tuple)):
        assert len(x) == len(y), what
        for i, (p, q) in enumerate(zip(x, y)):
            assert_state_dicts(p, q, f"{what}[{i}]")
    elif torch.is_tensor(x):
        assert torch.equal(x, y), what
    else:
        assert x == y, what


def rng_state():
    return random.getstate(), np.random.get_state()[1].copy(), torch.get_rng_state().clone()


@pytest.mark.parametrize("device_rng", [False, True])
@pytest.mark.parametrize("kind", ["td3", "ddpg", "sac"])
def test_learner_group_train_matches_solo_train(kind, device_rng):
    from rl_replicas_b200.algorithms import LearnerGroup
    from rl_replicas_b200.utils import set_seed_for_libraries
    seeds = (0, 1, 2)
    calls = ((6, 32), (5, 32), (3, 16))

    def setup(s):
        algo = build(kind, s, fill_rows=400 + 150 * s)
        algo.metrics_manager, algo.current_total_steps = Recorder(), 1000 + s
        algo.use_device_rng, algo.device_rng_seed = device_rng, 7 + s
        return algo

    solo = {}
    for s in seeds:
        set_seed_for_libraries(s)
        a = setup(s)
        for S, B in calls:
            a.train(a.replay_buffer, S, B)
        solo[s] = a
    group = LearnerGroup()
    members = {}
    for s in seeds:
        set_seed_for_libraries(s)
        members[s] = setup(s)
        group.add(members[s])
    set_seed_for_libraries(99)
    before = rng_state()
    for S, B in calls:
        group.train(S, B)
    after = rng_state()
    assert after[0] == before[0] and np.array_equal(after[1], before[1]) and torch.equal(after[2], before[2])
    for s in seeds:
        a, b = members[s], solo[s]
        assert_same_learner(a, b, f"{kind} seed {s}")
        assert a.metrics_manager.rows == b.metrics_manager.rows
        assert_same(a.last_train_output, b.last_train_output, f"{kind} seed {s}")


@pytest.mark.parametrize("kind", ["td3", "sac"])
def test_learner_group_learn_matches_solo_learn(kind, tmp_path, monkeypatch):
    from rl_replicas_b200.algorithms import LearnerGroup
    from rl_replicas_b200.metrics_manager import MetricsManager
    from rl_replicas_b200.utils import set_seed_for_libraries
    recorded = {}
    orig = MetricsManager.record_scalar

    def record(self, tag, value, step=None, tensorboard=False):
        recorded.setdefault(id(self), []).append((tag, value, step))
        return orig(self, tag, value, step, tensorboard)
    monkeypatch.setattr(MetricsManager, "record_scalar", record)
    kw = dict(num_epochs=6, batch_size=50, minibatch_size=32, num_start_steps=100, num_steps_before_update=100,
              num_train_steps=5, num_evaluation_episodes=2, evaluation_interval=100, model_saving_interval=100)
    seeds = (0, 1, 2)
    solo = {}
    for s in seeds:
        set_seed_for_libraries(s)
        a = build(kind, s)
        a.learn(output_dir=str(tmp_path / f"solo-{s}"), **kw)
        solo[s] = a
    group = LearnerGroup()
    members = {}
    for s in seeds:
        set_seed_for_libraries(s)
        members[s] = build(kind, s)
        group.add(members[s])
    group.learn(output_dirs=[str(tmp_path / f"group-{s}") for s in seeds], **kw)
    for s in seeds:
        a, b = members[s], solo[s]
        assert_same_learner(a, b, f"{kind} seed {s}")
        ck_a = torch.load(os.path.join(tmp_path, f"group-{s}", "model.pt"), weights_only=False)
        ck_b = torch.load(os.path.join(tmp_path, f"solo-{s}", "model.pt"), weights_only=False)
        assert_state_dicts(ck_a, ck_b, f"{kind} seed {s} checkpoint")
        ra = [r for r in recorded[id(a.metrics_manager)] if r[0] != "time"]
        rb = [r for r in recorded[id(b.metrics_manager)] if r[0] != "time"]
        assert ra == rb and any(t.startswith("evaluation/") for t, _, _ in ra)
        assert any(t == "q-function_1/average_loss" for t, _, _ in ra)
