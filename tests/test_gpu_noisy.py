"""GPU: noisy networks on the off-policy engine (config noisy_layers; include/b200rl.h, "Noisy networks") -- DQN (Double
on and off), C51 and QR-DQN with a NoisyMLP and a noisy DuelingMLP against the float32 oracles fed the engine's draws
across calls and target copies, one step against the float64 reference (oracle/noisy.py) at edge shapes, sigma = 0
against a plain network bit for bit, the draws (normality, keys, streams), graph against plain launches, a group of 3
against solo engines, the stated launch counts, the engine's refusals and the checkpoint round trip."""
import os

import numpy as np
import pytest
import torch

from conftest import rel_err
from oracle import c51 as OC
from oracle import dqn as OD
from oracle import noisy as ON
from oracle import qr as OQ
from test_gpu_dqn import GAMMA, LR, adam_flat, fill, flat
from test_gpu_dueling import PER, _errs, _outputs, _state
from test_gpu_nstep import ring

pytestmark = pytest.mark.gpu

ATOMS = dict(n_atoms=51, v_min=-10.0, v_max=10.0)


def build(kind="dqn", dueling=False, O=8, n=4, K=None, hidden=(64, 64), seed=0, steps=0, per=None, plain=False,
          one_noisy=None, **kw):
    """A DQN / C51 / QR-DQN learner on a stub discrete environment with a NoisyMLP([O, *hidden, n K]) or a noisy
    DuelingMLP([O, *hidden], n, K) Q network (``plain``: the same shapes without noise; ``one_noisy`` = l: a NoisyMLP
    whose layers other than l are plain); ``steps`` > 0 gives its Adam a state at that step count."""
    import types
    from rl_replicas_b200.algorithms import C51, DQN, QRDQN
    from rl_replicas_b200.critics import CategoricalQFunction, DiscreteQFunction, QuantileQFunction
    from rl_replicas_b200.networks import MLP, DuelingMLP, NoisyMLP, reset_noise
    from rl_replicas_b200.replay_buffer import PrioritizedReplayBuffer, ReplayBuffer
    K = K or {"dqn": 1, "c51": ATOMS["n_atoms"], "qr": 32}[kind]
    torch.manual_seed(seed)
    if dueling:
        net = DuelingMLP([O, *hidden], n, K, noisy=not plain)
    elif plain:
        net = MLP([O, *hidden, n * K], torch.nn.ReLU)
    else:
        net = NoisyMLP([O, *hidden, n * K])
        if one_noisy is not None:
            for l, lin in enumerate(list(net.network)[::2]):
                if l != one_noisy:
                    net.network[2 * l] = torch.nn.Linear(lin.in_features, lin.out_features)
    opt = torch.optim.Adam(net.parameters(), lr=LR)
    for _ in range(steps):  # some arbitrary earlier steps, each under its own noise (sigma's Adam state is not fresh)
        reset_noise(net)
        opt.zero_grad()
        net(torch.randn(16, O)).pow(2).mean().backward()
        opt.step()
    env = types.SimpleNamespace(action_space=types.SimpleNamespace(n=n, shape=()), spec=types.SimpleNamespace(id="stub"),
                                observation_space=types.SimpleNamespace(shape=(O,)))
    rb = ReplayBuffer() if per is None else PrioritizedReplayBuffer(**per)
    if kind == "dqn":
        qf, cls = DiscreteQFunction(net, opt), DQN
    elif kind == "c51":
        qf, cls = CategoricalQFunction(net, opt, n_atoms=K, v_min=ATOMS["v_min"], v_max=ATOMS["v_max"]), C51
    else:
        qf, cls = QuantileQFunction(net, opt, n_quantiles=K), QRDQN
    algo = cls(qf, None, env, None, rb, None, gamma=GAMMA, **kw)
    with torch.no_grad():  # a target that differs from the online network
        for p in algo.target_q_function.network.parameters():
            p.add_(0.05 * torch.randn_like(p))
    algo.metrics_manager = None
    algo.current_total_steps = 0
    return algo


def oracle_for(algo, kind):
    q, qt = algo.q_function, algo.target_q_function
    kw = dict(gamma=algo.gamma, target_update_interval=algo.target_update_interval, double_q=algo.double_q)
    if kind == "c51":
        return OC.C51Oracle(q.network, qt.network, q.optimizer, **ATOMS, **kw)
    if kind == "qr":
        return OQ.QrDqnOracle(q.network, qt.network, q.optimizer, n_quantiles=q.n_quantiles, **kw)
    return OD.DqnOracle(q.network, qt.network, q.optimizer, **kw)


# The learners start from a few earlier Adam steps, as in tests/test_gpu_dueling.py.
@pytest.mark.parametrize("dueling", [False, True])
@pytest.mark.parametrize("kind,double_q", [("dqn", False), ("dqn", True), ("c51", True), ("qr", False), ("qr", True)])
def test_train_matches_the_oracle_across_calls_and_copies(kind, double_q, dueling):
    """Three train calls of 4 steps at interval 3 (copies inside a call and across calls) against the float32 oracle
    with the same minibatches and the engine's draws; 4 actions, 256 wide, C51 51 atoms, QR-DQN 200 quantiles."""
    S, B = 4, 64
    algo = build(kind, dueling, K=200 if kind == "qr" else None, hidden=(256, 256), double_q=double_q, steps=7,
                 target_update_interval=3)
    algo.device_rng_seed = 17
    fill(algo.replay_buffer, 8, 4)
    oracle = oracle_for(algo, kind)
    copies = 0
    for call in range(3):
        np.random.seed(20 + call)
        algo.train(algo.replay_buffer, S, B)
        draws = algo._engine.get_noisy_draws(S)
        np.random.seed(20 + call)
        logs = ON.train_f32(oracle, [algo.replay_buffer.sample_minibatch(B) for _ in range(S)], draws)
        copies += sum(logs["copied"])
        errs = _errs(algo, oracle, logs)
        print(f"{kind} dueling={dueling} double_q={double_q} call {call}:", {k: f"{v:.1e}" for k, v in errs.items()})
        for k, v in errs.items():
            assert v < 2e-5, (call, k, v, errs)
    assert copies == 4


# ---- one step against the float64 reference ------------------------------------------------------------------------
F64_CASES = {  # (kind, dueling, obs, (h1, h2), n actions, K, B, double_q, one noisy layer)
    "dqn_odd": ("dqn", False, 5, (33, 300), 4, 1, 256, True, None),
    "dqn_b1": ("dqn", False, 8, (300, 33), 6, 1, 1, True, None),
    "dqn_n1": ("dqn", False, 3, (33, 33), 1, 1, 256, False, None),
    "dqn_one_layer": ("dqn", False, 8, (64, 64), 4, 1, 128, True, 1),
    "dueling_odd": ("dqn", True, 5, (33, 300), 4, 1, 256, True, None),
    "c51_odd": ("c51", False, 6, (33, 300), 3, 51, 64, True, None),
    "c51_dueling_b1": ("c51", True, 6, (300, 33), 2, 51, 1, False, None),
    "qr_odd": ("qr", False, 6, (300, 33), 4, 32, 256, True, None),
    "qr_dueling_n1": ("qr", True, 6, (33, 33), 1, 16, 64, True, None),
}
KINK, NEAR_TIE = 1e-6, 1e-5
# Bars: about 4x the largest errors measured on an H100 80GB HBM3 (700 W).  The gradient of the noisy vector normwise
# (conftest.rel_err): 3.5e-6 (c51_dueling_b1; 3.3e-6 c51_odd, below 4.5e-7 elsewhere).  Entry by entry against its scale
# (which leaves out the cancellation inside the heads' sums): 6.5e-2 for C51 (c51_odd; 4.7e-4 c51_dueling_b1), 1.2e-4
# elsewhere (dqn_b1; below 2e-5 for the rest).  Q-values: 4.0e-6 of their maximum (c51_odd; below 7.5e-7 elsewhere);
# the loss: 2.6e-7 of its value (c51_dueling_b1).
BAR_GRAD_NORM, BAR_Q, BAR_LOSS = 1.4e-5, 1.6e-5, 1e-6
BAR_GRAD_ENTRY = dict(dqn=5e-4, qr=5e-4, c51=2.6e-1)


def _f64_case(name, seed=0):
    kind, dueling, O, hidden, n, K, B, double_q, one = F64_CASES[name]
    algo = build(kind, dueling, O=O, n=n, K=K, hidden=hidden, seed=seed, double_q=double_q,
                 target_update_interval=1000, one_noisy=one)
    sizes = [O, *hidden, n * K]
    layers = ON.layers_of(algo.q_function.network)
    q_flat, t_flat = flat(algo.q_function.network).astype(np.float64), flat(algo.target_q_function.network).astype(np.float64)
    rng = np.random.default_rng(100 + seed)
    pool = 2 * B + 64
    mb = dict(observations=rng.standard_normal((pool, O)).astype(np.float32),
              actions=rng.integers(0, n, pool).astype(np.float32),
              rewards=(2.0 * rng.standard_normal(pool)).astype(np.float32),
              next_observations=rng.standard_normal((pool, O)).astype(np.float32), dones=rng.random(pool) < 0.1)
    e = algo._ensure_engine(1, B)
    head = dict(dqn={}, c51=ATOMS, qr=dict(n_quantiles=K))[kind]

    def run(m):  # one step from the learner's state, noise keys (5, 1)
        trainable, targets, lins = algo._learner_nets()
        algo._upload_state(e, trainable, targets, lins)
        e.set_noise_keys([5], [1])
        return e.train(algo._hparams(False, 1), m["observations"][None], m["actions"][None], m["rewards"][None],
                       m["next_observations"][None], m["dones"].astype(np.float32)[None])
    run({k: v[:B] for k, v in mb.items()})  # the draws depend on the keys only: read them, then pick the rows
    draws = e.get_noisy_draws(1)[0]

    def ref(m):
        return ON.step_f64(kind, q_flat, t_flat, draws[0], draws[1], m, layers, sizes, K if dueling else 0, "relu",
                           GAMMA, double_q, **head)
    full = ref(mb)
    qmax = np.max(np.abs(full["q_values"])) + 1.0
    keep = (full["margin"] >= KINK) & (full["gap"] > NEAR_TIE * qmax)
    rows = np.flatnonzero(keep)[:B]
    assert len(rows) == B, (name, int(keep.sum()))
    mb = {k: v[rows] for k, v in mb.items()}
    out = run(mb)
    np.testing.assert_array_equal(e.get_noisy_draws(1)[0], draws)
    return algo, e, out, ref(mb)


@pytest.mark.parametrize("name", list(F64_CASES))
def test_one_step_against_the_float64_reference(name):
    algo, e, out, ref = _f64_case(name)
    blob, steps = e.get_state()
    layout, _ = e.state_layout()
    assert steps == [0, 1, 0]
    m = next(blob[o:o + c] for k, i, o, c in layout if k == "m")
    grad = m.astype(np.float64) / 0.1  # Adam's first exp_avg is (1 - beta1) g
    g_err = float(np.max(np.abs(grad - ref["grad"]) / np.maximum(ref["scale"], 1e-30)))
    g_norm = rel_err(grad, ref["grad"])
    q_err = rel_err(out["q1_values"][0], ref["q_values"])
    l_err = abs(float(out["q1_losses"][0]) - ref["loss"]) / max(abs(ref["loss"]), 1e-30)
    print(f"{name}: grad {g_norm:.2e} (entry / scale {g_err:.2e})  q {q_err:.2e}  loss {l_err:.2e}")
    bar_entry = BAR_GRAD_ENTRY[F64_CASES[name][0]]
    assert g_norm < BAR_GRAD_NORM and g_err < bar_entry and q_err < BAR_Q and l_err < BAR_LOSS, \
        (g_norm, g_err, q_err, l_err)


@pytest.mark.parametrize("kind", ["dqn", "c51", "qr"])
@pytest.mark.parametrize("dueling", [False, True])
def test_zero_sigma_is_the_plain_network_bit_for_bit(kind, dueling):
    """With sigma = 0 the composed weights are mu exactly: the first step's Q-values, loss and mu after Adam equal a
    plain network's step started from mu."""
    noisy = build(kind, dueling, double_q=True, target_update_interval=1)
    plain = build(kind, dueling, double_q=True, target_update_interval=1, plain=True)
    with torch.no_grad():
        for a in (noisy.q_function, noisy.target_q_function):
            for name, p in a.network.named_parameters():
                if name.endswith("_sigma"):
                    p.zero_()
        for a, b in ((noisy.q_function, plain.q_function), (noisy.target_q_function, plain.target_q_function)):
            src = {k.replace("weight_mu", "weight").replace("bias_mu", "bias"): v for k, v in a.network.state_dict().items()
                   if not k.endswith("_sigma")}
            b.network.load_state_dict(src)
    for a in (noisy, plain):
        fill(a.replay_buffer, 8, 4, seed=3)
        np.random.seed(4)
        a.train(a.replay_buffer, 1, 64)
    for k in ("q1_values", "q1_losses"):
        np.testing.assert_array_equal(noisy.last_train_output[k], plain.last_train_output[k], err_msg=k)
    mu = {k.replace("weight_mu", "weight").replace("bias_mu", "bias"): v
          for k, v in noisy.q_function.network.state_dict().items() if not k.endswith("_sigma")}
    for k, v in plain.q_function.network.state_dict().items():
        np.testing.assert_array_equal(mu[k].numpy(), v.numpy(), err_msg=k)
    assert any(p.abs().max() > 0 for n_, p in noisy.q_function.network.named_parameters() if n_.endswith("_sigma"))


# ---- the draws ----------------------------------------------------------------------------------------------------
def test_draws_are_standard_normal_and_keyed():
    from scipy import stats
    S, B = 8, 32

    def draws(seed, call, dueling=False):
        a = build("dqn", dueling, hidden=(256, 256), double_q=True)
        fill(a.replay_buffer, 8, 4, seed=2)
        a.device_rng_seed, a._noise_calls = seed, call - 1
        a.train(a.replay_buffer, S, B)
        return a._engine.get_noisy_draws(S)
    d = draws(11, 1)
    assert d.shape == (S, 2, 8 + 256 + 256 + 256 + 256 + 4) and np.isfinite(d).all()
    ks = stats.kstest(d.reshape(-1).astype(np.float64), "norm")
    print(f"{d.size} draws: KS statistic {ks.statistic:.2e}, p = {ks.pvalue:.3f}")
    assert ks.pvalue > 1e-3
    np.testing.assert_array_equal(d, draws(11, 1))  # the same (seed, call): the same draws
    assert not np.array_equal(d[:, 0], d[:, 1])  # online and target differ
    assert not np.array_equal(d[0], d[1])  # across steps
    assert not np.array_equal(d, draws(11, 2))  # across calls
    assert not np.array_equal(d, draws(12, 1))  # across learners' seeds
    for x, y in ((d[:, 0], d[:, 1]), (d[0], d[1])):
        assert abs(np.corrcoef(x.reshape(-1), y.reshape(-1))[0, 1]) < 0.02


# ---- execution paths and groups --------------------------------------------------------------------------------------
def _member(seed, steps, path, kind="qr", dueling=False):
    """path: host, gather, rng (uniform draws), per (prioritized) or nstep (n = 3 on uniform device draws)."""
    kw = dict(O=6, n=5, K=21 if kind != "dqn" else None, hidden=(48, 40), seed=seed, steps=steps, double_q=True,
              target_update_interval=3)
    algo = (build(kind, dueling, per=PER, **kw) if path == "per"
            else build(kind, dueling, n_step=3 if path == "nstep" else 1, **kw))
    if path == "nstep":
        ring(algo, O=6, seed=40 + seed)
    else:
        fill(algo.replay_buffer, 6, 5, rows=1500 + 100 * seed, seed=40 + seed)
    algo.use_device_replay = path != "host"
    algo.use_device_rng = path in ("rng", "nstep")
    algo.device_rng_seed = 1000 + seed
    return algo


@pytest.mark.parametrize("kind,path,dueling", [("dqn", "host", False), ("dqn", "per", True), ("c51", "gather", True),
                                               ("qr", "rng", False), ("qr", "nstep", True)])
def test_graph_and_plain_launches_are_bit_identical(kind, path, dueling):
    res = []
    for graph in ("1", "0"):
        os.environ["B200RL_OFFPOLICY_GRAPH"] = graph
        try:
            a = _member(0, 4, path, kind, dueling)
            runs = []
            for call in range(2):
                np.random.seed(30 + call)
                a.train(a.replay_buffer, 5 + call, 40)
                runs.append(_outputs(a) + _state(a) + [a._engine.get_noisy_draws(5 + call)])
            res.append(runs)
        finally:
            os.environ.pop("B200RL_OFFPOLICY_GRAPH", None)
    for call, (x, y) in enumerate(zip(*res)):
        for i, (u, v) in enumerate(zip(x, y)):
            np.testing.assert_array_equal(u, v, err_msg=f"{kind} {path}: call {call} tensor {i}")


@pytest.mark.parametrize("kind,path,dueling", [("dqn", "host", False), ("qr", "rng", True), ("qr", "per", False),
                                               ("c51", "nstep", True), ("dqn", "nstep", False)])
def test_group_of_three_is_bit_identical_to_solo_engines(kind, path, dueling):
    """Members at different Q step counts (interval 3: they copy on different steps) and noise keys, two calls."""
    from rl_replicas_b200.algorithms import LearnerGroup
    S, B, K = 4, 32, 3
    solo = [_member(k, 3 * k, path, kind, dueling) for k in range(K)]
    grouped = [_member(k, 3 * k, path, kind, dueling) for k in range(K)]
    g = LearnerGroup()
    for k, m in enumerate(grouped):
        np.random.seed(50 + k)
        g.add(m)
    for call in range(2):
        for k, m in enumerate(solo):
            np.random.seed(50 + k) if call == 0 else np.random.set_state(m._np_state)
            m.train(m.replay_buffer, S, B)
            m._np_state = np.random.get_state()
        g.train(S, B)
        assert g._engine.noisy_layers == solo[0]._engine.noisy_layers != 0
        gd = g._engine.get_noisy_draws(S)
        for k, (a, b) in enumerate(zip(solo, grouped)):
            np.testing.assert_array_equal(a._engine.get_noisy_draws(S), gd[k], err_msg=f"member {k} draws")
            for x, y, what in zip(_outputs(a) + _state(a), _outputs(b) + _state(b),
                                  ("q1_values", "q1_losses", "q", "target", "exp_avg", "exp_avg_sq")):
                np.testing.assert_array_equal(x, y, err_msg=f"{kind} {path}: member {k} {what} call {call}")


# ---- launches, refusals, checkpoints ------------------------------------------------------------------------------------
def _launches(algo, S=6, B=64, graph=True):
    from rl_replicas_b200 import _lib
    lib = _lib.load()
    os.environ["B200RL_OFFPOLICY_GRAPH"] = "1" if graph else "0"
    try:
        algo.train(algo.replay_buffer, S, B)  # builds the engine (and the graph)
        n0 = lib.b200rl_launch_count()
        algo.train(algo.replay_buffer, S, B)
        return lib.b200rl_launch_count() - n0
    finally:
        os.environ.pop("B200RL_OFFPOLICY_GRAPH", None)


def test_launches_per_step_are_the_stated_ones():
    """include/b200rl.h: 2 launches per step more than the same network without noise -- 16 (19 with double_q) for a
    plain 3-layer network, 26 (32) for a dueling one, + 2 with prioritized replay."""
    S = 6
    for kind in ("dqn", "qr", "c51"):
        for dueling in (False, True):
            for double_q in (False, True):
                for per in (False, True):
                    if per and kind == "c51":
                        continue
                    for graph in (False, True):
                        kw = dict(double_q=double_q, target_update_interval=3, per=PER if per else None)
                        a, b = build(kind, dueling, **kw), build(kind, dueling, plain=True, **kw)
                        for x in (a, b):
                            fill(x.replay_buffer, 8, 4, rows=1000, seed=6)
                        na, nb = _launches(a, S, graph=graph), _launches(b, S, graph=graph)
                        print(f"{kind} dueling={dueling} double_q={double_q} per={per} graph={graph}: noisy {na}, "
                              f"plain {nb}")
                        assert na - nb == 2 * S, (kind, dueling, double_q, per, graph, na, nb)


def test_engine_refusals():
    from rl_replicas_b200._lib import B200RLError
    from rl_replicas_b200.engine import OffPolicyEngine
    with pytest.raises(B200RLError, match="noisy_layers must be 0 unless"):
        OffPolicyEngine([4, 16, 2], [6, 16, 16, 1], 2, 8, 2, noisy_layers=1)
    with pytest.raises(B200RLError, match="noisy_layers must be 0 unless"):
        OffPolicyEngine([4, 16, 4], [6, 16, 16, 1], 2, 8, 2, algo=OffPolicyEngine.SAC, noisy_layers=1)
    with pytest.raises(B200RLError, match="beyond the Q network's 3 Linear"):
        OffPolicyEngine(None, [4, 16, 16, 3], 1, 8, 2, algo=OffPolicyEngine.DQN, noisy_layers=0b1000)
    with pytest.raises(B200RLError, match="beyond the Q network's 5 Linear"):
        OffPolicyEngine(None, [4, 16, 16, 3], 1, 8, 2, algo=OffPolicyEngine.DQN, dueling_k=1, noisy_layers=0b100000)
    with pytest.raises(B200RLError, match="beyond"):
        OffPolicyEngine(None, [4, 16, 16, 3], 1, 8, 2, algo=OffPolicyEngine.C51, noisy_layers=-1)
    plain = OffPolicyEngine(None, [4, 16, 3], 1, 8, 2, algo=OffPolicyEngine.DQN)
    with pytest.raises(B200RLError, match="no noisy layers"):
        plain.set_noise_keys([1], [1])
    e = OffPolicyEngine(None, [4, 16, 3], 1, 8, 2, algo=OffPolicyEngine.DQN, noisy_layers=0b10)
    P = 16 * 5 + 2 * 3 * 17
    assert e.n_qp == P and e.get_params(1).shape == (P,) and e.noise_width == 19
    e.set_dqn(1, False)
    from rl_replicas_b200._lib import OffPolicyHparams
    hp = OffPolicyHparams()
    hp.q1_lr, hp.q_beta1, hp.q_beta2, hp.q_eps = 1e-3, 0.9, 0.999, 1e-8
    z = np.zeros((1, 2, 4), np.float32)
    batch = (z, np.zeros((1, 2), np.float32), np.zeros((1, 2), np.float32), z, np.zeros((1, 2), np.float32))
    with pytest.raises(B200RLError, match="fresh keys"):
        e.train(hp, *batch)
    e.set_noise_keys([1], [1])
    e.train(hp, *batch)
    with pytest.raises(B200RLError, match="fresh keys"):  # a call consumes its keys
        e.train(hp, *batch)


def test_checkpoint_round_trip(tmp_path):
    a = build("qr", True, double_q=True, target_update_interval=2)
    fill(a.replay_buffer, 8, 4)
    np.random.seed(1)
    a.train(a.replay_buffer, 5, 64)
    path = str(tmp_path / "model.pt")
    a.save_model(1, path)
    b = build("qr", True, seed=9, double_q=True, target_update_interval=2)
    assert b.load_model(path) == 1
    for x, y in ((a.q_function, b.q_function), (a.target_q_function, b.target_q_function)):
        np.testing.assert_array_equal(flat(x.network), flat(y.network))
    for key in ("exp_avg", "exp_avg_sq"):
        np.testing.assert_array_equal(adam_flat(a.q_function.optimizer, key)[0], adam_flat(b.q_function.optimizer, key)[0])
    obs = np.random.default_rng(0).standard_normal((32, 8)).astype(np.float32)
    np.testing.assert_array_equal(a.evaluation_policy.get_action_numpy(obs), b.evaluation_policy.get_action_numpy(obs))
    # both continue identically on the device from the same keys
    for x in (a, b):
        x._noise_calls = 1
        np.random.seed(2)
        x.train(a.replay_buffer, 3, 64)
    np.testing.assert_array_equal(flat(a.q_function.network), flat(b.q_function.network))
