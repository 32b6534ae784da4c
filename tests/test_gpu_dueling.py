"""GPU: dueling Q networks on the off-policy engine (config dueling_k; include/b200rl.h, "Dueling Q networks") -- dueling
DQN (Double on and off), C51 and QR-DQN against their float32 oracles across calls and target copies, one step against
the float64 reference (oracle/dueling.py) at edge shapes, graph against plain launches, groups of 3 and 16 against solo
engines, prioritized replay replayed through oracle/per.py, n-step returns alone and with prioritized replay, the
engine's refusals, the stated launch count, and DQN.learn end to end."""
import os

import numpy as np
import pytest
import torch

from conftest import rel_err
from oracle import c51 as OC
from oracle import dqn as OD
from oracle import dueling as ODu
from oracle import nstep as ON
from oracle import per as OP
from oracle import qr as OQ
from test_dqn import LEARN, RETURN_BAR, evaluation_return
from test_dueling import DQN_KW, make
from test_gpu_dqn import GAMMA, LR, adam_flat, compare, fill, flat
from test_gpu_nstep import check_walk, fill_episodes, ring

pytestmark = pytest.mark.gpu

ATOMS = dict(n_atoms=51, v_min=-10.0, v_max=10.0)
PER = dict(buffer_size=8000, alpha=0.6, beta_start=0.4, beta_anneal_steps=50, eps=1e-6)


def build(kind="dqn", O=8, n=4, K=None, hidden=(64, 64), act=torch.nn.ReLU, seed=0, steps=0, per=None, **kw):
    """A dueling DQN / C51 / QR-DQN learner (DuelingMLP([O, *hidden], n, K)) on a stub discrete environment; ``steps`` >
    0 gives its Adam a state at that step count, ``per`` a PrioritizedReplayBuffer with those settings."""
    import types
    from rl_replicas_b200.algorithms import C51, DQN, QRDQN
    from rl_replicas_b200.critics import CategoricalQFunction, DiscreteQFunction, QuantileQFunction
    from rl_replicas_b200.networks import DuelingMLP
    from rl_replicas_b200.replay_buffer import PrioritizedReplayBuffer, ReplayBuffer
    K = K or {"dqn": 1, "c51": ATOMS["n_atoms"], "qr": 32}[kind]
    torch.manual_seed(seed)
    net = DuelingMLP([O, *hidden], n, K, act)
    opt = torch.optim.Adam(net.parameters(), lr=LR)
    for _ in range(steps):  # some arbitrary earlier steps
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


def kind_of(algo):
    return {"DQN": "dqn", "C51": "c51", "QRDQN": "qr"}[type(algo).__name__]


def oracle_for(algo):
    q, qt, rb = algo.q_function, algo.target_q_function, algo.replay_buffer
    kw = dict(gamma=algo.gamma, target_update_interval=algo.target_update_interval, double_q=algo.double_q)
    kind = kind_of(algo)
    nstep = algo.n_step > 1  # the oracles of oracle/nstep.py take each window's discount as gamma
    if kind == "c51":
        cls = ON.NStepC51Oracle if nstep else OC.C51Oracle
        return cls(q.network, qt.network, q.optimizer, n_atoms=q.n_atoms, v_min=q.v_min, v_max=q.v_max, **kw)
    if kind == "qr":  # takes a minibatch's discounts itself
        return OQ.QrDqnOracle(q.network, qt.network, q.optimizer, n_quantiles=q.n_quantiles,
                              alpha=getattr(rb, "alpha", 0.6), eps=getattr(rb, "eps", 1e-6), **kw)
    if hasattr(rb, "alpha"):
        cls = ON.NStepPerDqnOracle if nstep else OP.PerDqnOracle
        return cls(q.network, qt.network, q.optimizer, alpha=rb.alpha, eps=rb.eps, **kw)
    return (ON.NStepDqnOracle if nstep else OD.DqnOracle)(q.network, qt.network, q.optimizer, **kw)


def step_count(algo):
    from rl_replicas_b200.algorithms.dqn import describe_q_network
    return algo._adam_step_count(algo.q_function.optimizer, describe_q_network(algo.q_function.network)[3])


def _errs(algo, oracle, logs):
    errs = compare(algo, oracle)
    out = algo.last_train_output
    errs["q1_values"] = rel_err(out["q1_values"], np.stack(logs["q1_values"]))
    errs["q1_losses"] = rel_err(out["q1_losses"], np.asarray(logs["q1_losses"]))
    return errs


# The learners start from a few earlier Adam steps (a fresh Adam's first step turns float32 rounding of near-zero
# gradient entries into visible parameter differences); the first step itself is held against float64 below.
@pytest.mark.parametrize("kind,double_q", [("dqn", False), ("dqn", True), ("c51", True), ("qr", False), ("qr", True)])
def test_train_matches_the_oracle_across_calls_and_copies(kind, double_q):
    """Three train calls of 4 steps at interval 3 (copies inside a call and across calls) against the float32 oracle
    with the same minibatches; 4 actions, 256-wide trunk and streams, C51 51 atoms, QR-DQN 200 quantiles."""
    S, B = 4, 64
    algo = build(kind, K=200 if kind == "qr" else None, hidden=(256, 256), double_q=double_q, steps=7,
                 target_update_interval=3)
    fill(algo.replay_buffer, 8, 4)
    oracle = oracle_for(algo)
    copies = 0
    for call in range(3):
        np.random.seed(20 + call)
        algo.train(algo.replay_buffer, S, B)
        np.random.seed(20 + call)
        logs = oracle.train([algo.replay_buffer.sample_minibatch(B) for _ in range(S)])
        copies += sum(logs["copied"])
        errs = _errs(algo, oracle, logs)
        print(f"{kind} double_q={double_q} call {call}:", {k: f"{v:.1e}" for k, v in errs.items()})
        for k, v in errs.items():
            assert v < 2e-5, (call, k, v, errs)
    assert copies == 4


# ---- one step against the float64 reference ------------------------------------------------------------------------
F64_CASES = {  # (kind, obs, h1, h2, n actions, K, hidden, B, double_q)
    "dqn_lunar": ("dqn", 8, 256, 256, 4, 1, "relu", 256, True),
    "dqn_n1": ("dqn", 1, 33, 33, 1, 1, "relu", 256, False),
    "dqn_n18_wide": ("dqn", 128, 300, 256, 18, 1, "relu", 1000, True),
    "dqn_h1": ("dqn", 6, 1, 1, 4, 1, "relu", 256, True),
    "dqn_b1": ("dqn", 1, 300, 300, 18, 1, "relu", 1, True),
    "dqn_tanh": ("dqn", 8, 33, 300, 4, 1, "tanh", 256, False),
    "c51_lunar": ("c51", 8, 256, 256, 4, 51, "relu", 256, True),
    "c51_n18_b1": ("c51", 6, 33, 300, 18, 51, "relu", 1, False),
    "c51_n1": ("c51", 128, 256, 33, 1, 51, "relu", 256, True),
    "qr_lunar": ("qr", 8, 256, 256, 4, 200, "relu", 256, True),
    "qr_k256_n1": ("qr", 128, 300, 33, 1, 256, "relu", 64, False),
    "qr_n18": ("qr", 6, 33, 33, 18, 51, "relu", 256, True),
    "qr_k1": ("qr", 1, 256, 1, 4, 1, "relu", 1000, True),
}
KINK, NEAR_TIE = 1e-6, 1e-5
# Bars: about 4x the largest errors measured on an H100 80GB HBM3 (700 W).  The gradient normwise (conftest.rel_err):
# 2.8e-6 (qr_lunar; 1.7e-6 c51_n18_b1, below 1.3e-6 elsewhere).  Entry by entry against its scale (the sum over rows of
# |a row's contribution|, which leaves out the cancellation inside the aggregation's dQ - mean and inside the heads'
# sums): 3.1e-3 (c51_lunar; 2.5e-3 qr_lunar, 2.5e-4 c51_n18_b1, below 5e-5 elsewhere).  Q-values: 5.4e-6 of their
# maximum (c51_n1; 3.7e-6 c51_lunar, below 7e-7 elsewhere); the loss: 2.5e-7 of its value (dqn_b1).
BAR_GRAD_NORM, BAR_GRAD_ENTRY, BAR_Q, BAR_LOSS = 1.2e-5, 1.2e-2, 2e-5, 1e-6


def _ref(kind, q_flat, t_flat, mb, sizes, K, hidden, double_q):
    if kind == "dqn":
        return ODu.dqn_step_f64(q_flat, t_flat, mb, sizes, hidden, GAMMA, double_q)
    if kind == "c51":
        return ODu.c51_step_f64(q_flat, t_flat, mb, sizes, K, ATOMS["v_min"], ATOMS["v_max"], hidden, GAMMA, double_q)
    return ODu.qr_step_f64(q_flat, t_flat, mb, sizes, K, hidden, GAMMA, double_q)


def _f64_case(name, seed=0):
    kind, O, h1, h2, n, K, hidden, B, double_q = F64_CASES[name]
    sizes = [O, h1, h2, n * K]
    act = {"relu": torch.nn.ReLU, "tanh": torch.nn.Tanh}[hidden]
    algo = build(kind, O=O, n=n, K=K, hidden=(h1, h2), act=act, seed=seed, double_q=double_q,
                 target_update_interval=1000)
    q_flat, t_flat = flat(algo.q_function.network).astype(np.float64), flat(algo.target_q_function.network).astype(np.float64)
    rng = np.random.default_rng(100 + seed)
    pool = 2 * B + 64
    mb = dict(observations=rng.standard_normal((pool, O)).astype(np.float32),
              actions=rng.integers(0, n, pool).astype(np.float32),
              rewards=(2.0 * rng.standard_normal(pool)).astype(np.float32),
              next_observations=rng.standard_normal((pool, O)).astype(np.float32), dones=rng.random(pool) < 0.1)
    ref = _ref(kind, q_flat, t_flat, mb, sizes, K, hidden, double_q)
    qmax = np.max(np.abs(ref["q_values"])) + 1.0
    keep = (ref["margin"] >= KINK) & (ref["gap"] > NEAR_TIE * qmax)
    rows = np.flatnonzero(keep)[:B]
    assert len(rows) == B, (name, int(keep.sum()))
    mb = {k: v[rows] for k, v in mb.items()}
    return algo, mb, _ref(kind, q_flat, t_flat, mb, sizes, K, hidden, double_q)


@pytest.mark.parametrize("name", list(F64_CASES))
def test_one_step_against_the_float64_reference(name):
    algo, mb, ref = _f64_case(name)
    B = len(mb["rewards"])
    e = algo._ensure_engine(1, B)
    assert e.dueling_k == F64_CASES[name][5]
    trainable, targets, lins = algo._learner_nets()
    algo._upload_state(e, trainable, targets, lins)
    out = e.train(algo._hparams(False, 1), mb["observations"][None], mb["actions"][None], mb["rewards"][None],
                  mb["next_observations"][None], mb["dones"].astype(np.float32)[None])
    blob, steps = e.get_state()
    layout, _ = e.state_layout()
    assert steps == [0, 1, 0]
    m = next(blob[o:o + c] for k, i, o, c in layout if k == "m")
    grad = m.astype(np.float64) / 0.1
    g_err = float(np.max(np.abs(grad - ref["grad"]) / np.maximum(ref["scale"], 1e-30)))
    g_norm = rel_err(grad, ref["grad"])
    q_err = rel_err(out["q1_values"][0], ref["q_values"])
    l_err = abs(float(out["q1_losses"][0]) - ref["loss"]) / max(abs(ref["loss"]), 1e-30)
    print(f"{name}: grad {g_norm:.2e} (entry / scale {g_err:.2e})  q {q_err:.2e}  loss {l_err:.2e}")
    assert g_norm < BAR_GRAD_NORM and g_err < BAR_GRAD_ENTRY and q_err < BAR_Q and l_err < BAR_LOSS, \
        (g_norm, g_err, q_err, l_err)


# ---- prioritized replay and n-step returns ---------------------------------------------------------------------------
def _replay_prioritized(algo, calls, S, B, nstep=False):
    """`calls` train() calls replayed through oracle/per.py's draw and tree and the prioritized oracle."""
    rb = algo.replay_buffer
    oracle = oracle_for(algo)
    for call in range(calls):
        leaves = rb.priorities().astype(np.float32)
        t0 = step_count(algo)
        algo.train(rb, S, B)
        idx, w, newp = algo._engine.get_per_draws(S, B)
        if nstep:
            check_walk(algo, idx, S, B)
        mbs, ps, betas = [], [], []
        for st in range(S):
            want, dist = OP.stratified_draw(leaves, algo.device_rng_seed, algo._device_rng_calls, st, B)
            far = dist > 2e-6
            assert (want[far] == idx[st][far]).all(), (call, st)
            mbs.append(ON.nstep_minibatch(rb, idx[st], algo.n_step, algo.gamma) if nstep else
                       {k: rb._cols[k][idx[st]] for k in rb.COLUMNS})
            ps.append(leaves[idx[st]])
            betas.append(float(OP.beta_schedule(t0 + st, rb.beta_start, rb.beta_anneal_steps)))
            leaves = OP.apply_priorities(leaves, idx[st], newp[st]).astype(np.float32)
        np.testing.assert_array_equal(rb.priorities(), leaves)  # last occurrence wins, exactly
        logs = oracle.train(mbs, ps, betas)
        errs = _errs(algo, oracle, logs)
        w_err = float(np.max(np.abs(w - np.stack(logs["weights"])) / np.stack(logs["weights"])))
        p_ref = np.stack(logs["priorities"])
        p_err = float(np.max(np.abs(newp - p_ref) / p_ref))
        print(f"call {call}:", {k: f"{v:.1e}" for k, v in errs.items()}, f"weights {w_err:.1e} priorities {p_err:.1e}")
        for k, v in errs.items():
            assert v < 2e-5, (call, k, v)
        assert w_err < 1e-6 and p_err < 2e-5, (w_err, p_err)


@pytest.mark.parametrize("kind", ["dqn", "qr"])
def test_prioritized_draws_weights_and_priorities_match_the_oracle(kind):
    """3 calls of 4 steps on a half-full buffer (zero-priority leaves), target copies inside and across calls."""
    algo = build(kind, per=PER, double_q=True, steps=3, target_update_interval=3)
    fill(algo.replay_buffer, 8, 4, rows=4000, seed=11)
    algo.device_rng_seed = 91
    _replay_prioritized(algo, 3, 4, 64)


@pytest.mark.parametrize("kind", ["dqn", "c51", "qr"])
def test_nstep_matches_the_oracle(kind):
    """n = 3 on device draws from a wrapped ring, two calls, against the oracles of oracle/nstep.py."""
    S, B = 4, 64
    algo = ring(build(kind, steps=7, double_q=True, target_update_interval=3, n_step=3), seed=7)
    algo.use_device_rng, algo.device_rng_seed = True, 5
    oracle = oracle_for(algo)
    rb = algo.replay_buffer
    for call in range(2):
        algo.train(rb, S, B)
        idx, _ = algo._engine.get_draws(S, B)
        check_walk(algo, idx, S, B)
        logs = oracle.train([ON.nstep_minibatch(rb, idx[s], 3, algo.gamma) for s in range(S)])
        errs = _errs(algo, oracle, logs)
        print(f"{kind} n=3 call {call}:", {k: f"{v:.1e}" for k, v in errs.items()})
        for k, v in errs.items():
            assert v < 2e-5, (call, k, v, errs)


@pytest.mark.parametrize("kind", ["dqn", "qr"])
def test_prioritized_nstep_matches_the_oracle(kind):
    algo = build(kind, per=dict(PER, buffer_size=700), n_step=3, double_q=True, steps=2, target_update_interval=4)
    fill_episodes(algo.replay_buffer, 8, 1500, 9)
    algo.device_rng_seed = 9
    assert algo.replay_buffer._head > 0
    _replay_prioritized(algo, 2, 3, 64, nstep=True)


# ---- execution paths and groups --------------------------------------------------------------------------------------
def _state(algo):
    return [flat(algo.q_function.network), flat(algo.target_q_function.network),
            *[adam_flat(algo.q_function.optimizer, k)[0] for k in ("exp_avg", "exp_avg_sq")]]


def _member(seed, steps, path, kind="qr"):
    """path: host, gather, rng (uniform draws), per (prioritized) or nstep (n = 3 on uniform device draws)."""
    kw = dict(O=6, n=5, K=21 if kind != "dqn" else None, hidden=(48, 40), seed=seed, steps=steps, double_q=True,
              target_update_interval=3)
    algo = build(kind, per=PER, **kw) if path == "per" else build(kind, n_step=3 if path == "nstep" else 1, **kw)
    if path == "nstep":
        ring(algo, O=6, seed=40 + seed)
    else:
        fill(algo.replay_buffer, 6, 5, rows=1500 + 100 * seed, seed=40 + seed)
    algo.use_device_replay = path != "host"
    algo.use_device_rng = path in ("rng", "nstep")
    algo.device_rng_seed = 1000 + seed
    return algo


def _outputs(algo):
    return [algo.last_train_output[k] for k in ("q1_values", "q1_losses")]


@pytest.mark.parametrize("kind,path", [("dqn", "host"), ("dqn", "per"), ("c51", "gather"), ("qr", "rng"), ("qr", "per"),
                                       ("qr", "nstep")])
def test_graph_and_plain_launches_are_bit_identical(kind, path):
    res = []
    for graph in ("1", "0"):
        os.environ["B200RL_OFFPOLICY_GRAPH"] = graph
        try:
            a = _member(0, 4, path, kind)
            runs = []
            for call in range(2):
                np.random.seed(30 + call)
                a.train(a.replay_buffer, 5 + call, 40)
                runs.append(_outputs(a) + _state(a))
            res.append(runs)
        finally:
            os.environ.pop("B200RL_OFFPOLICY_GRAPH", None)
    for call, (x, y) in enumerate(zip(*res)):
        for i, (u, v) in enumerate(zip(x, y)):
            np.testing.assert_array_equal(u, v, err_msg=f"{kind} {path}: call {call} tensor {i}")


@pytest.mark.parametrize("K,kind,path", [(3, "dqn", "host"), (3, "c51", "gather"), (3, "qr", "per"), (3, "qr", "nstep"),
                                         (16, "dqn", "per"), (16, "qr", "gather")])
def test_group_is_bit_identical_to_solo_engines(K, kind, path):
    """Members at different Q step counts (interval 3: they copy on different steps), two calls."""
    from rl_replicas_b200.algorithms import LearnerGroup
    S, B = 4, 32
    solo = [_member(k, 3 * k, path, kind) for k in range(K)]
    grouped = [_member(k, 3 * k, path, kind) for k in range(K)]
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
        assert g._engine.dueling_k == solo[0].q_function.network.outputs_per_action
        for k, (a, b) in enumerate(zip(solo, grouped)):
            for x, y, what in zip(_outputs(a) + _state(a), _outputs(b) + _state(b),
                                  ("q1_values", "q1_losses", "q", "target", "exp_avg", "exp_avg_sq")):
                np.testing.assert_array_equal(x, y, err_msg=f"{kind} {path}: member {k} {what} call {call}")
            if path == "per":
                np.testing.assert_array_equal(a.replay_buffer.priorities(), b.replay_buffer.priorities())


# ---- refusals, launches and end to end --------------------------------------------------------------------------------
def test_engine_refuses_bad_dueling_configurations():
    from rl_replicas_b200._lib import B200RLError
    from rl_replicas_b200.engine import OffPolicyEngine
    with pytest.raises(B200RLError, match="dueling_k must be 0 unless"):
        OffPolicyEngine([4, 16, 2], [6, 16, 16, 1], 2, 8, 2, dueling_k=1)
    with pytest.raises(B200RLError, match="dueling_k must be 0 unless"):
        OffPolicyEngine([4, 16, 4], [6, 16, 16, 1], 2, 8, 2, algo=OffPolicyEngine.SAC, dueling_k=1)
    for sizes, k, msg in (([4, 16, 12], 1, "3 layers"), ([4, 16, 16, 16, 12], 1, "3 layers"),
                          ([4, 16, 16, 12], 5, "not n_actions x dueling_k"), ([4, 16, 16, 12], -1, ">= 1")):
        with pytest.raises(B200RLError, match=msg):
            OffPolicyEngine(None, sizes, 1, 8, 2, algo=OffPolicyEngine.DQN, dueling_k=k)
    with pytest.raises(B200RLError, match="out_act identity"):
        OffPolicyEngine(None, [4, 16, 16, 12], 1, 8, 2, q_acts=("relu", "tanh"), algo=OffPolicyEngine.DQN, dueling_k=3)
    e = OffPolicyEngine(None, [4, 16, 8, 12], 1, 8, 2, algo=OffPolicyEngine.C51, dueling_k=3)
    P = 16 * 5 + 2 * 8 * 17 + 3 * 9 + 12 * 9
    assert e.n_qp == P and e.get_params(1).shape == (P,)
    with pytest.raises(B200RLError, match=f"expects {P} floats"):
        e.set_params(1, np.zeros(P - 1, np.float32))


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
    """include/b200rl.h: 24 launches per step (30 with double_q) for DQN, QR-DQN and C51, + 2 with prioritized replay;
    a call adds what a plain network's call adds around its steps (staging, draws, the read-back)."""
    from test_gpu_dqn import build as build_plain
    S = 6
    for kind in ("dqn", "qr", "c51"):
        for double_q in (False, True):
            for per in (False, True):
                if per and kind == "c51":
                    continue
                for graph in (False, True):
                    kw = dict(double_q=double_q, target_update_interval=3)
                    d = build(kind, per=PER if per else None, **kw)
                    p = build_plain(**kw)
                    if per:
                        from rl_replicas_b200.replay_buffer import PrioritizedReplayBuffer
                        p.replay_buffer = PrioritizedReplayBuffer(**PER)
                    for a in (d, p):
                        fill(a.replay_buffer, 8, 4, rows=1000, seed=6)
                    nd, np_ = _launches(d, S, graph=graph), _launches(p, S, graph=graph)
                    print(f"{kind} double_q={double_q} per={per} graph={graph}: dueling {nd}, plain DQN {np_}")
                    plain_step, duel_step = (17, 30) if double_q else (14, 24)
                    assert nd - np_ == S * (duel_step - plain_step), (kind, double_q, per, graph, nd, np_)


def test_learn_solves_the_choice_task(tmp_path, capsys):
    """DQN.learn with a DuelingMLP end to end on tests/test_dqn.py's one-step choice task with the seeds of the
    oracle-driven loop in tests/test_dueling.py: the tags are recorded, model.pt is written and reloads, and the
    evaluation return clears the same bar."""
    np.random.seed(0)
    algo = make("dqn", **DQN_KW)
    algo.learn(output_dir=str(tmp_path), **LEARN)
    after = evaluation_return(algo)
    printed = capsys.readouterr().out
    with capsys.disabled():
        print(f"DQN.learn with a DuelingMLP on the choice task: evaluation return {after:.3f}")
    for tag in ("q-function/average_loss", "q-function/avarage_q-value", "exploration/epsilon",
                "evaluation/average_episode_return"):
        assert f"\n{tag}: " in printed, tag
    path = os.path.join(tmp_path, "model.pt")
    other = make("dqn", seed=5, **DQN_KW)
    other.load_model(path)
    assert evaluation_return(other) == after  # the reloaded networks act exactly as the trained ones
    assert after > RETURN_BAR
