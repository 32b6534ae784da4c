"""GPU: C51 on the off-policy engine -- C51.train against the float32 oracle (oracle/c51.py) across calls and target
copies, one step against the float64 reference at edge shapes, bit-identical execution paths, learner groups bit for bit
equal to solo engines, the invalid-action refusal, the engine's refusals, the launch budget, and C51.learn end to end."""
import os

import numpy as np
import pytest
import torch

from conftest import rel_err
from oracle import c51 as OC
from test_c51 import C51_KW, make_c51
from test_dqn import LEARN, RETURN_BAR, evaluation_return
from test_gpu_dqn import GAMMA, LR, adam_flat, compare, fill, flat

pytestmark = pytest.mark.gpu


def build(O=8, n=4, N=51, v=(-10.0, 10.0), hidden=(64, 64), act=torch.nn.ReLU, seed=0, steps=0, **kw):
    """A C51 learner on a stub discrete environment (test_gpu_dqn.build with a categorical critic)."""
    import types
    from rl_replicas_b200.algorithms import C51
    from rl_replicas_b200.critics import CategoricalQFunction
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    torch.manual_seed(seed)
    net = MLP([O, *hidden, n * N], act)
    opt = torch.optim.Adam(net.parameters(), lr=LR)
    for _ in range(steps):  # some arbitrary earlier steps
        opt.zero_grad()
        net(torch.randn(16, O)).pow(2).mean().backward()
        opt.step()
    env = types.SimpleNamespace(action_space=types.SimpleNamespace(n=n, shape=()), spec=types.SimpleNamespace(id="stub"),
                                observation_space=types.SimpleNamespace(shape=(O,)))
    qf = CategoricalQFunction(net, opt, n_atoms=N, v_min=v[0], v_max=v[1])
    algo = C51(qf, None, env, None, ReplayBuffer(), None, gamma=GAMMA, **kw)
    with torch.no_grad():  # a target that differs from the online network
        for p in algo.target_q_function.network.parameters():
            p.add_(0.05 * torch.randn_like(p))
    algo.metrics_manager = None
    algo.current_total_steps = 0
    return algo


def oracle_for(algo):
    q = algo.q_function
    return OC.C51Oracle(q.network, algo.target_q_function.network, q.optimizer, n_atoms=q.n_atoms, v_min=q.v_min,
                        v_max=q.v_max, gamma=algo.gamma, target_update_interval=algo.target_update_interval,
                        double_q=algo.double_q)


# From a fresh Adam the first step moves every parameter by lr g / (|g| + eps): entries whose gradient is at the scale
# of eps (C51's p_k sum m - m_k cancels on rows whose target matches p) turn float32 rounding into parameter
# differences of lr x error / eps, which says nothing about the head.  The first step itself is held against the
# float64 reference below; here the learners start from a few earlier Adam steps.
@pytest.mark.parametrize("start_steps", [7, 20])
@pytest.mark.parametrize("double_q", [False, True])
def test_train_matches_the_oracle_across_calls_and_copies(double_q, start_steps):
    """Three C51.train calls of 4 steps at interval 3 (copies inside a call and across calls) against the oracle with
    the same minibatches."""
    S, B = 4, 64
    algo = build(double_q=double_q, steps=start_steps, target_update_interval=3)
    fill(algo.replay_buffer, 8, 4)
    oracle = oracle_for(algo)
    copies = 0
    for call in range(3):
        np.random.seed(20 + call)
        algo.train(algo.replay_buffer, S, B)
        out = algo.last_train_output
        np.random.seed(20 + call)
        logs = oracle.train([algo.replay_buffer.sample_minibatch(B) for _ in range(S)])
        copies += sum(logs["copied"])
        errs = compare(algo, oracle)
        errs["q1_values"] = rel_err(out["q1_values"], np.stack(logs["q1_values"]))
        errs["q1_losses"] = rel_err(out["q1_losses"], np.asarray(logs["q1_losses"]))
        print(f"double_q={double_q} start={start_steps} call {call}:", {k: f"{v:.1e}" for k, v in errs.items()})
        for k, v in errs.items():
            assert v < 2e-5, (call, k, v, errs)
    assert copies == 4


# ---- one step against the float64 reference ------------------------------------------------------------------------
F64_CASES = {  # (sizes without the output layer, n actions, N atoms, (v_min, v_max), hidden, B, double_q)
    "lunar": ([8, 256, 256], 4, 51, (-10.0, 10.0), "relu", 256, True),
    "n1": ([6, 32, 32], 1, 51, (-10.0, 10.0), "relu", 33, False),
    "n18": ([6, 64, 64], 18, 51, (-10.0, 10.0), "relu", 257, True),
    "atoms2": ([6, 64, 64], 4, 2, (-1.0, 1.0), "relu", 100, True),
    "atoms101": ([6, 64, 64], 4, 101, (-5.0, 5.0), "relu", 1000, False),
    "b1": ([5, 31, 31], 3, 51, (-10.0, 10.0), "relu", 1, True),
    "two_layer": ([7, 48], 5, 51, (-10.0, 10.0), "relu", 64, True),
    "four_layer": ([7, 64, 48, 40], 3, 51, (-10.0, 10.0), "relu", 100, True),
    "tanh": ([8, 64, 64], 4, 51, (-10.0, 10.0), "tanh", 128, False),
    "tie": ([8, 64, 64], 4, 51, (-10.0, 10.0), "relu", 128, True),
}
KINK, NEAR_TIE = 1e-6, 1e-5
# Bars: about 4x the largest errors measured on an H100.  The gradient normwise (conftest.rel_err): 1.1e-6 (n18).  Entry
# by entry against its scale (the sum over rows of |a row's contribution|): 1.3e-2 (n18; 2.7e-3 atoms101, below 2.6e-3
# elsewhere) -- that scale leaves out the cancellation inside p_k sum m - m_k, which is where the float32 rounding sits.
# Q-values: 7.9e-6 of their maximum (four_layer; the expected values sit near 0 on a symmetric support); the loss:
# 8.8e-8 of its value (n1).
BAR_GRAD_NORM, BAR_GRAD_ENTRY, BAR_Q, BAR_LOSS = 5e-6, 5e-2, 3e-5, 4e-7


def _f64_case(name, seed=0):
    body, n, N, (v_min, v_max), hidden, B, double_q = F64_CASES[name]
    sizes = body + [n * N]
    act = {"relu": torch.nn.ReLU, "tanh": torch.nn.Tanh}[hidden]
    algo = build(O=sizes[0], n=n, N=N, v=(v_min, v_max), hidden=tuple(sizes[1:-1]), act=act, seed=seed,
                 double_q=double_q, target_update_interval=1000)
    if name == "tie":  # actions 1 and 2 of the online network have equal distributions on every row, and the largest
        lin = algo.q_function.network.network[-2]
        with torch.no_grad():
            lin.weight[2 * N:3 * N] = lin.weight[N:2 * N]
            lin.bias[N:3 * N] = torch.linspace(0.0, 8.0, N).repeat(2)
    q_flat, t_flat = flat(algo.q_function.network).astype(np.float64), flat(algo.target_q_function.network).astype(np.float64)
    rng = np.random.default_rng(100 + seed)
    pool = 4 * B + 64
    z = OC.support(N, v_min, v_max)
    rew = (2.0 * rng.standard_normal(pool)).astype(np.float32)
    done = rng.random(pool) < 0.1
    k = np.arange(pool)
    rew[k % 16 == 3] = 3.0 * v_max  # every Tz_j clamps at v_max
    rew[k % 16 == 7] = 3.0 * v_min - 3.0 * v_max  # ... at v_min
    on_atom = k % 16 == 11  # terminal rows whose target is an atom
    rew[on_atom], done[on_atom] = z[k[on_atom] % N], True
    mb = dict(observations=rng.standard_normal((pool, sizes[0])).astype(np.float32),
              actions=rng.integers(0, n, pool).astype(np.float32), rewards=rew,
              next_observations=rng.standard_normal((pool, sizes[0])).astype(np.float32), dones=done)
    ref = OC.c51_step_f64(q_flat, t_flat, mb, sizes, N, v_min, v_max, hidden, GAMMA, double_q)
    qmax = np.max(np.abs(ref["q_values"])) + 1.0
    keep = ref["margin"] >= KINK
    if name != "tie":
        keep &= ref["gap"] > NEAR_TIE * qmax
    rows = np.flatnonzero(keep)[:B]
    assert len(rows) == B, (name, int(keep.sum()))
    mb = {k: v[rows] for k, v in mb.items()}
    return algo, mb, OC.c51_step_f64(q_flat, t_flat, mb, sizes, N, v_min, v_max, hidden, GAMMA, double_q), sizes


@pytest.mark.parametrize("name", list(F64_CASES))
def test_one_step_against_the_float64_reference(name):
    algo, mb, ref, sizes = _f64_case(name)
    if name == "tie":
        with torch.no_grad():
            q = algo.q_function(torch.as_tensor(mb["next_observations"]))
        assert torch.equal(q[:, 1], q[:, 2]) and (q.argmax(1) == 1).all()
    B = len(mb["rewards"])
    e = algo._ensure_engine(1, B)
    trainable, targets, lins = algo._learner_nets()
    algo._upload_state(e, trainable, targets, lins)
    out = e.train(algo._hparams(False, 1), mb["observations"][None], mb["actions"][None], mb["rewards"][None],
                  mb["next_observations"][None], mb["dones"].astype(np.float32)[None])
    blob, steps = e.get_state()
    layout, _ = e.state_layout()
    assert [(k, i) for k, i, _, _ in layout] == [("params", 1), ("params", 4), ("m", 1), ("v", 1)]
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


# ---- execution paths -------------------------------------------------------------------------------------------------
def _run_paths(double_q, path, graph, calls=2, S=5, B=48):
    os.environ["B200RL_OFFPOLICY_GRAPH"] = "1" if graph else "0"
    try:
        algo = build(O=6, n=5, N=21, v=(-4.0, 4.0), double_q=double_q, target_update_interval=3, steps=1)
        fill(algo.replay_buffer, 6, 5, rows=2000, seed=3)
        algo.use_device_replay = path != "host"
        algo.use_device_rng, algo.device_rng_seed = path == "rng", 9
        outs = []
        for call in range(calls):
            np.random.seed(30 + call)
            algo.train(algo.replay_buffer, S + (call == calls - 1), B)
            outs.append(algo.last_train_output)
        return outs, [flat(algo.q_function.network), flat(algo.target_q_function.network),
                      adam_flat(algo.q_function.optimizer, "exp_avg")[0]]
    finally:
        os.environ.pop("B200RL_OFFPOLICY_GRAPH", None)


def _assert_same(got, ref, what):
    (outs, nets), (ref_outs, ref_nets) = got, ref
    for a, b in zip(outs, ref_outs):
        assert a.keys() == b.keys() == {"q1_values", "q1_losses"}
        for k in a:
            np.testing.assert_array_equal(a[k], b[k], err_msg=f"{k} {what}")
    for i, (a, b) in enumerate(zip(nets, ref_nets)):
        np.testing.assert_array_equal(a, b, err_msg=f"net {i} {what}")


@pytest.mark.parametrize("double_q", [False, True])
def test_host_staged_device_gather_and_graph_paths_are_bit_identical(double_q):
    ref = _run_paths(double_q, "host", False)
    for path, graph in (("gather", True), ("host", True), ("gather", False)):
        _assert_same(_run_paths(double_q, path, graph), ref, f"{path} graph={graph}")
    _assert_same(_run_paths(double_q, "rng", True), _run_paths(double_q, "rng", False), "rng")


def test_device_side_draws_replay_through_the_oracle():
    S, B = 6, 64
    algo = build(double_q=True, target_update_interval=4, steps=2)
    fill(algo.replay_buffer, 8, 4, seed=4)
    algo.use_device_rng, algo.device_rng_seed = True, 77
    oracle = oracle_for(algo)
    algo.train(algo.replay_buffer, S, B)
    idx, noise = algo._engine.get_draws(S, B)
    assert idx.shape == (S, B) and noise is None
    rb = algo.replay_buffer
    logs = oracle.train([{k: rb._cols[k][idx[s]] for k in rb.COLUMNS} for s in range(S)])
    errs = compare(algo, oracle)
    errs["q1_values"] = rel_err(algo.last_train_output["q1_values"], np.stack(logs["q1_values"]))
    for k, v in errs.items():
        assert v < 2e-5, (k, v, errs)


# ---- learner groups ----------------------------------------------------------------------------------------------------
def _member(seed, steps, path):
    algo = build(O=6, n=5, N=21, v=(-4.0, 4.0), seed=seed, steps=steps, double_q=True, target_update_interval=3)
    fill(algo.replay_buffer, 6, 5, rows=1500, seed=40 + seed)
    algo.use_device_replay = path != "host"
    algo.use_device_rng, algo.device_rng_seed = path == "rng", 1000 + seed
    return algo


def _state(algo):
    return [flat(algo.q_function.network), flat(algo.target_q_function.network),
            *[adam_flat(algo.q_function.optimizer, k)[0] for k in ("exp_avg", "exp_avg_sq")]]


@pytest.mark.parametrize("path", ["host", "gather", "rng"])
def test_group_of_three_is_bit_identical_to_solo_engines(path):
    """Members at Q step counts 0, 7 and 100 (interval 3: they copy on different steps), two calls."""
    from rl_replicas_b200.algorithms import LearnerGroup
    S, B, starts = 5, 40, (0, 7, 100)
    solo = [_member(k, st, path) for k, st in enumerate(starts)]
    grouped = [_member(k, st, path) for k, st in enumerate(starts)]
    g = LearnerGroup()
    for k, m in enumerate(grouped):
        np.random.seed(50 + k)
        torch.manual_seed(50 + k)
        g.add(m)
    for call in range(2):
        for k, m in enumerate(solo):
            np.random.seed(50 + k) if call == 0 else np.random.set_state(m._np_state)
            m.train(m.replay_buffer, S, B)
            m._np_state = np.random.get_state()
        g.train(S, B)
        for k, (a, b) in enumerate(zip(solo, grouped)):
            for key in ("q1_values", "q1_losses"):
                np.testing.assert_array_equal(a.last_train_output[key], b.last_train_output[key], err_msg=f"{key} {k}")
            for i, (x, y) in enumerate(zip(_state(a), _state(b))):
                np.testing.assert_array_equal(x, y, err_msg=f"member {k} tensor {i} call {call}")


def test_group_of_sixteen_is_bit_identical_to_solo_engines():
    from rl_replicas_b200.algorithms import LearnerGroup
    S, B = 4, 32
    solo = [_member(k, 3 * k, "gather") for k in range(16)]
    grouped = [_member(k, 3 * k, "gather") for k in range(16)]
    g = LearnerGroup()
    for k, m in enumerate(grouped):
        np.random.seed(70 + k)
        g.add(m)
    g.train(S, B)
    for k, m in enumerate(solo):
        np.random.seed(70 + k)
        m.train(m.replay_buffer, S, B)
        for i, (x, y) in enumerate(zip(_state(m), _state(grouped[k]))):
            np.testing.assert_array_equal(x, y, err_msg=f"member {k} tensor {i}")
        for key in ("q1_values", "q1_losses"):
            np.testing.assert_array_equal(m.last_train_output[key], grouped[k].last_train_output[key])


# ---- refusals, launches and end to end --------------------------------------------------------------------------------
@pytest.mark.parametrize("bad", [4.0, 1.5, -1.0, float("nan")])
def test_invalid_action_raises_and_leaves_the_host_modules_unchanged(bad):
    from rl_replicas_b200._lib import B200RLError
    algo = build(O=6, n=4, N=11, target_update_interval=2)
    fill(algo.replay_buffer, 6, 4, rows=64, seed=5, bad_action=bad)
    before = [flat(algo.q_function.network), flat(algo.target_q_function.network)]
    np.random.seed(0)
    with pytest.raises(B200RLError, match=r"C51 learner 0, step \d+: \d+ minibatch rows hold an action that is not "
                                          r"an integer in \[0, 4\)"):
        algo.train(algo.replay_buffer, 8, 64)  # 512 draws of 64 rows: the bad row is drawn
    for x, y in zip(before, [flat(algo.q_function.network), flat(algo.target_q_function.network)]):
        np.testing.assert_array_equal(x, y)
    assert algo._adam_step_count(algo.q_function.optimizer, list(algo.q_function.network.network)[::2]) == 0


def test_engine_refuses_bad_c51_configurations():
    from rl_replicas_b200._lib import B200RLError, OffPolicyHparams
    from rl_replicas_b200.engine import OffPolicyEngine
    dqn = OffPolicyEngine(None, [4, 16, 2], 1, 8, 2, algo=OffPolicyEngine.DQN)
    td3 = OffPolicyEngine([4, 16, 2], [6, 16, 1], 2, 8, 2)
    for e in (dqn, td3):
        with pytest.raises(B200RLError, match="algo = 3"):
            e.set_c51(51, -10.0, 10.0)
    with pytest.raises(B200RLError, match="algo must be"):
        OffPolicyEngine(None, [4, 16, 2], 1, 8, 2, algo=4)
    e = OffPolicyEngine(None, [4, 16, 3 * 11], 1, 8, 2, algo=OffPolicyEngine.C51)
    e.set_dqn(10, False)
    z = lambda *s: np.zeros(s, np.float32)
    with pytest.raises(B200RLError, match="set_c51"):
        e.train(OffPolicyHparams(), z(2, 8, 4), z(2, 8), z(2, 8), z(2, 8, 4), z(2, 8))
    for args, msg in (((1, -1.0, 1.0), "n_atoms must be 2"), ((257, -1.0, 1.0), "n_atoms must be 2"),
                      ((11, 1.0, 1.0), "v_min < v_max"), ((11, 0.0, float("inf")), "v_min < v_max"),
                      ((11, float("nan"), 1.0), "v_min < v_max"), ((10, -1.0, 1.0), "output width 33")):
        with pytest.raises(B200RLError, match=msg):
            e.set_c51(*args)
    e.set_c51(11, -1.0, 1.0)
    with pytest.raises(B200RLError, match="not implemented for C51"):
        e.set_per(0.6, 1e-6, 0.4, 100)
    cols = [torch.zeros(16, 4, device="cuda"), torch.zeros(16, device="cuda"), torch.zeros(16, device="cuda"),
            torch.zeros(16, 4, device="cuda"), torch.zeros(16, device="cuda")]
    tree = torch.zeros(int(e.lib.b200rl_per_tree_floats(16)), device="cuda")
    with pytest.raises(B200RLError, match="not implemented for C51"):
        e.train_prioritized(OffPolicyHparams(), cols, 16, tree, 2, 8, 0, 1)
    g = OffPolicyEngine(None, [4, 16, 3 * 11], 1, 8, 2, algo=OffPolicyEngine.C51, n_learners=2)
    g.set_dqn(10, False)
    g.set_c51(11, -1.0, 1.0)
    with pytest.raises(B200RLError, match="not implemented for C51"):
        g.train_prioritized_group(OffPolicyHparams(), [(cols, 16), (cols, 16)], [tree, tree.clone()], 2, 8, [0, 0],
                                  [1, 1])


def test_launches_per_step_at_most_one_more_than_dqn():
    from rl_replicas_b200 import _lib
    from test_gpu_dqn import build as build_dqn
    lib = _lib.load()
    S, B = 6, 64

    def launches(algo, graph):
        os.environ["B200RL_OFFPOLICY_GRAPH"] = "1" if graph else "0"
        try:
            fill(algo.replay_buffer, 8, 4, rows=1000, seed=6)
            algo.train(algo.replay_buffer, S, B)  # builds the engine (and the graph)
            n0 = lib.b200rl_launch_count()
            algo.train(algo.replay_buffer, S, B)
            return lib.b200rl_launch_count() - n0
        finally:
            os.environ.pop("B200RL_OFFPOLICY_GRAPH", None)
    for double_q in (False, True):
        for graph in (False, True):
            d = launches(build_dqn(double_q=double_q, target_update_interval=3), graph)
            c = launches(build(double_q=double_q, target_update_interval=3), graph)
            print(f"double_q={double_q} graph={graph}: DQN {d}, C51 {c} launches per call of {S} steps")
            assert c <= d + S, (c, d)


def test_learn_solves_the_choice_task(tmp_path, capsys):
    """C51.learn end to end on tests/test_dqn.py's one-step choice task with the seeds of the oracle-driven loop in
    tests/test_c51.py: DQN's tags are recorded, model.pt is written and reloads, and the evaluation return clears the
    same bar."""
    np.random.seed(0)
    algo = make_c51(**C51_KW)
    algo.learn(output_dir=str(tmp_path), **LEARN)
    after = evaluation_return(algo)
    printed = capsys.readouterr().out
    with capsys.disabled():
        print(f"C51.learn on the choice task: evaluation return {after:.3f}")
    for tag in ("q-function/average_loss", "q-function/avarage_q-value", "exploration/epsilon",
                "evaluation/average_episode_return"):
        assert f"\n{tag}: " in printed, tag
    path = os.path.join(tmp_path, "model.pt")
    assert os.path.exists(path)
    other = make_c51(seed=5, **C51_KW)
    other.load_model(path)
    assert evaluation_return(other) == after  # the reloaded networks act exactly as the trained ones
    assert after > RETURN_BAR
