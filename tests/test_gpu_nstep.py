"""GPU: n-step returns for DQN / C51 -- DQN.train against the float32 oracle fed oracle/nstep.py's minibatches, the
device's windows bit for bit equal to the float32 walk (gather, device-draw and prioritized paths, on wrapped rings), one
step against the float64 reference, C51 and prioritized DQN at n = 3, bit-identical execution paths and learner groups,
n = 5 equal to n = 1 where every row ends an episode, the engine's refusals and launch budget, and DQN.learn(n_step=3)
end to end on tests/test_nstep.py's delayed-reward task."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from conftest import rel_err
from oracle import dqn as OD
from oracle import nstep as ON
from oracle import per as OP
from test_gpu_dqn import BAR_GRAD_ENTRY, BAR_GRAD_NORM, BAR_LOSS, BAR_Q, KINK, NEAR_TIE, adam_flat, build, compare, flat
from test_nstep import LEARN, NSTEP_KW, RETURN_BAR, evaluation_return, make_nstep_dqn, nested

pytestmark = pytest.mark.gpu


def fill_episodes(rb, O, rows, seed, max_len=12, done_p=0.5):
    """Appends of a few episodes each (done or cut, some shorter than n) until ``rows`` rows went in."""
    rng = np.random.default_rng(seed)
    k = 0
    while rows > 0:
        eps = [(int(rng.integers(1, max_len + 1)), bool(rng.random() < done_p)) for _ in range(int(rng.integers(1, 5)))]
        e = nested(eps, O=O, seed=10000 * seed + k)
        rb.add_experience(e)
        rows -= sum(L for L, _ in eps)
        k += 1


def ring(algo, O=8, size=300, rows=700, seed=1, **kw):
    """A small ring (``size`` rows) that has wrapped several times."""
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    algo.replay_buffer = ReplayBuffer(buffer_size=size)
    fill_episodes(algo.replay_buffer, O, rows, seed, **kw)
    assert algo.replay_buffer._head > 0
    return algo


def check_walk(algo, idx, S, B):
    """get_nstep_draws equals the float32 walk from the start rows idx [S, B], bit for bit."""
    rb = algo.replay_buffer
    last, R, g = algo._engine.get_nstep_draws(S, B)
    want = ON.walk_f32(rb._cols["rewards"].astype(np.float32), rb._cols["dones"], rb._ends, idx, algo.n_step, algo.gamma)
    for got, exp, what in zip((last, R, g), want, ("last rows", "returns", "discounts")):
        np.testing.assert_array_equal(got, exp, err_msg=what)
    return last


def nstep_oracle(algo, cls=ON.NStepDqnOracle, **kw):
    return cls(algo.q_function.network, algo.target_q_function.network, algo.q_function.optimizer, gamma=algo.gamma,
               target_update_interval=algo.target_update_interval, double_q=algo.double_q, **kw)


@pytest.mark.parametrize("path", ["gather", "rng"])
@pytest.mark.parametrize("double_q", [False, True])
@pytest.mark.parametrize("n", [3, 32])
def test_train_matches_the_oracle_and_the_walk_is_exact(n, double_q, path):
    """Three DQN.train calls of 4 steps at interval 3 on a wrapped ring: the float32 oracle fed the n-step minibatches
    at the replayed rows, and the device's windows equal to the float32 walk bit for bit."""
    S, B = 4, 64
    algo = ring(build(double_q=double_q, steps=3, target_update_interval=3, n_step=n), seed=n)
    algo.use_device_rng, algo.device_rng_seed = path == "rng", 5
    oracle = nstep_oracle(algo)
    rb = algo.replay_buffer
    for call in range(3):
        np.random.seed(20 + call)
        algo.train(rb, S, B)
        if path == "rng":
            idx, _ = algo._engine.get_draws(S, B)
        else:
            np.random.seed(20 + call)
            idx = rb.physical_rows(np.stack([rb.sample_indices(B) for _ in range(S)]))
        last = check_walk(algo, idx, S, B)
        assert (last != idx).any()
        logs = oracle.train([ON.nstep_minibatch(rb, idx[s], n, algo.gamma) for s in range(S)])
        errs = compare(algo, oracle)
        out = algo.last_train_output
        errs["q1_values"] = rel_err(out["q1_values"], np.stack(logs["q1_values"]))
        errs["q1_losses"] = rel_err(out["q1_losses"], np.asarray(logs["q1_losses"]))
        print(f"n={n} double_q={double_q} {path} call {call}:", {k: f"{v:.1e}" for k, v in errs.items()})
        for k, v in errs.items():
            assert v < 2e-5, (call, k, v, errs)


# ---- one step against the float64 reference ------------------------------------------------------------------------
F64_CASES = {"lunar": ([8, 256, 256, 4], 256, True), "n33": ([6, 64, 64, 33], 33, False),
             "two_layer": ([7, 48, 5], 64, True)}


@pytest.mark.parametrize("n", [2, 5, 32])
@pytest.mark.parametrize("name", list(F64_CASES))
def test_one_step_against_the_float64_reference(name, n):
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    sizes, B, double_q = F64_CASES[name]
    algo = build(O=sizes[0], n=sizes[-1], hidden=tuple(sizes[1:-1]), double_q=double_q, target_update_interval=1000,
                 n_step=n)
    rb = algo.replay_buffer = ReplayBuffer(buffer_size=100000)
    fill_episodes(rb, sizes[0], 4 * B + 64, seed=200 + n, max_len=40, done_p=0.3)
    q_flat, t_flat = flat(algo.q_function.network).astype(np.float64), flat(algo.target_q_function.network).astype(np.float64)
    pool = rb.physical_rows(np.arange(rb.current_size))
    f64 = lambda mb: OD.dqn_step_f64(q_flat, t_flat, mb, sizes, "relu", torch.as_tensor(mb["discounts"], dtype=torch.float64),
                                     double_q)
    ref = f64(ON.nstep_minibatch(rb, pool, n, algo.gamma))
    qmax = np.max(np.abs(ref["q_values"])) + 1.0
    keep = (ref["margin"] >= KINK) & (np.abs(np.abs(ref["delta"]) - 1.0) > 1e-4) & (ref["gap"] > NEAR_TIE * qmax)
    idx = pool[np.flatnonzero(keep)[:B]]
    assert len(idx) == B, (name, int(keep.sum()))
    mb = ON.nstep_minibatch(rb, idx, n, algo.gamma)
    assert (mb["discounts"] < np.float32(algo.gamma)).any()
    ref = f64(mb)
    e = algo._ensure_engine(1, B)
    trainable, targets, lins = algo._learner_nets()
    algo._upload_state(e, trainable, targets, lins)
    e.set_nstep(n, [rb.device_episode_ends()])
    cols, rows = rb.device_columns()
    out = e.train_gather(algo._hparams(False, 1), cols, rows, idx[None])
    blob, steps = e.get_state()
    layout, _ = e.state_layout()
    m = next(blob[o:o + c] for k, i, o, c in layout if k == "m")
    grad = m.astype(np.float64) / 0.1
    g_err = float(np.max(np.abs(grad - ref["grad"]) / np.maximum(ref["scale"], 1e-30)))
    g_norm = rel_err(grad, ref["grad"])
    q_err = rel_err(out["q1_values"][0], ref["q_values"])
    l_err = abs(float(out["q1_losses"][0]) - ref["loss"]) / max(abs(ref["loss"]), 1e-30)
    print(f"{name} n={n}: grad {g_norm:.2e} (entry / scale {g_err:.2e})  q {q_err:.2e}  loss {l_err:.2e}")
    assert g_norm < BAR_GRAD_NORM and g_err < BAR_GRAD_ENTRY and q_err < BAR_Q and l_err < BAR_LOSS, \
        (g_norm, g_err, q_err, l_err)


# ---- C51 and prioritized replay at n = 3 -----------------------------------------------------------------------------
def test_c51_matches_the_oracle():
    from test_gpu_c51 import build as build_c51
    S, B = 4, 64
    algo = ring(build_c51(steps=7, double_q=True, target_update_interval=3, n_step=3), seed=7)
    q = algo.q_function
    oracle = nstep_oracle(algo, ON.NStepC51Oracle, n_atoms=q.n_atoms, v_min=q.v_min, v_max=q.v_max)
    rb = algo.replay_buffer
    for call in range(2):
        np.random.seed(40 + call)
        algo.train(rb, S, B)
        np.random.seed(40 + call)
        idx = rb.physical_rows(np.stack([rb.sample_indices(B) for _ in range(S)]))
        check_walk(algo, idx, S, B)
        logs = oracle.train([ON.nstep_minibatch(rb, idx[s], 3, algo.gamma) for s in range(S)])
        errs = compare(algo, oracle)
        errs["q1_values"] = rel_err(algo.last_train_output["q1_values"], np.stack(logs["q1_values"]))
        errs["q1_losses"] = rel_err(algo.last_train_output["q1_losses"], np.asarray(logs["q1_losses"]))
        print(f"C51 n=3 call {call}:", {k: f"{v:.1e}" for k, v in errs.items()})
        for k, v in errs.items():
            assert v < 2e-5, (call, k, v, errs)


def per_nstep(n=3, size=700, rows=1500, seed=9, **kw):
    from rl_replicas_b200.replay_buffer import PrioritizedReplayBuffer
    algo = build(n_step=n, **kw)
    algo.replay_buffer = PrioritizedReplayBuffer(size, alpha=0.6, beta_start=0.4, beta_anneal_steps=50, eps=1e-6)
    fill_episodes(algo.replay_buffer, 8, rows, seed)
    algo.device_rng_seed = seed
    return algo


@pytest.mark.parametrize("double_q", [False, True])
def test_prioritized_draws_weights_and_priorities_match_the_oracle(double_q):
    S, B = 3, 64
    algo = per_nstep(double_q=double_q, steps=2, target_update_interval=4)
    rb = algo.replay_buffer
    assert rb._head > 0
    oracle = nstep_oracle(algo, ON.NStepPerDqnOracle, alpha=rb.alpha, eps=rb.eps)
    for call in range(2):
        leaves = rb.priorities().astype(np.float32)
        t0 = algo._adam_step_count(algo.q_function.optimizer, list(algo.q_function.network.network)[::2])
        algo.train(rb, S, B)
        idx, w, newp = algo._engine.get_per_draws(S, B)
        check_walk(algo, idx, S, B)
        mbs, ps, betas = [], [], []
        for st in range(S):
            want, dist = OP.stratified_draw(leaves, algo.device_rng_seed, algo._device_rng_calls, st, B)
            far = dist > 2e-6
            assert (want[far] == idx[st][far]).all()
            mbs.append(ON.nstep_minibatch(rb, idx[st], 3, algo.gamma))
            ps.append(leaves[idx[st]])
            betas.append(float(OP.beta_schedule(t0 + st, rb.beta_start, rb.beta_anneal_steps)))
            leaves = OP.apply_priorities(leaves, idx[st], newp[st]).astype(np.float32)
        np.testing.assert_array_equal(rb.priorities(), leaves)
        logs = oracle.train(mbs, ps, betas)
        errs = compare(algo, oracle)
        errs["q1_values"] = rel_err(algo.last_train_output["q1_values"], np.stack(logs["q1_values"]))
        w_err = float(np.max(np.abs(w - np.stack(logs["weights"])) / np.stack(logs["weights"])))
        p_ref = np.stack(logs["priorities"])
        p_err = float(np.max(np.abs(newp - p_ref) / p_ref))
        print(f"PER n=3 double_q={double_q} call {call}:", {k: f"{v:.1e}" for k, v in errs.items()},
              f"weights {w_err:.1e} priorities {p_err:.1e}")
        for k, v in errs.items():
            assert v < 2e-5, (call, k, v)
        assert w_err < 1e-6 and p_err < 1e-4, (w_err, p_err)


# ---- bit identity ----------------------------------------------------------------------------------------------------
def _outputs_and_state(algo):
    return [algo.last_train_output[k] for k in ("q1_values", "q1_losses")] + [
        flat(algo.q_function.network), flat(algo.target_q_function.network),
        *[adam_flat(algo.q_function.optimizer, k)[0] for k in ("exp_avg", "exp_avg_sq")]]


def _run(make, graph, calls=2, S=5, B=48):
    os.environ["B200RL_OFFPOLICY_GRAPH"] = "1" if graph else "0"
    try:
        algo = make()
        res = []
        for call in range(calls):
            np.random.seed(30 + call)
            algo.train(algo.replay_buffer, S + (call == calls - 1), B)
            res.append(_outputs_and_state(algo))
        return res
    finally:
        os.environ.pop("B200RL_OFFPOLICY_GRAPH", None)


def _assert_runs_equal(a, b, what):
    for call, (x, y) in enumerate(zip(a, b)):
        for i, (u, v) in enumerate(zip(x, y)):
            np.testing.assert_array_equal(u, v, err_msg=f"{what}: call {call} tensor {i}")


@pytest.mark.parametrize("path", ["gather", "rng", "per"])
def test_graph_and_plain_launches_are_bit_identical(path):
    def make():
        if path == "per":
            return per_nstep(double_q=True, steps=1, target_update_interval=3)
        algo = ring(build(O=6, n=5, double_q=True, target_update_interval=3, steps=1, n_step=3), O=6, seed=3)
        algo.use_device_rng = path == "rng"
        return algo
    _assert_runs_equal(_run(make, True), _run(make, False), path)


def _member(seed, steps, path, n=3):
    algo = ring(build(O=6, n=5, seed=seed, steps=steps, double_q=True, target_update_interval=3, n_step=n), O=6,
                seed=40 + seed)
    algo.use_device_rng, algo.device_rng_seed = path == "rng", 1000 + seed
    return algo


@pytest.mark.parametrize("K,path", [(3, "gather"), (3, "rng"), (16, "gather")])
def test_group_is_bit_identical_to_solo_engines(K, path):
    from rl_replicas_b200.algorithms import LearnerGroup
    S, B = 4, 32
    solo = [_member(k, 3 * k, path) for k in range(K)]
    grouped = [_member(k, 3 * k, path) for k in range(K)]
    g = LearnerGroup()
    for k, m in enumerate(grouped):
        np.random.seed(70 + k)
        g.add(m)
    g.train(S, B)
    for k, m in enumerate(solo):
        np.random.seed(70 + k)
        m.train(m.replay_buffer, S, B)
        _assert_runs_equal([_outputs_and_state(m)], [_outputs_and_state(grouped[k])], f"member {k}")
        np.testing.assert_array_equal(m._engine.get_nstep_draws(S, B)[1], g._engine.get_nstep_draws(S, B)[1][k])


@pytest.mark.parametrize("kind", ["dqn", "c51", "per"])
def test_n5_equals_n1_where_every_row_ends_an_episode(kind):
    """Every append holds one-row episodes: every window stops at its start row, so n = 5 is the one-step update."""
    from test_gpu_c51 import build as build_c51
    from rl_replicas_b200.replay_buffer import PrioritizedReplayBuffer, ReplayBuffer

    def make(n):
        def f():
            if kind == "c51":
                algo = build_c51(steps=3, double_q=True, target_update_interval=3, n_step=n)
            else:
                algo = build(O=8, n=4, steps=3, double_q=True, target_update_interval=3, n_step=n)
            algo.replay_buffer = PrioritizedReplayBuffer(400) if kind == "per" else ReplayBuffer(400)
            fill_episodes(algo.replay_buffer, 8, 900, seed=11, max_len=1, done_p=0.3)
            assert all(algo.replay_buffer.episode_ends)
            return algo
        return f
    _assert_runs_equal(_run(make(5), True), _run(make(1), True), kind)


# ---- refusals, launches and end to end -------------------------------------------------------------------------------
def test_engine_refusals():
    from rl_replicas_b200._lib import B200RLError
    from rl_replicas_b200.engine import OffPolicyEngine
    td3 = OffPolicyEngine([3, 16, 2], [5, 16, 1], 2, 8, 2)
    with pytest.raises(B200RLError, match="DQN and C51 engines"):
        td3.set_nstep(1)
    algo = ring(build(n_step=3), seed=2)
    algo.train(algo.replay_buffer, 2, 16)
    e = algo._engine
    cols = (C.c_void_p * 1)(algo.replay_buffer.device_episode_ends().data_ptr())
    for bad in (0, 33):
        with pytest.raises(B200RLError, match="n_step must be 1..32"):
            _lib_set_nstep(e, bad, cols)
    with pytest.raises(B200RLError, match="needs the episode-end columns"):
        _lib_set_nstep(e, 3, None)
    with pytest.raises(ValueError, match="episode-end columns"):
        e.set_nstep(3, None)
    e.set_nstep(3, [algo.replay_buffer.device_episode_ends()])
    z = lambda *s: np.zeros(s, np.float32)
    with pytest.raises(B200RLError, match="need the device replay columns"):
        e.train(algo._hparams(False, 1), z(2, 16, 8), z(2, 16), z(2, 16), z(2, 16, 8), z(2, 16))
    algo.n_step = 1
    algo.train(algo.replay_buffer, 2, 16)
    with pytest.raises(B200RLError, match="not an n-step one"):
        e.get_nstep_draws(2, 16)


def _lib_set_nstep(e, n, ptrs):
    from rl_replicas_b200._lib import check
    check(e.lib.b200rl_offpolicy_set_nstep(e.h, n, ptrs), "set_nstep")


def test_launches_per_call_are_at_most_those_of_one_step():
    from rl_replicas_b200 import _lib
    lib = _lib.load()
    S, B = 6, 64

    def launches(make, graph):
        os.environ["B200RL_OFFPOLICY_GRAPH"] = "1" if graph else "0"
        try:
            algo = make()
            algo.train(algo.replay_buffer, S, B)  # builds the engine (and the graph)
            n0 = lib.b200rl_launch_count()
            algo.train(algo.replay_buffer, S, B)
            return lib.b200rl_launch_count() - n0
        finally:
            os.environ.pop("B200RL_OFFPOLICY_GRAPH", None)
    for path in ("gather", "rng", "per"):
        for graph in (False, True):
            def make(n):
                if path == "per":
                    return lambda: per_nstep(n=n, double_q=True)
                def f():
                    a = ring(build(double_q=True, n_step=n), seed=4)
                    a.use_device_rng = path == "rng"
                    return a
                return f
            one, three = launches(make(1), graph), launches(make(3), graph)
            print(f"{path} graph={graph}: n=1 {one}, n=3 {three} launches per call of {S} steps")
            assert three <= one, (path, graph, one, three)


def test_learn_solves_the_delayed_reward_task(tmp_path, capsys):
    """DQN.learn(n_step=3) end to end with the seeds of tests/test_nstep.py's oracle-driven loop."""
    np.random.seed(0)
    algo = make_nstep_dqn(**NSTEP_KW)
    algo.learn(output_dir=str(tmp_path), **LEARN)
    after = evaluation_return(algo)
    printed = capsys.readouterr().out
    with capsys.disabled():
        print(f"DQN.learn(n_step=3) on the delayed-reward task: evaluation return {after:.3f}")
    for tag in ("q-function/average_loss", "q-function/avarage_q-value", "exploration/epsilon",
                "evaluation/average_episode_return"):
        assert f"\n{tag}: " in printed, tag
    path = os.path.join(tmp_path, "model.pt")
    other = make_nstep_dqn(seed=5, **NSTEP_KW)
    other.load_model(path)
    assert evaluation_return(other) == after
    assert after > RETURN_BAR


def test_group_learn_matches_solo_learn(tmp_path):
    from rl_replicas_b200.algorithms import LearnerGroup
    from rl_replicas_b200.utils import set_seed_for_libraries
    kw = dict(LEARN, num_epochs=14)
    solo = []
    for seed in (0, 1):
        set_seed_for_libraries(seed)
        a = make_nstep_dqn(seed=seed, **NSTEP_KW)
        a.learn(output_dir=str(tmp_path / f"solo{seed}"), **kw)
        solo.append(a)
    g = LearnerGroup()
    for seed in (0, 1):
        set_seed_for_libraries(seed)
        g.add(make_nstep_dqn(seed=seed, **NSTEP_KW))
    g.learn([str(tmp_path / f"group{s}") for s in (0, 1)], **kw)
    for a, b in zip(solo, g.members):
        np.testing.assert_array_equal(flat(a.q_function.network), flat(b.q_function.network))
        np.testing.assert_array_equal(flat(a.target_q_function.network), flat(b.target_q_function.network))
