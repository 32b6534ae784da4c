"""GPU: prioritized experience replay for DQN -- the sum tree's builds and range sets, the device draws reproduced
through the oracle's Philox and float64 tree (oracle/per.py), the weighted update against PerDqnOracle on the engine's
indices (duplicates included), bit-identity with the unweighted DQN step at alpha = 0 and beta = 1, bit-identical
execution paths and learner groups, the non-finite refusal, DQN.learn end to end, and the launch budget."""
import os

import numpy as np
import pytest
import torch

from conftest import rel_err
from oracle import per as OP
from test_dqn import DQN_KW, LEARN, RETURN_BAR, evaluation_return, make_dqn
from test_gpu_dqn import adam_flat, build, compare, fill, flat

pytestmark = pytest.mark.gpu


def per_build(rows_capacity=8000, alpha=0.6, beta_start=0.4, beta_anneal_steps=50, eps=1e-6, **kw):
    from rl_replicas_b200.replay_buffer import PrioritizedReplayBuffer
    algo = build(**kw)
    algo.replay_buffer = PrioritizedReplayBuffer(rows_capacity, alpha=alpha, beta_start=beta_start,
                                                 beta_anneal_steps=beta_anneal_steps, eps=eps)
    return algo


def per_oracle(algo):
    rb = algo.replay_buffer
    return OP.PerDqnOracle(algo.q_function.network, algo.target_q_function.network, algo.q_function.optimizer,
                           gamma=algo.gamma, target_update_interval=algo.target_update_interval, double_q=algo.double_q,
                           alpha=rb.alpha, eps=rb.eps)


# ---- the tree --------------------------------------------------------------------------------------------------------
def _check_tree(tree, n):
    t = tree.double().cpu().numpy()
    offs, total = OP.tree_offsets(n)
    assert len(t) == total and np.isfinite(t).all()
    for k in range(1, len(offs)):
        cnt = -(-(offs[k] - offs[k - 1]) // 32) if k < len(offs) - 1 else 1
        child = t[offs[k - 1]:offs[k - 1] + 32 * cnt].reshape(-1, 32).sum(1)
        got = t[offs[k]:offs[k] + cnt]
        np.testing.assert_allclose(got, child, rtol=1e-6, atol=0, err_msg=f"n={n} level {k}")
    return t, offs


@pytest.mark.parametrize("n", [1, 31, 32, 33, 1025, 2 ** 20 + 1])
def test_tree_build_and_range_set(n):
    from rl_replicas_b200 import _lib
    from rl_replicas_b200.engine import current_stream_handle
    import ctypes as C
    lib = _lib.load()
    total = int(lib.b200rl_per_tree_floats(n))
    tree = torch.zeros(total, dtype=torch.float32, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(n)
    tree[:n] = torch.rand(n, device="cuda", generator=g) * 3.0
    tree[total - 31] = 2.5  # the running max
    ptr = C.c_void_p(tree.data_ptr())
    _lib.check(lib.b200rl_per_tree_build(ptr, n, current_stream_handle()), "build")
    _check_tree(tree, n)
    start, count = max(n - 7, 0), min(n, 20)  # wraps past the end when n > 7
    before = tree[:n].cpu().numpy()
    _lib.check(lib.b200rl_per_tree_set_range(ptr, n, start, count, current_stream_handle()), "set_range")
    t, offs = _check_tree(tree, n)
    rows = (start + np.arange(count)) % n
    want = before.copy()
    want[rows] = 2.5
    np.testing.assert_array_equal(t[:n].astype(np.float32), want)
    assert t[offs[-1] + 1] == 2.5


# ---- draws and update against the oracle -----------------------------------------------------------------------------
def _replay_calls(algo, calls, S, B, oracle=None, tol=2e-6):
    """Runs `calls` train() calls and replays every step through oracle/per.py; returns (exempt draws, total draws)."""
    rb = algo.replay_buffer
    exempt = total = 0
    for call in range(calls):
        leaves = rb.priorities().astype(np.float32)
        t0 = algo._adam_step_count(algo.q_function.optimizer, list(algo.q_function.network.network)[::2])
        algo.train(rb, S, B)
        idx, w, newp = algo._engine.get_per_draws(S, B)
        seed, ncall = algo.device_rng_seed, algo._device_rng_calls
        mbs, ps, betas = [], [], []
        for st in range(S):
            want, dist = OP.stratified_draw(leaves, seed, ncall, st, B)
            far = dist > tol
            exempt += int((~far).sum())
            total += B
            assert (want[far] == idx[st][far]).all(), (call, st, np.flatnonzero(far & (want != idx[st])))
            assert (leaves[idx[st]] > 0).all()  # a zero-priority leaf is never drawn
            mbs.append({k: rb._cols[k][idx[st]] for k in rb.COLUMNS})
            ps.append(leaves[idx[st]])
            betas.append(float(OP.beta_schedule(t0 + st, rb.beta_start, rb.beta_anneal_steps)))
            leaves = OP.apply_priorities(leaves, idx[st], newp[st]).astype(np.float32)
        np.testing.assert_array_equal(rb.priorities(), leaves)  # last occurrence wins, exactly
        if oracle is not None:
            logs = oracle.train(mbs, ps, betas)
            errs = compare(algo, oracle)
            out = algo.last_train_output
            errs["q1_values"] = rel_err(out["q1_values"], np.stack(logs["q1_values"]))
            errs["q1_losses"] = rel_err(out["q1_losses"], np.asarray(logs["q1_losses"]))
            w_err = float(np.max(np.abs(w - np.stack(logs["weights"])) / np.stack(logs["weights"])))
            p_ref = np.stack(logs["priorities"])
            p_err = float(np.max(np.abs(newp - p_ref) / p_ref))
            # |delta| itself against the oracle's, in units of the largest Q-value: delta = Q - y cancels, so its
            # relative error is not bounded; the priority is a function of it
            d_err = float(np.max(np.abs(np.abs(np.stack(logs["delta"])) - (newp.astype(np.float64) ** (1 / rb.alpha)
                                                                             - rb.eps))) / np.max(np.abs(p_ref)))
            print(f"call {call}:", {k: f"{v:.1e}" for k, v in errs.items()}, f"weights {w_err:.1e} priorities "
                  f"{p_err:.1e} |delta| {d_err:.1e}")
            for k, v in errs.items():
                assert v < 2e-5, (call, k, v)
            assert w_err < 1e-6, w_err
            assert p_err < 1e-6 and d_err < 2e-5, (p_err, d_err)
    return exempt, total


@pytest.mark.parametrize("double_q", [False, True])
def test_draws_and_update_match_the_oracle(double_q):
    """3 calls of 4 steps on a half-full buffer (zero-priority leaves), target copies inside and across calls."""
    algo = per_build(double_q=double_q, steps=3, target_update_interval=3)
    fill(algo.replay_buffer, 8, 4, rows=4000, seed=11)
    algo.device_rng_seed = 91
    exempt, total = _replay_calls(algo, 3, 4, 64, per_oracle(algo))
    print(f"draws within float tolerance of a boundary: {exempt} of {total}")
    # the band of 2e-6 M on either side of the ~4000 live leaves' boundaries covers about 1.6 % of [0, M)
    assert exempt <= 0.03 * total


@pytest.mark.parametrize("B", [256, 600])
def test_duplicate_draws_resolve_to_the_last_occurrence(B):
    """5 live rows: every leaf is drawn many times per step.  B = 600 is three chunks of the kernels' 256 threads, so a
    later chunk overwrites leaves an earlier chunk wrote."""
    algo = per_build(rows_capacity=64, target_update_interval=2)
    fill(algo.replay_buffer, 8, 4, rows=5, seed=12)
    algo.device_rng_seed = 5
    _replay_calls(algo, 2, 3, B, per_oracle(algo))


def test_alpha_zero_beta_one_is_the_unweighted_dqn_step():
    """Every priority is 1, so every weight is exactly 1: the step equals train_gather's on the same rows, bit for bit."""
    S, B = 5, 48
    algo = per_build(alpha=0.0, beta_start=1.0, double_q=True, steps=2, target_update_interval=3)
    ref = build(double_q=True, steps=2, target_update_interval=3)
    for a in (algo, ref):
        fill(a.replay_buffer, 8, 4, rows=3000, seed=13)
    algo.train(algo.replay_buffer, S, B)
    idx, w, newp = algo._engine.get_per_draws(S, B)
    assert (w == 1.0).all() and (newp == 1.0).all()
    e = ref._ensure_engine(S, B)
    trainable, targets, lins = ref._learner_nets()
    ref._upload_state(e, trainable, targets, lins)
    columns, rows = ref.replay_buffer.device_columns()
    out = e.train_gather(ref._hparams(False, 1), columns, rows, idx)
    ref._download_state(e, trainable, targets, lins)
    for k in ("q1_values", "q1_losses"):
        np.testing.assert_array_equal(algo.last_train_output[k], out[k], err_msg=k)
    for x, y in zip(_state(algo), _state(ref)):
        np.testing.assert_array_equal(x, y)


# ---- execution paths and groups --------------------------------------------------------------------------------------
def _state(algo):
    return [flat(algo.q_function.network), flat(algo.target_q_function.network),
            *[adam_flat(algo.q_function.optimizer, k)[0] for k in ("exp_avg", "exp_avg_sq")]]


def _member(seed, steps=0):
    algo = per_build(O=6, n=5, seed=seed, steps=steps, double_q=True, target_update_interval=3)
    fill(algo.replay_buffer, 6, 5, rows=1500 + 100 * seed, seed=40 + seed)
    algo.device_rng_seed = 1000 + seed
    return algo


def test_graph_and_plain_launches_are_bit_identical():
    res = []
    for graph in ("1", "0"):
        os.environ["B200RL_OFFPOLICY_GRAPH"] = graph
        try:
            a = _member(0, steps=4)
            outs = []
            for _ in range(2):
                a.train(a.replay_buffer, 5, 40)
                outs.append((a.last_train_output, a._engine.get_per_draws(5, 40)))
            res.append((outs, _state(a), a.replay_buffer.priorities()))
        finally:
            os.environ.pop("B200RL_OFFPOLICY_GRAPH", None)
    (o1, s1, p1), (o2, s2, p2) = res
    for (out_a, dr_a), (out_b, dr_b) in zip(o1, o2):
        for k in out_a:
            np.testing.assert_array_equal(out_a[k], out_b[k], err_msg=k)
        for x, y in zip(dr_a, dr_b):
            np.testing.assert_array_equal(x, y)
    for x, y in zip(s1, s2):
        np.testing.assert_array_equal(x, y)
    np.testing.assert_array_equal(p1, p2)


@pytest.mark.parametrize("K", [3, 16])
def test_group_is_bit_identical_to_solo_engines(K):
    from rl_replicas_b200.algorithms import LearnerGroup
    S, B = 4, 32
    solo = [_member(k, 3 * k) for k in range(K)]
    grouped = [_member(k, 3 * k) for k in range(K)]
    g = LearnerGroup()
    for m in grouped:
        g.add(m)
    for call in range(2):
        g.train(S, B)
        gd = g._engine.get_per_draws(S, B)
        for k, m in enumerate(solo):
            m.train(m.replay_buffer, S, B)
            sd = m._engine.get_per_draws(S, B)
            for x, y in zip(sd, gd):
                np.testing.assert_array_equal(x, y[k], err_msg=f"draws, member {k} call {call}")
            for i, (x, y) in enumerate(zip(_state(m), _state(grouped[k]))):
                np.testing.assert_array_equal(x, y, err_msg=f"member {k} tensor {i} call {call}")
            np.testing.assert_array_equal(m.replay_buffer.priorities(), grouped[k].replay_buffer.priorities())
            np.testing.assert_array_equal(m.last_train_output["q1_losses"], grouped[k].last_train_output["q1_losses"])


# ---- refusals, end to end, launches ----------------------------------------------------------------------------------
def test_non_finite_priorities_raise_and_leave_the_host_modules_unchanged():
    from rl_replicas_b200._lib import B200RLError
    algo = per_build(rows_capacity=128, O=6, n=4, target_update_interval=2)
    fill(algo.replay_buffer, 6, 4, rows=64, seed=5)
    algo.replay_buffer._cols["rewards"][10] = np.nan
    nets = lambda: [flat(algo.q_function.network), flat(algo.target_q_function.network)]
    before = nets()
    with pytest.raises(B200RLError, match=r"DQN learner 0, step \d+: \d+ minibatch rows gave a non-finite priority"):
        algo.train(algo.replay_buffer, 8, 64)
    for x, y in zip(before, nets()):
        np.testing.assert_array_equal(x, y)
    assert algo._adam_step_count(algo.q_function.optimizer, list(algo.q_function.network.network)[::2]) == 0
    t = algo.replay_buffer.device_tree().cpu().numpy()
    assert np.isfinite(t).all()


def test_engine_refusals():
    from rl_replicas_b200._lib import B200RLError, OffPolicyHparams
    from rl_replicas_b200.engine import OffPolicyEngine
    td3 = OffPolicyEngine([4, 16, 2], [6, 16, 1], 2, 8, 2)
    with pytest.raises(B200RLError, match="DQN engines"):
        td3.set_per(0.6, 1e-6, 0.4, 100)
    e = OffPolicyEngine(None, [4, 16, 2], 1, 8, 2, algo=OffPolicyEngine.DQN)
    e.set_dqn(10, False)
    cols = [torch.zeros(16, 4, device="cuda"), torch.zeros(16, device="cuda"), torch.zeros(16, device="cuda"),
            torch.zeros(16, 4, device="cuda"), torch.zeros(16, device="cuda")]
    tree = torch.zeros(64, device="cuda")
    with pytest.raises(B200RLError, match="set_per"):
        e.train_prioritized(OffPolicyHparams(), cols, 16, tree, 2, 8, 0, 1)
    with pytest.raises(B200RLError, match="alpha"):
        e.set_per(-1.0, 1e-6, 0.4, 100)
    e.set_per(0.6, 1e-6, 0.4, 100)
    for bad in (torch.zeros(32, device="cuda"), torch.zeros(64, device="cuda", dtype=torch.float64),
                torch.zeros(64), torch.zeros(128, device="cuda")[::2]):
        with pytest.raises(ValueError, match="contiguous float32 CUDA tensor"):
            e.train_prioritized(OffPolicyHparams(), cols, 16, bad, 2, 8, 0, 1)
    with pytest.raises(B200RLError, match="not a prioritized one"):
        e.get_per_draws(2, 8)  # no prioritized call yet
    g = OffPolicyEngine(None, [4, 16, 2], 1, 8, 2, algo=OffPolicyEngine.DQN, n_learners=2)
    g.set_dqn(10, False)
    g.set_per(0.6, 1e-6, 0.4, 100)
    with pytest.raises(B200RLError, match="learners 0 and 1 share one tree"):
        g.train_prioritized_group(OffPolicyHparams(), [(cols, 16), (cols, 16)], [tree, tree], 2, 8, [0, 0], [1, 1])


def test_get_per_draws_refuses_after_a_uniform_call():
    S, B = 3, 32
    algo = per_build(double_q=True)
    fill(algo.replay_buffer, 8, 4, rows=500)
    algo.train(algo.replay_buffer, S, B)
    algo._engine.get_per_draws(S, B)
    from rl_replicas_b200._lib import B200RLError
    columns, rows = algo.replay_buffer.device_columns()
    algo._engine.train_gather(algo._hparams(False, 1), columns, rows, np.zeros((S, B), np.int64))
    with pytest.raises(B200RLError, match="not a prioritized one"):
        algo._engine.get_per_draws(S, B)


def test_launches_per_step_within_two_of_the_uniform_device_draw_path():
    from rl_replicas_b200 import _lib
    lib = _lib.load()
    S, B = 6, 64

    def per_call(algo):
        algo.train(algo.replay_buffer, S, B)  # builds the engine and the graph
        n0 = lib.b200rl_launch_count()
        algo.train(algo.replay_buffer, S, B)
        return lib.b200rl_launch_count() - n0
    uni = build(double_q=True)
    fill(uni.replay_buffer, 8, 4, rows=2000)
    uni.use_device_rng = True
    per = per_build(double_q=True)
    fill(per.replay_buffer, 8, 4, rows=2000)
    n_uni, n_per = per_call(uni), per_call(per)
    print(f"launches per call of {S} steps: uniform device draws {n_uni}, prioritized {n_per}")
    assert n_per <= n_uni + 2 * S


def test_learn_solves_the_choice_task(tmp_path, capsys):
    from rl_replicas_b200.replay_buffer import PrioritizedReplayBuffer
    np.random.seed(0)
    algo = make_dqn(**DQN_KW)
    algo.replay_buffer = PrioritizedReplayBuffer(100000)
    algo.learn(output_dir=str(tmp_path), **LEARN)
    after = evaluation_return(algo)
    printed = capsys.readouterr().out
    with capsys.disabled():
        print(f"DQN.learn with prioritized replay on the choice task: evaluation return {after:.3f}")
    assert "\nreplay/beta: " in printed
    assert after > RETURN_BAR
