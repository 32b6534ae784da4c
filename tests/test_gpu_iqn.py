"""GPU: IQN on the off-policy engine -- IQN.train against the float32 oracle (oracle/iqn.py) across calls and target
copies, one step against the float64 reference at edge shapes, the device's fraction draws (their values, their
distribution and their keying), bit-identical execution paths, learner groups bit for bit equal to solo engines,
prioritized replay (draws and priorities replayed through oracle/per.py, unit weights against the uniform step, the
non-finite refusal), n-step returns alone and with prioritized replay, the invalid-action refusal, the stated launch
counts, the engine's refusals, and IQN.learn end to end."""
import os

import numpy as np
import pytest
import torch

from conftest import rel_err
from oracle import iqn as OI
from oracle import nstep as ON
from oracle import per as OP
from test_dqn import LEARN, RETURN_BAR, evaluation_return
from test_gpu_dqn import GAMMA, LR, adam_flat, compare, fill, flat
from test_gpu_nstep import check_walk, fill_episodes, ring
from test_iqn import IQN_KW, make_iqn

pytestmark = pytest.mark.gpu


def build(O=8, n=4, d=64, hidden=64, n_cos=16, N=8, Nt=12, K=4, act=torch.nn.ReLU, seed=0, steps=0, per=None, **kw):
    """An IQN learner on a stub discrete environment (test_gpu_dqn.build with an implicit quantile critic); ``per`` = a
    dict of PrioritizedReplayBuffer settings gives it a prioritized buffer."""
    import types
    from rl_replicas_b200.algorithms import IQN
    from rl_replicas_b200.critics import ImplicitQuantileQFunction
    from rl_replicas_b200.networks import ImplicitQuantileMLP
    from rl_replicas_b200.replay_buffer import PrioritizedReplayBuffer, ReplayBuffer
    torch.manual_seed(seed)
    net = ImplicitQuantileMLP([O, d, hidden], n, n_cos=n_cos, activation_function=act)
    opt = torch.optim.Adam(net.parameters(), lr=LR)
    for _ in range(steps):  # some arbitrary earlier steps
        opt.zero_grad()
        net(torch.randn(16, O), torch.rand(16, 3)).pow(2).mean().backward()
        opt.step()
    env = types.SimpleNamespace(action_space=types.SimpleNamespace(n=n, shape=()), spec=types.SimpleNamespace(id="stub"),
                                observation_space=types.SimpleNamespace(shape=(O,)))
    rb = ReplayBuffer() if per is None else PrioritizedReplayBuffer(**per)
    qf = ImplicitQuantileQFunction(net, opt, n_quantiles=N, n_target_quantiles=Nt, n_policy_quantiles=K)
    algo = IQN(qf, None, env, None, rb, None, gamma=GAMMA, **kw)
    with torch.no_grad():  # a target that differs from the online network
        for p in algo.target_q_function.network.parameters():
            p.add_(0.05 * torch.randn_like(p))
    algo.metrics_manager = None
    algo.current_total_steps = 0
    algo.device_rng_seed = 1000 + seed
    return algo


PER = dict(buffer_size=8000, alpha=0.6, beta_start=0.4, beta_anneal_steps=50, eps=1e-6)


def oracle_for(algo):
    q, rb = algo.q_function, algo.replay_buffer
    return OI.IqnOracle(q.network, algo.target_q_function.network, q.optimizer, q.n_quantiles, q.n_target_quantiles,
                        q.n_policy_quantiles, gamma=algo.gamma, target_update_interval=algo.target_update_interval,
                        double_q=algo.double_q, alpha=getattr(rb, "alpha", 0.6), eps=getattr(rb, "eps", 1e-6))


def host_taus(algo, S, B):
    """The fractions of the learner's last call, from its keys, on the host."""
    q = algo.q_function
    Mt = q.n_quantiles + q.n_target_quantiles + q.n_policy_quantiles
    seed, call = algo.noise_key
    return np.stack([OI.iqn_taus(seed, call, s, B, Mt) for s in range(S)])


def _errs(algo, oracle, logs):
    errs = compare(algo, oracle)
    out = algo.last_train_output
    errs["q1_values"] = rel_err(out["q1_values"], np.stack(logs["q1_values"]))
    errs["q1_losses"] = rel_err(out["q1_losses"], np.asarray(logs["q1_losses"]))
    return errs


def _lins(algo):
    return algo._learner_nets()[2][0]


# From a fresh Adam the first step moves every parameter by lr g / (|g| + eps), which turns float32 rounding in
# near-zero gradient entries into visible parameter differences; the learners start from a few earlier Adam steps, and
# the first step itself is held against the float64 reference below.
@pytest.mark.parametrize("path", ["host", "gather"])
@pytest.mark.parametrize("double_q", [False, True])
def test_train_matches_the_oracle_across_calls_and_copies(double_q, path):
    """Three IQN.train calls of 4 steps at interval 3 (copies inside a call and across calls) against the oracle with
    the same minibatches and the engine's fractions, N = 32, N' = 24, K = 8."""
    S, B = 4, 64
    algo = build(N=32, Nt=24, K=8, n_cos=64, double_q=double_q, steps=7, target_update_interval=3)
    algo.use_device_replay = path == "gather"
    fill(algo.replay_buffer, 8, 4)
    oracle = oracle_for(algo)
    copies = 0
    for call in range(3):
        np.random.seed(20 + call)
        algo.train(algo.replay_buffer, S, B)
        taus = algo._engine.get_iqn_draws(S)
        np.testing.assert_array_equal(taus, host_taus(algo, S, B))
        np.random.seed(20 + call)
        logs = oracle.train([algo.replay_buffer.sample_minibatch(B) for _ in range(S)], taus)
        copies += sum(logs["copied"])
        errs = _errs(algo, oracle, logs)
        print(f"double_q={double_q} {path} call {call}:", {k: f"{v:.1e}" for k, v in errs.items()})
        for k, v in errs.items():
            assert v < 2e-5, (call, k, v, errs)
    assert copies == 4


# ---- one step against the float64 reference ------------------------------------------------------------------------
F64_CASES = {  # ([obs, d, h], n actions, n_cos, N, N', K, hidden, B, double_q)
    "lunar": ([8, 256, 256], 4, 64, 64, 64, 32, "relu", 64, True),
    "N1": ([6, 32, 32], 3, 16, 1, 1, 1, "relu", 33, False),
    "N31": ([6, 64, 64], 4, 32, 31, 31, 31, "relu", 77, False),
    "N32": ([6, 64, 64], 4, 32, 32, 32, 32, "relu", 64, True),
    "N33": ([6, 64, 64], 4, 32, 33, 33, 33, "relu", 65, True),
    "N8_Nt64_K1": ([6, 64, 64], 4, 32, 8, 64, 1, "relu", 100, True),
    "cos1": ([6, 64, 48], 4, 1, 16, 16, 8, "relu", 64, True),
    "cos256": ([6, 64, 48], 4, 256, 16, 16, 8, "relu", 64, True),
    "b1": ([5, 31, 31], 3, 64, 64, 64, 32, "relu", 1, True),
    "n18": ([6, 64, 64], 18, 32, 16, 16, 8, "relu", 129, True),
    "tanh": ([8, 64, 64], 4, 32, 32, 32, 16, "tanh", 128, False),
}
# Every row runs N + N' + K samples through two 256-wide ReLU layers and phi, so nearly every row of a large minibatch
# has some unit within 1e-6 (relative) of its kink: the margin kept is 1e-7, about the float32 rounding of a 256-term sum.
KINK, NEAR_TIE = 1e-7, 1e-5
# Bars: about 4x the largest errors measured on an H100.  The gradient normwise (conftest.rel_err): 8.3e-7 (N31;
# below 6.5e-7 elsewhere, 4.6e-7 lunar).  Entry by entry against its scale (the sum over rows of |a row's contribution|, which leaves
# out the cancellation inside each sample's sum over j and inside the dX chain): 4.8e-3 (N33; 1.5e-3 b1, below 1e-5
# elsewhere).  Q-values: 2.0e-7 of their maximum (lunar); the loss: 6.0e-8 of its value (cos256).
BAR_GRAD_NORM, BAR_GRAD_ENTRY, BAR_Q, BAR_LOSS = 3.5e-6, 2e-2, 8e-7, 2.5e-7


def _phi_margin(flat_p, sizes, n_cos, taus, hidden):
    """The smallest relative distance of phi's pre-activations to the ReLU kink over every fraction of ``taus``."""
    if hidden != "relu":
        return np.inf
    _, (Wc, bc), _, _ = OI._iqn_params(torch.as_tensor(flat_p), sizes, n_cos)
    x = OI._features_f64(torch.as_tensor(taus).reshape(-1), n_cos)
    z, scale = x @ Wc.T + bc, x.abs() @ Wc.abs().T + bc.abs()
    return float((z.abs() / scale.clamp_min(1e-300)).min())


def _f64_case(name, seed=0):
    """The learner, a minibatch whose rows keep every ReLU and argmax decision clear of a tie at their row positions'
    fractions, the fractions and the float64 reference."""
    body, n, n_cos, N, Nt, K, hidden, B, double_q = F64_CASES[name]
    sizes = body + [n]
    act = {"relu": torch.nn.ReLU, "tanh": torch.nn.Tanh}[hidden]
    algo = build(O=body[0], n=n, d=body[1], hidden=body[2], n_cos=n_cos, N=N, Nt=Nt, K=K, act=act, seed=seed,
                 double_q=double_q, target_update_interval=1000)
    q_flat, t_flat = flat(algo.q_function.network).astype(np.float64), flat(algo.target_q_function.network).astype(np.float64)
    rng = np.random.default_rng(100 + seed)
    pool = 8 * B + 64
    cols = dict(observations=rng.standard_normal((pool, body[0])).astype(np.float32),
                actions=rng.integers(0, n, pool).astype(np.float32),
                rewards=(2.0 * rng.standard_normal(pool)).astype(np.float32),
                next_observations=rng.standard_normal((pool, body[0])).astype(np.float32), dones=rng.random(pool) < 0.1)
    # phi depends on the fractions alone: keys whose fractions keep every phi unit of both networks clear of its kink
    seed_key, call_key = 77 + seed, 5
    while True:
        taus = OI.iqn_taus(seed_key, call_key, 0, B, N + Nt + K)
        if min(_phi_margin(f, sizes, n_cos, taus, hidden) for f in (q_flat, t_flat)) >= KINK:
            break
        call_key += 1
    rows, spare = np.arange(B), B
    for _ in range(40):  # replace the rows that sit near a kink or a tie at their position's fractions
        mb = {k: v[rows] for k, v in cols.items()}
        ref = OI.iqn_step_f64(q_flat, t_flat, mb, taus, sizes, n_cos, N, Nt, K, hidden, GAMMA, double_q)
        qmax = np.max(np.abs(ref["q_values"])) + 1.0
        bad = np.flatnonzero((ref["margin"] < KINK) | (ref["gap"] <= NEAR_TIE * qmax))
        if bad.size == 0:
            return algo, mb, taus, (seed_key, call_key), ref, sizes
        assert spare + bad.size <= pool, name
        rows[bad] = np.arange(spare, spare + bad.size)
        spare += bad.size
    raise AssertionError(f"{name}: no clear minibatch")


@pytest.mark.parametrize("name", list(F64_CASES))
def test_one_step_against_the_float64_reference(name):
    algo, mb, taus, keys, ref, sizes = _f64_case(name)
    B = len(mb["rewards"])
    e = algo._ensure_engine(1, B)
    trainable, targets, lins = algo._learner_nets()
    algo._upload_state(e, trainable, targets, lins)
    e.set_noise_keys([keys[0]], [keys[1]])
    out = e.train(algo._hparams(False, 1), mb["observations"][None], mb["actions"][None], mb["rewards"][None],
                  mb["next_observations"][None], mb["dones"].astype(np.float32)[None])
    np.testing.assert_array_equal(e.get_iqn_draws(1)[0], taus)
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


# ---- the draws -------------------------------------------------------------------------------------------------------
def test_draws_values_distribution_and_keys():
    """Odd multiples of 2^-24 in (0, 1), the host Philox's values bit for bit, uniform by a KS test; the same keys give
    the same draws, a new call new ones."""
    from scipy import stats
    S, B = 3, 256
    algo = build(N=64, Nt=64, K=32, steps=1)
    fill(algo.replay_buffer, 8, 4)
    e = algo._ensure_engine(S, B)
    algo._upload_state(e, *algo._learner_nets())
    hp = algo._hparams(False, 1)
    columns, rows = algo.replay_buffer.device_columns()
    idx = np.random.default_rng(0).integers(0, rows, (S, B))
    draws = []
    for call in (1, 1, 2):
        e.set_noise_keys([42], [call])
        e.train_gather(hp, columns, rows, idx)
        draws.append(e.get_iqn_draws(S))
    t = draws[0]
    assert t.shape == (S, B, 160)
    m = t.astype(np.float64) * 2.0 ** 24
    assert (m == np.round(m)).all() and (np.round(m) % 2 == 1).all() and (t > 0).all() and (t < 1).all()
    np.testing.assert_array_equal(t, np.stack([OI.iqn_taus(42, 1, s, B, 160) for s in range(S)]))
    p = stats.kstest(t.reshape(-1).astype(np.float64), "uniform").pvalue
    print(f"KS p-value over {t.size} draws: {p:.3f}")
    assert p > 1e-3
    np.testing.assert_array_equal(draws[1], t)
    assert (draws[2] != t).mean() > 0.99
    assert len(np.unique(t)) > 0.99 * t.size


def test_train_without_fresh_keys_is_refused():
    from rl_replicas_b200._lib import B200RLError
    algo = build()
    fill(algo.replay_buffer, 8, 4)
    e = algo._ensure_engine(2, 16)
    algo._upload_state(e, *algo._learner_nets())
    columns, rows = algo.replay_buffer.device_columns()
    idx = np.zeros((2, 16), np.int64)
    e.set_noise_keys([1], [1])
    e.train_gather(algo._hparams(False, 1), columns, rows, idx)
    with pytest.raises(B200RLError, match="IQN engine needs fresh keys"):
        e.train_gather(algo._hparams(False, 1), columns, rows, idx)


# ---- prioritized replay ----------------------------------------------------------------------------------------------
def _replay_prioritized(algo, calls, S, B, nstep=False):
    """`calls` train() calls replayed through oracle/per.py's draw and tree and the prioritized IQN oracle."""
    rb = algo.replay_buffer
    oracle = oracle_for(algo)
    for call in range(calls):
        leaves = rb.priorities().astype(np.float32)
        t0 = algo._adam_step_count(algo.q_function.optimizer, _lins(algo))
        algo.train(rb, S, B)
        idx, w, newp = algo._engine.get_per_draws(S, B)
        taus = algo._engine.get_iqn_draws(S)
        np.testing.assert_array_equal(taus, host_taus(algo, S, B))
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
        logs = oracle.train(mbs, taus, ps, betas)
        errs = _errs(algo, oracle, logs)
        w_err = float(np.max(np.abs(w - np.stack(logs["weights"])) / np.stack(logs["weights"])))
        p_ref = np.stack(logs["priorities"])
        p_err = float(np.max(np.abs(newp - p_ref) / p_ref))
        print(f"call {call}:", {k: f"{v:.1e}" for k, v in errs.items()}, f"weights {w_err:.1e} priorities {p_err:.1e}")
        for k, v in errs.items():
            assert v < 2e-5, (call, k, v)
        assert w_err < 1e-6 and p_err < 2e-5, (w_err, p_err)


@pytest.mark.parametrize("double_q", [False, True])
def test_prioritized_draws_weights_and_priorities_match_the_oracle(double_q):
    """3 calls of 4 steps on a half-full buffer (zero-priority leaves), target copies inside and across calls."""
    algo = build(per=PER, double_q=double_q, steps=3, target_update_interval=3)
    fill(algo.replay_buffer, 8, 4, rows=4000, seed=11)
    algo.device_rng_seed = 91
    _replay_prioritized(algo, 3, 4, 64)


def test_alpha_zero_beta_one_is_the_uniform_step():
    """Every priority is 1, so every weight is exactly 1: the step equals train_gather's on the same rows and
    fractions, bit for bit."""
    S, B = 5, 48
    algo = build(per=dict(PER, alpha=0.0, beta_start=1.0), double_q=True, steps=2, target_update_interval=3)
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
    e.set_noise_keys([algo.noise_key[0]], [algo.noise_key[1]])
    out = e.train_gather(ref._hparams(False, 1), columns, rows, idx)
    ref._download_state(e, trainable, targets, lins)
    for k in ("q1_values", "q1_losses"):
        np.testing.assert_array_equal(algo.last_train_output[k], out[k], err_msg=k)
    for x, y in zip(_state(algo), _state(ref)):
        np.testing.assert_array_equal(x, y)


def test_nan_reward_raises_and_leaves_the_host_modules_unchanged():
    from rl_replicas_b200._lib import B200RLError
    algo = build(O=6, n=4, per=dict(PER, buffer_size=128), target_update_interval=2)
    fill(algo.replay_buffer, 6, 4, rows=64, seed=5)
    algo.replay_buffer._cols["rewards"][10] = np.nan
    nets = lambda: [flat(algo.q_function.network), flat(algo.target_q_function.network)]
    before = nets()
    leaf = algo.replay_buffer.priorities()[10]
    with pytest.raises(B200RLError, match=r"IQN learner 0, step \d+: \d+ minibatch rows gave a non-finite priority"):
        algo.train(algo.replay_buffer, 8, 64)
    for x, y in zip(before, nets()):
        np.testing.assert_array_equal(x, y)
    assert algo._adam_step_count(algo.q_function.optimizer, _lins(algo)) == 0
    assert np.isfinite(algo.replay_buffer.device_tree().cpu().numpy()).all()
    assert algo.replay_buffer.priorities()[10] == leaf  # the NaN row never wrote its leaf


# ---- n-step returns --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", ["gather", "rng"])
def test_nstep_matches_the_oracle(path):
    S, B = 4, 64
    algo = ring(build(steps=7, double_q=True, target_update_interval=3, n_step=3), seed=7)
    algo.use_device_rng, algo.device_rng_seed = path == "rng", 5
    oracle = oracle_for(algo)
    rb = algo.replay_buffer
    for call in range(2):
        np.random.seed(40 + call)
        algo.train(rb, S, B)
        if path == "rng":
            idx, _ = algo._engine.get_draws(S, B)
        else:
            np.random.seed(40 + call)
            idx = rb.physical_rows(np.stack([rb.sample_indices(B) for _ in range(S)]))
        check_walk(algo, idx, S, B)
        logs = oracle.train([ON.nstep_minibatch(rb, idx[s], 3, algo.gamma) for s in range(S)],
                            algo._engine.get_iqn_draws(S))
        errs = _errs(algo, oracle, logs)
        print(f"n=3 {path} call {call}:", {k: f"{v:.1e}" for k, v in errs.items()})
        for k, v in errs.items():
            assert v < 2e-5, (call, k, v, errs)


def test_prioritized_nstep_matches_the_oracle():
    algo = build(per=dict(PER, buffer_size=700), n_step=3, double_q=True, steps=2, target_update_interval=4)
    fill_episodes(algo.replay_buffer, 8, 1500, 9)
    algo.device_rng_seed = 9
    assert algo.replay_buffer._head > 0
    _replay_prioritized(algo, 2, 3, 64, nstep=True)


# ---- execution paths and groups --------------------------------------------------------------------------------------
def _state(algo):
    return [flat(algo.q_function.network), flat(algo.target_q_function.network),
            *[adam_flat(algo.q_function.optimizer, k)[0] for k in ("exp_avg", "exp_avg_sq")]]


def _member(seed, steps, path):
    """path: host, gather, rng (uniform draws), per (prioritized) or nstep (n = 3 on uniform device draws)."""
    kw = dict(O=6, n=5, N=9, Nt=7, K=5, n_cos=12, seed=seed, steps=steps, double_q=True, target_update_interval=3)
    if path == "per":
        algo = build(per=PER, **kw)
    else:
        algo = build(n_step=3 if path == "nstep" else 1, **kw)
    if path == "nstep":
        ring(algo, O=6, seed=40 + seed)
    else:
        fill(algo.replay_buffer, 6, 5, rows=1500 + 100 * seed, seed=40 + seed)
    algo.use_device_replay = path != "host"
    algo.use_device_rng = path in ("rng", "nstep")
    return algo


def _outputs(algo):
    return [algo.last_train_output[k] for k in ("q1_values", "q1_losses")]


@pytest.mark.parametrize("path", ["host", "gather", "per", "nstep"])
def test_graph_and_plain_launches_are_bit_identical(path):
    res = []
    for graph in ("1", "0"):
        os.environ["B200RL_OFFPOLICY_GRAPH"] = graph
        try:
            a = _member(0, 4, path)
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
            np.testing.assert_array_equal(u, v, err_msg=f"{path}: call {call} tensor {i}")


@pytest.mark.parametrize("K,path", [(3, "host"), (3, "rng"), (3, "per"), (3, "nstep"), (16, "gather")])
def test_group_is_bit_identical_to_solo_engines(K, path):
    """Members at different Q step counts (interval 3: they copy on different steps) and with their own draw keys, two
    calls; each member's fractions equal its solo engine's."""
    from rl_replicas_b200.algorithms import LearnerGroup
    S, B = 4, 32
    solo = [_member(k, 3 * k, path) for k in range(K)]
    grouped = [_member(k, 3 * k, path) for k in range(K)]
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
        taus = g._engine.get_iqn_draws(S)
        for k, (a, b) in enumerate(zip(solo, grouped)):
            np.testing.assert_array_equal(taus[k], a._engine.get_iqn_draws(S), err_msg=f"{path}: member {k} draws")
            for x, y, what in zip(_outputs(a) + _state(a), _outputs(b) + _state(b),
                                  ("q1_values", "q1_losses", "q", "target", "exp_avg", "exp_avg_sq")):
                np.testing.assert_array_equal(x, y, err_msg=f"{path}: member {k} {what} call {call}")
            if path == "per":
                np.testing.assert_array_equal(a.replay_buffer.priorities(), b.replay_buffer.priorities())


# ---- refusals, launches and end to end --------------------------------------------------------------------------------
@pytest.mark.parametrize("bad", [4.0, 1.5, -1.0, float("nan")])
def test_invalid_action_raises_and_leaves_the_host_modules_unchanged(bad):
    from rl_replicas_b200._lib import B200RLError
    algo = build(O=6, n=4, target_update_interval=2)
    fill(algo.replay_buffer, 6, 4, rows=64, seed=5, bad_action=bad)
    before = [flat(algo.q_function.network), flat(algo.target_q_function.network)]
    np.random.seed(0)
    with pytest.raises(B200RLError, match=r"IQN learner 0, step \d+: \d+ minibatch rows hold an action that is "
                                          r"not an integer in \[0, 4\)"):
        algo.train(algo.replay_buffer, 8, 64)  # 512 draws of 64 rows: the bad row is drawn
    for x, y in zip(before, [flat(algo.q_function.network), flat(algo.target_q_function.network)]):
        np.testing.assert_array_equal(x, y)
    assert algo._adam_step_count(algo.q_function.optimizer, _lins(algo)) == 0


def test_engine_refuses_bad_iqn_configurations():
    from rl_replicas_b200._lib import B200RLError
    from rl_replicas_b200.engine import OffPolicyEngine as E
    q = [4, 16, 16, 3]
    for algo, sizes in ((E.DQN, q), (E.C51, [4, 16, 33])):
        with pytest.raises(B200RLError, match="the config's algo must be 4"):
            E(None, sizes, 1, 8, 2, algo=algo, iqn=(8, 8, 8, 4))
    with pytest.raises(B200RLError, match="the config's algo must be 4"):
        E([4, 16, 2], [6, 16, 1], 2, 8, 2, iqn=(8, 8, 8, 4))
    for kw in (dict(dueling_k=1), dict(noisy_layers=1)):
        with pytest.raises(B200RLError, match="dueling and noisy IQN networks are not implemented"):
            E(None, q, 1, 8, 2, algo=E.IQN, iqn=(8, 8, 8, 4), **kw)
    for bad in ((0, 8, 8, 4), (8, 257, 8, 4), (8, 8, 0, 4), (8, 8, 8, 257), (257, 8, 8, 4)):
        with pytest.raises(B200RLError, match="must each be 1..256"):
            E(None, q, 1, 8, 2, algo=E.IQN, iqn=bad)
    with pytest.raises(B200RLError, match="algo 4, IQN, is created by b200rl_offpolicy_create_iqn"):
        E(None, q, 1, 8, 2, algo=E.IQN)  # create_group without the counts
    with pytest.raises(B200RLError, match="3 layers"):
        E(None, [4, 16, 3], 1, 8, 2, algo=E.IQN, iqn=(8, 8, 8, 4))
    with pytest.raises(B200RLError, match="out_act identity"):
        E(None, q, 1, 8, 2, q_acts=("relu", "tanh"), algo=E.IQN, iqn=(8, 8, 8, 4))
    e = E(None, q, 1, 8, 2, algo=E.IQN, iqn=(8, 8, 8, 4))
    with pytest.raises(B200RLError, match="algo = 2"):
        e.set_qr(1)
    with pytest.raises(B200RLError, match="has not run a train step"):
        e.get_iqn_draws(1)
    e.set_per(0.6, 1e-6, 0.4, 100)  # prioritized replay is available
    E(None, q, 1, 8, 2, algo=E.IQN, iqn=(256, 256, 256, 256), n_learners=2)


def _launches(algo, graph, S=6, B=64):
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
    """b200rl.h: 21 launches per step, 26 with Double DQN, 2 more with prioritized replay (host minibatches: nothing
    else is launched per call)."""
    S = 6
    for per in (False, True):
        for double_q in (False, True):
            for graph in (False, True):
                algo = build(per=PER if per else None, double_q=double_q, target_update_interval=3)
                fill(algo.replay_buffer, 8, 4, rows=1000, seed=6)
                algo.use_device_replay = per
                got = _launches(algo, graph, S)
                want = S * ((26 if double_q else 21) + (2 if per else 0))
                print(f"per={per} double_q={double_q} graph={graph}: {got} launches per call of {S} steps")
                assert got == want, (per, double_q, graph, got, want)


def test_learn_solves_the_choice_task(tmp_path, capsys):
    """IQN.learn end to end on tests/test_dqn.py's one-step choice task with the seeds of the oracle-driven loop in
    tests/test_iqn.py: DQN's tags are recorded, model.pt is written and reloads, and the evaluation return clears the
    same bar."""
    np.random.seed(0)
    algo = make_iqn(**IQN_KW)
    algo.learn(output_dir=str(tmp_path), **LEARN)
    after = evaluation_return(algo)
    printed = capsys.readouterr().out
    with capsys.disabled():
        print(f"IQN.learn on the choice task: evaluation return {after:.3f}")
    for tag in ("q-function/average_loss", "q-function/avarage_q-value", "exploration/epsilon",
                "evaluation/average_episode_return"):
        assert f"\n{tag}: " in printed, tag
    path = os.path.join(tmp_path, "model.pt")
    assert os.path.exists(path)
    other = make_iqn(seed=5, **IQN_KW)
    other.load_model(path)
    assert evaluation_return(other) == after  # the reloaded networks act exactly as the trained ones
    assert after > RETURN_BAR
