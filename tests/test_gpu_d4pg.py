"""GPU: D4PG on the off-policy engine -- D4PG.train against the float32 oracle (oracle/d4pg.py) across calls on
host-drawn and device-drawn indices, one step against the float64 reference at edge shapes, n-step windows, prioritized
replay reproduced from the Philox keys, bit-identical execution paths and learner groups, the engine's refusals, the
launch budget, and D4PG.learn end to end."""
import os
import types

import numpy as np
import pytest
import torch

from conftest import rel_err
from oracle import d4pg as OD
from oracle import nstep as ON
from oracle import per as OP
from test_d4pg import LEARN, RETURN_BAR, evaluation_return, make_d4pg
from test_gpu_dqn import adam_flat, flat

pytestmark = pytest.mark.gpu
LR = 1e-3


def build(O=8, A=3, N=51, v=(-10.0, 10.0), policy_hidden=(64, 64), q_hidden=(64, 64), act=torch.nn.ReLU, seed=0,
          steps=0, replay_buffer=None, **kw):
    """A D4PG learner on a stub continuous environment; ``steps`` > 0 gives both Adams a state at that step count."""
    from rl_replicas_b200.algorithms import D4PG
    from rl_replicas_b200.critics import DistributionalQFunction
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import DeterministicPolicy
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    torch.manual_seed(seed)
    pnet = MLP([O, *policy_hidden, A], act, torch.nn.Tanh)
    qnet = MLP([O + A, *q_hidden, N], act)
    popt, qopt = torch.optim.Adam(pnet.parameters(), lr=LR), torch.optim.Adam(qnet.parameters(), lr=LR)
    for _ in range(steps):  # some arbitrary earlier steps
        for net, opt, w in ((pnet, popt, O), (qnet, qopt, O + A)):
            opt.zero_grad()
            net(torch.randn(16, w)).pow(2).mean().backward()
            opt.step()
    hi = np.ones(A, np.float32)
    env = types.SimpleNamespace(action_space=types.SimpleNamespace(high=hi, low=-hi, shape=(A,)),
                                observation_space=types.SimpleNamespace(shape=(O,)), spec=types.SimpleNamespace(id="stub"))
    qf = DistributionalQFunction(qnet, qopt, n_atoms=N, v_min=v[0], v_max=v[1])
    algo = D4PG(DeterministicPolicy(pnet, popt), None, qf, env, None,
                replay_buffer if replay_buffer is not None else ReplayBuffer(), None, **kw)
    with torch.no_grad():  # targets that differ from the online networks
        for m in (algo.target_policy, algo.target_q_function):
            for p in m.network.parameters():
                p.add_(0.05 * torch.randn_like(p))
    algo.metrics_manager = None
    algo.current_total_steps = 0
    return algo


def fill(rb, O, A, rows=4000, seed=1, ep=(20, 60)):
    """Episodes of random lengths in ``ep``, about half of them ending in a done row (the others cut off)."""
    from rl_replicas_b200.experience import Experience
    rng = np.random.default_rng(seed)
    e = Experience()
    e.observations, e.actions, e.rewards, e.dones, e.last_observations = [], [], [], [], []
    left = rows
    while left > 0:
        L = min(left, int(rng.integers(*ep)))
        obs = rng.standard_normal((L + 1, O)).astype(np.float32)
        e.observations.append([obs[i] for i in range(L)])
        e.actions.append([a for a in rng.uniform(-1, 1, (L, A)).astype(np.float32)])
        e.rewards.append([float(x) for x in 2.0 * rng.standard_normal(L)])
        e.dones.append([False] * (L - 1) + [bool(rng.random() < 0.5)])
        e.last_observations.append(obs[L])
        left -= L
    rb.add_experience(e)


def oracle_for(algo):
    q = algo.q_function
    rb = algo.replay_buffer
    return OD.D4pgOracle(algo.policy.network, q.network, algo.target_policy.network, algo.target_q_function.network,
                         algo.policy.optimizer, q.optimizer, n_atoms=q.n_atoms, v_min=q.v_min, v_max=q.v_max,
                         gamma=algo.gamma, rho=algo.polyak_rho, alpha=getattr(rb, "alpha", 0.6),
                         eps=getattr(rb, "eps", 1e-6))


def compare(algo, oracle, out=None, logs=None):
    errs = {}
    for name, a, b in (("policy", algo.policy.network, oracle.pi), ("q", algo.q_function.network, oracle.q),
                       ("target_policy", algo.target_policy.network, oracle.pi_t),
                       ("target_q", algo.target_q_function.network, oracle.q_t)):
        errs[name] = rel_err(flat(a), flat(b))
    for name, opt, oopt in (("pi", algo.policy.optimizer, oracle.opt_pi), ("q", algo.q_function.optimizer, oracle.opt_q)):
        for key in ("exp_avg", "exp_avg_sq"):
            got, step = adam_flat(opt, key)
            want, step_o = adam_flat(oopt, key)
            errs[f"{name} {key}"] = rel_err(got, want)
            assert step == step_o, (name, step, step_o)
    if out is not None:
        for key in ("q1_values", "q1_losses", "policy_losses"):
            errs[key] = rel_err(np.asarray(out[key]), np.stack(logs[key]) if key == "q1_values" else np.asarray(logs[key]))
    return errs


# From a fresh Adam the first step moves every parameter by lr g / (|g| + eps) (see tests/test_gpu_c51.py): the
# learners start from a few earlier Adam steps; the first step itself is held against the float64 reference below.
@pytest.mark.parametrize("path", ["gather", "rng"])
def test_train_matches_the_oracle_across_calls(path):
    """Three D4PG.train calls of 4 steps against the oracle with the same minibatches: host-drawn indices (the numpy
    stream) or device-drawn ones (replayed from get_draws)."""
    S, B = 4, 64
    algo = build(steps=5)
    fill(algo.replay_buffer, 8, 3)
    algo.use_device_rng, algo.device_rng_seed = path == "rng", 21
    oracle = oracle_for(algo)
    rb = algo.replay_buffer
    for call in range(3):
        np.random.seed(20 + call)
        algo.train(rb, S, B)
        out = algo.last_train_output
        if path == "rng":
            idx, _ = algo._engine.get_draws(S, B, with_noise=False)
            mbs = [{k: rb._cols[k][idx[s]] for k in rb.COLUMNS} for s in range(S)]
        else:
            np.random.seed(20 + call)
            mbs = [rb.sample_minibatch(B) for _ in range(S)]
        logs = oracle.train(mbs)
        errs = compare(algo, oracle, out, logs)
        print(f"{path} call {call}:", {k: f"{v:.1e}" for k, v in errs.items()})
        for k, v in errs.items():
            assert v < 2e-5, (call, k, v, errs)


# ---- one step against the float64 reference ------------------------------------------------------------------------
F64_CASES = {  # (policy sizes, critic hidden, N atoms, (v_min, v_max), hidden act, B)
    "cheetah": ([17, 256, 256, 6], [256, 256], 51, (-10.0, 10.0), "relu", 256),
    "atoms2": ([6, 64, 64, 2], [64, 64], 2, (-1.0, 1.0), "relu", 100),
    "atoms101_b257": ([6, 64, 64, 3], [64, 64], 101, (-5.0, 5.0), "relu", 257),
    "atoms256_b1": ([6, 32, 32, 4], [64, 64], 256, (-10.0, 10.0), "relu", 1),
    "a1": ([5, 64, 64, 1], [64, 64], 51, (-10.0, 10.0), "relu", 64),
    "a17": ([9, 64, 64, 17], [64, 64], 51, (-10.0, 10.0), "relu", 64),
    "two_layer": ([7, 48, 3], [48], 51, (-10.0, 10.0), "relu", 64),
    "four_layer": ([7, 64, 48, 40, 3], [64, 48, 40], 51, (-10.0, 10.0), "relu", 100),
    "tanh": ([8, 64, 64, 3], [64, 64], 51, (-10.0, 10.0), "tanh", 128),
}
KINK = 1e-5
# Bars: about 4x the largest errors measured on an H100 80GB HBM3 (700 W).  Both gradients normwise (conftest.rel_err):
# 8.7e-7 (atoms256_b1; the policy's 4.9e-7).  Entry by entry against its scale (the sum over rows of |a row's
# contribution|): the critic's 3.5e-3 (atoms256_b1; below 9e-4 elsewhere), the policy's 1.2e-3 (four_layer; below 5e-5
# elsewhere).  Q-values: 1.6e-5 of their maximum (atoms256_b1).  The critic's loss: 4.1e-8 of its value
# (atoms101_b257).  The policy loss -mean Q against max(|loss|, 1): 2.1e-6 (atoms256_b1: one row, 256 atoms).
BAR_GRAD_NORM, BAR_CRITIC_ENTRY, BAR_POLICY_ENTRY = 4e-6, 1.5e-2, 5e-3
BAR_Q, BAR_LOSS, BAR_POLICY_LOSS = 6e-5, 1.6e-7, 8e-6


def _f64_case(name, seed=0):
    psz, qh, N, (v_min, v_max), hidden, B = F64_CASES[name]
    O, A = psz[0], psz[-1]
    qsz = [O + A, *qh, N]
    act = {"relu": torch.nn.ReLU, "tanh": torch.nn.Tanh}[hidden]
    algo = build(O=O, A=A, N=N, v=(v_min, v_max), policy_hidden=tuple(psz[1:-1]), q_hidden=tuple(qh), act=act,
                 seed=seed)
    nets = dict(policy=flat(algo.policy.network), q1=flat(algo.q_function.network),
                target_policy=flat(algo.target_policy.network), target_q1=flat(algo.target_q_function.network))
    rng = np.random.default_rng(100 + seed)
    pool = 4 * B + 64
    z = OD.support(N, v_min, v_max)
    rew = (2.0 * rng.standard_normal(pool)).astype(np.float32)
    done = rng.random(pool) < 0.1
    k = np.arange(pool)
    rew[k % 16 == 3] = 3.0 * v_max  # every Tz_j clamps at v_max
    rew[k % 16 == 7] = 3.0 * v_min - 3.0 * v_max  # ... at v_min
    on_atom = k % 16 == 11  # terminal rows whose target is an atom
    rew[on_atom], done[on_atom] = z[k[on_atom] % N], True
    mb = dict(observations=rng.standard_normal((pool, O)).astype(np.float32),
              actions=rng.uniform(-1, 1, (pool, A)).astype(np.float32), rewards=rew,
              next_observations=rng.standard_normal((pool, O)).astype(np.float32), dones=done)
    ref = OD.d4pg_step_f64(nets, mb, psz, qsz, N, v_min, v_max, hidden, algo.gamma)
    keep = (ref["margin"] >= KINK) & (ref["margin_pi"] >= KINK) & (ref["margin_q"] >= KINK)
    rows = np.flatnonzero(keep)[:B]
    assert len(rows) == B, (name, int(keep.sum()))
    return algo, {k: v[rows] for k, v in mb.items()}, nets, psz, qsz


@pytest.mark.parametrize("name", list(F64_CASES))
def test_one_step_against_the_float64_reference(name):
    algo, mb, nets, psz, qsz = _f64_case(name)
    _, _, N, (v_min, v_max), hidden, B = F64_CASES[name]
    e = algo._ensure_engine(1, B)
    trainable, targets, lins = algo._learner_nets()
    algo._upload_state(e, trainable, targets, lins)
    out = e.train(algo._hparams(False, 1), mb["observations"][None], mb["actions"][None], mb["rewards"][None],
                  mb["next_observations"][None], mb["dones"].astype(np.float32)[None])
    blob, steps = e.get_state()
    layout, _ = e.state_layout()
    assert [(k, i) for k, i, _, _ in layout] == [("params", 0), ("params", 1), ("params", 3), ("params", 4), ("m", 0),
                                                 ("v", 0), ("m", 1), ("v", 1)]
    assert steps == [1, 1, 0]
    seg = {(k, i): blob[o:o + c].astype(np.float64) for k, i, o, c in layout}
    ref = OD.d4pg_step_f64(nets, mb, psz, qsz, N, v_min, v_max, hidden, algo.gamma, q_after=seg[("params", 1)])
    errs = {}
    for what, g, want, scale in (("critic", seg[("m", 1)] / 0.1, ref["grad_q"], ref["scale_q"]),
                                 ("policy", seg[("m", 0)] / 0.1, ref["grad_pi"], ref["scale_pi"])):
        errs[f"{what} grad"] = rel_err(g, want)
        errs[f"{what} entry"] = float(np.max(np.abs(g - want) / np.maximum(scale, 1e-30)))
    errs["q"] = rel_err(out["q1_values"][0], ref["q_values"])
    errs["loss"] = abs(float(out["q1_losses"][0]) - ref["loss"]) / max(abs(ref["loss"]), 1e-30)
    errs["policy loss"] = abs(float(out["policy_losses"][0]) - ref["policy_loss"]) / max(abs(ref["policy_loss"]), 1.0)
    print(f"{name}:", {k: f"{v:.2e}" for k, v in errs.items()})
    assert errs["critic grad"] < BAR_GRAD_NORM and errs["policy grad"] < BAR_GRAD_NORM, errs
    assert errs["critic entry"] < BAR_CRITIC_ENTRY and errs["policy entry"] < BAR_POLICY_ENTRY, errs
    assert errs["q"] < BAR_Q and errs["loss"] < BAR_LOSS and errs["policy loss"] < BAR_POLICY_LOSS, errs


# ---- n-step returns ----------------------------------------------------------------------------------------------------
def test_nstep_windows_are_bit_exact_and_the_step_matches_the_oracle():
    S, B, n = 4, 64, 5
    algo = build(steps=5, n_step=n)
    fill(algo.replay_buffer, 8, 3, rows=3000, seed=2)
    rb = algo.replay_buffer
    oracle = oracle_for(algo)
    for call in range(2):
        np.random.seed(40 + call)
        algo.train(rb, S, B)
        np.random.seed(40 + call)
        idx = rb.physical_rows(np.stack([rb.sample_indices(B) for _ in range(S)]))
        last, R, g = algo._engine.get_nstep_draws(S, B)
        want_last, want_R, want_g = ON.walk_f32(rb._cols["rewards"].astype(np.float32), rb._cols["dones"], rb._ends,
                                                idx, n, algo.gamma)
        np.testing.assert_array_equal(last, want_last)
        np.testing.assert_array_equal(R, want_R)
        np.testing.assert_array_equal(g, want_g)
        assert (g < np.float32(algo.gamma)).any()  # some windows are longer than one row
        logs = oracle.train([ON.nstep_minibatch(rb, idx[s], n, algo.gamma) for s in range(S)])
        errs = compare(algo, oracle, algo.last_train_output, logs)
        print(f"n-step call {call}:", {k: f"{v:.1e}" for k, v in errs.items()})
        for k, v in errs.items():
            assert v < 2e-5, (call, k, v)


# ---- prioritized replay --------------------------------------------------------------------------------------------------
def per_build(rows_capacity=8000, alpha=0.6, beta_start=0.4, beta_anneal_steps=50, eps=1e-6, **kw):
    from rl_replicas_b200.replay_buffer import PrioritizedReplayBuffer
    return build(replay_buffer=PrioritizedReplayBuffer(rows_capacity, alpha=alpha, beta_start=beta_start,
                                                       beta_anneal_steps=beta_anneal_steps, eps=eps), **kw)


def test_prioritized_draws_weights_and_priorities_match_the_oracle():
    S, B, tol = 4, 64, 2e-6
    algo = per_build(steps=5)
    fill(algo.replay_buffer, 8, 3, rows=3000, seed=3)
    rb = algo.replay_buffer
    oracle = oracle_for(algo)
    exempt = total = 0
    for call in range(3):
        leaves = rb.priorities().astype(np.float32)
        t0 = algo._adam_step_count(algo.q_function.optimizer, list(algo.q_function.network.network)[::2])
        algo.train(rb, S, B)
        idx, w, newp = algo._engine.get_per_draws(S, B)
        seed, ncall = algo.device_rng_seed, algo._device_rng_calls
        mbs, ps, betas = [], [], []
        for st in range(S):
            want, dist = OP.stratified_draw(leaves, seed, ncall, st, B)
            far = dist > tol
            exempt, total = exempt + int((~far).sum()), total + B
            assert (want[far] == idx[st][far]).all(), (call, st)
            mbs.append({k: rb._cols[k][idx[st]] for k in rb.COLUMNS})
            ps.append(leaves[idx[st]])
            betas.append(float(OP.beta_schedule(t0 + st, rb.beta_start, rb.beta_anneal_steps)))
            leaves = OP.apply_priorities(leaves, idx[st], newp[st]).astype(np.float32)
        np.testing.assert_array_equal(rb.priorities(), leaves)  # last occurrence wins, exactly
        logs = oracle.train(mbs, ps, betas)
        errs = compare(algo, oracle, algo.last_train_output, logs)
        w_ref, p_ref = np.stack(logs["weights"]), np.stack(logs["priorities"])
        errs["weights"] = float(np.max(np.abs(w - w_ref) / w_ref))
        # KL against the oracle's in units of the largest KL: KL = CE - H(m) cancels, so its relative error is not
        # bounded; the priority is a function of it
        kl_dev = newp.astype(np.float64) ** (1 / rb.alpha) - rb.eps
        errs["kl"] = float(np.max(np.abs(kl_dev - np.maximum(np.stack(logs["kl"]), 0))) / np.max(np.stack(logs["kl"])))
        print(f"prioritized call {call}:", {k: f"{v:.1e}" for k, v in errs.items()})
        for k, v in errs.items():
            assert v < (1e-6 if k == "weights" else 2e-5), (call, k, v)
    assert exempt <= total // 100, (exempt, total)


def test_non_finite_priorities_raise_and_leave_the_host_modules_and_the_row_unchanged():
    from rl_replicas_b200._lib import B200RLError
    algo = per_build(rows_capacity=128)
    fill(algo.replay_buffer, 8, 3, rows=64, seed=5)
    algo.replay_buffer._cols["rewards"][10] = np.nan
    nets = lambda: [flat(m.network) for m in (algo.policy, algo.q_function, algo.target_policy, algo.target_q_function)]
    before, leaf = nets(), float(algo.replay_buffer.priorities()[10])
    with pytest.raises(B200RLError, match=r"D4PG learner 0, step \d+: \d+ minibatch rows gave a non-finite priority"):
        algo.train(algo.replay_buffer, 8, 64)
    for x, y in zip(before, nets()):
        np.testing.assert_array_equal(x, y)
    assert float(algo.replay_buffer.priorities()[10]) == leaf
    assert np.isfinite(algo.replay_buffer.device_tree().cpu().numpy()).all()


# ---- execution paths and learner groups ---------------------------------------------------------------------------------
def _learner(path, seed=0, steps=1):
    from rl_replicas_b200.replay_buffer import PrioritizedReplayBuffer, ReplayBuffer
    rb = PrioritizedReplayBuffer(3000, beta_anneal_steps=20) if path == "per" else ReplayBuffer()
    algo = build(O=6, A=2, N=21, v=(-4.0, 4.0), seed=seed, steps=steps, replay_buffer=rb,
                 n_step=5 if path == "nstep" else 1)
    fill(algo.replay_buffer, 6, 2, rows=2000, seed=3 + seed)
    algo.use_device_rng, algo.device_rng_seed = path == "rng", 9 + seed
    return algo


def _state(algo):
    out = [flat(m.network) for m in (algo.policy, algo.q_function, algo.target_policy, algo.target_q_function)]
    for opt in (algo.policy.optimizer, algo.q_function.optimizer):
        out += [adam_flat(opt, k)[0] for k in ("exp_avg", "exp_avg_sq")]
    if hasattr(algo.replay_buffer, "priorities"):
        out.append(algo.replay_buffer.priorities())
    return out


def _run(path, graph, calls=2, S=5, B=48):
    os.environ["B200RL_OFFPOLICY_GRAPH"] = "1" if graph else "0"
    try:
        algo = _learner(path)
        outs = []
        for call in range(calls):
            np.random.seed(30 + call)
            algo.train(algo.replay_buffer, S + (call == calls - 1), B)
            outs.append(algo.last_train_output)
        return outs, _state(algo)
    finally:
        os.environ.pop("B200RL_OFFPOLICY_GRAPH", None)


@pytest.mark.parametrize("path", ["gather", "rng", "nstep", "per"])
def test_graph_and_plain_launches_are_bit_identical(path):
    (a_outs, a_state), (b_outs, b_state) = _run(path, True), _run(path, False)
    for a, b in zip(a_outs, b_outs):
        assert a.keys() == b.keys() and "policy_losses" in a
        for k in a:
            np.testing.assert_array_equal(a[k], b[k], err_msg=f"{path} {k}")
    for i, (x, y) in enumerate(zip(a_state, b_state)):
        np.testing.assert_array_equal(x, y, err_msg=f"{path} tensor {i}")


@pytest.mark.parametrize("path", ["gather", "nstep", "per"])
def test_group_of_three_is_bit_identical_to_solo_learners(path):
    from rl_replicas_b200.algorithms import LearnerGroup
    S, B, starts = 5, 40, (0, 7, 30)
    solo = [_learner(path, k, st) for k, st in enumerate(starts)]
    grouped = [_learner(path, k, st) for k, st in enumerate(starts)]
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
            for key in ("q1_values", "q1_losses", "policy_losses"):
                np.testing.assert_array_equal(a.last_train_output[key], b.last_train_output[key], err_msg=f"{key} {k}")
            for i, (x, y) in enumerate(zip(_state(a), _state(b))):
                np.testing.assert_array_equal(x, y, err_msg=f"{path} member {k} tensor {i} call {call}")


# ---- refusals, launches and end to end --------------------------------------------------------------------------------
def test_engine_refusals():
    from rl_replicas_b200._lib import B200RLError, OffPolicyHparams
    from rl_replicas_b200.engine import OffPolicyEngine
    P, Q = [4, 16, 2], [6, 16, 11]
    mk = lambda **kw: OffPolicyEngine(kw.pop("p", P), kw.pop("q", Q), kw.pop("n_q", 1), 8, 2,
                                      algo=kw.pop("algo", OffPolicyEngine.D4PG), **kw)
    with pytest.raises(B200RLError, match="algo must be"):
        mk(algo=6)  # plain create
    with pytest.raises(B200RLError, match="algo must be 6"):
        mk(algo=OffPolicyEngine.TD3, d4pg=(11, -1.0, 1.0))
    for kw, msg in ((dict(n_q=2), "n_q = 1"), (dict(q=[5, 16, 11]), "critic must map"),
                    (dict(q=[6, 16, 12]), "critic must map"), (dict(q=[6, 16, 1], d4pg=(1, -1.0, 1.0)), "n_atoms"),
                    (dict(q=[6, 16, 257], d4pg=(257, -1.0, 1.0)), "n_atoms"), (dict(d4pg=(11, 1.0, 1.0)), "v_min < v_max"),
                    (dict(d4pg=(11, 0.0, float("inf"))), "v_min < v_max"), (dict(d4pg=(11, float("nan"), 1.0)), "v_min"),
                    (dict(dueling_k=1), "dueling"), (dict(noisy_layers=1), "noisy")):
        kw.setdefault("d4pg", (11, -1.0, 1.0))
        with pytest.raises(B200RLError, match=msg):
            mk(**kw)
    e = mk(d4pg=(11, -1.0, 1.0))
    with pytest.raises(B200RLError, match="takes its support at create"):
        e.set_c51(11, -1.0, 1.0)
    with pytest.raises(B200RLError, match="algo = 2"):
        e.set_qr(11)
    with pytest.raises(B200RLError, match="algo = 2"):
        e.set_dqn(10, False)
    with pytest.raises(B200RLError, match="algo = 1"):
        e.set_sac(__import__("rl_replicas_b200._lib", fromlist=["SacHparams"]).SacHparams())
    with pytest.raises(B200RLError, match="no noisy layers"):
        e.set_noise_keys([0], [1])
    hp = OffPolicyHparams()
    hp.policy_delay, hp.use_target_noise = 1, 1
    z = lambda *s: np.zeros(s, np.float32)
    with pytest.raises(B200RLError, match="no target-policy smoothing"):
        e.train(hp, z(2, 8, 4), z(2, 8, 2), z(2, 8), z(2, 8, 4), z(2, 8), z(2, 8, 2))
    # DDPG / TD3 keep their refusals
    td3 = OffPolicyEngine(P, [6, 16, 1], 2, 8, 2)
    with pytest.raises(B200RLError, match="DQN engines"):
        td3.set_per(0.6, 1e-6, 0.4, 100)
    with pytest.raises(B200RLError, match="DQN and C51 engines"):
        td3.set_nstep(3, [torch.zeros(4, device="cuda")])
    with pytest.raises(B200RLError, match="algo = 3"):
        td3.set_c51(11, -1.0, 1.0)


def test_launches_per_step():
    """Uniform device draws: no more launches than DDPG at the same S; prioritized: at most 2 more per step."""
    from rl_replicas_b200 import _lib
    from rl_replicas_b200.algorithms import DDPG
    from rl_replicas_b200.critics import QFunction
    lib = _lib.load()
    S, B = 6, 64

    def per_call(algo):
        algo.train(algo.replay_buffer, S, B)  # builds the engine and the graph
        n0 = lib.b200rl_launch_count()
        algo.train(algo.replay_buffer, S, B)
        return lib.b200rl_launch_count() - n0
    d4pg = build()
    fill(d4pg.replay_buffer, 8, 3, rows=2000)
    d4pg.use_device_rng = True
    ref = build()
    qnet = type(ref.q_function.network)([11, 64, 64, 1], torch.nn.ReLU)
    ddpg = DDPG(ref.policy, None, QFunction(qnet, torch.optim.Adam(qnet.parameters(), lr=LR)), ref.env, None,
                ref.replay_buffer, None)
    ddpg.metrics_manager, ddpg.current_total_steps = None, 0
    fill(ddpg.replay_buffer, 8, 3, rows=2000)
    ddpg.use_device_rng = True
    per = per_build()
    fill(per.replay_buffer, 8, 3, rows=2000)
    n_ddpg, n_d4pg, n_per = per_call(ddpg), per_call(d4pg), per_call(per)
    print(f"launches per call of {S} steps: DDPG {n_ddpg}, D4PG {n_d4pg}, D4PG prioritized {n_per}")
    assert n_d4pg <= n_ddpg and n_per <= n_d4pg + 2 * S


def test_learn_solves_the_bandit(tmp_path, capsys):
    """D4PG.learn end to end on tests/test_sac.py's bandit with the seeds of the oracle-driven loop in
    tests/test_d4pg.py: DDPG's tags are recorded, model.pt is written and reloads, and the return clears the bar."""
    np.random.seed(0)
    algo = make_d4pg(polyak_rho=0.95)
    algo.learn(output_dir=str(tmp_path), **LEARN)
    after = evaluation_return(algo)
    printed = capsys.readouterr().out
    with capsys.disabled():
        print(f"D4PG.learn on the bandit: evaluation return {after:.3f}")
    for tag in ("policy/average_loss", "q-function/average_loss", "q-function/avarage_q-value",
                "evaluation/average_episode_return"):
        assert f"\n{tag}: " in printed, tag
    path = os.path.join(tmp_path, "model.pt")
    assert os.path.exists(path)
    other = make_d4pg(seed=5)
    other.load_model(path)
    assert evaluation_return(other) == after  # the reloaded networks act exactly as the trained ones
    assert after > RETURN_BAR
