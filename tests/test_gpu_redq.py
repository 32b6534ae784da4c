"""GPU: REDQ.train on the off-policy engine against the torch-autograd oracle (oracle/redq.py), N = M = 2 against a SAC
engine, bit-identical results across its execution paths and in learner groups, the device-side subset draws, the
engine's refusals, the launches per step b200rl.h states, and REDQ.learn end to end."""
import os
import types

import numpy as np
import pytest
import torch

from conftest import rel_err
from oracle import redq as OR
from test_gpu_sac import SHAPES, adam_flat, fill, flat
from test_gpu_sac import build as build_sac
from test_redq import REDQ_LEARN, make_redq
from test_sac import RETURN_BAR, evaluation_return

pytestmark = pytest.mark.gpu


def build(shape, n=10, n_min=2, delay=20, seed=0, learn_alpha=False):
    from rl_replicas_b200.algorithms import REDQ
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import RandomPolicy, SquashedGaussianPolicy
    from rl_replicas_b200.q_function import QFunction
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    O, A, H, act, L, _ = SHAPES[shape]
    torch.manual_seed(seed)
    pnet = MLP([O, H, H, 2 * A], act)
    qs = [MLP([O + A, H, H, 1], act) for _ in range(n)]
    hi = np.full(A, L, np.float32)
    env = types.SimpleNamespace(action_space=types.SimpleNamespace(high=hi, low=-hi, shape=(A,)),
                                spec=types.SimpleNamespace(id="stub"))
    algo = REDQ(SquashedGaussianPolicy(pnet, torch.optim.Adam(pnet.parameters(), lr=1e-3), action_limit=L),
                RandomPolicy(None), [QFunction(q, torch.optim.Adam(q.parameters(), lr=1e-3)) for q in qs], env, None,
                ReplayBuffer(), None, learn_alpha=learn_alpha, alpha_lr=3e-3, n_min=n_min, policy_delay=delay)
    algo.metrics_manager = None
    algo.current_total_steps = 0
    return algo


def oracle_for(algo):
    return OR.RedqOracle(algo.policy.network, [q.network for q in algo.q_functions], gamma=algo.gamma,
                         rho=algo.polyak_rho, alpha=algo.alpha, learn_alpha=algo.learn_alpha,
                         target_entropy=algo.target_entropy, alpha_lr=3e-3, limit=algo.policy.action_limit,
                         policy_delay=algo.policy_delay)


def compare(algo, oracle, logs, out):
    """{name: norm-wise error} of every logged quantity and every tensor of the learner against the oracle."""
    errs = {"q_values": rel_err(out["redq_q_values"], np.asarray(logs["q_values"])),
            "q_losses": rel_err(out["redq_q_losses"], np.asarray(logs["q_losses"]))}
    for k in ("policy_losses", "log_prob_means", "alphas"):
        errs[k] = rel_err(out[k], np.asarray(logs[k]))
    errs["q1_values"] = rel_err(out["q1_values"], np.asarray(logs["q_values"][0]))
    errs["q2_losses"] = rel_err(out["q2_losses"], np.asarray(logs["q_losses"][1]))
    pairs = [("policy", algo.policy, oracle.pi, oracle.pi_opt)]
    pairs += [(f"q{i}", q, o, opt) for i, (q, o, opt) in enumerate(zip(algo.q_functions, oracle.qs, oracle.q_opts))]
    for name, m, o, opt in pairs:
        errs[name] = rel_err(flat(m.network), flat(o))
        for key in ("exp_avg", "exp_avg_sq"):
            got, step = adam_flat(m.optimizer, key)
            want, step_o = adam_flat(opt, key)
            errs[f"{name}.{key}"] = rel_err(got, want)
            assert step == step_o, (name, step, step_o)
    for i, (t, o) in enumerate(zip(algo.target_q_functions, oracle.q_targs)):
        errs[f"target_q{i}"] = rel_err(flat(t.network), flat(o))
    errs["log_alpha"] = rel_err(float(algo.log_alpha.detach()), float(oracle.log_alpha.detach()))
    return errs


def _train_and_replay(algo, S, B, seed=7):
    """algo.train, then the oracle on the same minibatches, noise and subsets (the host streams replayed)."""
    oracle = oracle_for(algo)
    np.random.seed(seed)
    torch.manual_seed(seed)
    state_np, state_t = np.random.get_state(), torch.get_rng_state()
    algo.train(algo.replay_buffer, S, B)
    np.random.set_state(state_np)
    torch.set_rng_state(state_t)
    mbs = [algo.replay_buffer.sample_minibatch(B) for _ in range(S)]
    noise, subsets = algo._noise(S, B)
    return oracle, oracle.train(mbs, noise, subsets)


# (shape, N, M, G, S, learn_alpha): the paper's setting at the HalfCheetah shape, then N = M (a deterministic subset),
# M = 1, the largest N and G = 1 at small_tanh
CASES = [("halfcheetah", 10, 2, 20, 25, True), ("small_tanh", 10, 2, 20, 25, True), ("small_tanh", 4, 4, 3, 10, False),
         ("small_tanh", 5, 1, 2, 9, True), ("small_tanh", 32, 2, 4, 8, False), ("small_tanh", 3, 2, 1, 6, True)]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "-".join(str(x) for x in c))
def test_train_matches_the_oracle(case):
    shape, N, M, G, S, learn_alpha = case
    O, A, H, act, L, B = SHAPES[shape]
    algo = build(shape, n=N, n_min=M, delay=G, learn_alpha=learn_alpha)
    fill(algo.replay_buffer, O, A, L)
    oracle, logs = _train_and_replay(algo, S, B)
    out = algo.last_train_output
    assert len(out["policy_losses"]) == len(OR.policy_steps(S, G)) == len(logs["policy_losses"])
    errs = compare(algo, oracle, logs, out)
    print(case, {k: f"{v:.2e}" for k, v in errs.items() if v > 1e-6})
    # At the 256-wide ReLU shape a pre-activation within float rounding of the ReLU kink can decide whether one row's
    # gradient passes, and Adam turns such a one-row difference on a unit with a tiny exp_avg_sq into an lr-sized step
    # (the mechanism test_gpu_sac.py and test_gpu_tqc.py trace).  Measured on H100 over these 25 steps: critic 0 drifts
    # by 8.4e-4 of its maximum and its exp_avg by 2.0e-3, every other tensor stays below 8e-5 and the logged values
    # below 7.5e-5.  Bounded at 1e-2 for tensors and 2e-4 for logged values; small_tanh stays within 2e-5 throughout.
    kink = shape == "halfcheetah"
    for k, v in errs.items():
        logged = k in ("q_values", "q_losses", "policy_losses", "log_prob_means", "alphas", "q1_values", "q2_losses",
                       "log_alpha")
        assert v < ((2e-4 if logged else 1e-2) if kink else 2e-5), (k, v)
    if not learn_alpha:
        assert (out["alphas"] == np.float32(0.2)).all()


def test_two_critics_two_drawn_match_a_sac_engine_on_the_first_step():
    """N = M = 2: the first step's critic step is SAC's -- q-values, critic losses, critic parameters, their Adam
    moments and the target critics equal a SAC engine's bit for bit on the same inputs."""
    O, A, _, _, L, _ = SHAPES["halfcheetah"]
    B = 256
    redq, sac = build("halfcheetah", n=2, n_min=2, delay=1), build_sac("halfcheetah")
    for a in (redq, sac):
        fill(a.replay_buffer, O, A, L, n=3000, seed=5)
        np.random.seed(3)
        torch.manual_seed(3)
        a.train(a.replay_buffer, 1, B)
    r, s = redq.last_train_output, sac.last_train_output
    for k in ("q1_values", "q2_values", "q1_losses", "q2_losses"):
        np.testing.assert_array_equal(r[k], s[k], err_msg=k)
    for qr, qs in ((redq.q_functions[0], sac.q_function_1), (redq.q_functions[1], sac.q_function_2),
                   (redq.target_q_functions[0], sac.target_q_function_1),
                   (redq.target_q_functions[1], sac.target_q_function_2)):
        np.testing.assert_array_equal(flat(qr.network), flat(qs.network))
    for qr, qs in ((redq.q_functions[0], sac.q_function_1), (redq.q_functions[1], sac.q_function_2)):
        for key in ("exp_avg", "exp_avg_sq"):
            np.testing.assert_array_equal(adam_flat(qr.optimizer, key)[0], adam_flat(qs.optimizer, key)[0])


def test_one_step_against_the_float64_reference():
    """One step at the HalfCheetah shape: every critic's values and loss, and the policy loss and mean log pi (with the
    critics the engine updated), against float64 stages at the engine's parameters and draws."""
    O, A, H, _, L, B = SHAPES["halfcheetah"]
    algo = build("halfcheetah", n=10, n_min=2, delay=1)
    fill(algo.replay_buffer, O, A, L, n=3000, seed=8)
    f64 = lambda m: flat(m.network).astype(np.float64)
    nets = dict(policy=f64(algo.policy), q=[f64(q) for q in algo.q_functions],
                target_q=[f64(q) for q in algo.target_q_functions])
    np.random.seed(9)
    torch.manual_seed(9)
    state_np, state_t = np.random.get_state(), torch.get_rng_state()
    algo.train(algo.replay_buffer, 1, B)
    out = algo.last_train_output
    np.random.set_state(state_np)
    torch.set_rng_state(state_t)
    mb = algo.replay_buffer.sample_minibatch(B)
    noise, subsets = algo._noise(1, B)
    psz, qsz = [O, H, H, 2 * A], [O + A, H, H, 1]
    c = OR.critic_stage_f64(nets, mb, noise[0, 0], subsets[0], 0.2, psz, qsz, gamma=algo.gamma, action_limit=L)
    for k in range(10):
        assert rel_err(out["redq_q_values"][k][0], c["values"][k]) < 1e-5
        assert rel_err(out["redq_q_losses"][k][0], c["losses"][k]) < 1e-5
    qs_new = [flat(q.network).astype(np.float64) for q in algo.q_functions]
    p = OR.policy_stage_f64(nets["policy"], qs_new, mb["observations"], noise[0, 1], 0.2, psz, qsz, action_limit=L)
    assert rel_err(out["policy_losses"][0], p["loss"]) < 1e-5
    assert rel_err(out["log_prob_means"][0], p["logp_mean"]) < 1e-5


def _run_paths(device_replay, graph, rng=False):
    O, A, _, _, L, _ = SHAPES["small_tanh"]
    os.environ["B200RL_OFFPOLICY_GRAPH"] = "1" if graph else "0"
    try:
        algo = build("small_tanh", n=6, n_min=2, delay=3, learn_alpha=True)
        fill(algo.replay_buffer, O, A, L, n=3000, seed=3)
        algo.use_device_replay = device_replay
        algo.use_device_rng, algo.device_rng_seed = rng, 41
        outs = []
        for call in range(3):
            np.random.seed(10 + call)
            torch.manual_seed(10 + call)
            algo.train(algo.replay_buffer, 7 + (call == 2), 32)
            outs.append(algo.last_train_output)
        nets = [flat(m.network) for m in [algo.policy] + algo.q_functions + algo.target_q_functions]
        return outs, nets + [algo.log_alpha.detach().numpy().reshape(1)]
    finally:
        os.environ.pop("B200RL_OFFPOLICY_GRAPH", None)


def test_execution_paths_are_bit_identical():
    """Plain launches on host-staged minibatches, the captured graph replayed across calls (the third call changes S
    and recaptures) and the device-replay gather all agree bit for bit; so do device draws with and without a graph."""
    for ref, others in (((False, False), ((True, True), (False, True), (True, False))),
                        ((True, False, True), ((True, True, True),))):
        ref_outs, ref_nets = _run_paths(*ref)
        for args in others:
            outs, nets = _run_paths(*args)
            for a, b in zip(outs, ref_outs):
                assert a.keys() == b.keys()
                for k in a:
                    np.testing.assert_array_equal(a[k], b[k], err_msg=f"{k} {args}")
            for i, (a, b) in enumerate(zip(nets, ref_nets)):
                np.testing.assert_array_equal(a, b, err_msg=f"net {i} {args}")


def test_device_subsets_replay_through_the_oracle():
    O, A, _, _, L, _ = SHAPES["small_tanh"]
    S, B, N, M = 12, 64, 8, 3
    algo = build("small_tanh", n=N, n_min=M, delay=4, learn_alpha=True)
    fill(algo.replay_buffer, O, A, L, n=3000, seed=4)
    algo.use_device_rng, algo.device_rng_seed = True, 77
    oracle = oracle_for(algo)
    algo.train(algo.replay_buffer, S, B)
    idx, noise = algo._engine.get_draws(S, B)
    sub = algo._engine.get_redq_subsets(S)
    assert sub.shape == (S, M) and sub.min() >= 0 and sub.max() < N
    assert all(len(set(row)) == M for row in sub.tolist())
    rb = algo.replay_buffer
    logs = oracle.train([{k: rb._cols[k][idx[s]] for k in rb.COLUMNS} for s in range(S)], noise, sub)
    errs = compare(algo, oracle, logs, algo.last_train_output)
    for k, v in errs.items():
        assert v < 2e-5, (k, v, errs)
    algo.train(rb, 400, 16)  # every critic is drawn about equally often
    counts = np.bincount(algo._engine.get_redq_subsets(400).ravel(), minlength=N)
    assert counts.min() > 0.7 * 400 * M / N and counts.max() < 1.3 * 400 * M / N, counts


# ---- learner groups -------------------------------------------------------------------------------------------------
def _member(k, path):
    O, A, _, _, L, _ = SHAPES["small_tanh"]
    algo = build("small_tanh", n=5, n_min=2, delay=2, seed=k, learn_alpha=True)
    fill(algo.replay_buffer, O, A, L, n=2000, seed=30 + k)
    algo.use_device_replay = path != "host"
    algo.use_device_rng, algo.device_rng_seed = path == "rng", 90 + k
    if k % 2:  # members at different Adam step counts
        np.random.seed(k)
        torch.manual_seed(k)
        algo.train(algo.replay_buffer, k, 16)
    return algo


def _state(algo):
    out = [flat(m.network) for m in [algo.policy] + algo.q_functions + algo.target_q_functions]
    for m in [algo.policy] + algo.q_functions:
        out += [adam_flat(m.optimizer, k)[0] for k in ("exp_avg", "exp_avg_sq")]
    return out + [np.asarray(algo._alpha_state(), np.float64)]


def _check_group(path, K, S, B, calls):
    from rl_replicas_b200.algorithms import LearnerGroup
    from rl_replicas_b200.utils import set_seed_for_libraries
    solo = []
    for k in range(K):
        m = _member(k, path)
        set_seed_for_libraries(50 + k)
        for _ in range(calls):
            m.train(m.replay_buffer, S, B)
        solo.append(m)
    g = LearnerGroup()
    grouped = [_member(k, path) for k in range(K)]
    for k, m in enumerate(grouped):
        set_seed_for_libraries(50 + k)
        g.add(m)
    for _ in range(calls):
        g.train(S, B)
    for k, (a, b) in enumerate(zip(solo, grouped)):
        assert a.last_train_output.keys() == b.last_train_output.keys()
        for key in a.last_train_output:
            np.testing.assert_array_equal(a.last_train_output[key], b.last_train_output[key], err_msg=f"{key} {k}")
        for i, (x, y) in enumerate(zip(_state(a), _state(b))):
            np.testing.assert_array_equal(x, y, err_msg=f"member {k} tensor {i}")


@pytest.mark.parametrize("path", ["host", "gather", "rng"])
def test_group_of_three_is_bit_identical_to_solo_engines(path):
    _check_group(path, 3, 5, 40, 2)


def test_group_of_sixteen_is_bit_identical_to_solo_engines():
    _check_group("gather", 16, 3, 32, 1)


# ---- refusals, launches and end to end ------------------------------------------------------------------------------
def test_engine_refuses_bad_redq_configurations():
    from rl_replicas_b200 import _lib
    from rl_replicas_b200._lib import B200RLError, OffPolicyHparams
    from rl_replicas_b200.engine import OffPolicyEngine as E
    acts = ("relu", "identity")
    P, Q = [5, 16, 4], [7, 16, 1]
    with pytest.raises(B200RLError, match="algo must be"):
        E(P, Q, 2, 8, 2, acts, acts, algo=E.REDQ)  # create / create_group refuse algo 10
    with pytest.raises(B200RLError, match="algo must be 10"):
        E(P, Q, 2, 8, 2, acts, acts, algo=E.SAC, redq=(4, 2))
    with pytest.raises(B200RLError, match="REDQ needs n_q = 2"):
        E(P, Q, 1, 8, 2, acts, acts, algo=E.REDQ, redq=(4, 2))
    for N, M in ((1, 1), (33, 2), (4, 0), (4, 5)):
        with pytest.raises(B200RLError, match="offpolicy_create_redq"):
            E(P, Q, 2, 8, 2, acts, acts, algo=E.REDQ, redq=(N, M))
    with pytest.raises(B200RLError, match="critics must map"):
        E(P, [7, 16, 3], 2, 8, 2, acts, acts, algo=E.REDQ, redq=(4, 2))
    with pytest.raises(B200RLError, match="policy must map"):
        E([5, 16, 3], Q, 2, 8, 2, acts, acts, algo=E.REDQ, redq=(4, 2))
    with pytest.raises(B200RLError, match="REDQ takes neither dueling_k"):
        E(P, Q, 2, 8, 2, acts, acts, algo=E.REDQ, redq=(4, 2), noisy_layers=1)
    e = E(P, Q, 2, 8, 2, acts, acts, algo=E.REDQ, redq=(4, 2))
    layout, _ = e.state_layout()
    assert [i for kind, i, _, _ in layout if kind == "params"] == list(range(9))
    assert [i for kind, i, _, _ in layout if kind == "m"] == list(range(5))
    z = lambda *s: np.zeros(s, np.float32)
    hp = OffPolicyHparams()
    hp.policy_delay = 1
    with pytest.raises(B200RLError, match="set_sac"):
        e.train(hp, z(2, 8, 5), z(2, 8, 2), z(2, 8), z(2, 8, 5), z(2, 8), z(2, 2, 8, 2))
    from rl_replicas_b200._lib import SacHparams
    sp = SacHparams()
    sp.alpha, sp.log_std_min, sp.log_std_max = 0.2, -20.0, 2.0
    e.set_sac(sp)
    with pytest.raises(B200RLError, match="set_redq_subsets"):
        e.train(hp, z(2, 8, 5), z(2, 8, 2), z(2, 8), z(2, 8, 5), z(2, 8), z(2, 2, 8, 2))
    with pytest.raises(B200RLError, match="distinct"):
        e.set_redq_subsets(np.array([[1, 1], [0, 2]], np.int32))
    with pytest.raises(B200RLError, match="distinct"):
        e.set_redq_subsets(np.array([[0, 4], [0, 2]], np.int32))
    e.set_redq_subsets(np.array([[0, 3], [2, 1]], np.int32))
    hp.q1_lr, hp.q2_lr = 1e-3, 3e-4
    with pytest.raises(B200RLError, match="one learning rate"):
        e.train(hp, z(2, 8, 5), z(2, 8, 2), z(2, 8), z(2, 8, 5), z(2, 8), z(2, 2, 8, 2))
    e.set_adam(3, None, None, 5)
    hp.q2_lr = hp.q1_lr
    with pytest.raises(B200RLError, match="one Adam step count"):
        e.train(hp, z(2, 8, 5), z(2, 8, 2), z(2, 8), z(2, 8, 5), z(2, 8), (z(2, 2, 8, 2), np.array([[0, 3], [2, 1]])))
    for call in (lambda: e.set_dqn(1, False), lambda: e.set_c51(5, -1.0, 1.0), lambda: e.set_qr(3),
                 lambda: e.set_per(0.6, 1e-6, 0.4, 100), lambda: e.set_nstep(1), lambda: e.set_noise_keys([1], [1]),
                 lambda: e.set_cql(1.0, 1.0), lambda: e.set_iql(0.7, 3.0, 100.0, -5.0, 2.0, 3e-4)):
        with pytest.raises(B200RLError, match="REDQ"):
            call()
    rows = 16
    cols = [torch.zeros(rows, 5, device="cuda"), torch.zeros(rows, 2, device="cuda"), torch.zeros(rows, device="cuda"),
            torch.zeros(rows, 5, device="cuda"), torch.zeros(rows, device="cuda")]
    tree = torch.zeros(int(_lib.load().b200rl_per_tree_floats(rows)), device="cuda")
    with pytest.raises(B200RLError, match="REDQ engines"):
        e.train_prioritized(OffPolicyHparams(), cols, rows, tree, 2, 8, 0, 1)
    sac = E(P, Q, 2, 8, 2, acts, acts, algo=E.SAC)
    sac.redq = (4, 2)  # lets the binding shape the call: the engine itself must refuse
    with pytest.raises(B200RLError, match="algo = 10"):
        sac.set_redq_subsets(np.array([[0, 1]], np.int32))


def _launches(algo, S, B, graph):
    from rl_replicas_b200 import _lib
    lib = _lib.load()
    os.environ["B200RL_OFFPOLICY_GRAPH"] = "1" if graph else "0"
    try:
        np.random.seed(0)
        algo.train(algo.replay_buffer, S, B)  # builds the engine (and the graph)
        n0 = lib.b200rl_launch_count()
        algo.train(algo.replay_buffer, S, B)
        return lib.b200rl_launch_count() - n0
    finally:
        os.environ.pop("B200RL_OFFPOLICY_GRAPH", None)


def test_launches_per_step_are_the_stated_ones():
    """b200rl.h: 1 per call, then 4 Lq + Lp + 4 per step plus 2 Lq + 3 Lp + 3 (+1 with a learned temperature) per
    policy step, whatever N and M; host-staged minibatches launch nothing else."""
    S, B = 7, 32
    O, A, _, _, L, _ = SHAPES["small_tanh"]
    for learn_alpha in (False, True):
        for graph in (False, True):
            for N, M in ((3, 1), (12, 5)):
                algo = build("small_tanh", n=N, n_min=M, delay=3, learn_alpha=learn_alpha)
                fill(algo.replay_buffer, O, A, L, n=500, seed=6)
                algo.use_device_replay = False
                n_pol = len(OR.policy_steps(S, 3))  # steps 2, 5 and 6
                want = 1 + S * (4 * 3 + 3 + 4) + n_pol * (2 * 3 + 3 * 3 + 3 + int(learn_alpha))
                assert _launches(algo, S, B, graph) == want, (learn_alpha, graph, N, M)


def test_learn_solves_the_bandit(tmp_path, capsys):
    """REDQ.learn end to end on the one-step bandit of tests/test_sac.py with the seeds the oracle-driven loop in
    tests/test_redq.py used: the per-critic tags are recorded, model.pt is written and reloads, and the evaluation
    return clears the same bar."""
    np.random.seed(0)
    algo = make_redq(n=5, n_min=2, policy_delay=5, learn_alpha=True)
    algo.learn(output_dir=str(tmp_path), **REDQ_LEARN)
    after = evaluation_return(algo)
    printed = capsys.readouterr().out
    with capsys.disabled():
        print(f"REDQ.learn on the bandit: evaluation return {after:.3f}")
    for tag in ("policy/average_loss", "policy/average_log_prob", "alpha/value", "q-function_1/average_loss",
                "q-function_5/average_loss", "q-function_5/avarage_q-value", "evaluation/average_episode_return"):
        assert f"\n{tag}: " in printed, tag
    path = os.path.join(tmp_path, "model.pt")
    assert os.path.exists(path)
    other = make_redq(n=5, n_min=2, policy_delay=5, seed=5, learn_alpha=True)
    other.load_model(path)
    assert evaluation_return(other) == after
    assert after > RETURN_BAR
