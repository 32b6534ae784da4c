"""GPU: EDAC.train on the off-policy engine against the torch-autograd oracle (oracle/edac.py), one step against the
float64 stages, eta = 0 against a REDQ engine with every critic in the target, bit-identical results across its
execution paths and in learner groups, the engine's refusals, the launches per step b200rl.h states, and
EDAC.learn_offline end to end."""
import os
import types

import numpy as np
import pytest
import torch

from conftest import rel_err
from oracle import edac as OE
from test_edac import OFFLINE_BAR, OFFLINE_ETA, OFFLINE_N, make_edac
from test_cql import OFFLINE
from test_gpu_sac import adam_flat, fill, flat
from test_sac import evaluation_return

pytestmark = pytest.mark.gpu

SHAPES = {  # (obs, act, hidden widths, hidden activation, action limit, minibatch)
    "halfcheetah": (17, 6, (256, 256), torch.nn.ReLU, 1.0, 256),
    "small_relu": (5, 2, (64, 64), torch.nn.ReLU, 2.0, 64),
    "ragged": (7, 3, (50, 37), torch.nn.ReLU, 1.0, 45),  # widths and minibatch off the 32-wide GEMM tiles
    "deep": (5, 2, (64, 48, 40), torch.nn.ReLU, 1.0, 64),  # three hidden layers: three ones-backward buffers
    "small_tanh": (5, 2, (64, 64), torch.nn.Tanh, 2.0, 64),
}


def _env(A, L):
    hi = np.full(A, L, np.float32)
    return types.SimpleNamespace(action_space=types.SimpleNamespace(high=hi, low=-hi, shape=(A,)),
                                 spec=types.SimpleNamespace(id="stub"))


def build(shape, n=10, eta=1.0, seed=0, learn_alpha=True, cls=None, **kw):
    from rl_replicas_b200.algorithms import EDAC
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import RandomPolicy, SquashedGaussianPolicy
    from rl_replicas_b200.q_function import QFunction
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    O, A, H, act, L, _ = SHAPES[shape]
    torch.manual_seed(seed)
    pnet = MLP([O, 64, 64, 2 * A], torch.nn.ReLU) if shape == "deep" else MLP([O, *H, 2 * A], act)
    qs = [MLP([O + A, *H, 1], act) for _ in range(n)]
    policy = SquashedGaussianPolicy(pnet, torch.optim.Adam(pnet.parameters(), lr=1e-3), action_limit=L)
    critics = [QFunction(q, torch.optim.Adam(q.parameters(), lr=1e-3)) for q in qs]
    if cls is None:
        algo = EDAC(policy, RandomPolicy(None), critics, _env(A, L), None, ReplayBuffer(), None, learn_alpha=learn_alpha,
                    alpha_lr=3e-3, eta=eta)
    else:
        algo = cls(policy, RandomPolicy(None), critics, _env(A, L), None, ReplayBuffer(), None, learn_alpha=learn_alpha,
                   alpha_lr=3e-3, **kw)
    algo.metrics_manager = None
    algo.current_total_steps = 0
    return algo


def oracle_for(algo):
    return OE.EdacOracle(algo.policy.network, [q.network for q in algo.q_functions], gamma=algo.gamma,
                         rho=algo.polyak_rho, alpha=algo.alpha, learn_alpha=algo.learn_alpha,
                         target_entropy=algo.target_entropy, alpha_lr=3e-3, limit=algo.policy.action_limit,
                         eta=algo.eta)


def compare(algo, oracle, logs, out):
    """{name: norm-wise error} of every logged quantity and every tensor of the learner against the oracle."""
    errs = {"q_values": rel_err(out["redq_q_values"], np.asarray(logs["q_values"])),
            "q_losses": rel_err(out["redq_q_losses"], np.asarray(logs["q_losses"]))}
    for k in ("policy_losses", "log_prob_means", "alphas"):
        errs[k] = rel_err(out[k], np.asarray(logs[k]))
    if algo.eta > 0:
        errs["diversity"] = rel_err(out["edac_diversity"], np.asarray(logs["diversity"]))
    else:
        assert (out["edac_diversity"] == 0).all()
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
    """algo.train, then the oracle on the same minibatches and noise (the host streams replayed)."""
    oracle = oracle_for(algo)
    np.random.seed(seed)
    torch.manual_seed(seed)
    state_np, state_t = np.random.get_state(), torch.get_rng_state()
    algo.train(algo.replay_buffer, S, B)
    np.random.set_state(state_np)
    torch.set_rng_state(state_t)
    mbs = [algo.replay_buffer.sample_minibatch(B) for _ in range(S)]
    return oracle, oracle.train(mbs, algo._noise(S, B))


LOGGED = ("q_values", "q_losses", "policy_losses", "log_prob_means", "alphas", "diversity", "log_alpha")
# (shape, N, eta, S, learn_alpha, tensor bound, logged bound).  The engine and the oracle round differently (fma chains,
# a double-precision diversity head against float32 autograd), and at ReLU shapes a pre-activation within rounding of
# its kink can decide whether one row's gradient passes; Adam turns such a one-row difference on a unit with a tiny
# exp_avg_sq into an lr-sized step (test_gpu_sac.py, test_gpu_redq.py).  The diversity term adds a second way in: its
# u_k carries 1 / |g_k|, so a row whose action gradient is near 0 amplifies rounding.  Measured on an H100 (700 W): at
# the HalfCheetah shape the largest tensor error over 12 steps was 3.9e-3 (eta = 1, critic 1 and the policy's exp_avg,
# the kink mechanism) and 2.9e-3 (eta = 5), the logged values 1.2e-4 and 2.1e-5; every smaller shape stayed below
# 6.4e-6 for tensors and 4.4e-7 for logged values, small_tanh (eta = 0) below 1.3e-6.  Bounded at about 3x / 10x those.
CASES = [("halfcheetah", 10, 1.0, 12, True, 1e-2, 5e-4), ("halfcheetah", 10, 5.0, 12, True, 1e-2, 5e-4),
         ("small_relu", 5, 1.0, 10, True, 5e-5, 5e-6), ("ragged", 4, 2.0, 8, True, 5e-5, 5e-6),
         ("deep", 4, 1.0, 8, False, 5e-5, 5e-6), ("small_relu", 2, 1.0, 8, True, 5e-5, 5e-6),
         ("small_relu", 32, 1.0, 6, False, 5e-5, 5e-6), ("small_tanh", 6, 0.0, 10, True, 2e-5, 5e-6)]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "-".join(str(x) for x in c[:5]))
def test_train_matches_the_oracle(case):
    shape, N, eta, S, learn_alpha, tol, tol_logged = case
    O, A, H, act, L, B = SHAPES[shape]
    algo = build(shape, n=N, eta=eta, learn_alpha=learn_alpha)
    fill(algo.replay_buffer, O, A, L)
    oracle, logs = _train_and_replay(algo, S, B)
    out = algo.last_train_output
    assert len(out["policy_losses"]) == S == len(logs["policy_losses"])
    errs = compare(algo, oracle, logs, out)
    print(case[:5], "max tensor", max(v for k, v in errs.items() if k not in LOGGED),
          "max logged", max(v for k, v in errs.items() if k in LOGGED),
          {k: f"{v:.2e}" for k, v in errs.items() if v > 1e-6})
    for k, v in errs.items():
        assert v < (tol_logged if k in LOGGED else tol), (k, v)
    if eta > 0:  # sum_{i != j} gh_i . gh_j = |sum_i gh_i|^2 - sum_i |gh_i|^2 lies in [-N, N (N - 1)] per row
        assert np.all(out["edac_diversity"] >= -N / (N - 1) - 1e-5) and np.all(out["edac_diversity"] <= N + 1e-5)
    if not learn_alpha:
        assert (out["alphas"] == np.float32(0.2)).all()


def test_one_step_against_the_float64_reference():
    """One step at the HalfCheetah shape: every critic's values, TD loss and first Adam step (the sign of the float64
    gradient of TD loss + eta D), D, and the policy loss and mean log pi (with
    the critics the engine updated), against float64 stages at the engine's parameters and draws."""
    O, A, H, _, L, B = SHAPES["halfcheetah"]
    N, eta = 10, 1.0
    algo = build("halfcheetah", n=N, eta=eta, learn_alpha=False)
    fill(algo.replay_buffer, O, A, L, n=3000, seed=8)
    f64 = lambda m: flat(m.network).astype(np.float64)
    nets = dict(policy=f64(algo.policy), q=[f64(q) for q in algo.q_functions],
                target_q=[f64(q) for q in algo.target_q_functions])
    before = [flat(q.network).copy() for q in algo.q_functions]
    np.random.seed(9)
    torch.manual_seed(9)
    state_np, state_t = np.random.get_state(), torch.get_rng_state()
    algo.train(algo.replay_buffer, 1, B)
    out = algo.last_train_output
    np.random.set_state(state_np)
    torch.set_rng_state(state_t)
    mb = algo.replay_buffer.sample_minibatch(B)
    noise = algo._noise(1, B)
    psz, qsz = [O, *H, 2 * A], [O + A, *H, 1]
    c = OE.critic_stage_f64(nets, mb, noise[0, 0], 0.2, eta, psz, qsz, gamma=algo.gamma, action_limit=L)
    assert rel_err(out["edac_diversity"][0], c["diversity"]) < 1e-5
    for k in range(N):
        assert rel_err(out["redq_q_values"][k][0], c["values"][k]) < 1e-5
        assert rel_err(out["redq_q_losses"][k][0], c["losses"][k]) < 1e-5
        # a first Adam step moves each parameter by -lr g / (|g| + eps): lr sign(g) wherever g is clearly nonzero
        moved = flat(algo.q_functions[k].network).astype(np.float64) - before[k]
        g = c["grads"][k]
        clear = np.abs(g) > 1e-3 * np.abs(g).max()
        np.testing.assert_allclose(moved[clear], -1e-3 * np.sign(g[clear]), rtol=1e-3, atol=1e-6)
    qs_new = [flat(q.network).astype(np.float64) for q in algo.q_functions]
    p = OE.policy_stage_f64(nets["policy"], qs_new, mb["observations"], noise[0, 1], 0.2, psz, qsz, action_limit=L)
    assert rel_err(out["policy_losses"][0], p["loss"]) < 1e-5
    assert rel_err(out["log_prob_means"][0], p["logp_mean"]) < 1e-5


def test_eta_zero_first_critic_step_is_redq_with_every_critic_bit_for_bit():
    """eta = 0 (SAC-N) against a REDQ engine with N = M, G = 1 and the subsets 0..N-1: the first step's critic values,
    losses, critics, their Adam moments and the target critics agree bit for bit."""
    from rl_replicas_b200.algorithms import REDQ
    O, A, _, _, L, B = SHAPES["halfcheetah"]
    N = 6
    edac = build("halfcheetah", n=N, eta=0.0)
    redq = build("halfcheetah", n=N, cls=REDQ, n_min=N, policy_delay=1)
    redq._noise = lambda S, B_: (edac._noise(S, B_), np.tile(np.arange(N, dtype=np.int32), (S, 1)))
    for a in (edac, redq):
        fill(a.replay_buffer, O, A, L, n=3000, seed=5)
        np.random.seed(3)
        torch.manual_seed(3)
        a.train(a.replay_buffer, 1, B)
    e, r = edac.last_train_output, redq.last_train_output
    for k in ("q1_values", "q2_values", "q1_losses", "q2_losses", "redq_q_values", "redq_q_losses"):
        np.testing.assert_array_equal(e[k], r[k], err_msg=k)
    for qe, qr in zip(edac.q_functions + edac.target_q_functions, redq.q_functions + redq.target_q_functions):
        np.testing.assert_array_equal(flat(qe.network), flat(qr.network))
    for qe, qr in zip(edac.q_functions, redq.q_functions):
        for key in ("exp_avg", "exp_avg_sq"):
            np.testing.assert_array_equal(adam_flat(qe.optimizer, key)[0], adam_flat(qr.optimizer, key)[0])


def _run_paths(device_replay, graph, rng=False):
    O, A, _, _, L, _ = SHAPES["small_relu"]
    os.environ["B200RL_OFFPOLICY_GRAPH"] = "1" if graph else "0"
    try:
        algo = build("small_relu", n=6, eta=2.0, learn_alpha=True)
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


# ---- learner groups -------------------------------------------------------------------------------------------------
def _member(k, path):
    O, A, _, _, L, _ = SHAPES["small_relu"]
    algo = build("small_relu", n=5, eta=1.5, seed=k, learn_alpha=True)
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


def test_group_members_share_one_dataset_buffer():
    """Offline members may share one ReplayBuffer.from_dataset: each still ends where it would alone."""
    from rl_replicas_b200.algorithms import LearnerGroup
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    from test_iql import mixed_dataset
    from rl_replicas_b200.utils import set_seed_for_libraries
    rb = ReplayBuffer.from_dataset(mixed_dataset(4000))
    solo = []
    for k in range(2):
        m = make_edac(n=4, hidden=32, seed=k, eta=2.0)
        m.replay_buffer = rb
        set_seed_for_libraries(60 + k)
        m.train(rb, 6, 32)
        solo.append(m)
    g = LearnerGroup()
    grouped = []
    for k in range(2):
        m = make_edac(n=4, hidden=32, seed=k, eta=2.0)
        m.replay_buffer = rb
        set_seed_for_libraries(60 + k)
        g.add(m)
        grouped.append(m)
    g.train(6, 32)
    for a, b in zip(solo, grouped):
        for x, y in zip(_state(a), _state(b)):
            np.testing.assert_array_equal(x, y)


# ---- refusals, launches and end to end ------------------------------------------------------------------------------
def test_engine_refuses_bad_edac_configurations():
    from rl_replicas_b200 import _lib
    from rl_replicas_b200._lib import B200RLError, OffPolicyHparams, SacHparams
    from rl_replicas_b200.engine import OffPolicyEngine as E
    acts = ("relu", "identity")
    P, Q = [5, 16, 4], [7, 16, 1]
    with pytest.raises(B200RLError, match="algo must be"):
        E(P, Q, 2, 8, 2, acts, acts, algo=E.EDAC)  # create / create_group refuse algo 11
    with pytest.raises(B200RLError, match="algo must be"):
        E(P, Q, 2, 8, 2, acts, acts, algo=E.EDAC, redq=(4, 4))  # so does create_redq
    with pytest.raises(B200RLError, match="algo must be 11"):
        E(P, Q, 2, 8, 2, acts, acts, algo=E.SAC, edac=(4, 1.0))
    with pytest.raises(B200RLError, match="EDAC needs n_q = 2"):
        E(P, Q, 1, 8, 2, acts, acts, algo=E.EDAC, edac=(4, 1.0))
    for N, eta in ((1, 1.0), (33, 1.0), (4, -0.5), (4, float("nan")), (4, float("inf"))):
        with pytest.raises(B200RLError, match="offpolicy_create_edac"):
            E(P, Q, 2, 8, 2, acts, acts, algo=E.EDAC, edac=(N, eta))
    with pytest.raises(B200RLError, match="critics must map"):
        E(P, [7, 16, 3], 2, 8, 2, acts, acts, algo=E.EDAC, edac=(4, 1.0))
    with pytest.raises(B200RLError, match="policy must map"):
        E([5, 16, 3], Q, 2, 8, 2, acts, acts, algo=E.EDAC, edac=(4, 1.0))
    with pytest.raises(B200RLError, match="EDAC takes neither dueling_k"):
        E(P, Q, 2, 8, 2, acts, acts, algo=E.EDAC, edac=(4, 1.0), noisy_layers=1)
    with pytest.raises(B200RLError, match="ReLU hidden layers"):
        E(P, Q, 2, 8, 2, acts, ("tanh", "identity"), algo=E.EDAC, edac=(4, 1.0))
    with pytest.raises(B200RLError, match="ReLU hidden layers"):
        E(P, Q, 2, 8, 2, acts, ("relu", "tanh"), algo=E.EDAC, edac=(4, 1.0))
    E(P, Q, 2, 8, 2, acts, ("tanh", "identity"), algo=E.EDAC, edac=(4, 0.0)).close()  # SAC-N takes any
    e = E(P, Q, 2, 8, 2, acts, acts, algo=E.EDAC, edac=(4, 1.0))
    layout, _ = e.state_layout()
    assert [i for kind, i, _, _ in layout if kind == "params"] == list(range(9))
    assert [i for kind, i, _, _ in layout if kind == "m"] == list(range(5))
    z = lambda *s: np.zeros(s, np.float32)
    hp = OffPolicyHparams()
    hp.policy_delay = 1
    with pytest.raises(B200RLError, match="set_sac"):
        e.train(hp, z(2, 8, 5), z(2, 8, 2), z(2, 8), z(2, 8, 5), z(2, 8), z(2, 2, 8, 2))
    sp = SacHparams()
    sp.alpha, sp.log_std_min, sp.log_std_max = 0.2, -20.0, 2.0
    e.set_sac(sp)
    hp.q1_lr, hp.q2_lr = 1e-3, 3e-4
    with pytest.raises(B200RLError, match="one learning rate"):
        e.train(hp, z(2, 8, 5), z(2, 8, 2), z(2, 8), z(2, 8, 5), z(2, 8), z(2, 2, 8, 2))
    hp.q2_lr = hp.q1_lr
    e.train(hp, z(2, 8, 5), z(2, 8, 2), z(2, 8), z(2, 8, 5), z(2, 8), z(2, 2, 8, 2))  # no subsets needed
    assert e.edac_outputs(2).shape == (2,)
    e.redq = (4, 4)  # lets the binding shape the calls: the engine itself must refuse
    for call in (lambda: e.set_redq_subsets(np.array([[0, 1, 2, 3]], np.int32)), lambda: e.get_redq_subsets(1),
                 lambda: e.set_dqn(1, False), lambda: e.set_c51(5, -1.0, 1.0), lambda: e.set_qr(3),
                 lambda: e.set_per(0.6, 1e-6, 0.4, 100), lambda: e.set_nstep(1), lambda: e.set_noise_keys([1], [1]),
                 lambda: e.set_cql(1.0, 1.0), lambda: e.set_iql(0.7, 3.0, 100.0, -5.0, 2.0, 3e-4)):
        with pytest.raises(B200RLError, match="EDAC|algo = 10"):
            call()
    rows = 16
    cols = [torch.zeros(rows, 5, device="cuda"), torch.zeros(rows, 2, device="cuda"), torch.zeros(rows, device="cuda"),
            torch.zeros(rows, 5, device="cuda"), torch.zeros(rows, device="cuda")]
    tree = torch.zeros(int(_lib.load().b200rl_per_tree_floats(rows)), device="cuda")
    with pytest.raises(B200RLError, match="EDAC engines"):
        e.train_prioritized(OffPolicyHparams(), cols, rows, tree, 2, 8, 0, 1)
    sac = E(P, Q, 2, 8, 2, acts, acts, algo=E.SAC)
    with pytest.raises(B200RLError, match="EDAC engine"):
        sac.edac_outputs(0)


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
    """b200rl.h: 1 per call, then 6 Lq + 4 Lp + 7 per step (+1 with a learned temperature), plus 3 Lq with eta > 0:
    37 (38) and 46 (47) at two hidden layers, whatever N; host-staged minibatches launch nothing else."""
    S, B = 5, 32
    for shape, Lq, Lp in (("small_relu", 3, 3), ("deep", 4, 3)):
        O, A, _, _, L, _ = SHAPES[shape]
        for learn_alpha in (False, True):
            for eta in (0.0, 1.0):
                for graph in (False, True):
                    for N in (3, 12):
                        algo = build(shape, n=N, eta=eta, learn_alpha=learn_alpha)
                        fill(algo.replay_buffer, O, A, L, n=500, seed=6)
                        algo.use_device_replay = False
                        per_step = 6 * Lq + 4 * Lp + 7 + int(learn_alpha) + (3 * Lq if eta > 0 else 0)
                        if shape == "small_relu":
                            assert per_step == (37 if eta == 0 else 46) + int(learn_alpha)
                        assert _launches(algo, S, B, graph) == 1 + S * per_step, (shape, learn_alpha, eta, graph, N)


def _mean_gradient_cosine(algo, n=2000):
    """The mean pairwise cosine similarity of the critics' action gradients at n dataset rows."""
    d = algo.replay_buffer
    idx = np.arange(n)
    cols = d.gather(idx)
    o = torch.as_tensor(np.asarray(cols["observations"], np.float32))
    a = torch.as_tensor(np.asarray(cols["actions"], np.float32))
    _, g = OE.action_gradients([q.network for q in algo.q_functions], o, a, create_graph=False)
    gh = g / (g.norm(dim=2, keepdim=True) + OE.NORM_EPS)
    N = g.shape[0]
    cos = torch.einsum("ibk,jbk->bij", gh, gh) * (1 - torch.eye(N))
    return float(cos.sum() / (n * N * (N - 1)))


def test_learn_offline_diversifies_the_critics(tmp_path, capsys):
    """EDAC.learn_offline end to end on tests/test_iql.py's mixed dataset with the seeds the oracle-driven run in
    tests/test_edac.py used: the tags are recorded, model.pt is written, the return clears that run's bar, and the
    critics' dataset-action gradients end less aligned than SAC-N's (eta = 0) under the same seeds."""
    runs = {}
    for eta in (OFFLINE_ETA, 0.0):
        np.random.seed(0)
        torch.manual_seed(0)
        algo = make_edac(n=OFFLINE_N, eta=eta)
        algo.learn_offline(output_dir=str(tmp_path / str(eta)), **OFFLINE)
        runs[eta] = (algo, evaluation_return(algo), _mean_gradient_cosine(algo))
    printed = capsys.readouterr().out
    with capsys.disabled():
        print("EDAC.learn_offline: return / mean gradient cosine", {k: v[1:] for k, v in runs.items()})
    for tag in ("policy/average_loss", "alpha/value", "q-function_5/average_loss", "edac/diversity_loss",
                "evaluation/average_episode_return"):
        assert f"\n{tag}: " in printed, tag
    assert os.path.exists(tmp_path / str(OFFLINE_ETA) / "model.pt")
    assert runs[OFFLINE_ETA][1] > OFFLINE_BAR
    assert runs[OFFLINE_ETA][2] < runs[0.0][2]
