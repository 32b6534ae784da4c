"""GPU: TQC.train on the off-policy engine against the torch-autograd oracle (oracle/tqc.py) and the float64
reference, bit-identical results across its execution paths and in learner groups, the device-side draws, the
engine's refusals, the launches per step b200rl.h states, and TQC.learn end to end."""
import os

import numpy as np
import pytest
import torch

from conftest import rel_err
from oracle import tqc as OT
from test_gpu_sac import adam_flat, compare, fill, flat
from test_sac import LEARN, RETURN_BAR, evaluation_return
from test_tqc import make_tqc, oracle_for

pytestmark = pytest.mark.gpu

SHAPES = {  # (obs, act, hidden, hidden activation, action limit, minibatch, M, d)
    "halfcheetah": (17, 6, 256, torch.nn.ReLU, 1.0, 256, 25, 2),
    "small_tanh": (5, 2, 64, torch.nn.Tanh, 2.0, 64, 5, 1),
}


def build(shape, seed=0, learn_alpha=False, clamp_rows=False, M=None, d=None, **kw):
    from rl_replicas_b200.algorithms import TQC
    from rl_replicas_b200.critics import ContinuousQuantileQFunction
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import RandomPolicy, SquashedGaussianPolicy
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    import types
    O, A, H, act, L, _, M0, d0 = SHAPES[shape]
    M, d = M0 if M is None else M, d0 if d is None else d
    torch.manual_seed(seed)
    pnet = MLP([O, H, H, 2 * A], act)
    if clamp_rows:  # log_std above log_std_max = 2 on part of the batch: the clamp's zero gradient is exercised
        with torch.no_grad():
            pnet.network[-2].weight[A:] *= 8.0
            pnet.network[-2].bias[A:] = 1.9
    q1, q2 = MLP([O + A, H, H, M], act), MLP([O + A, H, H, M], act)
    hi = np.full(A, L, np.float32)
    env = types.SimpleNamespace(action_space=types.SimpleNamespace(high=hi, low=-hi, shape=(A,)),
                                spec=types.SimpleNamespace(id="stub"))
    algo = TQC(SquashedGaussianPolicy(pnet, torch.optim.Adam(pnet.parameters(), lr=1e-3), action_limit=L),
               RandomPolicy(None),
               ContinuousQuantileQFunction(q1, torch.optim.Adam(q1.parameters(), lr=1e-3), n_quantiles=M),
               ContinuousQuantileQFunction(q2, torch.optim.Adam(q2.parameters(), lr=1e-3), n_quantiles=M), env, None,
               ReplayBuffer(), None, learn_alpha=learn_alpha, alpha_lr=3e-3, top_quantiles_to_drop_per_net=d, **kw)
    algo.metrics_manager = None
    algo.current_total_steps = 0
    return algo


def run_against_oracle(algo, S, B, calls=3):
    """``calls`` TQC.train calls of S steps and the oracle fed the same minibatches and noise; the worst error of each
    logged or stored quantity over the calls."""
    A = algo.action_dim
    oracle = OT.TqcOracle(algo.policy.network, algo.q_function_1.network, algo.q_function_2.network,
                          n_quantiles=algo.q_function_1.n_quantiles, n_drop=algo.top_quantiles_to_drop_per_net,
                          gamma=algo.gamma, rho=algo.polyak_rho, alpha=algo.alpha, learn_alpha=algo.learn_alpha,
                          target_entropy=algo.target_entropy, alpha_lr=3e-3, limit=algo.policy.action_limit)
    worst = {}
    for call in range(calls):
        np.random.seed(7 + call)
        torch.manual_seed(7 + call)
        state_np, state_t = np.random.get_state(), torch.get_rng_state()
        algo.train(algo.replay_buffer, S, B)
        out = algo.last_train_output
        np.random.set_state(state_np)
        torch.set_rng_state(state_t)
        mbs = [algo.replay_buffer.sample_minibatch(B) for _ in range(S)]
        noise = torch.stack([torch.stack([torch.randn(B, A), torch.randn(B, A)]) for _ in range(S)]).numpy()
        logs = oracle.train(mbs, noise)
        assert len(out["policy_losses"]) == S
        for k, v in compare(algo, oracle, logs, out).items():
            worst[k] = max(worst.get(k, 0.0), v)
    return worst


@pytest.mark.parametrize("learn_alpha", [False, True])
@pytest.mark.parametrize("shape", ["halfcheetah", "small_tanh"])
def test_train_matches_the_oracle(shape, learn_alpha):
    """Three calls of six steps through TQC.train (device replay, graph replay) against the autograd oracle with the
    same minibatches and noise.  small_tanh starts with log_std above the clamp on part of the batch."""
    O, A, H, act, L, B, M, d = SHAPES[shape]
    algo = build(shape, learn_alpha=learn_alpha, clamp_rows=shape == "small_tanh")
    fill(algo.replay_buffer, O, A, L)
    worst = run_against_oracle(algo, 6, B)
    print(f"{shape} learn_alpha={learn_alpha}:", {k: f"{v:.1e}" for k, v in worst.items()})
    # Measured on H100 at the HalfCheetah shape (256-wide ReLU layers): every logged quantity (losses, Q-values, log pi,
    # alpha) stays below 3e-7 of its maximum, but the networks and their Adam moments drift to 2.3e-5 (learned alpha)
    # and 1.0e-3 (fixed alpha) of their maximum over the 18 steps.  Rows of these minibatches have hidden
    # pre-activations within 2e-8 (relative) of a ReLU kink, where float rounding decides whether a row's gradient
    # passes, and Adam's first steps normalise each entry by its own magnitude, so a rounding-level difference in a
    # small gradient entry becomes a difference of a fraction of lr in its step.  The Tanh shape has no kinks and stays
    # below 1e-6 here; test_one_step_against_the_float64_reference holds every gradient to 2e-5 on rows clear of the kinks.
    drift = {"policy", "q1", "q2", "target_q1", "target_q2"} | {f"{n}.{m}" for n in ("policy", "q1", "q2")
                                                                  for m in ("exp_avg", "exp_avg_sq")}
    for k, v in worst.items():
        assert v < (1e-2 if shape == "halfcheetah" and k in drift else 2e-5), (k, v, worst)
    if not learn_alpha:
        assert (algo.last_train_output["alphas"] == np.float32(0.2)).all()


@pytest.mark.parametrize("M,d", [(5, 0), (5, 4), (1, 0), (256, 3)])
def test_quantile_count_edges_match_the_oracle(M, d):
    """d = 0 (nothing dropped), d = M - 1 (one atom kept per critic), M = 1 and M = 256 (the largest head)."""
    O, A, _, _, L, _, _, _ = SHAPES["small_tanh"]
    algo = build("small_tanh", learn_alpha=True, M=M, d=d)
    fill(algo.replay_buffer, O, A, L, n=3000, seed=11)
    worst = run_against_oracle(algo, 4, 48, calls=2)
    print(f"M={M} d={d}:", {k: f"{v:.1e}" for k, v in worst.items()})
    for k, v in worst.items():
        assert v < 2e-5, (k, v, worst)


def test_one_step_against_the_float64_reference():
    """One step from fresh Adam states at the HalfCheetah shape: the critics' gradients (Adam's first moment over
    1 - beta1), losses and Q-values, the policy's loss, gradient and mean log pi, and the temperature's gradient
    against oracle/tqc.py's float64 stages, the policy stage fed the engine's own post-step critics.  The replay holds
    only rows whose ReLU pre-activations in every pass the step differentiates are at least 1e-5 (relative) away from
    0: a row at rounding distance from a kink may be gated differently by a float32 kernel, which is not an error of
    the kernel."""
    from oracle.offpolicy_f64 import _t, mlp, squash
    O, A, H, _, L, B, M, d = SHAPES["halfcheetah"]
    algo = build("halfcheetah", learn_alpha=True)
    psz, qsz = [O, H, H, 2 * A], [O + A, H, H, M]
    nets = dict(policy=flat(algo.policy.network), q1=flat(algo.q_function_1.network),
                q2=flat(algo.q_function_2.network), target_q1=flat(algo.target_q_function_1.network),
                target_q2=flat(algo.target_q_function_2.network))
    nets = {k: v.astype(np.float64) for k, v in nets.items()}
    rng = np.random.default_rng(2)
    n = 6 * B
    o, a = rng.standard_normal((n, O)), rng.uniform(-L, L, (n, A))
    o2, e2, e1 = rng.standard_normal((n, O)), rng.standard_normal((n, A)), rng.standard_normal((n, A))
    with torch.no_grad():  # margins of pi(s), pi(s'), the critics at (s, a), (s', a') and (s, a_pi)
        out2, m = mlp(_t(nets["policy"]), psz, _t(o2), "relu", "identity")
        a2, _ = squash(out2, _t(e2), L, -20.0, 2.0)
        out1, m1 = mlp(_t(nets["policy"]), psz, _t(o), "relu", "identity")
        a1, _ = squash(out1, _t(e1), L, -20.0, 2.0)
        m = torch.minimum(m, m1)
        for k in ("q1", "q2", "target_q1", "target_q2"):
            for x in (torch.cat([_t(o), _t(a)], -1), torch.cat([_t(o2), a2], -1), torch.cat([_t(o), a1], -1)):
                m = torch.minimum(m, mlp(_t(nets[k]), qsz, x, "relu", "identity")[1])
    keep = np.flatnonzero(m.numpy() >= 1e-5)[:B]
    assert len(keep) == B, len(keep)
    f32 = lambda x: np.asarray(x, np.float32)
    mb = dict(observations=f32(o[keep]), actions=f32(a[keep]), rewards=f32(rng.standard_normal(B)),
              next_observations=f32(o2[keep]), dones=rng.random(B) < 0.1)
    noise = np.stack([f32(e2[keep]), f32(e1[keep])])[None]
    e = algo._ensure_engine(1, B)
    algo._upload_state(e, *algo._learner_nets())
    hp = algo._hparams(True, 1)
    out = e.train(hp, mb["observations"][None], mb["actions"][None], mb["rewards"][None],
                  mb["next_observations"][None], mb["dones"].astype(np.float32)[None], noise)
    algo._download_state(e, *algo._learner_nets())
    alpha = float(np.float32(0.2))
    c = OT.critic_stage_f64(nets, mb, noise[0, 0].astype(np.float64), alpha, psz, qsz, M, d, action_limit=L)
    errs = {}
    for k, m_ in ((1, algo.q_function_1), (2, algo.q_function_2)):
        errs[f"q{k}_values"] = rel_err(out[f"q{k}_values"][0], c[f"q{k}_values"])
        errs[f"q{k}_loss"] = rel_err(out[f"q{k}_losses"][0], c[f"q{k}_loss"])
        errs[f"q{k}_grad"] = rel_err(adam_flat(m_.optimizer, "exp_avg")[0] / 0.1, c[f"q{k}_grad"])
    p = OT.policy_stage_f64(nets["policy"], flat(algo.q_function_1.network), flat(algo.q_function_2.network),
                            mb["observations"], noise[0, 1].astype(np.float64), alpha, psz, qsz, action_limit=L,
                            target_entropy=algo.target_entropy)
    errs["policy_loss"] = rel_err(out["policy_losses"][0], p["loss"])
    errs["logp_mean"] = rel_err(out["log_prob_means"][0], p["logp_mean"])
    errs["policy_grad"] = rel_err(adam_flat(algo.policy.optimizer, "exp_avg")[0] / 0.1, p["grad"])
    errs["alpha_grad"] = rel_err(adam_flat(algo.alpha_optimizer, "exp_avg")[0] / 0.1, p["alpha_grad"])
    print({k: f"{v:.1e}" for k, v in errs.items()})
    for k, v in errs.items():
        assert v < 2e-5, (k, v, errs)


def _run_paths(device_replay, graph, S=5, B=48):
    os.environ["B200RL_OFFPOLICY_GRAPH"] = "1" if graph else "0"
    try:
        O, A, _, _, L, _, _, _ = SHAPES["small_tanh"]
        algo = build("small_tanh", learn_alpha=True)
        fill(algo.replay_buffer, O, A, L, n=3000, seed=3)
        algo.use_device_replay = device_replay
        outs = []
        for call in range(3):
            np.random.seed(10 + call)
            torch.manual_seed(10 + call)
            algo.train(algo.replay_buffer, S + (call == 2), B)
            outs.append(algo.last_train_output)
        nets = [flat(m.network) for m in (algo.policy, algo.q_function_1, algo.q_function_2, algo.target_q_function_1,
                                          algo.target_q_function_2)]
        return outs, nets + [algo.log_alpha.detach().numpy().reshape(1)]
    finally:
        os.environ.pop("B200RL_OFFPOLICY_GRAPH", None)


def test_host_staged_graph_replay_and_device_gather_are_bit_identical():
    """Plain launches on host-staged minibatches, the captured graph replayed across calls (the third call changes S
    and recaptures) and the device-replay gather all agree bit for bit."""
    ref_outs, ref_nets = _run_paths(False, False)
    for dev, graph in ((True, True), (False, True), (True, False)):
        outs, nets = _run_paths(dev, graph)
        for a, b in zip(outs, ref_outs):
            assert a.keys() == b.keys()
            for k in a:
                np.testing.assert_array_equal(a[k], b[k], err_msg=f"{k} dev={dev} graph={graph}")
        for i, (a, b) in enumerate(zip(nets, ref_nets)):
            np.testing.assert_array_equal(a, b, err_msg=f"net {i} dev={dev} graph={graph}")


def test_device_side_draws_replay_through_the_oracle():
    O, A, _, _, L, _, _, _ = SHAPES["small_tanh"]
    S, B = 8, 64
    algo = build("small_tanh", learn_alpha=True)
    fill(algo.replay_buffer, O, A, L, n=3000, seed=4)
    algo.use_device_rng, algo.device_rng_seed = True, 77
    oracle = oracle_for(algo, alpha_lr=3e-3)
    algo.train(algo.replay_buffer, S, B)
    idx, noise = algo._engine.get_draws(S, B)
    assert idx.shape == (S, B) and noise.shape == (S, 2, B, A)
    rb = algo.replay_buffer
    logs = oracle.train([{k: rb._cols[k][idx[s]] for k in rb.COLUMNS} for s in range(S)], noise)
    errs = compare(algo, oracle, logs, algo.last_train_output)
    for k, v in errs.items():
        assert v < 2e-5, (k, v, errs)


# ---- learner groups -------------------------------------------------------------------------------------------------
def _member(k, path):
    O, A, _, _, L, _, _, _ = SHAPES["small_tanh"]
    algo = build("small_tanh", seed=k, learn_alpha=True)
    fill(algo.replay_buffer, O, A, L, n=2000, seed=30 + k)
    algo.use_device_replay = path != "host"
    algo.use_device_rng, algo.device_rng_seed = path == "rng", 90 + k
    if k % 2:  # members at different Adam step counts
        np.random.seed(k)
        torch.manual_seed(k)
        algo.train(algo.replay_buffer, k, 16)
    return algo


def _state(algo):
    out = [flat(m.network) for m in (algo.policy, algo.q_function_1, algo.q_function_2, algo.target_q_function_1,
                                     algo.target_q_function_2)]
    for m in (algo.policy, algo.q_function_1, algo.q_function_2):
        out += [adam_flat(m.optimizer, k)[0] for k in ("exp_avg", "exp_avg_sq")]
    return out + [np.asarray(algo._alpha_state(), np.float64)]


def _check_group(path, K, S, B, calls):
    """LearnerGroup.train against each member's own train: member k's private random stream starts from seed 50 + k,
    which is what the solo learner trains from."""
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
    _check_group(path, 3, 4, 40, 2)


def test_group_of_sixteen_is_bit_identical_to_solo_engines():
    _check_group("gather", 16, 3, 32, 1)


# ---- refusals, launches and end to end ------------------------------------------------------------------------------
def test_engine_refuses_bad_tqc_configurations():
    from rl_replicas_b200 import _lib
    from rl_replicas_b200._lib import B200RLError, OffPolicyHparams
    from rl_replicas_b200.engine import OffPolicyEngine as E
    acts = ("relu", "identity")
    P, Q = [5, 16, 4], [7, 16, 6]
    with pytest.raises(B200RLError, match="algo must be"):
        E(P, Q, 2, 8, 2, acts, acts, algo=E.TQC)  # create / create_group refuse algo 7
    with pytest.raises(B200RLError, match="algo must be 7"):
        E(P, [7, 16, 1], 2, 8, 2, acts, acts, algo=E.SAC, tqc=(6, 1))
    with pytest.raises(B200RLError, match="TQC needs n_q = 2"):
        E(P, Q, 1, 8, 2, acts, acts, algo=E.TQC, tqc=(6, 1))
    for M, d in ((0, 0), (257, 0), (6, 6), (6, -1)):
        with pytest.raises(B200RLError, match="offpolicy_create_tqc"):
            E(P, [7, 16, max(M, 1)], 2, 8, 2, acts, acts, algo=E.TQC, tqc=(M, d))
    with pytest.raises(B200RLError, match="critics must map"):
        E(P, [7, 16, 5], 2, 8, 2, acts, acts, algo=E.TQC, tqc=(6, 1))
    with pytest.raises(B200RLError, match="TQC takes neither dueling_k"):
        E(P, [7, 16, 16, 6], 2, 8, 2, acts, acts, algo=E.TQC, tqc=(6, 1), dueling_k=1)
    with pytest.raises(B200RLError, match="TQC takes neither dueling_k"):
        E(P, Q, 2, 8, 2, acts, acts, algo=E.TQC, tqc=(6, 1), noisy_layers=1)
    e = E(P, Q, 2, 8, 2, acts, acts, algo=E.TQC, tqc=(6, 1))
    layout, _ = e.state_layout()
    assert [i for kind, i, _, _ in layout if kind == "params"] == [0, 1, 2, 4, 5]
    z = lambda *s: np.zeros(s, np.float32)
    hp = OffPolicyHparams()
    hp.policy_delay = 1
    with pytest.raises(B200RLError, match="set_sac"):
        e.train(hp, z(2, 8, 5), z(2, 8, 2), z(2, 8), z(2, 8, 5), z(2, 8), z(2, 2, 8, 2))
    for call in (lambda: e.set_dqn(1, False), lambda: e.set_c51(5, -1.0, 1.0), lambda: e.set_qr(3),
                 lambda: e.set_per(0.6, 1e-6, 0.4, 100), lambda: e.set_nstep(1),
                 lambda: e.set_noise_keys([1], [1])):
        with pytest.raises(B200RLError, match="TQC engine"):
            call()
    rows = 16
    cols = [torch.zeros(rows, 5, device="cuda"), torch.zeros(rows, 2, device="cuda"), torch.zeros(rows, device="cuda"),
            torch.zeros(rows, 5, device="cuda"), torch.zeros(rows, device="cuda")]
    tree = torch.zeros(int(_lib.load().b200rl_per_tree_floats(rows)), device="cuda")
    with pytest.raises(B200RLError, match="TQC engines"):
        e.train_prioritized(OffPolicyHparams(), cols, rows, tree, 2, 8, 0, 1)


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
    """b200rl.h: 1 per call, then SAC's 12 Lq + 4 Lp + 7 per step (+1 with a learned temperature) plus the target
    kernel; host-staged minibatches launch nothing else.  SAC at the same shape launches exactly one fewer per step."""
    from test_gpu_sac import build as build_sac
    S, B = 5, 32
    O, A, _, _, L, _, _, _ = SHAPES["small_tanh"]
    for learn_alpha in (False, True):
        for graph in (False, True):
            algo = build("small_tanh", learn_alpha=learn_alpha)
            sac = build_sac("small_tanh", learn_alpha=learn_alpha)
            for a in (algo, sac):
                fill(a.replay_buffer, O, A, L, n=500, seed=6)
                a.use_device_replay = False
            want = 1 + S * (12 * 3 + 4 * 3 + 7 + int(learn_alpha) + 1)
            assert _launches(algo, S, B, graph) == want, (learn_alpha, graph)
            assert _launches(sac, S, B, graph) == want - S, (learn_alpha, graph)


def test_learn_solves_the_bandit(tmp_path, capsys):
    """TQC.learn end to end on the one-step bandit of tests/test_sac.py with the seeds the oracle-driven loop in
    tests/test_tqc.py used: the tags are recorded, model.pt is written and reloads, and the evaluation return clears
    the same bar."""
    np.random.seed(0)
    algo = make_tqc(learn_alpha=True)
    algo.learn(output_dir=str(tmp_path), **LEARN)
    after = evaluation_return(algo)
    printed = capsys.readouterr().out
    with capsys.disabled():
        print(f"TQC.learn on the bandit: evaluation return {after:.3f}")
    for tag in ("policy/average_loss", "policy/average_log_prob", "alpha/value", "q-function_1/average_loss",
                "q-function_2/average_loss", "q-function_1/avarage_q-value", "evaluation/average_episode_return"):
        assert f"\n{tag}: " in printed, tag
    path = os.path.join(tmp_path, "model.pt")
    assert os.path.exists(path)
    other = make_tqc(seed=5, learn_alpha=True)
    other.load_model(path)
    assert evaluation_return(other) == after
    assert after > RETURN_BAR
