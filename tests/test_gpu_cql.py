"""GPU: CQL.train on the off-policy engine against the torch-autograd oracle (oracle/cql.py) and the float64 stage,
cql_weight = 0 against a SAC engine bit for bit, bit-identical execution paths and learner groups, the device-side
draws, the engine's refusals, the launches per step b200rl.h states, and CQL.learn_offline end to end."""
import os

import numpy as np
import pytest
import torch

from conftest import rel_err
from oracle import cql as OC
from test_cql import GAP_MARGIN, OFFLINE, make_offline, q_gap
from test_gpu_sac import adam_flat, compare, fill, flat
from test_gpu_sac import build as build_sac
from test_sac import RETURN_BAR, evaluation_return

pytestmark = pytest.mark.gpu

SHAPES = {  # (obs, act, hidden, hidden activation, action limit, minibatch)
    "halfcheetah": (17, 6, 256, torch.nn.ReLU, 1.0, 256),
    "small_tanh": (5, 2, 64, torch.nn.Tanh, 2.0, 50),
}


def build(shape, seed=0, learn_alpha=False, **kw):
    from rl_replicas_b200.algorithms import CQL
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import SquashedGaussianPolicy
    from rl_replicas_b200.q_function import QFunction
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    import types
    O, A, H, act, L, _ = SHAPES[shape]
    torch.manual_seed(seed)
    pnet = MLP([O, H, H, 2 * A], act)
    q1, q2 = MLP([O + A, H, H, 1], act), MLP([O + A, H, H, 1], act)
    hi = np.full(A, L, np.float32)
    env = types.SimpleNamespace(action_space=types.SimpleNamespace(high=hi, low=-hi, shape=(A,)),
                                spec=types.SimpleNamespace(id="stub"))
    algo = CQL(SquashedGaussianPolicy(pnet, torch.optim.Adam(pnet.parameters(), lr=1e-3), action_limit=L), None,
               QFunction(q1, torch.optim.Adam(q1.parameters(), lr=1e-3)),
               QFunction(q2, torch.optim.Adam(q2.parameters(), lr=1e-3)), env, None, ReplayBuffer(), None,
               learn_alpha=learn_alpha, alpha_lr=3e-3, **kw)
    algo.metrics_manager = None
    algo.current_total_steps = 0
    return algo


def oracle_for(algo):
    return OC.CqlOracle(algo.policy.network, algo.q_function_1.network, algo.q_function_2.network,
                        cql_weight=algo.cql_weight, cql_n_actions=algo.cql_n_actions,
                        cql_temperature=algo.cql_temperature, cql_target_action_gap=algo.cql_target_action_gap,
                        cql_alpha_lr=3e-4, backup_entropy=algo.backup_entropy, gamma=algo.gamma, rho=algo.polyak_rho,
                        alpha=algo.alpha, learn_alpha=algo.learn_alpha, target_entropy=algo.target_entropy,
                        alpha_lr=3e-3, limit=algo.policy.action_limit)


def compare_cql(algo, oracle, logs, out):
    errs = compare(algo, oracle, logs, out)
    for k in ("cql_gap_1", "cql_gap_2", "alpha_primes"):
        errs[k] = rel_err(out[k], np.asarray(logs[k]))
    errs["log_alpha_prime"] = rel_err(float(algo.log_alpha_prime.detach()), float(oracle.log_alpha_prime.detach()))
    return errs


def run_against_oracle(algo, S, B, calls=3):
    oracle = oracle_for(algo)
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
        logs = oracle.train(mbs, algo._noise(S, B))
        for k, v in compare_cql(algo, oracle, logs, out).items():
            worst[k] = max(worst.get(k, 0.0), v)
    return worst


@pytest.mark.parametrize("case", [
    dict(shape="small_tanh", cql_n_actions=10),
    dict(shape="small_tanh", cql_n_actions=1, learn_alpha=True, backup_entropy=True),
    dict(shape="small_tanh", cql_n_actions=64, cql_temperature=0.5),
    dict(shape="small_tanh", cql_n_actions=10, cql_target_action_gap=1.0, learn_alpha=True),
    dict(shape="halfcheetah", cql_n_actions=10),
], ids=["N10", "N1_entropy_learned_alpha", "N64_T05", "lagrange", "halfcheetah"])
def test_train_matches_the_oracle(case):
    """Three calls of four steps through CQL.train (device replay, graph replay) against the autograd oracle on the
    same minibatches and draws."""
    case = dict(case)
    shape = case.pop("shape")
    O, A, _, _, L, B = SHAPES[shape]
    algo = build(shape, **case)
    fill(algo.replay_buffer, O, A, L)
    worst = run_against_oracle(algo, 4, B)
    print(shape, case, {k: f"{v:.1e}" for k, v in worst.items()})
    # At the ReLU HalfCheetah shape rows near a ReLU kink let parameters and Adam moments drift (test_gpu_tqc.py
    # explains it).  Measured on H100: the networks and moments drift to 4e-3 over the 12 steps, and the values the
    # next calls compute from the drifted networks follow (Q-values 2.6e-4, policy loss 3e-5, mean log pi 3e-6), while
    # the critic losses and gaps stay below 3e-7.  The Tanh shape has no kinks and holds everything to 1e-4.
    drift = {"policy", "q1", "q2", "target_q1", "target_q2", "q1_values", "q2_values", "policy_losses",
             "log_prob_means"} | {f"{n}.{m}" for n in ("policy", "q1", "q2") for m in ("exp_avg", "exp_avg_sq")}
    for k, v in worst.items():
        assert v < (1e-2 if shape == "halfcheetah" and k in drift else 1e-4), (k, v, worst)


def test_one_step_against_the_float64_reference():
    O, A, _, _, L, B = SHAPES["small_tanh"]
    psz, qsz = [O, 64, 64, 2 * A], [O + A, 64, 64, 1]
    algo = build("small_tanh", cql_n_actions=10, backup_entropy=True)
    nets = dict(policy=flat(algo.policy.network), q1=flat(algo.q_function_1.network),
                q2=flat(algo.q_function_2.network), target_q1=flat(algo.target_q_function_1.network),
                target_q2=flat(algo.target_q_function_2.network))
    nets = {k: v.astype(np.float64) for k, v in nets.items()}
    rng = np.random.default_rng(2)
    f32 = lambda x: np.asarray(x, np.float32)
    mb = dict(observations=f32(rng.standard_normal((B, O))), actions=f32(rng.uniform(-L, L, (B, A))),
              rewards=f32(rng.standard_normal(B)), next_observations=f32(rng.standard_normal((B, O))),
              dones=rng.random(B) < 0.1)
    torch.manual_seed(3)
    sac, draws = algo._noise(1, B)
    e = algo._ensure_engine(1, B)
    algo._upload_state(e, *algo._learner_nets())
    out = e.train(algo._hparams(True, 1), mb["observations"][None], mb["actions"][None], mb["rewards"][None],
                  mb["next_observations"][None], mb["dones"].astype(np.float32)[None], (sac, draws))
    algo._download_state(e, *algo._learner_nets())
    c = OC.critic_stage_f64(nets, mb, sac[0, 0].astype(np.float64), draws[0].astype(np.float64),
                            float(np.float32(0.2)), psz, qsz, algo.cql_weight, algo.cql_temperature,
                            backup_entropy=True, hidden="tanh", action_limit=L)
    errs = {}
    for k, m_ in ((1, algo.q_function_1), (2, algo.q_function_2)):
        errs[f"q{k}_values"] = rel_err(out[f"q{k}_values"][0], c[f"q{k}_values"])
        errs[f"q{k}_loss"] = rel_err(out[f"q{k}_losses"][0], c[f"q{k}_loss"])
        errs[f"q{k}_gap"] = rel_err(out[f"cql_gap_{k}"][0], c[f"q{k}_gap"])
        errs[f"q{k}_grad"] = rel_err(adam_flat(m_.optimizer, "exp_avg")[0] / 0.1, c[f"q{k}_grad"])
    print({k: f"{v:.1e}" for k, v in errs.items()})
    for k, v in errs.items():
        assert v < 2e-5, (k, v, errs)


def _sac_state(algo):
    out = [flat(m.network) for m in (algo.policy, algo.q_function_1, algo.q_function_2, algo.target_q_function_1,
                                     algo.target_q_function_2)]
    for m in (algo.policy, algo.q_function_1, algo.q_function_2):
        out += [adam_flat(m.optimizer, k)[0] for k in ("exp_avg", "exp_avg_sq")]
    return out + [np.asarray(algo._alpha_state(), np.float64)]


@pytest.mark.parametrize("device_rng", [False, True])
def test_zero_weight_is_sac_bit_for_bit(device_rng):
    """cql_weight = 0 with backup_entropy: the same parameters, Adam states, Q-values and losses as a SAC engine on
    the same draws, through the fanned-out critic step.  Host draws: the SAC learner gets the SAC part of the CQL
    learner's noise; device draws: the same device_rng_seed."""
    O, A, _, _, L, B = SHAPES["halfcheetah"]
    cql = build("halfcheetah", learn_alpha=True, cql_weight=0.0, backup_entropy=True)
    sac = build_sac("halfcheetah", learn_alpha=True)
    for a in (cql, sac):
        fill(a.replay_buffer, O, A, L)
        a.use_device_rng, a.device_rng_seed = device_rng, 5
    if not device_rng:
        cql_noise = cql._noise
        sac._noise = lambda S, B_: cql_noise(S, B_)[0]
    for call in range(2):
        outs = []
        for a in (cql, sac):
            np.random.seed(20 + call)
            torch.manual_seed(20 + call)
            a.train(a.replay_buffer, 5, B)
            outs.append(a.last_train_output)
        for k in outs[1]:
            np.testing.assert_array_equal(outs[0][k], outs[1][k], err_msg=k)
        assert (outs[0]["cql_gap_1"] != 0).all()  # the penalty ran
    for i, (x, y) in enumerate(zip(_sac_state(cql), _sac_state(sac))):
        np.testing.assert_array_equal(x, y, err_msg=f"tensor {i}")


def _run_paths(device_replay, graph, S=4, B=40):
    os.environ["B200RL_OFFPOLICY_GRAPH"] = "1" if graph else "0"
    try:
        O, A, _, _, L, _ = SHAPES["small_tanh"]
        algo = build("small_tanh", learn_alpha=True, cql_n_actions=6, cql_target_action_gap=0.5)
        fill(algo.replay_buffer, O, A, L, n=3000, seed=3)
        algo.use_device_replay = device_replay
        outs = []
        for call in range(3):
            np.random.seed(10 + call)
            torch.manual_seed(10 + call)
            algo.train(algo.replay_buffer, S + (call == 2), B)
            outs.append(algo.last_train_output)
        return outs, _sac_state(algo) + [np.asarray(algo._alpha_prime_state(), np.float64)]
    finally:
        os.environ.pop("B200RL_OFFPOLICY_GRAPH", None)


def test_host_staged_graph_replay_and_device_gather_are_bit_identical():
    ref_outs, ref_state = _run_paths(False, False)
    for dev, graph in ((True, True), (False, True), (True, False)):
        outs, state = _run_paths(dev, graph)
        for a, b in zip(outs, ref_outs):
            assert a.keys() == b.keys()
            for k in a:
                np.testing.assert_array_equal(a[k], b[k], err_msg=f"{k} dev={dev} graph={graph}")
        for i, (a, b) in enumerate(zip(state, ref_state)):
            np.testing.assert_array_equal(a, b, err_msg=f"tensor {i} dev={dev} graph={graph}")


def test_device_side_draws_replay_through_the_oracle():
    O, A, _, _, L, _ = SHAPES["small_tanh"]
    S, B, N = 6, 64, 8
    algo = build("small_tanh", learn_alpha=True, cql_n_actions=N, cql_target_action_gap=1.0)
    fill(algo.replay_buffer, O, A, L, n=3000, seed=4)
    algo.use_device_rng, algo.device_rng_seed = True, 77
    oracle = oracle_for(algo)
    algo.train(algo.replay_buffer, S, B)
    idx, noise = algo._engine.get_draws(S, B)
    draws = algo._engine.get_cql_draws(S, B)
    assert draws.shape == (S, 3, B, N, A)
    assert (draws[:, 0] >= 0).all() and (draws[:, 0] < 1).all() and abs(draws[:, 1:].std() - 1) < 0.05
    rb = algo.replay_buffer
    logs = oracle.train([{k: rb._cols[k][idx[s]] for k in rb.COLUMNS} for s in range(S)], (noise, draws))
    errs = compare_cql(algo, oracle, logs, algo.last_train_output)
    for k, v in errs.items():
        assert v < 1e-4, (k, v, errs)


# ---- learner groups -------------------------------------------------------------------------------------------------
def _check_group(path, K, S, B):
    """K members on ONE shared dataset buffer, LearnerGroup.train against each member's own train."""
    from rl_replicas_b200.algorithms import LearnerGroup
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    from rl_replicas_b200.utils import set_seed_for_libraries
    from test_cql import bandit_dataset
    shared = ReplayBuffer.from_dataset(bandit_dataset(3000))

    def member(k):
        algo = make_offline(seed=k, hidden=32, cql_n_actions=4, cql_target_action_gap=1.0, learn_alpha=True)
        algo.replay_buffer = shared
        algo.use_device_replay = path != "host"
        algo.use_device_rng, algo.device_rng_seed = path == "rng", 90 + k
        return algo

    solo = []
    for k in range(K):
        m = member(k)
        set_seed_for_libraries(50 + k)
        for _ in range(2):
            m.train(m.replay_buffer, S, B)
        solo.append(m)
    g = LearnerGroup()
    grouped = [member(k) for k in range(K)]
    for k, m in enumerate(grouped):
        set_seed_for_libraries(50 + k)
        g.add(m)
    for _ in range(2):
        g.train(S, B)
    for k, (a, b) in enumerate(zip(solo, grouped)):
        for key in a.last_train_output:
            np.testing.assert_array_equal(a.last_train_output[key], b.last_train_output[key], err_msg=f"{key} {k}")
        for i, (x, y) in enumerate(zip(_sac_state(a) + [np.asarray(a._alpha_prime_state())],
                                       _sac_state(b) + [np.asarray(b._alpha_prime_state())])):
            np.testing.assert_array_equal(x, y, err_msg=f"member {k} tensor {i}")


@pytest.mark.parametrize("path", ["host", "gather", "rng"])
def test_group_of_three_on_one_dataset_is_bit_identical_to_solo_engines(path):
    _check_group(path, 3, 3, 32)


def test_group_of_sixteen_on_one_dataset_is_bit_identical_to_solo_engines():
    _check_group("gather", 16, 2, 32)


# ---- refusals, launches and end to end ------------------------------------------------------------------------------
def test_engine_refuses_bad_cql_configurations():
    from rl_replicas_b200._lib import B200RLError, OffPolicyHparams
    from rl_replicas_b200.engine import OffPolicyEngine as E
    acts = ("relu", "identity")
    P, Q = [5, 16, 4], [7, 16, 1]
    with pytest.raises(B200RLError, match="algo must be"):
        E(P, Q, 2, 8, 2, acts, acts, algo=E.CQL)
    with pytest.raises(B200RLError, match="algo must be 8"):
        E(P, Q, 2, 8, 2, acts, acts, algo=E.SAC, cql=(4, 0))
    with pytest.raises(B200RLError, match="CQL needs n_q = 2"):
        E(P, Q, 1, 8, 2, acts, acts, algo=E.CQL, cql=(4, 0))
    for N in (0, 65):
        with pytest.raises(B200RLError, match="n_actions must be"):
            E(P, Q, 2, 8, 2, acts, acts, algo=E.CQL, cql=(N, 0))
    with pytest.raises(B200RLError, match="stacked rows"):
        E(P, Q, 2, 20000, 2, acts, acts, algo=E.CQL, cql=(64, 0))
    with pytest.raises(B200RLError, match="CQL takes neither"):
        E(P, [7, 16, 16, 1], 2, 8, 2, acts, acts, algo=E.CQL, cql=(4, 0), dueling_k=1)
    with pytest.raises(B200RLError, match="CQL takes neither"):
        E(P, Q, 2, 8, 2, acts, acts, algo=E.CQL, cql=(4, 0), noisy_layers=1)
    e = E(P, Q, 2, 8, 2, acts, acts, algo=E.CQL, cql=(4, 0))
    z = lambda *s: np.zeros(s, np.float32)
    hp = OffPolicyHparams()
    hp.policy_delay, hp.action_limit = 1, 1.0
    from rl_replicas_b200._lib import SacHparams
    sp = SacHparams()
    sp.alpha, sp.log_std_min, sp.log_std_max = 0.2, -20.0, 2.0
    e.set_sac(sp)
    with pytest.raises(B200RLError, match="set_cql"):
        e.train(hp, z(2, 8, 5), z(2, 8, 2), z(2, 8), z(2, 8, 5), z(2, 8), (z(2, 2, 8, 2), z(2, 3, 8, 4, 2)))
    for kw in (dict(weight=-1.0, temperature=1.0), dict(weight=1.0, temperature=0.0)):
        with pytest.raises(B200RLError, match="offpolicy_set_cql"):
            e.set_cql(**kw)
    e.set_cql(1.0, 1.0)
    with pytest.raises(B200RLError, match="set_cql_draws"):  # the draws staged above are for S = 2, not 1
        e.train(hp, z(1, 8, 5), z(1, 8, 2), z(1, 8), z(1, 8, 5), z(1, 8), z(1, 2, 8, 2))
    for call in (lambda: e.set_dqn(1, False), lambda: e.set_per(0.6, 1e-6, 0.4, 100), lambda: e.set_nstep(2, None)):
        with pytest.raises(Exception):
            call()


def _launches(algo, S, B, graph):
    from rl_replicas_b200 import _lib
    lib = _lib.load()
    os.environ["B200RL_OFFPOLICY_GRAPH"] = "1" if graph else "0"
    try:
        np.random.seed(0)
        algo.train(algo.replay_buffer, S, B)
        n0 = lib.b200rl_launch_count()
        algo.train(algo.replay_buffer, S, B)
        return lib.b200rl_launch_count() - n0
    finally:
        os.environ.pop("B200RL_OFFPOLICY_GRAPH", None)


def test_launches_per_step_are_the_stated_ones():
    """b200rl.h: 1 per call (+1 with the Lagrange step), then SAC's 12 Lq + 4 Lp + 7 per step (+1 with a learned
    temperature) plus the staging kernel and the two penalty heads (+1 with the Lagrange step)."""
    S, B = 5, 32
    O, A, _, _, L, _ = SHAPES["small_tanh"]
    for learn_alpha in (False, True):
        for lag in (None, 1.0):
            for graph in (False, True):
                algo = build("small_tanh", learn_alpha=learn_alpha, cql_n_actions=3, cql_target_action_gap=lag)
                fill(algo.replay_buffer, O, A, L, n=500, seed=6)
                algo.use_device_replay = False
                on = lag is not None
                want = 1 + int(on) + S * (12 * 3 + 4 * 3 + 7 + int(learn_alpha) + 3 + int(on))
                assert _launches(algo, S, B, graph) == want, (learn_alpha, lag, graph)


def test_learn_offline_on_the_bandit_dataset(tmp_path, capsys):
    """CQL.learn_offline end to end on tests/test_cql.py's bandit dataset with its seeds: the bars that test set,
    model.pt written, and a reload evaluating to the same return."""
    np.random.seed(0)
    torch.manual_seed(0)
    algo = make_offline()
    algo.learn_offline(output_dir=str(tmp_path), **OFFLINE)
    printed = capsys.readouterr().out
    ret, gap = evaluation_return(algo), q_gap(algo)
    np.random.seed(0)
    torch.manual_seed(0)
    sac = make_offline("SAC")
    sac.learn_offline(output_dir=str(tmp_path / "sac"), **OFFLINE)
    gap_sac = q_gap(sac)
    with capsys.disabled():
        print(f"CQL.learn_offline on the bandit dataset: return {ret:.3f}, Q gap {gap:.3f} (offline SAC {gap_sac:.3f})")
    for tag in ("epoch", "total_train_steps", "cql/penalty_1", "cql/penalty_2", "q-function_1/average_loss",
                "evaluation/average_episode_return"):
        assert f"\n{tag}: " in printed, tag
    assert ret > RETURN_BAR and gap > GAP_MARGIN and gap > gap_sac
    path = os.path.join(tmp_path, "model.pt")
    assert os.path.exists(path)
    other = make_offline(seed=5)
    other.load_model(path)
    assert evaluation_return(other) == ret
