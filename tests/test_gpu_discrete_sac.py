"""GPU: DiscreteSAC.train on the off-policy engine against the float32 autograd oracle (oracle/discrete_sac.py) across
calls, one step against the float64 reference, bit-identical execution paths, learner groups bit for bit equal to solo
engines, the invalid-action refusal, the engine's refusals, the launches per step b200rl.h states, and
DiscreteSAC.learn end to end."""
import os
import types

import numpy as np
import pytest
import torch

from conftest import rel_err
from oracle import discrete_sac as OD
from test_discrete_sac import LEARN, RETURN_BAR, evaluation_return, make_dsac

pytestmark = pytest.mark.gpu

GAMMA, LR, ALPHA_LR = 0.99, 1e-3, 3e-3


def build(O=8, n=4, hidden=64, seed=0, learn_alpha=False, **kw):
    """A DiscreteSAC learner on a stub discrete environment with two ReLU hidden layers of width ``hidden``."""
    from rl_replicas_b200.algorithms import DiscreteSAC
    from rl_replicas_b200.critics import DiscreteQFunction
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import CategoricalPolicy
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    torch.manual_seed(seed)
    pnet, q1, q2 = (MLP([O, hidden, hidden, n], torch.nn.ReLU) for _ in range(3))
    env = types.SimpleNamespace(action_space=types.SimpleNamespace(n=n, shape=()), spec=types.SimpleNamespace(id="stub"),
                                observation_space=types.SimpleNamespace(shape=(O,)))
    algo = DiscreteSAC(CategoricalPolicy(pnet, torch.optim.Adam(pnet.parameters(), lr=LR)), None,
                       DiscreteQFunction(q1, torch.optim.Adam(q1.parameters(), lr=LR)),
                       DiscreteQFunction(q2, torch.optim.Adam(q2.parameters(), lr=LR)), env, None, ReplayBuffer(), None,
                       gamma=GAMMA, learn_alpha=learn_alpha, alpha_lr=ALPHA_LR, **kw)
    with torch.no_grad():  # targets that differ from the online critics
        for t in (algo.target_q_function_1, algo.target_q_function_2):
            for p in t.network.parameters():
                p.add_(0.05 * torch.randn_like(p))
    algo.metrics_manager = None
    algo.current_total_steps = 0
    return algo


def fill(rb, O, n, rows=4000, seed=1, bad_action=None, obs=None):
    """``rows`` random transitions (``obs`` [rows + 1, O]: the observations to use) into ``rb``."""
    from rl_replicas_b200.experience import Experience
    rng = np.random.default_rng(seed)
    e = Experience()
    obs = rng.standard_normal((rows + 1, O)).astype(np.float32) if obs is None else obs
    e.observations = [[obs[i] for i in range(rows)]]
    e.actions = [[a for a in rng.integers(0, n, rows).astype(np.int64)]]
    e.rewards = [[float(x) for x in rng.standard_normal(rows)]]
    e.dones = [[bool(x) for x in (rng.random(rows) < 0.1)]]
    e.last_observations = [obs[rows]]
    rb.add_experience(e)
    if bad_action is not None:
        rb._cols["actions"][rows // 2] = bad_action


def flat(m):
    return torch.nn.utils.parameters_to_vector(m.parameters()).detach().numpy()


def adam_flat(opt, key):
    ps = opt.param_groups[0]["params"]
    return np.concatenate([opt.state[p][key].reshape(-1).numpy() for p in ps]), int(float(opt.state[ps[0]]["step"]))


def oracle_for(algo):
    o = OD.DiscreteSacOracle(algo.policy.network, algo.q_function_1.network, algo.q_function_2.network, pi_lr=LR,
                             q_lr=LR, gamma=algo.gamma, rho=algo.polyak_rho, alpha=algo.alpha,
                             learn_alpha=algo.learn_alpha, target_entropy=algo.target_entropy, alpha_lr=ALPHA_LR)
    o.q1_targ.load_state_dict(algo.target_q_function_1.network.state_dict())
    o.q2_targ.load_state_dict(algo.target_q_function_2.network.state_dict())
    return o


def compare(algo, oracle, logs, out):
    errs = {}
    for k in ("q1_values", "q2_values"):
        errs[k] = rel_err(out[k], np.stack(logs[k]))
    for k in ("q1_losses", "q2_losses", "policy_losses", "log_prob_means", "alphas"):
        errs[k] = rel_err(out[k], np.asarray(logs[k]))
    pairs = {"policy": (algo.policy, oracle.pi, oracle.pi_opt), "q1": (algo.q_function_1, oracle.q1, oracle.q1_opt),
             "q2": (algo.q_function_2, oracle.q2, oracle.q2_opt)}
    for name, (m, o, opt) in pairs.items():
        errs[name] = rel_err(flat(m.network), flat(o))
        for key in ("exp_avg", "exp_avg_sq"):
            got, step = adam_flat(m.optimizer, key)
            want, step_o = adam_flat(opt, key)
            errs[f"{name}.{key}"] = rel_err(got, want)
            assert step == step_o, (name, step, step_o)
    errs["target_q1"] = rel_err(flat(algo.target_q_function_1.network), flat(oracle.q1_targ))
    errs["target_q2"] = rel_err(flat(algo.target_q_function_2.network), flat(oracle.q2_targ))
    errs["log_alpha"] = rel_err(float(algo.log_alpha.detach()), float(oracle.log_alpha.detach()))
    if algo.learn_alpha:
        for key in ("exp_avg", "exp_avg_sq"):
            got, step = adam_flat(algo.alpha_optimizer, key)
            want, step_o = adam_flat(oracle.alpha_opt, key)
            errs[f"alpha.{key}"] = rel_err(got, want)
            assert step == step_o
    return errs


SHAPES = {"n2_h64_b50": (2, 64, 50), "n3_h256_b256": (3, 256, 256), "n18_h64_b256": (18, 64, 256),
          "n18_h256_b50": (18, 256, 50)}


@pytest.mark.parametrize("learn_alpha", [False, True])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_train_matches_the_oracle_across_calls(shape, learn_alpha):
    """Three DiscreteSAC.train calls of 4 steps (device replay, graph replay) against the autograd oracle with the same
    minibatches: Q-values, losses, mean E, alpha, every network, its Adam moments and the temperature's."""
    n, H, B = SHAPES[shape]
    O, S = 8, 4
    algo = build(O=O, n=n, hidden=H, learn_alpha=learn_alpha)
    fill(algo.replay_buffer, O, n)
    oracle = oracle_for(algo)
    worst = {}
    for call in range(3):
        np.random.seed(20 + call)
        algo.train(algo.replay_buffer, S, B)
        out = algo.last_train_output
        np.random.seed(20 + call)
        logs = oracle.train([algo.replay_buffer.sample_minibatch(B) for _ in range(S)])
        assert len(out["policy_losses"]) == S
        errs = compare(algo, oracle, logs, out)
        worst = {k: max(v, worst.get(k, 0.0)) for k, v in errs.items()}
    print(f"{shape} learn_alpha={learn_alpha}:", {k: f"{v:.1e}" for k, v in worst.items()})
    for k, v in worst.items():
        assert v < 2e-5, (k, v, worst)
    if not learn_alpha:
        assert (out["alphas"] == np.float32(0.2)).all()


def test_one_step_against_the_float64_reference():
    """One step from fresh Adam states at 18 actions, 256-wide layers and B = 256: the gradients (Adam's first moment
    over 1 - beta1), losses, Q-values and mean E against oracle/discrete_sac.py's float64 stages, the policy stage fed
    the engine's own post-step critics.  The replay holds only observations whose ReLU pre-activations in Q1, Q2 and
    pi are at least 1e-6 (relative) away from 0: a row at rounding distance from a kink may be gated differently by a
    float32 kernel, which is not an error of the kernel.  Every pass whose gradient the step takes reads them."""
    from oracle.offpolicy_f64 import _t, mlp
    n, H, B, O = 18, 256, 256, 8
    algo = build(O=O, n=n, hidden=H, learn_alpha=True)
    sizes = [O, H, H, n]
    before = {k: flat(m.network).astype(np.float64) for k, m in (("pi", algo.policy), ("q1", algo.q_function_1),
              ("q2", algo.q_function_2), ("t1", algo.target_q_function_1), ("t2", algo.target_q_function_2))}
    pool = np.random.default_rng(2).standard_normal((4 * B, O)).astype(np.float32)
    margin = np.min([mlp(_t(before[k]), sizes, _t(pool), "relu", "identity")[1].numpy() for k in ("pi", "q1", "q2")], 0)
    keep = pool[margin >= 1e-6][:B + 1]
    assert len(keep) == B + 1, len(keep)
    fill(algo.replay_buffer, O, n, rows=B, seed=2, obs=keep)
    la0 = float(algo.log_alpha.detach())
    np.random.seed(3)
    algo.train(algo.replay_buffer, 1, B)
    out = algo.last_train_output
    np.random.seed(3)
    mb = algo.replay_buffer.sample_minibatch(B)
    alpha = float(np.float32(np.exp(np.float32(la0))))
    c = OD.critic_stage_f64(before["q1"], before["q2"], before["t1"], before["t2"], before["pi"], sizes, sizes,
                            mb["observations"], mb["actions"], mb["rewards"], mb["next_observations"], mb["dones"],
                            alpha, GAMMA)
    errs = {}
    for k, m in ((1, algo.q_function_1), (2, algo.q_function_2)):
        errs[f"q{k}_values"] = rel_err(out[f"q{k}_values"][0], c[f"q{k}_values"])
        errs[f"q{k}_loss"] = rel_err(out[f"q{k}_losses"][0], c[f"q{k}_loss"])
        errs[f"q{k}_grad"] = rel_err(adam_flat(m.optimizer, "exp_avg")[0] / 0.1, c[f"q{k}_grad"])
    p = OD.policy_stage_f64(before["pi"], flat(algo.q_function_1.network), flat(algo.q_function_2.network), sizes, sizes,
                            mb["observations"], alpha, algo.target_entropy, log_alpha=la0)
    errs["policy_loss"] = rel_err(out["policy_losses"][0], p["loss"])
    errs["ent_mean"] = rel_err(out["log_prob_means"][0], p["ent_mean"])
    errs["policy_grad"] = rel_err(adam_flat(algo.policy.optimizer, "exp_avg")[0] / 0.1, p["grad"])
    errs["alpha_grad"] = rel_err(adam_flat(algo.alpha_optimizer, "exp_avg")[0] / 0.1, p["alpha_grad"])
    print({k: f"{v:.1e}" for k, v in errs.items()})
    for k, v in errs.items():
        assert v < 2e-5, (k, v, errs)


def _run_paths(device_replay, graph, S=5, B=48):
    os.environ["B200RL_OFFPOLICY_GRAPH"] = "1" if graph else "0"
    try:
        algo = build(O=6, n=5, learn_alpha=True)
        fill(algo.replay_buffer, 6, 5, rows=3000, seed=3)
        algo.use_device_replay = device_replay
        outs = []
        for call in range(3):
            np.random.seed(10 + call)
            algo.train(algo.replay_buffer, S + (call == 2), B)
            outs.append(algo.last_train_output)
        nets = [flat(m.network) for m in (algo.policy, algo.q_function_1, algo.q_function_2, algo.target_q_function_1,
                                          algo.target_q_function_2)]
        return outs, nets + [algo.log_alpha.detach().numpy().reshape(1)]
    finally:
        os.environ.pop("B200RL_OFFPOLICY_GRAPH", None)


def test_host_staged_device_gather_and_graph_paths_are_bit_identical():
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
    S, B, n = 6, 64, 5
    algo = build(O=6, n=n, learn_alpha=True)
    fill(algo.replay_buffer, 6, n, rows=3000, seed=4)
    algo.use_device_rng, algo.device_rng_seed = True, 77
    oracle = oracle_for(algo)
    algo.train(algo.replay_buffer, S, B)
    idx, noise = algo._engine.get_draws(S, B)
    assert idx.shape == (S, B) and noise is None  # indices only
    rb = algo.replay_buffer
    logs = oracle.train([{k: rb._cols[k][idx[s]] for k in rb.COLUMNS} for s in range(S)])
    errs = compare(algo, oracle, logs, algo.last_train_output)
    for k, v in errs.items():
        assert v < 2e-5, (k, v, errs)


# ---- learner groups -------------------------------------------------------------------------------------------------
def _member(k, path, n=4):
    algo = build(O=6, n=n, seed=k, learn_alpha=True)
    fill(algo.replay_buffer, 6, n, rows=2000, seed=30 + k)
    algo.use_device_replay = path != "host"
    algo.use_device_rng, algo.device_rng_seed = path == "rng", 90 + k
    if k % 2:  # members at different Adam step counts
        np.random.seed(k)
        algo.train(algo.replay_buffer, k, 16)
    return algo


def _state(algo):
    out = [flat(m.network) for m in (algo.policy, algo.q_function_1, algo.q_function_2, algo.target_q_function_1,
                                     algo.target_q_function_2)]
    for m in (algo.policy, algo.q_function_1, algo.q_function_2):
        out += [adam_flat(m.optimizer, k)[0] for k in ("exp_avg", "exp_avg_sq")]
    return out + [np.asarray(algo._alpha_state(), np.float64)]


def _check_group(solo, grouped, seeds, S, B, calls):
    from rl_replicas_b200.algorithms import LearnerGroup
    g = LearnerGroup()
    for k, m in enumerate(grouped):
        np.random.seed(seeds[k])
        torch.manual_seed(seeds[k])
        g.add(m)
    for call in range(calls):
        for k, m in enumerate(solo):
            np.random.seed(seeds[k]) if call == 0 else np.random.set_state(m._np_state)
            m.train(m.replay_buffer, S, B)
            m._np_state = np.random.get_state()
        g.train(S, B)
        for k, (a, b) in enumerate(zip(solo, grouped)):
            assert a.last_train_output.keys() == b.last_train_output.keys()
            for key in a.last_train_output:
                np.testing.assert_array_equal(a.last_train_output[key], b.last_train_output[key], err_msg=f"{key} {k}")
            for i, (x, y) in enumerate(zip(_state(a), _state(b))):
                np.testing.assert_array_equal(x, y, err_msg=f"member {k} tensor {i} call {call}")


@pytest.mark.parametrize("path", ["host", "gather", "rng"])
def test_group_of_three_is_bit_identical_to_solo_engines(path):
    """LearnerGroup.train against each member's own train, two calls, members at different step counts."""
    solo = [_member(k, path) for k in range(3)]
    grouped = [_member(k, path) for k in range(3)]
    _check_group(solo, grouped, [50, 51, 52], 4, 40, 2)


def test_group_of_sixteen_is_bit_identical_to_solo_engines():
    solo = [_member(k, "gather", n=3) for k in range(16)]
    grouped = [_member(k, "gather", n=3) for k in range(16)]
    _check_group(solo, grouped, [70 + k for k in range(16)], 3, 32, 1)


# ---- refusals, launches and end to end ------------------------------------------------------------------------------
@pytest.mark.parametrize("bad", [4.0, 1.5, -1.0, float("nan")])
def test_invalid_action_raises_and_leaves_the_host_modules_unchanged(bad):
    from rl_replicas_b200._lib import B200RLError
    algo = build(O=6, n=4, learn_alpha=True)
    fill(algo.replay_buffer, 6, 4, rows=64, seed=5, bad_action=bad)
    before = _state_nets(algo)
    np.random.seed(0)
    with pytest.raises(B200RLError, match=r"discrete SAC learner 0, step \d+: \d+ minibatch rows hold an action"):
        algo.train(algo.replay_buffer, 8, 64)  # 512 draws of 64 rows: the bad row is drawn
    for x, y in zip(before, _state_nets(algo)):
        np.testing.assert_array_equal(x, y)
    assert algo._alpha_state()[3] == 0


def _state_nets(algo):
    return [flat(m.network) for m in (algo.policy, algo.q_function_1, algo.q_function_2, algo.target_q_function_1,
                                      algo.target_q_function_2)] + [algo.log_alpha.detach().numpy().copy()]


def test_engine_refuses_bad_discrete_sac_configurations():
    from rl_replicas_b200._lib import B200RLError, OffPolicyHparams
    from rl_replicas_b200.engine import OffPolicyEngine as E
    acts = ("relu", "identity")
    with pytest.raises(B200RLError, match="n_q = 2"):
        E([4, 16, 3], [4, 16, 3], 1, 8, 2, acts, acts, algo=E.DSAC)
    with pytest.raises(B200RLError, match="n >= 2 actions"):
        E([4, 16, 3], [4, 16, 4], 2, 8, 2, acts, acts, algo=E.DSAC)
    with pytest.raises(B200RLError, match="n >= 2 actions"):
        E([4, 16, 1], [4, 16, 1], 2, 8, 2, acts, acts, algo=E.DSAC)
    with pytest.raises(B200RLError, match="n >= 2 actions"):
        E([4, 16, 3], [7, 16, 3], 2, 8, 2, acts, acts, algo=E.DSAC)
    with pytest.raises(B200RLError, match="algo = 5.*dueling"):
        E([4, 16, 3], [4, 16, 16, 3], 2, 8, 2, acts, acts, algo=E.DSAC, dueling_k=1)
    with pytest.raises(B200RLError, match="algo = 5.*noisy"):
        E([4, 16, 3], [4, 16, 3], 2, 8, 2, acts, acts, algo=E.DSAC, noisy_layers=1)
    with pytest.raises(B200RLError, match="algo must be"):
        E([4, 16, 3], [4, 16, 3], 2, 8, 2, acts, acts, algo=6)
    e = E([4, 16, 3], [4, 16, 3], 2, 8, 2, acts, acts, algo=E.DSAC)
    layout, _ = e.state_layout()
    assert [i for kind, i, _, _ in layout if kind == "params"] == [0, 1, 2, 4, 5]
    z = lambda *s: np.zeros(s, np.float32)
    with pytest.raises(B200RLError, match="set_sac"):
        e.train(OffPolicyHparams(), z(2, 8, 4), z(2, 8), z(2, 8), z(2, 8, 4), z(2, 8))
    with pytest.raises(B200RLError, match="algo = 5"):
        e.set_dqn(1, False)
    with pytest.raises(B200RLError, match="algo = 5"):
        e.set_c51(5, -1.0, 1.0)
    with pytest.raises(B200RLError, match="algo = 5"):
        e.set_qr(3)
    with pytest.raises(B200RLError, match="algo = 5"):
        e.set_per(0.6, 1e-6, 0.4, 100)
    with pytest.raises(B200RLError, match="algo = 5"):
        e.set_nstep(1)
    with pytest.raises(B200RLError, match="algo = 5"):
        e.set_noise_keys([1], [1])
    from rl_replicas_b200 import _lib
    rows = 16
    cols = [torch.zeros(rows, 4, device="cuda"), torch.zeros(rows, device="cuda"), torch.zeros(rows, device="cuda"),
            torch.zeros(rows, 4, device="cuda"), torch.zeros(rows, device="cuda")]
    tree = torch.zeros(int(_lib.load().b200rl_per_tree_floats(rows)), device="cuda")
    with pytest.raises(B200RLError, match="algo = 5"):
        e.train_prioritized(OffPolicyHparams(), cols, rows, tree, 2, 8, 0, 1)


def _launches(algo, graph, S, B):
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
    """b200rl.h: 10 Lq + 4 Lp + 4 launches per step (+1 with a learned temperature) and 1 per call, Lq and Lp the
    critics' and the policy's Linear layers; host-staged minibatches launch nothing else."""
    S, B = 5, 32
    for learn_alpha in (False, True):
        for graph in (False, True):
            algo = build(O=6, n=4, learn_alpha=learn_alpha)
            fill(algo.replay_buffer, 6, 4, rows=500, seed=6)
            algo.use_device_replay = False
            want = 1 + S * (10 * 3 + 4 * 3 + 4 + int(learn_alpha))
            assert _launches(algo, graph, S, B) == want, (learn_alpha, graph)


def test_learn_solves_the_choice_task(tmp_path, capsys):
    """DiscreteSAC.learn end to end on tests/test_dqn.py's one-step choice task with the seeds of the oracle-driven loop
    in tests/test_discrete_sac.py: the tags are recorded, model.pt is written and reloads, and the evaluation return
    clears the same bar."""
    np.random.seed(0)
    algo = make_dsac(learn_alpha=True)
    algo.learn(output_dir=str(tmp_path), **LEARN)
    after = evaluation_return(algo)
    printed = capsys.readouterr().out
    with capsys.disabled():
        print(f"DiscreteSAC.learn on the choice task: evaluation return {after:.3f}")
    for tag in ("policy/average_loss", "policy/average_log_prob", "alpha/value", "q-function_1/average_loss",
                "q-function_2/average_loss", "q-function_1/avarage_q-value", "evaluation/average_episode_return"):
        assert f"\n{tag}: " in printed, tag
    path = os.path.join(tmp_path, "model.pt")
    assert os.path.exists(path)
    other = make_dsac(seed=5, learn_alpha=True)
    other.load_model(path)
    assert evaluation_return(other) == after
    assert after > RETURN_BAR
