"""GPU: DQN on the off-policy engine -- DQN.train against the float32 oracle (oracle/dqn.py) across calls and target
copies, one step against the float64 reference at edge shapes, bit-identical execution paths, learner groups bit for bit
equal to solo engines, the invalid-action refusal, and DQN.learn end to end."""
import os

import numpy as np
import pytest
import torch

from conftest import rel_err
from oracle import dqn as OD
from test_dqn import DQN_KW, LEARN, N_ACT, O_DIM, RETURN_BAR, evaluation_return, make_dqn

pytestmark = pytest.mark.gpu

GAMMA, LR = 0.99, 1e-3


def build(O=8, n=4, hidden=(64, 64), act=torch.nn.ReLU, seed=0, steps=0, **kw):
    """A DQN learner on a stub discrete environment; ``steps`` > 0 gives its Adam a state at that step count."""
    import types
    from rl_replicas_b200.algorithms import DQN
    from rl_replicas_b200.critics import DiscreteQFunction
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    torch.manual_seed(seed)
    net = MLP([O, *hidden, n], act)
    opt = torch.optim.Adam(net.parameters(), lr=LR)
    for _ in range(steps):  # some arbitrary earlier steps
        opt.zero_grad()
        net(torch.randn(16, O)).pow(2).mean().backward()
        opt.step()
    env = types.SimpleNamespace(action_space=types.SimpleNamespace(n=n, shape=()), spec=types.SimpleNamespace(id="stub"),
                                observation_space=types.SimpleNamespace(shape=(O,)))
    algo = DQN(DiscreteQFunction(net, opt), None, env, None, ReplayBuffer(), None, gamma=GAMMA, **kw)
    with torch.no_grad():  # a target that differs from the online network
        for p in algo.target_q_function.network.parameters():
            p.add_(0.05 * torch.randn_like(p))
    algo.metrics_manager = None
    algo.current_total_steps = 0
    return algo


def fill(rb, O, n, rows=4000, seed=1, bad_action=None):
    from rl_replicas_b200.experience import Experience
    rng = np.random.default_rng(seed)
    e = Experience()
    obs = rng.standard_normal((rows + 1, O)).astype(np.float32)
    acts = rng.integers(0, n, rows).astype(np.int64)
    e.observations = [[obs[i] for i in range(rows)]]
    e.actions = [[a for a in acts]]
    e.rewards = [[float(x) for x in 2.0 * rng.standard_normal(rows)]]  # |delta| on both sides of 1
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
    return OD.DqnOracle(algo.q_function.network, algo.target_q_function.network, algo.q_function.optimizer,
                        gamma=algo.gamma, target_update_interval=algo.target_update_interval, double_q=algo.double_q)


def compare(algo, oracle):
    errs = {"q": rel_err(flat(algo.q_function.network), flat(oracle.q)),
            "target_q": rel_err(flat(algo.target_q_function.network), flat(oracle.q_targ))}
    for key in ("exp_avg", "exp_avg_sq"):
        got, step = adam_flat(algo.q_function.optimizer, key)
        want, step_o = adam_flat(oracle.opt, key)
        errs[key] = rel_err(got, want)
        assert step == step_o, (step, step_o)
    return errs


@pytest.mark.parametrize("start_steps", [0, 7])
@pytest.mark.parametrize("double_q", [False, True])
def test_train_matches_the_oracle_across_calls_and_copies(double_q, start_steps):
    """Three DQN.train calls of 4 steps at interval 3 (copies inside a call and across calls) against the oracle with the
    same minibatches."""
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
F64_CASES = {  # (sizes, hidden, B, double_q)
    "cartpole": ([4, 64, 64, 2], "relu", 256, True),
    "lunar": ([8, 256, 256, 4], "relu", 256, True),
    "n1": ([6, 32, 32, 1], "relu", 33, False),
    "n18": ([6, 64, 64, 18], "relu", 257, True),
    "n33": ([6, 64, 64, 33], "relu", 33, False),
    "w31": ([5, 31, 31, 3], "relu", 1, True),
    "w33": ([5, 33, 33, 3], "relu", 1000, False),
    "two_layer": ([7, 48, 5], "relu", 64, True),
    "four_layer": ([7, 64, 48, 40, 5], "relu", 100, True),
    "tanh": ([8, 64, 64, 4], "tanh", 128, True),
    "tie": ([8, 64, 64, 4], "relu", 128, True),
}
KINK, NEAR_TIE = 1e-6, 1e-5
# Bars: about 4x the largest errors measured on an H100.  The gradient normwise (conftest.rel_err): 3.5e-7 (n1).  Entry
# by entry against its scale (the sum over rows of |a row's contribution|): 4.8e-4 (four_layer; 1.6e-4 lunar, 8.4e-5
# n33, below 7e-6 elsewhere) -- that scale leaves out the cancellation inside the dX chain of a deep ReLU network.
# Q-values: 2.5e-7 of their maximum; the loss: 9.7e-8 of its value.
BAR_GRAD_NORM, BAR_GRAD_ENTRY, BAR_Q, BAR_LOSS = 1.5e-6, 2e-3, 1e-6, 4e-7


def _f64_case(name, seed=0):
    sizes, hidden, B, double_q = F64_CASES[name]
    act = {"relu": torch.nn.ReLU, "tanh": torch.nn.Tanh}[hidden]
    algo = build(O=sizes[0], n=sizes[-1], hidden=tuple(sizes[1:-1]), act=act, seed=seed, double_q=double_q,
                 target_update_interval=1000)
    if name == "tie":  # actions 1 and 2 of the online network are equal on every row, and the largest
        lin = algo.q_function.network.network[-2]
        with torch.no_grad():
            lin.weight[2] = lin.weight[1]
            lin.bias[1] = lin.bias[2] = 10.0
    q_flat, t_flat = flat(algo.q_function.network).astype(np.float64), flat(algo.target_q_function.network).astype(np.float64)
    rng = np.random.default_rng(100 + seed)
    pool = 4 * B + 64
    mb = dict(observations=rng.standard_normal((pool, sizes[0])).astype(np.float32),
              actions=rng.integers(0, sizes[-1], pool).astype(np.float32),
              rewards=(2.0 * rng.standard_normal(pool)).astype(np.float32),
              next_observations=rng.standard_normal((pool, sizes[0])).astype(np.float32),
              dones=rng.random(pool) < 0.1)
    ref = OD.dqn_step_f64(q_flat, t_flat, mb, sizes, hidden, GAMMA, double_q)
    qmax = np.max(np.abs(ref["q_values"])) + 1.0
    keep = (ref["margin"] >= KINK) & (np.abs(np.abs(ref["delta"]) - 1.0) > 1e-4)
    if name != "tie":
        keep &= ref["gap"] > NEAR_TIE * qmax
    rows = np.flatnonzero(keep)[:B]
    assert len(rows) == B, (name, int(keep.sum()))
    mb = {k: v[rows] for k, v in mb.items()}
    return algo, mb, OD.dqn_step_f64(q_flat, t_flat, mb, sizes, hidden, GAMMA, double_q), sizes


@pytest.mark.parametrize("name", list(F64_CASES))
def test_one_step_against_the_float64_reference(name):
    algo, mb, ref, sizes = _f64_case(name)
    if name == "tie":
        with torch.no_grad():
            q = algo.q_function.network(torch.as_tensor(mb["next_observations"]))
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
    both = (np.abs(ref["delta"]) < 1).any() and (np.abs(ref["delta"]) > 1).any()
    print(f"{name}: grad {g_norm:.2e} (entry / scale {g_err:.2e})  q {q_err:.2e}  loss {l_err:.2e}  "
          f"both Huber branches: {both}")
    assert g_norm < BAR_GRAD_NORM and g_err < BAR_GRAD_ENTRY and q_err < BAR_Q and l_err < BAR_LOSS, \
        (g_norm, g_err, q_err, l_err)
    if B >= 33:
        assert both


# ---- execution paths -------------------------------------------------------------------------------------------------
def _run_paths(double_q, device_replay, graph, calls=2, S=5, B=48):
    os.environ["B200RL_OFFPOLICY_GRAPH"] = "1" if graph else "0"
    try:
        algo = build(O=6, n=5, double_q=double_q, target_update_interval=3, steps=1)
        fill(algo.replay_buffer, 6, 5, rows=2000, seed=3)
        algo.use_device_replay = device_replay
        outs = []
        for call in range(calls):
            np.random.seed(30 + call)
            algo.train(algo.replay_buffer, S + (call == calls - 1), B)
            outs.append(algo.last_train_output)
        return outs, [flat(algo.q_function.network), flat(algo.target_q_function.network),
                      adam_flat(algo.q_function.optimizer, "exp_avg")[0]]
    finally:
        os.environ.pop("B200RL_OFFPOLICY_GRAPH", None)


@pytest.mark.parametrize("double_q", [False, True])
def test_host_staged_device_gather_and_graph_paths_are_bit_identical(double_q):
    ref_outs, ref_nets = _run_paths(double_q, False, False)
    for dev, graph in ((True, True), (False, True), (True, False)):
        outs, nets = _run_paths(double_q, dev, graph)
        for a, b in zip(outs, ref_outs):
            assert a.keys() == b.keys() == {"q1_values", "q1_losses"}
            for k in a:
                np.testing.assert_array_equal(a[k], b[k], err_msg=f"{k} dev={dev} graph={graph}")
        for i, (a, b) in enumerate(zip(nets, ref_nets)):
            np.testing.assert_array_equal(a, b, err_msg=f"net {i} dev={dev} graph={graph}")


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
    algo = build(O=6, n=5, seed=seed, steps=steps, double_q=True, target_update_interval=3)
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
        np.testing.assert_array_equal(m.last_train_output["q1_values"], grouped[k].last_train_output["q1_values"])


def test_group_learn_matches_solo_learn(tmp_path):
    from rl_replicas_b200.algorithms import LearnerGroup
    from rl_replicas_b200.utils import set_seed_for_libraries
    kw = dict(LEARN, num_epochs=14)
    solo = []
    for seed in (0, 1):
        set_seed_for_libraries(seed)
        a = make_dqn(seed=seed, **DQN_KW)
        a.learn(output_dir=str(tmp_path / f"solo{seed}"), **kw)
        solo.append(a)
    g = LearnerGroup()
    for seed in (0, 1):
        set_seed_for_libraries(seed)
        g.add(make_dqn(seed=seed, **DQN_KW))
    g.learn([str(tmp_path / f"group{s}") for s in (0, 1)], **kw)
    for a, b in zip(solo, g.members):
        np.testing.assert_array_equal(flat(a.q_function.network), flat(b.q_function.network))
        np.testing.assert_array_equal(flat(a.target_q_function.network), flat(b.target_q_function.network))


# ---- refusals and end to end ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bad", [4.0, 1.5, -1.0, float("nan")])
def test_invalid_action_raises_and_leaves_the_host_modules_unchanged(bad):
    from rl_replicas_b200._lib import B200RLError
    algo = build(O=6, n=4, target_update_interval=2)
    fill(algo.replay_buffer, 6, 4, rows=64, seed=5, bad_action=bad)
    before = [flat(algo.q_function.network), flat(algo.target_q_function.network)]
    np.random.seed(0)
    with pytest.raises(B200RLError, match=r"DQN learner 0, step \d+: \d+ minibatch rows hold an action"):
        algo.train(algo.replay_buffer, 8, 64)  # 512 draws of 64 rows: the bad row is drawn
    for x, y in zip(before, [flat(algo.q_function.network), flat(algo.target_q_function.network)]):
        np.testing.assert_array_equal(x, y)
    assert algo._adam_step_count(algo.q_function.optimizer, list(algo.q_function.network.network)[::2]) == 0


def test_engine_refuses_bad_dqn_configurations():
    from rl_replicas_b200._lib import B200RLError
    from rl_replicas_b200.engine import OffPolicyEngine
    with pytest.raises(B200RLError, match="n_q = 1"):
        OffPolicyEngine(None, [4, 16, 2], 2, 8, 2, algo=OffPolicyEngine.DQN)
    with pytest.raises(B200RLError, match="policy description must be zeroed"):
        OffPolicyEngine([4, 16, 2], [4, 16, 2], 1, 8, 2, algo=OffPolicyEngine.DQN)
    e = OffPolicyEngine(None, [4, 16, 2], 1, 8, 2, q_acts=("relu", "identity"), algo=OffPolicyEngine.DQN)
    z = lambda *s: np.zeros(s, np.float32)
    from rl_replicas_b200._lib import OffPolicyHparams
    with pytest.raises(B200RLError, match="set_dqn"):
        e.train(OffPolicyHparams(), z(2, 8, 4), z(2, 8), z(2, 8), z(2, 8, 4), z(2, 8))
    with pytest.raises(B200RLError, match="target_update_interval"):
        e.set_dqn(0, False)


def test_learn_solves_the_choice_task(tmp_path, capsys):
    """DQN.learn end to end on tests/test_dqn.py's one-step choice task with the seeds of the oracle-driven loop there:
    the tags are recorded, model.pt is written and reloads, and the evaluation return clears the same bar."""
    np.random.seed(0)
    algo = make_dqn(**DQN_KW)
    algo.learn(output_dir=str(tmp_path), **LEARN)
    after = evaluation_return(algo)
    printed = capsys.readouterr().out
    with capsys.disabled():
        print(f"DQN.learn on the choice task: evaluation return {after:.3f}")
    for tag in ("q-function/average_loss", "q-function/avarage_q-value", "exploration/epsilon",
                "evaluation/average_episode_return"):
        assert f"\n{tag}: " in printed, tag
    path = os.path.join(tmp_path, "model.pt")
    assert os.path.exists(path)
    other = make_dqn(seed=5, **DQN_KW)
    other.load_model(path)
    assert evaluation_return(other) == after  # the reloaded networks act exactly as the trained ones
    assert after > RETURN_BAR
