"""GPU parity of TD3.train / DDPG.train through the reference-facing classes (C ABI underneath) against the
reference's own outputs (golden: same replay content, same numpy / torch seeds -> same minibatches and noise) and the
numpy oracle at the benchmark shape (256-256 nets, B = 256)."""
import types

import numpy as np
import pytest
import torch

from conftest import load_golden, rel_err
from oracle import offpolicy as OP
from oracle import onpolicy as O

pytestmark = pytest.mark.gpu
O_DIM, A_DIM = 11, 3


class Rec:
    def __init__(self):
        self.s = {}

    def record_scalar(self, tag, scalar, total_steps=None, tensorboard=False):
        self.s[tag] = float(scalar)


def flat(m):
    return torch.nn.utils.parameters_to_vector(m.parameters()).detach().numpy()


def build(twin, hidden, pflat, qflats):
    from rl_replicas_b200.algorithms import DDPG, TD3
    from rl_replicas_b200.algorithms._onpolicy import describe_mlp, write_flat
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import DeterministicPolicy, RandomPolicy
    from rl_replicas_b200.q_function import QFunction
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    pnet = MLP([O_DIM, hidden, hidden, A_DIM], torch.nn.ReLU, torch.nn.Tanh)
    write_flat(describe_mlp(pnet)[3], pflat)
    policy = DeterministicPolicy(pnet, torch.optim.Adam(pnet.parameters(), lr=1e-3))
    qfs = []
    for qf in qflats:
        n = MLP([O_DIM + A_DIM, hidden, hidden, 1], torch.nn.ReLU)
        write_flat(describe_mlp(n)[3], qf)
        qfs.append(QFunction(n, torch.optim.Adam(n.parameters(), lr=1e-3)))
    env = types.SimpleNamespace(action_space=types.SimpleNamespace(high=np.ones(A_DIM, np.float32), shape=(A_DIM,)),
                                spec=types.SimpleNamespace(id="stub"))
    rb = ReplayBuffer()
    algo = TD3(policy, RandomPolicy(None), qfs[0], qfs[1], env, None, rb, None) if twin else \
        DDPG(policy, RandomPolicy(None), qfs[0], env, None, rb, None)
    algo.metrics_manager = Rec()
    algo.current_total_steps = 0
    return algo, rb


def fill_buffer(rb, g):
    """Rebuild the reference run's replay content from the raw arrays stored in the fixture."""
    from rl_replicas_b200.experience import Experience
    obs, act, rew, dones = g["raw_obs"], g["raw_act"], g["raw_rew"], g["raw_dones"]
    e, start, n = Experience(), 0, len(rew)
    for t in range(n):
        if dones[t] or t == n - 1:
            e.observations.append([obs[i] for i in range(start, t + 1)])
            e.actions.append([act[i] for i in range(start, t + 1)])
            e.rewards.append([float(x) for x in rew[start:t + 1]])
            d = [False] * (t + 1 - start)
            d[-1] = bool(dones[t])
            e.dones.append(d)
            e.last_observations.append(obs[t + 1])
            start = t + 1
    rb.add_experience(e)


@pytest.mark.parametrize("case,twin", [("td3_small", True), ("ddpg_small", False)])
def test_train_matches_reference_golden(case, twin):
    g = load_golden(case)
    algo, rb = build(twin, 64, g["policy_flat0"], [g["q1_flat0"]] + ([g["q2_flat0"]] if twin else []))
    fill_buffer(rb, g)
    np.random.seed(int(g["seed_train"]))
    torch.manual_seed(int(g["seed_train"]))
    algo.train(rb, int(g["S"]), int(g["B"]))
    out = algo.last_train_output
    # the host side reproduced the reference's random streams exactly
    q_nets = [algo.q_function_1, algo.q_function_2] if twin else [algo.q_function]
    t_nets = [algo.target_q_function_1, algo.target_q_function_2] if twin else [algo.target_q_function]
    assert rel_err(flat(algo.policy.network), g["policy_flat_final"]) < 2e-5
    assert rel_err(flat(algo.target_policy.network), g["target_policy_flat_final"]) < 2e-5
    for i, (q, t) in enumerate(zip(q_nets, t_nets)):
        assert rel_err(flat(q.network), g[f"q{i + 1}_flat_final"]) < 2e-5
        assert rel_err(flat(t.network), g[f"target_q{i + 1}_flat_final"]) < 2e-5
    m = algo.metrics_manager.s
    for k, v in g.items():
        if k.startswith("metric:"):
            assert abs(m[k[7:]] - float(v)) < 1e-5 * max(1.0, abs(float(v))), k
    assert len(out["policy_losses"]) == (4 if twin else 7)
    p0 = algo.policy.optimizer.param_groups[0]["params"][0]
    assert float(algo.policy.optimizer.state[p0]["step"]) == float(g["policy_adam_step"])


@pytest.mark.parametrize("twin", [True, False])
def test_train_vs_oracle_benchmark_shape(twin):
    """BASELINE config 4 shape: 256-256 nets, minibatch 256, 10 steps, against the numpy oracle."""
    rng = np.random.default_rng(1)
    H = 256
    mk = lambda sz: [(rng.standard_normal((o, i)).astype(np.float32) / np.sqrt(i), 0.05 * rng.standard_normal(o).astype(np.float32))
                     for i, o in zip(sz[:-1], sz[1:])]
    PS, QS = [O_DIM, H, H, A_DIM], [O_DIM + A_DIM, H, H, 1]
    pl, q1l, q2l = mk(PS), mk(QS), mk(QS)
    algo, rb = build(twin, H, O.flatten_layers(pl), [O.flatten_layers(q1l)] + ([O.flatten_layers(q2l)] if twin else []))
    from rl_replicas_b200.experience import Experience
    n = 5000
    e = Experience()
    obs = rng.standard_normal((n + 1, O_DIM)).astype(np.float32)
    e.observations = [[obs[i] for i in range(n)]]
    e.actions = [[rng.uniform(-1, 1, A_DIM).astype(np.float32) for _ in range(n)]]
    e.rewards = [[float(x) for x in rng.standard_normal(n)]]
    e.dones = [[bool(x) for x in (rng.random(n) < 0.01)]]
    e.last_observations = [obs[n]]
    rb.add_experience(e)
    S, B = 10, 256
    np.random.seed(7)
    torch.manual_seed(7)
    state_np, state_t = np.random.get_state(), torch.get_rng_state()
    algo.train(rb, S, B)
    # replay the same random streams for the oracle
    np.random.set_state(state_np)
    torch.set_rng_state(state_t)
    mbs = [rb.sample_minibatch(B) for _ in range(S)]
    noise = torch.stack([torch.randn(B, A_DIM) for _ in range(S)]).numpy() if twin else None
    nets = {"policy": pl, "q1": q1l, "target_policy": [(w.copy(), b.copy()) for w, b in pl],
            "target_q1": [(w.copy(), b.copy()) for w, b in q1l]}
    names = ["policy", "q1"]
    if twin:
        nets["q2"], nets["target_q2"] = q2l, [(w.copy(), b.copy()) for w, b in q2l]
        names.append("q2")
    adams = {k: O.AdamState(O.flatten_layers(nets[k]).size, 1e-3) for k in names}
    logs = OP.offpolicy_train(nets, adams, mbs, noise, policy_delay=2 if twin else 1, twin=twin)
    out = algo.last_train_output
    q_nets = [algo.q_function_1, algo.q_function_2] if twin else [algo.q_function]
    errs = {"q1_values": rel_err(out["q1_values"], np.stack(logs["q1_values"])),
            "q1_losses": rel_err(out["q1_losses"], np.asarray(logs["q1_losses"])),
            "policy_losses": rel_err(out["policy_losses"], np.asarray(logs["policy_losses"])),
            "policy": rel_err(flat(algo.policy.network), O.flatten_layers(nets["policy"])),
            "target_policy": rel_err(flat(algo.target_policy.network), O.flatten_layers(nets["target_policy"]))}
    for i, q in enumerate(q_nets):
        errs[f"q{i + 1}"] = rel_err(flat(q.network), O.flatten_layers(nets[f"q{i + 1}"]))
    print("benchmark-shape errors:", {k: f"{v:.2e}" for k, v in errs.items()})
    for k, v in errs.items():
        assert v < 2e-5, (k, v, errs)  # north_star: 1e-5 per tensor; 2e-5 after ten Adam steps of three networks


@pytest.mark.parametrize("twin", [True, False])
def test_device_replay_and_graph_replay_match_the_staged_path(twin):
    """b200rl_offpolicy_train_gather (replay columns in HBM, only indices uploaded) and the CUDA-graph replay of the
    S-step loop give BIT-IDENTICAL results to host-staged minibatches run with plain launches of one kernel per
    operation.  TD3 (twin critics, delayed policy step, smoothing noise) and DDPG."""
    import os
    from rl_replicas_b200.experience import Experience
    rng = np.random.default_rng(3)
    H, S, B = 64, 6, 32
    mk = lambda sz: O.flatten_layers([(rng.standard_normal((o, i)).astype(np.float32) / np.sqrt(i), np.zeros(o, np.float32))
                                      for i, o in zip(sz[:-1], sz[1:])])
    p0, q10, q20 = mk([O_DIM, H, H, A_DIM]), mk([O_DIM + A_DIM, H, H, 1]), mk([O_DIM + A_DIM, H, H, 1])
    n = 3000
    ex = Experience()
    obs = rng.standard_normal((n + 1, O_DIM)).astype(np.float32)
    ex.observations = [[obs[i] for i in range(n)]]
    ex.actions = [[a for a in rng.uniform(-1, 1, (n, A_DIM)).astype(np.float32)]]
    ex.rewards = [[float(x) for x in rng.standard_normal(n)]]
    ex.dones = [[bool(x) for x in (rng.random(n) < 0.01)]]
    ex.last_observations = [obs[n]]

    def run(device_replay, graph):
        os.environ["B200RL_OFFPOLICY_GRAPH"] = "1" if graph else "0"
        algo, rb = build(twin, H, p0, [q10, q20] if twin else [q10])
        rb.add_experience(ex)
        algo.use_device_replay = device_replay  # False: minibatches gathered on the host and uploaded
        outs = []
        for call in range(3):  # the 2nd call replays the captured graph
            np.random.seed(10 + call)
            torch.manual_seed(10 + call)
            algo.train(rb, S + (call == 2), B)  # the third call changes the shape: the graph is recaptured
            outs.append(algo.last_train_output)
        qs = (algo.q_function_1, algo.q_function_2) if twin else (algo.q_function,)
        tq = (algo.target_q_function_1, algo.target_q_function_2) if twin else (algo.target_q_function,)
        nets = [flat(m.network) for m in (algo.policy, algo.target_policy) + qs + tq]
        return outs, nets

    try:
        ref_outs, ref_nets = run(False, False)
        for dev, graph in ((True, True), (False, True), (True, False)):
            outs, nets = run(dev, graph)
            for a, b in zip(outs, ref_outs):
                for k in a:
                    np.testing.assert_array_equal(a[k], b[k], err_msg=f"{k} dev={dev} graph={graph}")
            for i, (a, b) in enumerate(zip(nets, ref_nets)):
                np.testing.assert_array_equal(a, b, err_msg=f"net {i} dev={dev} graph={graph}")
    finally:
        os.environ.pop("B200RL_OFFPOLICY_GRAPH", None)


def test_train_gather_rejects_indices_outside_the_replay_columns():
    from rl_replicas_b200._lib import B200RLError
    rng = np.random.default_rng(0)
    H = 32
    mk = lambda sz: O.flatten_layers([(rng.standard_normal((o, i)).astype(np.float32) / np.sqrt(i), np.zeros(o, np.float32))
                                      for i, o in zip(sz[:-1], sz[1:])])
    algo, rb = build(True, H, mk([O_DIM, H, H, A_DIM]), [mk([O_DIM + A_DIM, H, H, 1]), mk([O_DIM + A_DIM, H, H, 1])])
    eng = algo._ensure_engine(2, 8)
    rows = 100
    cols = (torch.zeros(rows, O_DIM, device="cuda"), torch.zeros(rows, A_DIM, device="cuda"), torch.zeros(rows, device="cuda"),
            torch.zeros(rows, O_DIM, device="cuda"), torch.zeros(rows, device="cuda"))
    idx = np.zeros((2, 8), np.int64)
    idx[1, 3] = rows  # one past the end
    with pytest.raises(B200RLError, match="outside"):
        eng.train_gather(algo._hparams(True, 2), cols, rows, idx, np.zeros((2, 8, A_DIM), np.float32))


@pytest.mark.parametrize("n_q", [1, 2])
def test_state_blob_round_trip_matches_the_per_network_accessors(n_q):
    """b200rl_offpolicy_get_state / set_state move every network and Adam state in one copy (segments padded to 64
    floats); the per-network accessors see the same values, and a blob written back reproduces itself."""
    from rl_replicas_b200.engine import OffPolicyEngine
    rng = np.random.default_rng(n_q)
    e = OffPolicyEngine([11, 40, 24, 3], [14, 40, 24, 1], n_q, 32, 4)
    layout, total = e.state_layout()
    assert total % 64 == 0 and all(off % 64 == 0 for _, _, off, _ in layout)
    blob = np.full(total, np.nan, np.float32)  # padding stays NaN: it must never be read
    want = {}
    for kind, i, off, n in layout:
        x = rng.standard_normal(n).astype(np.float32)
        if kind == "v":
            x = np.abs(x)
        blob[off:off + n] = x
        want[(kind, i)] = x
    steps = [3, 5, 7 if n_q == 2 else 0]
    e.set_state(blob, steps)
    for (kind, i), x in want.items():
        if kind == "params":
            np.testing.assert_array_equal(e.get_params(i), x)
    for i in range(1 + n_q):
        m, v, step = e.get_adam(i)
        np.testing.assert_array_equal(m, want[("m", i)])
        np.testing.assert_array_equal(v, want[("v", i)])
        assert step == steps[i]
    # per-network writes show up in the blob
    newp = rng.standard_normal(want[("params", 1)].size).astype(np.float32)
    e.set_params(1, newp)
    back, steps_back = e.get_state()
    assert steps_back[:1 + n_q] == steps[:1 + n_q]
    for kind, i, off, n in layout:
        np.testing.assert_array_equal(back[off:off + n], newp if (kind, i) == ("params", 1) else want[(kind, i)])
    e.close()


@pytest.mark.parametrize("twin", [True, False])
def test_device_side_draws_opt_in(twin):
    """use_device_rng: indices (uniform over the live rows of the replay ring, physical addressing across the wrap) and
    target-smoothing noise come from a Philox generator on the device.  The draws are read back and replayed through
    the numpy oracle (2e-5 like the host-drawn path); they are reproducible per (seed, call), differ between calls, and
    have the right distributions."""
    from rl_replicas_b200.experience import Experience
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    rng = np.random.default_rng(11)
    H, S, B = 64, 8, 64
    mk = lambda sz: [(rng.standard_normal((o, i)).astype(np.float32) / np.sqrt(i), 0.05 * rng.standard_normal(o).astype(np.float32))
                     for i, o in zip(sz[:-1], sz[1:])]
    pl, q1l, q2l = mk([O_DIM, H, H, A_DIM]), mk([O_DIM + A_DIM, H, H, 1]), mk([O_DIM + A_DIM, H, H, 1])

    def fresh():
        algo, _ = build(twin, H, O.flatten_layers(pl), [O.flatten_layers(q1l)] + ([O.flatten_layers(q2l)] if twin else []))
        rb = ReplayBuffer(buffer_size=3000)  # 4000 rows into 3000: the ring has wrapped, head != 0
        r2 = np.random.default_rng(5)
        for chunk in range(4):
            n = 1000
            e = Experience()
            obs = r2.standard_normal((n + 1, O_DIM)).astype(np.float32)
            e.observations = [[obs[i] for i in range(n)]]
            e.actions = [[r2.uniform(-1, 1, A_DIM).astype(np.float32) for _ in range(n)]]
            e.rewards = [[float(x) for x in r2.standard_normal(n)]]
            e.dones = [[bool(x) for x in (r2.random(n) < 0.01)]]
            e.last_observations = [obs[n]]
            rb.add_experience(e)
        algo.use_device_rng, algo.device_rng_seed = True, 1234
        return algo, rb

    algo, rb = fresh()
    start, size, cap = rb.ring()
    assert size == 3000 and start != 0
    algo.train(rb, S, B)
    idx, noise = algo._engine.get_draws(S, B, with_noise=twin)
    assert (((idx - start) % cap) < size).all() and idx.min() >= 0 and idx.max() < cap
    # the oracle on exactly these draws
    mbs = [{k: rb._cols[k][idx[s]] for k in rb.COLUMNS} for s in range(S)]
    nets = {"policy": [(w.copy(), b.copy()) for w, b in pl], "q1": [(w.copy(), b.copy()) for w, b in q1l],
            "target_policy": [(w.copy(), b.copy()) for w, b in pl], "target_q1": [(w.copy(), b.copy()) for w, b in q1l]}
    names = ["policy", "q1"]
    if twin:
        nets["q2"], nets["target_q2"] = [(w.copy(), b.copy()) for w, b in q2l], [(w.copy(), b.copy()) for w, b in q2l]
        names.append("q2")
    adams = {k: O.AdamState(O.flatten_layers(nets[k]).size, 1e-3) for k in names}
    logs = OP.offpolicy_train(nets, adams, mbs, noise, policy_delay=2 if twin else 1, twin=twin)
    out = algo.last_train_output
    assert rel_err(out["q1_values"], np.stack(logs["q1_values"])) < 2e-5
    assert rel_err(out["q1_losses"], np.asarray(logs["q1_losses"])) < 2e-5
    assert rel_err(flat(algo.policy.network), O.flatten_layers(nets["policy"])) < 2e-5
    q_nets = [algo.q_function_1, algo.q_function_2] if twin else [algo.q_function]
    for i, q in enumerate(q_nets):
        assert rel_err(flat(q.network), O.flatten_layers(nets[f"q{i + 1}"])) < 2e-5
    # reproducible per (seed, call); the next call draws a different block
    algo2, rb2 = fresh()
    algo2.train(rb2, S, B)
    idx2, noise2 = algo2._engine.get_draws(S, B, with_noise=twin)
    np.testing.assert_array_equal(idx, idx2)
    if twin:
        np.testing.assert_array_equal(noise, noise2)
    algo2.train(rb2, S, B)
    idx3, _ = algo2._engine.get_draws(S, B, with_noise=False)
    assert (idx3 != idx).mean() > 0.9
    algo2.device_rng_seed = 99
    algo2._device_rng_calls = 0
    algo2.train(rb2, S, B)
    assert (algo2._engine.get_draws(S, B, with_noise=False)[0] != idx).mean() > 0.9
    # distributions over a larger block: 50 x 256 indices, 38400 normal draws
    algo2.train(rb2, 50, 256)
    big, eps = algo2._engine.get_draws(50, 256, with_noise=twin)
    logical = (big - rb2.ring()[0]) % cap
    assert abs(logical.mean() / size - 0.5) < 0.02 and logical.min() < 30 and logical.max() > size - 30
    counts = np.bincount(logical.ravel() * 10 // size, minlength=10)
    assert counts.min() > 0.85 * big.size / 10 and counts.max() < 1.15 * big.size / 10
    if twin:
        assert abs(eps.mean()) < 0.03 and abs(eps.std() - 1.0) < 0.03 and np.abs(eps).max() < 6.5
        assert abs(np.mean(eps ** 3)) < 0.1 and abs(np.mean(eps ** 4) - 3.0) < 0.25  # skewness, kurtosis of N(0, 1)
