"""CPU: dueling Q networks' host side -- networks.DuelingMLP against eq. 9 of Wang et al. (2016), its flat parameter
layout and checkpoint keys, the DQN / C51 / QRDQN constructors' acceptances and refusals (and the refusals of the
algorithms that take plain MLPs only), the LearnerGroup signature, the checkpoint round trip, the float64 dueling
oracle (oracle/dueling.py) against the torch module and against the float32 oracles, and the oracle-driven learn()
loop that sets the bar for the GPU end-to-end test (tests/test_gpu_dueling.py)."""
import types

import numpy as np
import pytest
import torch

from oracle import c51 as OC
from oracle import dqn as OD
from oracle import dueling as ODu
from oracle import qr as OQ
from test_c51 import ATOMS
from test_dqn import DQN_KW, LEARN, N_ACT, O_DIM, RETURN_BAR, ChooseEnv, OracleDQN, evaluation_return, flat, \
    random_minibatch

HIDDEN = 64


def make(kind="dqn", hidden=HIDDEN, seed=0, lr=1e-3, n_actions=N_ACT, k=None, n_quantiles=32, atoms=ATOMS,
         replay_buffer=None, **kw):
    """A DQN / C51 / QRDQN learner on ChooseEnv with a DuelingMLP([obs, hidden, hidden], n_actions, k) Q network (k
    defaults to what the algorithm needs)."""
    from rl_replicas_b200.algorithms import C51, DQN, QRDQN
    from rl_replicas_b200.critics import CategoricalQFunction, DiscreteQFunction, QuantileQFunction
    from rl_replicas_b200.evaluator import Evaluator
    from rl_replicas_b200.networks import DuelingMLP
    from rl_replicas_b200.policies import RandomPolicy
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    from rl_replicas_b200.samplers import BatchSampler
    torch.manual_seed(seed)
    env = ChooseEnv()
    need = {"dqn": 1, "c51": atoms["n_atoms"], "qr": n_quantiles}[kind]
    net = DuelingMLP([O_DIM, hidden, hidden], n_actions, need if k is None else k)
    opt = torch.optim.Adam(net.parameters(), lr=lr)
    qf, cls = {"dqn": lambda: (DiscreteQFunction(net, opt), DQN),
               "c51": lambda: (CategoricalQFunction(net, opt, **atoms), C51),
               "qr": lambda: (QuantileQFunction(net, opt, n_quantiles=n_quantiles), QRDQN)}[kind]()
    return cls(qf, RandomPolicy(env.action_space), env, BatchSampler(env, seed=0),
               replay_buffer if replay_buffer is not None else ReplayBuffer(buffer_size=100000), Evaluator(seed=0), **kw)


def test_forward_is_eq_9_per_output_column():
    from rl_replicas_b200.networks import DuelingMLP
    torch.manual_seed(0)
    net = DuelingMLP([5, 16, 8], 4, 3)
    x = torch.randn(7, 5)
    h = torch.relu(x @ net.trunk[0].weight.T + net.trunk[0].bias)
    v = net.value(h)  # [7, 3]
    a = net.advantage(h).reshape(7, 4, 3)
    want = torch.stack([v + (a[:, j] - a.mean(1)) for j in range(4)], 1).reshape(7, 12)
    torch.testing.assert_close(net(x), want, rtol=0, atol=1e-6)
    # the mean advantage of every column is zero: the action-mean of Q is V
    torch.testing.assert_close(net(x).reshape(7, 4, 3).mean(1), v, rtol=0, atol=1e-6)
    one = DuelingMLP([5, 16, 8], 1, 3)
    assert torch.equal(one(x), one.value(one.trunk(x)))  # n = 1: A - mean(A) is exactly 0
    assert net(torch.randn(2, 6, 5)).shape == (2, 6, 12)


def test_flat_layout_state_dict_keys_and_parameter_count():
    from rl_replicas_b200.algorithms._onpolicy import describe_mlp, flat_params, write_flat
    from rl_replicas_b200.algorithms.dqn import describe_q_network
    from rl_replicas_b200.networks import MLP, DuelingMLP
    net = DuelingMLP([6, 20, 12], 5, 7, torch.nn.Tanh)
    assert list(net.state_dict()) == ["trunk.0.weight", "trunk.0.bias", "value.0.weight", "value.0.bias",
                                      "value.2.weight", "value.2.bias", "advantage.0.weight", "advantage.0.bias",
                                      "advantage.2.weight", "advantage.2.bias"]
    sizes, hid, out, lins, k = describe_q_network(net)
    assert (sizes, hid, out, k) == ([6, 20, 12, 35], "tanh", "identity", 7)
    f = flat_params(lins)
    np.testing.assert_array_equal(f, torch.nn.utils.parameters_to_vector(net.parameters()).detach().numpy())
    O, h1, h2, K, n = 6, 20, 12, 7, 5
    assert f.size == h1 * (O + 1) + 2 * h2 * (h1 + 1) + K * (h2 + 1) + n * K * (h2 + 1)
    write_flat(lins, f * 2)
    np.testing.assert_array_equal(flat_params(lins), f * 2)
    with pytest.raises(NotImplementedError):
        describe_mlp(net)  # the plain describer keeps refusing it
    assert describe_q_network(MLP([2, 8, 3], torch.nn.ReLU))[4] == 0
    with pytest.raises(NotImplementedError, match="activations"):
        describe_q_network(DuelingMLP([2, 8, 8], 3, 1, torch.nn.ELU))
    for bad in (dict(sizes=[2, 8], n_actions=3), dict(sizes=[2, 8, 8], n_actions=0),
                dict(sizes=[2, 8, 8], n_actions=3, outputs_per_action=0)):
        with pytest.raises(ValueError):
            DuelingMLP(**bad)


@pytest.mark.parametrize("kind", ["dqn", "c51", "qr"])
def test_constructors_accept_matching_and_refuse_mismatched_dueling_networks(kind):
    algo = make(kind)
    assert algo.n_actions == N_ACT
    with pytest.raises(ValueError, match="n_actions = 4"):
        make(kind, n_actions=N_ACT + 1)
    want = {"dqn": "outputs_per_action = 1", "c51": "outputs_per_action = 51", "qr": "outputs_per_action = 32"}[kind]
    with pytest.raises(ValueError, match=want):
        make(kind, k=2)


def test_td3_sac_and_ppo_keep_refusing_a_dueling_network():
    from rl_replicas_b200.algorithms import PPO, SAC
    from rl_replicas_b200.networks import MLP, DuelingMLP
    from rl_replicas_b200.policies import CategoricalPolicy, SquashedGaussianPolicy
    from rl_replicas_b200.q_function import QFunction
    from rl_replicas_b200.value_function import ValueFunction
    from test_offpolicy_group import td3
    t = td3(0)
    net = DuelingMLP([5, 16, 16], 1)
    t.q_function_1 = QFunction(net, torch.optim.Adam(net.parameters()))
    with pytest.raises(NotImplementedError):
        t._learner_nets()
    env = types.SimpleNamespace(action_space=types.SimpleNamespace(shape=(2,), high=np.ones(2, np.float32)),
                                spec=types.SimpleNamespace(id="synthetic"))
    pnet = MLP([3, 16, 4], torch.nn.ReLU)
    policy = SquashedGaussianPolicy(pnet, torch.optim.Adam(pnet.parameters()), action_limit=1.0)
    qs = [QFunction(n, torch.optim.Adam(n.parameters())) for n in (DuelingMLP([5, 16, 16], 1), MLP([5, 16, 1]))]
    with pytest.raises(NotImplementedError):
        SAC(policy, None, qs[0], qs[1], env, None, None, None)
    vnet = DuelingMLP([3, 16, 16], 1)
    cnet = MLP([3, 16, 2])
    ppo = PPO(CategoricalPolicy(cnet, torch.optim.Adam(cnet.parameters())),
              ValueFunction(vnet, torch.optim.Adam(vnet.parameters())), env, None)
    with pytest.raises(NotImplementedError):
        ppo._describe()


def test_group_signature_refuses_mixed_kinds_and_differing_shapes():
    from rl_replicas_b200.algorithms import LearnerGroup
    from test_dqn import make_dqn
    from test_qr import make_qr
    g = LearnerGroup()
    g.add(make("dqn", seed=0, **DQN_KW))
    g.add(make("dqn", seed=1, **DQN_KW))
    with pytest.raises(ValueError, match="network kind"):
        g.add(make_dqn(seed=2, **DQN_KW))  # a plain MLP of the same widths
    with pytest.raises(ValueError, match="dueling"):
        g.add(make("dqn", seed=2, hidden=32, **DQN_KW))
    p = LearnerGroup()
    p.add(make_dqn(seed=0, **DQN_KW))
    with pytest.raises(ValueError, match="network kind"):
        p.add(make("dqn", seed=1, **DQN_KW))
    q = LearnerGroup()
    q.add(make("qr", seed=0, n_quantiles=32))
    with pytest.raises(ValueError, match=r"dueling .*\(64, 64, 16\) != \(64, 64, 32\)"):
        q.add(make("qr", seed=1, n_quantiles=16))
    with pytest.raises(ValueError, match="network kind"):
        q.add(make_qr(seed=1))


def test_save_and_load_round_trip(tmp_path):
    algo = make("qr", seed=1)
    algo.current_total_steps = 99
    algo.q_function.network(torch.randn(8, O_DIM)).sum().backward()
    algo.q_function.optimizer.step()
    with torch.no_grad():
        for p in algo.target_q_function.network.parameters():
            p.add_(0.5)
    path = str(tmp_path / "model.pt")
    algo.save_model(3, path)
    ckpt = torch.load(path, weights_only=True)
    assert list(ckpt["q_function_state_dict"])[:2] == ["trunk.0.weight", "trunk.0.bias"]
    other = make("qr", seed=2)
    assert other.load_model(path) == 3 and other.current_total_steps == 99
    for a, b in ((algo.q_function.network, other.q_function.network),
                 (algo.target_q_function.network, other.target_q_function.network)):
        for (k, x), (_, y) in zip(a.state_dict().items(), b.state_dict().items()):
            assert torch.equal(x, y), k
    from rl_replicas_b200.algorithms.dqn import describe_q_network
    assert other._adam_step_count(other.q_function.optimizer, describe_q_network(other.q_function.network)[3]) == 1


@pytest.mark.parametrize("n,k,hidden", [(1, 1, "relu"), (4, 3, "relu"), (18, 1, "tanh"), (2, 51, "relu")])
def test_float64_forward_matches_the_torch_module(n, k, hidden):
    from rl_replicas_b200.networks import DuelingMLP
    torch.manual_seed(n + k)
    net = DuelingMLP([5, 33, 17], n, k, {"relu": torch.nn.ReLU, "tanh": torch.nn.Tanh}[hidden]).double()
    x = torch.randn(11, 5, dtype=torch.float64)
    q, margin = ODu.dueling_mlp(torch.nn.utils.parameters_to_vector(net.parameters()).detach(), [5, 33, 17, n * k], k,
                                x, hidden)
    torch.testing.assert_close(q, net(x).detach(), rtol=1e-14, atol=1e-14)
    assert margin.shape == (11,) and (np.isinf(margin.numpy()).all() == (hidden == "tanh"))
    if n == 1:
        assert torch.equal(q, net.value(net.trunk(x)).detach())


def _networks(kind, seed):
    algo = make(kind, seed=seed, hidden=32)
    with torch.no_grad():  # a target that differs from the online network
        for p in algo.target_q_function.network.parameters():
            p.add_(0.05 * torch.randn_like(p))
    return algo


@pytest.mark.parametrize("double_q", [False, True])
@pytest.mark.parametrize("kind", ["dqn", "c51", "qr"])
def test_float32_oracles_take_a_dueling_network_and_agree_with_the_float64_step(kind, double_q):
    """The float32 oracles are used as they are: one step's Q-values, loss and parameter update against the float64
    step of oracle/dueling.py."""
    algo = _networks(kind, seed=3)
    q, qt, opt = algo.q_function, algo.target_q_function, algo.q_function.optimizer
    sizes = [O_DIM, 32, 32, q.network.n_actions * q.network.outputs_per_action]
    mb = random_minibatch(np.random.default_rng(5), 64)
    p0, t0 = flat(q.network), flat(qt.network)
    if kind == "dqn":
        oracle = OD.DqnOracle(q.network, qt.network, opt, gamma=0.99, double_q=double_q)
        ref = ODu.dqn_step_f64(p0, t0, mb, sizes, "relu", 0.99, double_q)
    elif kind == "c51":
        oracle = OC.C51Oracle(q.network, qt.network, opt, gamma=0.99, double_q=double_q, **ATOMS)
        ref = ODu.c51_step_f64(p0, t0, mb, sizes, ATOMS["n_atoms"], ATOMS["v_min"], ATOMS["v_max"], "relu", 0.99,
                               double_q)
    else:
        oracle = OQ.QrDqnOracle(q.network, qt.network, opt, n_quantiles=q.n_quantiles, gamma=0.99, double_q=double_q)
        ref = ODu.qr_step_f64(p0, t0, mb, sizes, q.n_quantiles, "relu", 0.99, double_q)
    logs = oracle.train([mb])
    np.testing.assert_allclose(logs["q1_values"][0], ref["q_values"], rtol=1e-5, atol=1e-5)
    assert abs(logs["q1_losses"][0] - ref["loss"]) <= 1e-5 * max(1.0, abs(ref["loss"]))
    # Adam's first step moves every parameter by lr * g / (|g| + eps): compare the update's direction entry by entry
    # where the float64 gradient is clear of zero
    step = flat(oracle.q) - p0
    clear = np.abs(ref["grad"]) > 1e-3 * np.abs(ref["grad"]).max()
    assert clear.sum() > 100
    np.testing.assert_array_equal(np.sign(step[clear]), -np.sign(ref["grad"][clear]))
    assert np.all(ref["scale"] >= np.abs(ref["grad"]) * (1 - 1e-12))


def test_oracle_driven_learn_loop_solves_the_choice_task(tmp_path):
    """The bar the GPU learn() loop must clear (tests/test_gpu_dueling.py) is one the oracle reaches with the same
    seeds."""
    np.random.seed(0)
    algo = make("dqn", **DQN_KW)
    OracleDQN.patch(algo)
    before = evaluation_return(algo)
    algo.learn(output_dir=str(tmp_path), **LEARN)
    after = evaluation_return(algo)
    print(f"oracle-driven learn: evaluation return {before:.3f} -> {after:.3f}")
    assert before < 0.6 and after > RETURN_BAR, (before, after)
