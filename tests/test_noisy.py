"""CPU: noisy networks' host side -- networks.NoisyLinear against the factorized-noise formulas (f, the rounding order,
eval mode, initialization, parameter order and checkpoint keys), reset_noise under torch.manual_seed,
NoisyGreedyPolicy's draws, the DQN / C51 / QRDQN acceptances and the refusals of the other algorithms, the
LearnerGroup signature, the float32 noisy oracle against the float64 one (oracle/noisy.py), the oracle-driven learn()
loop without epsilon, and the engine config's size."""
import ctypes as C
import types

import numpy as np
import pytest
import torch

from oracle import c51 as OC
from oracle import dqn as OD
from oracle import noisy as ON
from oracle import qr as OQ
from test_c51 import ATOMS
from test_dqn import DQN_KW, LEARN, N_ACT, O_DIM, ChooseEnv, evaluation_return, flat, random_minibatch

HIDDEN = 32


def make(kind="dqn", dueling=False, hidden=HIDDEN, seed=0, lr=1e-3, n_quantiles=32, replay_buffer=None, **kw):
    """A DQN / C51 / QRDQN learner on ChooseEnv with a NoisyMLP([obs, hidden, hidden, n K]) or a noisy
    DuelingMLP([obs, hidden, hidden], n, K) Q network."""
    from rl_replicas_b200.algorithms import C51, DQN, QRDQN
    from rl_replicas_b200.critics import CategoricalQFunction, DiscreteQFunction, QuantileQFunction
    from rl_replicas_b200.evaluator import Evaluator
    from rl_replicas_b200.networks import DuelingMLP, NoisyMLP
    from rl_replicas_b200.policies import RandomPolicy
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    from rl_replicas_b200.samplers import BatchSampler
    torch.manual_seed(seed)
    env = ChooseEnv()
    k = {"dqn": 1, "c51": ATOMS["n_atoms"], "qr": n_quantiles}[kind]
    net = (DuelingMLP([O_DIM, hidden, hidden], N_ACT, k, noisy=True) if dueling
           else NoisyMLP([O_DIM, hidden, hidden, N_ACT * k]))
    opt = torch.optim.Adam(net.parameters(), lr=lr)
    qf, cls = {"dqn": lambda: (DiscreteQFunction(net, opt), DQN),
               "c51": lambda: (CategoricalQFunction(net, opt, **ATOMS), C51),
               "qr": lambda: (QuantileQFunction(net, opt, n_quantiles=n_quantiles), QRDQN)}[kind]()
    return cls(qf, RandomPolicy(env.action_space), env, BatchSampler(env, seed=0),
               replay_buffer if replay_buffer is not None else ReplayBuffer(buffer_size=100000), Evaluator(seed=0), **kw)


def test_noisy_linear_follows_the_formulas_in_float32():
    from rl_replicas_b200.networks import NoisyLinear
    torch.manual_seed(0)
    layer = NoisyLinear(7, 5)
    layer.reset_noise()
    f = lambda x: np.copysign(np.sqrt(np.abs(x)), x).astype(np.float32)
    fi, fo = f(layer.eps_in.numpy()), f(layer.eps_out.numpy())
    assert np.array_equal(f(np.float32([-4.0, 0.0, 2.25])), np.float32([-2.0, 0.0, 1.5]))
    e = (fo[:, None] * fi[None, :]).astype(np.float32)  # one rounding each
    W = (layer.weight_mu.detach().numpy() + (layer.weight_sigma.detach().numpy() * e).astype(np.float32))
    b = layer.bias_mu.detach().numpy() + (layer.bias_sigma.detach().numpy() * fo).astype(np.float32)
    Wt, bt = layer.composed()
    assert np.array_equal(Wt.detach().numpy(), W.astype(np.float32)) and np.array_equal(bt.detach().numpy(), b)
    x = torch.randn(3, 7)
    torch.testing.assert_close(layer(x), x @ torch.from_numpy(W).T + torch.from_numpy(b), rtol=0, atol=0)
    # the gradient of the composition: d mu = dW, d sigma = dW e
    layer(x).sum().backward()
    torch.testing.assert_close(layer.weight_sigma.grad, layer.weight_mu.grad * torch.from_numpy(e), rtol=0, atol=0)
    torch.testing.assert_close(layer.bias_sigma.grad, layer.bias_mu.grad * torch.from_numpy(fo), rtol=0, atol=0)
    layer.eval()  # the mean weights
    torch.testing.assert_close(layer(x), torch.nn.functional.linear(x, layer.weight_mu, layer.bias_mu), rtol=0, atol=0)


def test_initialization_parameter_order_and_checkpoint_keys():
    from rl_replicas_b200.networks import DuelingMLP, NoisyLinear, NoisyMLP
    torch.manual_seed(1)
    layer = NoisyLinear(64, 300, sigma_0=0.4)
    bound = 1 / 8
    assert [n for n, _ in layer.named_parameters()] == ["weight_mu", "weight_sigma", "bias_mu", "bias_sigma"]
    assert layer.weight_mu.abs().max() <= bound and layer.bias_mu.abs().max() <= bound
    assert layer.weight_mu.std() > 0.5 * bound / np.sqrt(3)
    assert torch.all(layer.weight_sigma == np.float32(0.4 * bound)) and torch.all(layer.bias_sigma == np.float32(0.4 * bound))
    assert list(layer.state_dict()) == ["weight_mu", "weight_sigma", "bias_mu", "bias_sigma"]  # eps_* not persistent
    assert not isinstance(layer, torch.nn.Linear)
    net = NoisyMLP([4, 8, 3])
    assert list(net.state_dict())[:4] == ["network.0.weight_mu", "network.0.weight_sigma", "network.0.bias_mu",
                                         "network.0.bias_sigma"]
    assert sum(p.numel() for p in net.parameters()) == 2 * (8 * 5 + 3 * 9)
    d = DuelingMLP([4, 8, 6], 3, 2, noisy=True)
    assert isinstance(d.trunk[0], torch.nn.Linear)
    assert all(isinstance(m, NoisyLinear) for m in (d.value[0], d.value[2], d.advantage[0], d.advantage[2]))
    assert list(d.state_dict())[2:4] == ["value.0.weight_mu", "value.0.weight_sigma"]
    torch.manual_seed(2)
    plain = DuelingMLP([4, 8, 6], 3, 2)
    torch.manual_seed(2)
    again = DuelingMLP([4, 8, 6], 3, 2, noisy=False)  # the default is unchanged
    assert all(torch.equal(a, b) for a, b in zip(plain.parameters(), again.parameters()))


def test_reset_noise_is_reproducible_under_manual_seed():
    from rl_replicas_b200.networks import NoisyMLP, reset_noise
    net = NoisyMLP([3, 5, 2])
    draws = []
    for _ in range(2):
        torch.manual_seed(7)
        reset_noise(net)
        draws.append([t.clone() for t in net.buffers()])
    assert all(torch.equal(a, b) for a, b in zip(*draws))
    reset_noise(net)
    assert not torch.equal(draws[0][0], next(net.buffers()))


def test_noisy_greedy_policy_resamples_and_leaves_numpy_alone():
    from rl_replicas_b200.critics import DiscreteQFunction
    from rl_replicas_b200.networks import NoisyMLP
    from rl_replicas_b200.policies import NoisyGreedyPolicy
    torch.manual_seed(0)
    net = NoisyMLP([O_DIM, 16, N_ACT], sigma_0=4.0)
    q = DiscreteQFunction(net, torch.optim.Adam(net.parameters()))
    policy = NoisyGreedyPolicy(q)
    obs = np.random.default_rng(0).uniform(-1, 1, (64, O_DIM)).astype(np.float32)
    np.random.seed(3)
    before = np.random.get_state()[1].copy()
    seen = []
    for _ in range(4):
        a = policy.get_action_numpy(obs)
        assert a.shape == (64,)
        seen.append(net.network[0].eps_in.clone())
        # the batch shares the sample just drawn: greedy under the module's current noise
        assert np.array_equal(a, torch.argmax(q(torch.from_numpy(obs)), -1).numpy())
    assert all(not torch.equal(seen[0], s) for s in seen[1:])
    assert np.array_equal(np.random.get_state()[1], before)
    mean = policy.deterministic()
    assert np.array_equal(mean.get_action_numpy(obs), torch.argmax(
        torch.nn.functional.linear(torch.relu(torch.nn.functional.linear(
            torch.from_numpy(obs), net.network[0].weight_mu, net.network[0].bias_mu)),
            net.network[2].weight_mu, net.network[2].bias_mu), -1).numpy())
    assert q.training  # the mode is restored


@pytest.mark.parametrize("kind", ["dqn", "c51", "qr"])
@pytest.mark.parametrize("dueling", [False, True])
def test_constructors_accept_noisy_networks(kind, dueling):
    from rl_replicas_b200.algorithms.dqn import describe_q_network, noisy_mask
    from rl_replicas_b200.policies import NoisyGreedyPolicy
    algo = make(kind, dueling)
    assert algo.noisy and isinstance(algo.noised_policy, NoisyGreedyPolicy)
    lins = describe_q_network(algo.q_function.network)[3]
    assert noisy_mask(lins) == (0b11110 if dueling else 0b111)
    algo.current_total_steps = 10 ** 6
    assert algo.noised_policy is algo.noisy_policy  # epsilon plays no part
    # prioritized replay (DQN / QR-DQN) and n-step returns are accepted as for plain networks
    from rl_replicas_b200.replay_buffer import PrioritizedReplayBuffer
    if kind != "c51":
        make(kind, dueling, replay_buffer=PrioritizedReplayBuffer(buffer_size=1000), n_step=3)
    else:
        make(kind, dueling, n_step=3)


def test_other_algorithms_refuse_noisy_networks():
    from rl_replicas_b200.algorithms import DDPG, PPO, SAC, TD3, TRPO, VPG
    from rl_replicas_b200.networks import MLP, NoisyMLP
    from rl_replicas_b200.policies import CategoricalPolicy, DeterministicPolicy, SquashedGaussianPolicy
    from rl_replicas_b200.q_function import QFunction
    from rl_replicas_b200.value_function import ValueFunction
    env = types.SimpleNamespace(action_space=types.SimpleNamespace(shape=(2,), high=np.ones(2, np.float32)),
                                spec=types.SimpleNamespace(id="synthetic"))
    adam = lambda n: torch.optim.Adam(n.parameters())
    noisy_q, plain_q = NoisyMLP([5, 16, 1]), MLP([5, 16, 1])
    pol = MLP([3, 16, 2])
    match = "noisy layers"
    with pytest.raises(NotImplementedError, match=match):
        TD3(DeterministicPolicy(pol, adam(pol)), None, QFunction(noisy_q, adam(noisy_q)),
            QFunction(plain_q, adam(plain_q)), env, None, None, None)
    npol = NoisyMLP([3, 16, 2])
    with pytest.raises(NotImplementedError, match=match):
        DDPG(DeterministicPolicy(npol, adam(npol)), None, QFunction(plain_q, adam(plain_q)), env, None, None, None)
    spol = MLP([3, 16, 4])
    with pytest.raises(NotImplementedError, match=match):
        SAC(SquashedGaussianPolicy(spol, adam(spol)), None, QFunction(noisy_q, adam(noisy_q)),
            QFunction(plain_q, adam(plain_q)), env, None, None, None)
    cnet, vnet = MLP([3, 16, 2]), NoisyMLP([3, 16, 1])
    for cls in (PPO, VPG, TRPO):
        with pytest.raises(NotImplementedError, match=match):
            cls(CategoricalPolicy(cnet, adam(cnet)), ValueFunction(vnet, adam(vnet)), env, None)
    from rl_replicas_b200.algorithms._onpolicy import describe_mlp
    with pytest.raises(NotImplementedError, match="NoisyLinear"):
        describe_mlp(vnet)


def test_group_signature_refuses_mixed_noisy_and_plain_members():
    from rl_replicas_b200.algorithms import LearnerGroup
    from test_dqn import make_dqn
    from test_dueling import make as make_dueling
    g = LearnerGroup()
    g.add(make("dqn", hidden=64, seed=0, **DQN_KW))
    g.add(make("dqn", hidden=64, seed=1, **DQN_KW))
    with pytest.raises(ValueError, match="noisy layers"):
        g.add(make_dqn(seed=2, **DQN_KW))  # a plain MLP of the same widths
    d = LearnerGroup()
    d.add(make("dqn", dueling=True, hidden=64, seed=0, **DQN_KW))
    with pytest.raises(ValueError, match="noisy layers .*0 != 30"):
        d.add(make_dueling("dqn", seed=1, **DQN_KW))


def _step_case(kind, dueling, double_q, seed=3):
    algo = make(kind, dueling, seed=seed)
    q, qt = algo.q_function, algo.target_q_function
    with torch.no_grad():
        for p in qt.network.parameters():
            p.add_(0.05 * torch.randn_like(p))
    layers = ON.layers_of(q.network)
    E = sum(i + o for i, o, n in layers if n)
    draws = np.random.default_rng(seed).standard_normal((1, 2, E)).astype(np.float32)
    return algo, q, qt, layers, draws


@pytest.mark.parametrize("double_q", [False, True])
@pytest.mark.parametrize("dueling", [False, True])
@pytest.mark.parametrize("kind", ["dqn", "c51", "qr"])
def test_float32_oracle_agrees_with_the_float64_step(kind, dueling, double_q):
    algo, q, qt, layers, draws = _step_case(kind, dueling, double_q)
    opt = q.optimizer
    mb = random_minibatch(np.random.default_rng(5), 64)
    net = q.network
    k = {"dqn": 1, "c51": ATOMS["n_atoms"], "qr": q.n_quantiles if kind == "qr" else 1}[kind]
    sizes = ([O_DIM, HIDDEN, HIDDEN, N_ACT * k])
    kw = dict(gamma=0.99, double_q=double_q)
    if kind == "dqn":
        oracle, head = OD.DqnOracle(net, qt.network, opt, **kw), {}
    elif kind == "c51":
        oracle, head = OC.C51Oracle(net, qt.network, opt, **kw, **ATOMS), ATOMS
    else:
        oracle, head = OQ.QrDqnOracle(net, qt.network, opt, n_quantiles=q.n_quantiles, **kw), \
            dict(n_quantiles=q.n_quantiles)
    p0, t0 = flat(net), flat(qt.network)
    ref = ON.step_f64(kind, p0, t0, draws[0, 0], draws[0, 1], mb, layers, sizes, k if dueling else 0, "relu", **kw,
                      **head)
    logs = ON.train_f32(oracle, [mb], draws)
    np.testing.assert_allclose(logs["q1_values"][0], ref["q_values"], rtol=1e-5, atol=1e-5)
    assert abs(logs["q1_losses"][0] - ref["loss"]) <= 1e-5 * max(1.0, abs(ref["loss"]))
    step = flat(oracle.q) - p0  # Adam's first step: the sign of each clear gradient entry
    clear = np.abs(ref["grad"]) > 1e-3 * np.abs(ref["grad"]).max()
    assert clear.sum() > 100
    np.testing.assert_array_equal(np.sign(step[clear]), -np.sign(ref["grad"][clear]))
    assert np.all(ref["scale"] >= np.abs(ref["grad"]) * (1 - 1e-12))
    # the online sample drives Q(s): the composed float64 weights reproduce the logged values
    assert not np.array_equal(ON.compose_f64(p0, layers, draws[0, 0]), ON.compose_f64(p0, layers, draws[0, 1]))


def test_oracle_driven_learn_loop_explores_without_epsilon(tmp_path):
    """learn() with the float32 oracle and host-drawn weight noise in place of the engine: acting after warm-up is the
    NoisyGreedyPolicy, epsilon is never consulted nor logged, and the loop solves the task."""
    np.random.seed(0)
    algo = make("dqn", hidden=64, **DQN_KW)
    oracle = OD.DqnOracle(algo.q_function.network, algo.target_q_function.network, algo.q_function.optimizer,
                          gamma=algo.gamma, target_update_interval=algo.target_update_interval, double_q=algo.double_q)
    E = sum(i + o for i, o, n in ON.layers_of(algo.q_function.network) if n)
    rng = np.random.default_rng(0)

    def train(replay_buffer, num_train_steps, minibatch_size):
        S, B = num_train_steps, minibatch_size
        idx = np.stack([replay_buffer.sample_indices(B) for _ in range(S)])
        ON.train_f32(oracle, [replay_buffer.gather(idx[s]) for s in range(S)],
                     rng.standard_normal((S, 2, E)).astype(np.float32))
        algo.q_function.network.load_state_dict(oracle.q.state_dict())
        algo.target_q_function.network.load_state_dict(oracle.q_targ.state_dict())
    algo.train = train

    def no_epsilon():
        raise AssertionError("epsilon consulted")
    algo.epsilon = no_epsilon
    before = evaluation_return(algo)
    algo.learn(output_dir=str(tmp_path), **LEARN)
    after = evaluation_return(algo)
    print(f"oracle-driven noisy learn: evaluation return {before:.3f} -> {after:.3f}")
    assert before < 0.6 and after > NOISY_RETURN_BAR, (before, after)
    tags = []
    algo.metrics_manager = types.SimpleNamespace(record_scalar=lambda tag, *a, **k: tags.append(tag))
    algo._record_train(dict(q1_values=np.zeros((2, 4), np.float32), q1_losses=np.zeros(2, np.float32)))
    assert "q-function/average_loss" in tags and "exploration/epsilon" not in tags


NOISY_RETURN_BAR = 0.85  # a uniform random policy scores 1/3 on ChooseEnv


def test_config_struct_size():
    from rl_replicas_b200 import _lib
    assert C.sizeof(_lib.OffPolicyConfig) == 88
    assert _lib.OffPolicyConfig.noisy_layers.offset == 84
