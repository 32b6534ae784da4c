"""CPU: IQN's host side -- ImplicitQuantileMLP's shapes, parameter order, flat layout and checkpoint keys, the critic's
midpoint mean, the host copy of the device's fraction draws, the float32 oracle (oracle/iqn.py) and the float64 step
against the paper's double loop with N != N', the IQN constructor's refusals and the other trainers' refusals of the
network, the LearnerGroup signature for IQN members, the checkpoint round trip, the IQN counts' struct layout and the
oracle-driven learn() loop that sets the bar for the GPU end-to-end test (tests/test_gpu_iqn.py)."""
import ctypes as C
import types

import numpy as np
import pytest
import torch

from oracle import iqn as OI
from test_dqn import DQN_KW, LEARN, N_ACT, O_DIM, RETURN_BAR, ChooseEnv, evaluation_return, flat, random_minibatch

IQN_KW = dict(DQN_KW)


def make_iqn(hidden=64, seed=0, lr=1e-3, replay_buffer=None, n_cos=32, n_quantiles=32, n_target_quantiles=32,
             n_policy_quantiles=16, **kw):
    from rl_replicas_b200.algorithms import IQN
    from rl_replicas_b200.critics import ImplicitQuantileQFunction
    from rl_replicas_b200.evaluator import Evaluator
    from rl_replicas_b200.networks import ImplicitQuantileMLP
    from rl_replicas_b200.policies import RandomPolicy
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    from rl_replicas_b200.samplers import BatchSampler
    torch.manual_seed(seed)
    env = ChooseEnv()
    net = ImplicitQuantileMLP([O_DIM, hidden, hidden], N_ACT, n_cos=n_cos)
    qf = ImplicitQuantileQFunction(net, torch.optim.Adam(net.parameters(), lr=lr), n_quantiles=n_quantiles,
                                   n_target_quantiles=n_target_quantiles, n_policy_quantiles=n_policy_quantiles)
    return IQN(qf, RandomPolicy(env.action_space), env, BatchSampler(env, seed=0),
               replay_buffer if replay_buffer is not None else ReplayBuffer(buffer_size=100000), Evaluator(seed=0),
               **kw)


def test_network_shapes_parameter_order_and_checkpoint_keys():
    from rl_replicas_b200.networks import ImplicitQuantileMLP
    from rl_replicas_b200.networks.iqn import cosine_features
    torch.manual_seed(0)
    net = ImplicitQuantileMLP([5, 24, 16], 3, n_cos=7, activation_function=torch.nn.Tanh)
    names = [k for k, _ in net.named_parameters()]
    assert names == ["embedding.0.weight", "embedding.0.bias", "tau_embedding.0.weight", "tau_embedding.0.bias",
                     "head.0.weight", "head.0.bias", "head.2.weight", "head.2.bias"]
    assert list(net.state_dict()) == names
    shapes = [tuple(p.shape) for p in net.parameters()]
    assert shapes == [(24, 5), (24,), (24, 7), (24,), (16, 24), (16,), (3, 16), (3,)]
    obs, taus = torch.randn(4, 5), torch.rand(4, 6)
    z = net(obs, taus)
    assert z.shape == (4, 6, 3)
    x = cosine_features(taus, 7)
    assert x.shape == (4, 6, 7) and (x[..., 0] == 1).all()
    want = torch.cos(np.pi * torch.arange(7, dtype=torch.float64) * taus.double()[..., None])
    torch.testing.assert_close(x.double(), want, rtol=0, atol=1e-6)
    by_hand = net.head(torch.tanh(obs @ net.embedding[0].weight.T + net.embedding[0].bias)[:, None]
                       * torch.tanh(x @ net.tau_embedding[0].weight.T + net.tau_embedding[0].bias))
    assert torch.equal(z, by_hand)
    # the flat vector (parameters_to_vector) is W_psi, b_psi, W_phi, b_phi, W_h, b_h, W_out, b_out
    v = torch.nn.utils.parameters_to_vector(net.parameters())
    o = 0
    for p in (net.embedding[0].weight, net.embedding[0].bias, net.tau_embedding[0].weight, net.tau_embedding[0].bias,
              net.head[0].weight, net.head[0].bias, net.head[2].weight, net.head[2].bias):
        assert torch.equal(v[o:o + p.numel()], p.reshape(-1))
        o += p.numel()
    assert o == v.numel() == 24 * 6 + 24 * 8 + 16 * 25 + 3 * 17
    from rl_replicas_b200.algorithms.dqn import describe_q_network
    sizes, hidden, out, lins, k = describe_q_network(net)
    assert (sizes, hidden, out, k) == ([5, 24, 16, 3], "tanh", "identity", 0)
    assert lins == [net.embedding[0], net.tau_embedding[0], net.head[0], net.head[2]]
    for bad in ([5, 24], [5, 0, 16]):
        with pytest.raises(ValueError, match="sizes"):
            ImplicitQuantileMLP(bad, 3)


def test_critic_is_the_mean_over_the_midpoints():
    from rl_replicas_b200.critics import ImplicitQuantileQFunction
    from rl_replicas_b200.networks import ImplicitQuantileMLP
    from rl_replicas_b200.policies import EpsilonGreedyPolicy, GreedyPolicy
    from rl_replicas_b200.q_function import ImplicitQuantileQFunction as Exported
    assert Exported is ImplicitQuantileQFunction
    torch.manual_seed(1)
    net = ImplicitQuantileMLP([3, 16, 16], 4, n_cos=8)
    qf = ImplicitQuantileQFunction(net, None, n_policy_quantiles=5)
    d = ImplicitQuantileQFunction(net, None)
    assert (d.n_quantiles, d.n_target_quantiles, d.n_policy_quantiles) == (64, 64, 32)
    mids = np.asarray([np.float32(2 * k + 1) / np.float32(10) for k in range(5)], np.float32)
    np.testing.assert_array_equal(qf.policy_taus.numpy(), mids)
    obs = torch.randn(9, 3)
    z = qf.quantiles(obs, torch.rand(9, 6))
    assert z.shape == (9, 4, 6)
    q = qf(obs)
    assert q.shape == (9, 4)
    want = net(obs, torch.as_tensor(mids).expand(9, 5)).sum(1) / 5
    assert torch.equal(q, want)
    assert qf(obs[0]).shape == (4,)
    assert torch.equal(qf(obs), qf(obs))  # deterministic
    assert (GreedyPolicy(qf).get_action_numpy(obs.numpy()) == q.argmax(-1).numpy()).all()
    EpsilonGreedyPolicy(qf, types.SimpleNamespace(n=4, sample=lambda: 0), 0.0).get_action_numpy(obs.numpy()[0])
    for name in ("n_quantiles", "n_target_quantiles", "n_policy_quantiles"):
        for bad in (0, 257, 2.5, True):
            with pytest.raises(ValueError, match=f"{name} must be an integer from 1 to 256"):
                ImplicitQuantileQFunction(net, None, **{name: bad})


def test_host_draws_are_odd_multiples_of_two_to_the_minus_24():
    t = OI.iqn_taus(7, 3, 2, 33, 13)
    assert t.shape == (33, 13) and t.dtype == np.float32
    m = t.astype(np.float64) * 2.0 ** 24
    assert (m == np.round(m)).all() and (np.round(m) % 2 == 1).all()
    assert (t > 0).all() and (t < 1).all()
    # the draw of a row position does not depend on the minibatch size; other keys give other draws
    np.testing.assert_array_equal(OI.iqn_taus(7, 3, 2, 5, 13), t[:5])
    for other in (OI.iqn_taus(8, 3, 2, 33, 13), OI.iqn_taus(7, 4, 2, 33, 13), OI.iqn_taus(7, 3, 1, 33, 13)):
        assert (other != t).mean() > 0.99


@pytest.mark.parametrize("N,Nt", [(1, 1), (3, 8), (8, 3), (5, 5)])
def test_tensor_forms_match_the_double_loop(N, Nt):
    """Both tensor forms of the row loss (float64 and float32) against the explicit loop, N != N' included, on rows
    with |u| below, at and above 1 and with u = 0."""
    rng = np.random.default_rng(N * 10 + Nt)
    B = 9
    theta, target = rng.standard_normal((B, N)) * 1.5, rng.standard_normal((B, Nt)) * 1.5
    tau = rng.random((B, N)).astype(np.float32)
    target[0] = theta[0, 0]  # u = 0 on every pair of sample 0
    target[1, 0] = theta[1, 0] + 1.0  # |u| = 1 exactly
    want = np.asarray([OI.rho_loop_f64(theta[b], target[b], tau[b]) for b in range(B)])
    got64 = OI.sampled_quantile_huber(*(torch.as_tensor(x, dtype=torch.float64) for x in (theta, target, tau))).numpy()
    np.testing.assert_allclose(got64, want, rtol=1e-13, atol=0)
    got32 = OI.sampled_quantile_huber(*(torch.as_tensor(x, dtype=torch.float32) for x in (theta, target, tau))).numpy()
    np.testing.assert_allclose(got32, want, rtol=2e-6, atol=1e-7)


def _nets(seed, sizes=(4, 32, 24), n=5, n_cos=9, act=torch.nn.Tanh):
    from rl_replicas_b200.networks import ImplicitQuantileMLP
    torch.manual_seed(seed)
    return (ImplicitQuantileMLP(list(sizes), n, n_cos=n_cos, activation_function=act),
            ImplicitQuantileMLP(list(sizes), n, n_cos=n_cos, activation_function=act))


@pytest.mark.parametrize("double_q", [False, True])
@pytest.mark.parametrize("per_row", [False, True])
def test_float32_oracle_agrees_with_the_float64_reference(double_q, per_row):
    """One step with N = 7, N' = 11, K = 4: loss, row losses, Q(s, a) and the gradient (read from Adam's first moment)
    of the float32 autograd oracle within 1e-5 of the float64 reference; the reference's row losses equal the double
    loop; per_row: n-step discounts."""
    N, Nt, K, n, n_cos = 7, 11, 4, 5, 9
    net, targ = _nets(3)
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    rng = np.random.default_rng(0)
    mb = random_minibatch(rng, 64, n=n, O=4)
    taus = OI.iqn_taus(5, 1, 0, 64, N + Nt + K)
    gamma = torch.tensor(0.99, dtype=torch.float64)
    if per_row:
        mb["discounts"] = (0.99 ** rng.integers(1, 4, 64)).astype(np.float32)
        gamma = torch.as_tensor(mb["discounts"], dtype=torch.float64)
    ref = OI.iqn_step_f64(flat(net), flat(targ), mb, taus, [4, 32, 24, n], n_cos, N, Nt, K, "tanh", gamma, double_q)
    o = OI.IqnOracle(net, targ, opt, N, Nt, K, gamma=0.99, target_update_interval=100, double_q=double_q)
    logs = o.train([mb], [taus])
    grad = torch.cat([o.opt.state[p]["exp_avg"].reshape(-1) for p in o.q.parameters()]).numpy() / 0.1
    rel = lambda x, r: float(np.max(np.abs(np.asarray(x, np.float64) - r)) / np.max(np.abs(r)))
    assert rel(logs["q1_values"][0], ref["q_values"]) < 1e-5
    assert abs(logs["q1_losses"][0] - ref["loss"]) <= 1e-5 * abs(ref["loss"])
    assert rel(logs["row_losses"][0], ref["row_loss"]) < 1e-5
    assert rel(grad, ref["grad"]) < 1e-5
    assert (ref["scale"] >= np.abs(ref["grad"]) * (1 - 1e-12)).all()
    with torch.no_grad():
        z = net(torch.as_tensor(mb["observations"]), torch.as_tensor(taus[:, :N])).double()
    th = z[torch.arange(64), :, torch.as_tensor(mb["actions"]).long()].numpy()
    loop = np.asarray([OI.rho_loop_f64(th[b], ref["target"][b], taus[b, :N]) for b in range(64)])
    np.testing.assert_allclose(ref["row_loss"], loop, rtol=1e-5)


def test_prioritized_oracle_with_unit_weights_is_the_unweighted_one():
    net, targ = _nets(4, act=torch.nn.ReLU)
    mb = random_minibatch(np.random.default_rng(1), 32, n=5, O=4)
    taus = [OI.iqn_taus(1, 1, 0, 32, 6 + 5 + 3)]
    a = OI.IqnOracle(net, targ, torch.optim.Adam(net.parameters()), 6, 5, 3, alpha=0.5, eps=1e-3)
    b = OI.IqnOracle(net, targ, torch.optim.Adam(net.parameters()), 6, 5, 3)
    la = a.train([mb], taus, [np.full(32, 2.0)], [1.0])
    lb = b.train([mb], taus)
    assert (la["weights"][0] == 1.0).all()
    assert la["q1_losses"] == lb["q1_losses"]
    for x, y in zip(a.q.parameters(), b.q.parameters()):
        assert torch.equal(x, y)
    np.testing.assert_allclose(la["priorities"][0], (lb["row_losses"][0].astype(np.float64) + 1e-3) ** 0.5, rtol=1e-15)


def test_constructor_refusals():
    from rl_replicas_b200.algorithms import IQN
    from rl_replicas_b200.critics import DiscreteQFunction, ImplicitQuantileQFunction, QuantileQFunction
    from rl_replicas_b200.networks import MLP, DuelingMLP, ImplicitQuantileMLP, NoisyLinear
    from rl_replicas_b200.replay_buffer import PrioritizedReplayBuffer
    env = ChooseEnv()
    net = ImplicitQuantileMLP([O_DIM, 16, 16], N_ACT, n_cos=8)
    opt = torch.optim.Adam(net.parameters())
    qf = ImplicitQuantileQFunction(net, opt, 8, 8, 4)
    mlp = MLP([O_DIM, 16, N_ACT * 8], torch.nn.ReLU)
    for other in (DiscreteQFunction(mlp, opt), QuantileQFunction(mlp, opt, n_quantiles=8)):
        with pytest.raises(ValueError, match="ImplicitQuantileQFunction"):
            IQN(other, None, env, None, None, None)
    duel = DuelingMLP([O_DIM, 16, 16], N_ACT)
    with pytest.raises(NotImplementedError, match="dueling IQN networks are not implemented"):
        IQN(ImplicitQuantileQFunction(duel, opt), None, env, None, None, None)
    noisy = ImplicitQuantileMLP([O_DIM, 16, 16], N_ACT, n_cos=8)
    noisy.head[2] = NoisyLinear(16, N_ACT)
    with pytest.raises(NotImplementedError, match="noisy IQN networks are not implemented"):
        IQN(ImplicitQuantileQFunction(noisy, opt), None, env, None, None, None)
    with pytest.raises(ValueError, match="ImplicitQuantileMLP"):
        IQN(ImplicitQuantileQFunction(mlp, opt), None, env, None, None, None)
    wrong = ImplicitQuantileMLP([O_DIM, 16, 16], N_ACT + 1)
    with pytest.raises(ValueError, match=r"must map 2 -> 3 \(one value per action\), got 2 -> 4"):
        IQN(ImplicitQuantileQFunction(wrong, torch.optim.Adam(wrong.parameters())), None, env, None, None, None)
    cont = types.SimpleNamespace(action_space=types.SimpleNamespace(shape=(2,), high=np.ones(2)),
                                 observation_space=env.observation_space, spec=env.spec)
    with pytest.raises(ValueError, match="discrete"):
        IQN(qf, None, cont, None, None, None)
    with pytest.raises(ValueError, match="n_step"):
        IQN(qf, None, env, None, None, None, n_step=33)
    with pytest.raises(NotImplementedError, match="torch.optim.Adam"):
        IQN(ImplicitQuantileQFunction(net, torch.optim.SGD(net.parameters(), lr=0.1)), None, env, None, None, None)
    algo = IQN(qf, None, env, None, PrioritizedReplayBuffer(1000), None, target_update_interval=5, double_q=True,
               n_step=3)
    assert (algo.target_update_interval, algo.double_q, algo.gamma, algo.epsilon_end, algo.n_step) == \
        (5, True, 0.99, 0.05, 3)
    assert algo.iqn_config == (8, 8, 8, 4) and algo._needs_draw_keys() and not algo.noisy
    sizes, acts, kw = algo._engine_config()
    assert (sizes, acts, kw) == ([O_DIM, 16, 16, N_ACT], ("relu", "identity"),
                                 dict(dueling_k=0, noisy_layers=0, iqn=(8, 8, 8, 4)))


def test_other_trainers_refuse_the_network():
    from rl_replicas_b200.algorithms import DDPG, PPO, SAC, TD3, TRPO, VPG
    from rl_replicas_b200.networks import MLP, ImplicitQuantileMLP
    from rl_replicas_b200.policies import CategoricalPolicy, DeterministicPolicy, SquashedGaussianPolicy
    from rl_replicas_b200.q_function import QFunction
    from rl_replicas_b200.value_function import ValueFunction
    env = types.SimpleNamespace(action_space=types.SimpleNamespace(shape=(2,), high=np.ones(2, np.float32)),
                                spec=types.SimpleNamespace(id="synthetic"))
    adam = lambda n: torch.optim.Adam(n.parameters())
    iqn_net = ImplicitQuantileMLP([5, 16, 16], 1, n_cos=4)
    plain_q, pol = MLP([5, 16, 1]), MLP([3, 16, 2])
    match = "MLP"
    td3 = TD3(DeterministicPolicy(pol, adam(pol)), None, QFunction(iqn_net, adam(iqn_net)),
              QFunction(plain_q, adam(plain_q)), env, None, None, None)
    ddpg = DDPG(DeterministicPolicy(pol, adam(pol)), None, QFunction(iqn_net, adam(iqn_net)), env, None, None, None)
    for algo in (td3, ddpg):  # the engine is described (and refused) before it is built
        with pytest.raises(NotImplementedError, match=match):
            algo._ensure_engine(1, 8)
    spol = MLP([3, 16, 4])
    with pytest.raises(NotImplementedError, match=match):
        SAC(SquashedGaussianPolicy(spol, adam(spol)), None, QFunction(iqn_net, adam(iqn_net)),
            QFunction(plain_q, adam(plain_q)), env, None, None, None)
    cnet = MLP([3, 16, 2])
    for cls in (PPO, VPG, TRPO):
        algo = cls(CategoricalPolicy(cnet, adam(cnet)), ValueFunction(iqn_net, adam(iqn_net)), env, None)
        with pytest.raises(NotImplementedError, match=match):
            algo._describe()


def test_save_and_load_round_trip(tmp_path):
    algo = make_iqn(seed=1)
    algo.current_total_steps = 77
    algo.q_function(torch.randn(8, O_DIM)).sum().backward()
    algo.q_function.optimizer.step()
    with torch.no_grad():
        for p in algo.target_q_function.network.parameters():
            p.add_(0.5)
    path = str(tmp_path / "model.pt")
    algo.save_model(3, path)
    ckpt = torch.load(path, weights_only=True)
    assert set(ckpt) == {"epoch", "total_steps", "q_function_state_dict", "q_function_optimizer_state_dict",
                         "target_q_function_state_dict"}  # DQN's keys
    assert list(ckpt["q_function_state_dict"]) == [f"{m}.{k}" for m in ("embedding.0", "tau_embedding.0", "head.0",
                                                                         "head.2") for k in ("weight", "bias")]
    other = make_iqn(seed=2)
    assert other.load_model(path) == 3 and other.current_total_steps == 77
    for a, b in ((algo.q_function.network, other.q_function.network),
                 (algo.target_q_function.network, other.target_q_function.network)):
        for (k, x), (_, y) in zip(a.state_dict().items(), b.state_dict().items()):
            assert torch.equal(x, y), k
    lins = algo._learner_nets()[2][0]
    assert other._adam_step_count(other.q_function.optimizer, other._learner_nets()[2][0]) == 1 and len(lins) == 4
    obs = torch.randn(5, O_DIM)
    assert torch.equal(algo.q_function(obs), other.q_function(obs))


def test_group_signature_refuses_differing_sizes_and_mixes():
    from rl_replicas_b200.algorithms import LearnerGroup
    from rl_replicas_b200.replay_buffer import PrioritizedReplayBuffer
    from test_dqn import make_dqn
    from test_qr import make_qr
    g = LearnerGroup()
    g.add(make_iqn(seed=0))
    g.add(make_iqn(seed=1))
    for kw in (dict(n_cos=16), dict(n_quantiles=16), dict(n_target_quantiles=8), dict(n_policy_quantiles=8)):
        with pytest.raises(ValueError, match="IQN \\(n_cos|n_quantiles differs"):
            g.add(make_iqn(seed=2, **kw))
    with pytest.raises(ValueError, match="network"):
        g.add(make_iqn(seed=2, hidden=32))
    for other in (make_dqn(seed=2), make_qr(seed=2)):
        with pytest.raises(ValueError, match="class"):
            g.add(other)
    with pytest.raises(ValueError, match="target_update_interval"):
        g.add(make_iqn(seed=2, target_update_interval=7))
    with pytest.raises(ValueError, match="prioritized replay"):
        g.add(make_iqn(seed=2, replay_buffer=PrioritizedReplayBuffer(1000)))
    assert len(g) == 2


def test_iqn_config_struct_layout():
    """IQN's counts travel in a struct of their own (b200rl_offpolicy_create_iqn); the off-policy config keeps its
    88 bytes."""
    from rl_replicas_b200 import _lib
    ic = _lib.IqnConfig
    assert C.sizeof(ic) == 16
    assert [getattr(ic, f).offset for f in ("n_cos", "n", "n_target", "k")] == [0, 4, 8, 12]
    assert C.sizeof(_lib.OffPolicyConfig) == 88
    assert _lib.SIGNATURES["b200rl_offpolicy_create_iqn"][1][1] is C.POINTER(ic)


class OracleIQN:
    """IQN.train with the float32 oracle in place of the engine: the same host random stream for the indices, the
    device's fractions from their keys (device_rng_seed, the learner's call count), the oracle's networks written back
    into the learner's."""

    @staticmethod
    def patch(algo):
        q = algo.q_function
        oracle = OI.IqnOracle(q.network, algo.target_q_function.network, q.optimizer, q.n_quantiles,
                              q.n_target_quantiles, q.n_policy_quantiles, gamma=algo.gamma,
                              target_update_interval=algo.target_update_interval, double_q=algo.double_q)
        Mt = q.n_quantiles + q.n_target_quantiles + q.n_policy_quantiles

        def train(replay_buffer, num_train_steps, minibatch_size):
            S, B = num_train_steps, minibatch_size
            algo._noise_calls = getattr(algo, "_noise_calls", 0) + 1
            idx = np.stack([replay_buffer.sample_indices(B) for _ in range(S)])
            taus = [OI.iqn_taus(algo.device_rng_seed, algo._noise_calls, s, B, Mt) for s in range(S)]
            oracle.train([replay_buffer.gather(idx[s]) for s in range(S)], taus)
            algo.q_function.network.load_state_dict(oracle.q.state_dict())
            algo.target_q_function.network.load_state_dict(oracle.q_targ.state_dict())
        algo.train = train
        return oracle


def test_oracle_driven_learn_loop_solves_the_choice_task(tmp_path):
    """The bar the GPU learn() loop must clear (tests/test_gpu_iqn.py) is one the oracle reaches with the same seeds."""
    np.random.seed(0)
    algo = make_iqn(**IQN_KW)
    OracleIQN.patch(algo)
    before = evaluation_return(algo)
    algo.learn(output_dir=str(tmp_path), **LEARN)
    after = evaluation_return(algo)
    print(f"oracle-driven learn: evaluation return {before:.3f} -> {after:.3f}")
    assert before < 0.6 and after > RETURN_BAR, (before, after)
