"""CPU: QR-DQN's host side -- the float32 oracle (oracle/qr.py) and the float64 step against the paper's double loop and
against each other (prioritized and per-row discounted forms included), QuantileQFunction, the QRDQN constructor's
refusals, its checkpoint round trip, the LearnerGroup signature for QR-DQN members, and the oracle-driven learn() loop
that sets the bar for the GPU end-to-end test (tests/test_gpu_qr.py)."""
import types

import numpy as np
import pytest
import torch

from oracle import qr as OQ
from test_dqn import DQN_KW, LEARN, N_ACT, O_DIM, RETURN_BAR, ChooseEnv, evaluation_return, flat, random_minibatch

QR_KW = dict(DQN_KW)
N_QUANT = 32  # the choice task's returns are 0 and 1: a few quantiles describe them


def make_qr(hidden=64, seed=0, lr=1e-3, n_quantiles=N_QUANT, replay_buffer=None, **kw):
    from rl_replicas_b200.algorithms import QRDQN
    from rl_replicas_b200.critics import QuantileQFunction
    from rl_replicas_b200.evaluator import Evaluator
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import RandomPolicy
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    from rl_replicas_b200.samplers import BatchSampler
    torch.manual_seed(seed)
    env = ChooseEnv()
    net = MLP([O_DIM, hidden, hidden, N_ACT * n_quantiles], torch.nn.ReLU)
    qf = QuantileQFunction(net, torch.optim.Adam(net.parameters(), lr=lr), n_quantiles=n_quantiles)
    return QRDQN(qf, RandomPolicy(env.action_space), env, BatchSampler(env, seed=0),
                 replay_buffer if replay_buffer is not None else ReplayBuffer(buffer_size=100000), Evaluator(seed=0),
                 **kw)


def test_taus_are_one_float32_division():
    for N in (1, 2, 7, 200, 256):
        t = OQ.taus(N)
        assert t.dtype == torch.float32 and t.shape == (N,)
        want = np.asarray([np.float32(2 * i + 1) / np.float32(2 * N) for i in range(N)], np.float32)
        np.testing.assert_array_equal(t.numpy(), want)
    assert OQ.taus(1).tolist() == [0.5]


@pytest.mark.parametrize("N", [1, 2, 5, 16])
def test_tensor_forms_match_the_double_loop(N):
    """Both tensor forms of the row loss (float64 and float32) against the explicit loop, on rows with |u| below, at and
    above 1 and with u = 0."""
    rng = np.random.default_rng(N)
    B = 9
    theta = rng.standard_normal((B, N)) * 1.5
    target = rng.standard_normal((B, N)) * 1.5
    target[0] = theta[0, 0]  # u = 0 on every pair of quantile 0
    target[1, 0] = theta[1, 0] + 1.0  # |u| = 1 exactly
    want = np.asarray([OQ.rho_loop_f64(theta[b], target[b]) for b in range(B)])
    got64 = OQ.quantile_huber(torch.as_tensor(theta), torch.as_tensor(target), OQ.taus(N, torch.float64)).numpy()
    np.testing.assert_allclose(got64, want, rtol=1e-13, atol=0)
    t32 = lambda x: torch.as_tensor(x, dtype=torch.float32)
    got32 = OQ.quantile_huber(t32(theta), t32(target), OQ.taus(N)).numpy()
    np.testing.assert_allclose(got32, want, rtol=2e-6, atol=1e-7)


def test_autograd_gradient_is_the_stated_output_gradient():
    """d L / d theta_i = -(1/N) sum_j |tau_i - 1{u_ij < 0}| clamp(u_ij, -1, 1), written out with loops."""
    rng = np.random.default_rng(3)
    N = 6
    theta = torch.as_tensor(rng.standard_normal(N) * 2, dtype=torch.float64).requires_grad_()
    target = torch.as_tensor(rng.standard_normal(N) * 2, dtype=torch.float64)
    OQ.quantile_huber(theta[None], target[None], OQ.taus(N, torch.float64))[0].backward()
    want = np.zeros(N)
    for i in range(N):
        tau = (2 * i + 1) / (2 * N)
        for j in range(N):
            u = float(target[j] - theta.detach()[i])
            want[i] -= abs(tau - (u < 0)) * min(max(u, -1.0), 1.0) / N
    np.testing.assert_allclose(theta.grad.numpy(), want, rtol=1e-13, atol=1e-15)


@pytest.mark.parametrize("double_q", [False, True])
@pytest.mark.parametrize("per_row", [False, True])
def test_float32_oracle_agrees_with_the_float64_reference(double_q, per_row):
    """One step: loss, row losses, Q(s, a) and the gradient (read from Adam's first moment) of the float32 autograd
    oracle within 1e-5 of the float64 reference; the reference's row losses equal the double loop; per_row: n-step
    discounts."""
    from rl_replicas_b200.networks import MLP
    torch.manual_seed(3)
    n, N, sizes = 5, 13, [4, 32, 32, 5 * 13]
    net, targ = MLP(sizes, torch.nn.Tanh), MLP(sizes, torch.nn.Tanh)
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    rng = np.random.default_rng(0)
    mb = random_minibatch(rng, 64, n=n, O=4)
    gamma = torch.tensor(0.99, dtype=torch.float64)
    if per_row:
        mb["discounts"] = (0.99 ** rng.integers(1, 4, 64)).astype(np.float32)
        gamma = torch.as_tensor(mb["discounts"], dtype=torch.float64)
    ref = OQ.qr_step_f64(flat(net), flat(targ), mb, sizes, N, "tanh", gamma, double_q)
    o = OQ.QrDqnOracle(net, targ, opt, n_quantiles=N, gamma=0.99, target_update_interval=100, double_q=double_q)
    logs = o.train([mb])
    grad = torch.cat([o.opt.state[p]["exp_avg"].reshape(-1) for p in o.q.parameters()]).numpy() / 0.1
    rel = lambda x, r: float(np.max(np.abs(np.asarray(x, np.float64) - r)) / np.max(np.abs(r)))
    assert rel(logs["q1_values"][0], ref["q_values"]) < 1e-5
    assert abs(logs["q1_losses"][0] - ref["loss"]) <= 1e-5 * abs(ref["loss"])
    assert rel(logs["row_losses"][0], ref["row_loss"]) < 1e-5
    assert rel(grad, ref["grad"]) < 1e-5
    assert (ref["scale"] >= np.abs(ref["grad"]) * (1 - 1e-12)).all()
    q_theta = ref["target"]  # the loop form from the reference's own targets and a fresh forward pass
    with torch.no_grad():
        th = net(torch.as_tensor(mb["observations"])).double().unflatten(-1, (n, N))
    th = th[torch.arange(64), torch.as_tensor(mb["actions"]).long()].numpy()
    loop = np.asarray([OQ.rho_loop_f64(th[b], q_theta[b]) for b in range(64)])
    np.testing.assert_allclose(ref["row_loss"], loop, rtol=1e-5)


def test_prioritized_oracle_with_unit_weights_is_the_unweighted_one():
    """Equal priorities at beta = 1: every weight is 1, the step is the unweighted one and the new priorities are
    (L_b + eps)^alpha of the row losses."""
    from rl_replicas_b200.networks import MLP
    torch.manual_seed(4)
    sizes = [4, 16, 3 * 8]
    net, targ = MLP(sizes, torch.nn.ReLU), MLP(sizes, torch.nn.ReLU)
    mb = random_minibatch(np.random.default_rng(1), 32, n=3, O=4)
    a = OQ.QrDqnOracle(net, targ, torch.optim.Adam(net.parameters()), n_quantiles=8, alpha=0.5, eps=1e-3)
    b = OQ.QrDqnOracle(net, targ, torch.optim.Adam(net.parameters()), n_quantiles=8)
    la = a.train([mb], [np.full(32, 2.0)], [1.0])
    lb = b.train([mb])
    assert (la["weights"][0] == 1.0).all()
    assert la["q1_losses"] == lb["q1_losses"]
    for x, y in zip(a.q.parameters(), b.q.parameters()):
        assert torch.equal(x, y)
    np.testing.assert_allclose(la["priorities"][0], (lb["row_losses"][0].astype(np.float64) + 1e-3) ** 0.5, rtol=1e-15)


def test_quantile_q_function():
    from rl_replicas_b200.critics import QuantileQFunction
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import GreedyPolicy
    from rl_replicas_b200.q_function import QuantileQFunction as Exported
    assert Exported is QuantileQFunction and QuantileQFunction.MAX_QUANTILES == 256
    torch.manual_seed(0)
    net = MLP([3, 16, 4 * 7], torch.nn.ReLU)
    qf = QuantileQFunction(net, torch.optim.Adam(net.parameters()), n_quantiles=7)
    assert QuantileQFunction(net, None).n_quantiles == 200  # the default
    assert torch.equal(qf.taus, OQ.taus(7))
    obs = torch.randn(9, 3)
    th = qf.quantiles(obs)
    assert th.shape == (9, 4, 7)
    assert torch.equal(th.reshape(9, -1), net(obs))
    q = qf(obs)
    assert q.shape == (9, 4)
    torch.testing.assert_close(q, th.mean(-1))
    assert (GreedyPolicy(qf).get_action_numpy(obs.numpy()) == q.argmax(-1).numpy()).all()


def test_constructor_refusals():
    from rl_replicas_b200.algorithms import QRDQN
    from rl_replicas_b200.critics import CategoricalQFunction, DiscreteQFunction, QuantileQFunction
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.replay_buffer import PrioritizedReplayBuffer
    env = ChooseEnv()
    net = MLP([O_DIM, 16, N_ACT * 11], torch.nn.ReLU)
    opt = torch.optim.Adam(net.parameters())
    qf = QuantileQFunction(net, opt, n_quantiles=11)
    with pytest.raises(ValueError, match=r"must map 2 -> 36 \(3 actions x 12 quantiles\)"):
        QRDQN(QuantileQFunction(net, opt, n_quantiles=12), None, env, None, None, None)
    for bad in (0, 257, -1, 2.5, True):
        with pytest.raises(ValueError, match="n_quantiles must be an integer from 1 to 256"):
            QuantileQFunction(net, opt, n_quantiles=bad)
    cont = types.SimpleNamespace(action_space=types.SimpleNamespace(shape=(2,), high=np.ones(2)),
                                 observation_space=env.observation_space, spec=env.spec)
    with pytest.raises(ValueError, match="discrete"):
        QRDQN(qf, None, cont, None, None, None)
    for other in (DiscreteQFunction(net, opt), CategoricalQFunction(net, opt, n_atoms=11)):
        with pytest.raises(ValueError, match="QuantileQFunction"):
            QRDQN(other, None, env, None, None, None)
    with pytest.raises(ValueError, match="n_step"):
        QRDQN(qf, None, env, None, None, None, n_step=33)
    algo = QRDQN(qf, None, env, None, PrioritizedReplayBuffer(1000), None, target_update_interval=5, double_q=True,
                 n_step=3)
    assert (algo.target_update_interval, algo.double_q, algo.gamma, algo.epsilon_end, algo.n_step) == \
        (5, True, 0.99, 0.05, 3)
    one = MLP([O_DIM, 16, N_ACT], torch.nn.ReLU)
    QRDQN(QuantileQFunction(one, torch.optim.Adam(one.parameters()), n_quantiles=1), None, env, None, None, None)


def test_save_and_load_round_trip(tmp_path):
    algo = make_qr(seed=1)
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
    other = make_qr(seed=2)
    assert other.load_model(path) == 3 and other.current_total_steps == 77
    for a, b in ((algo.q_function.network, other.q_function.network),
                 (algo.target_q_function.network, other.target_q_function.network)):
        for (k, x), (_, y) in zip(a.state_dict().items(), b.state_dict().items()):
            assert torch.equal(x, y), k
    assert other._adam_step_count(other.q_function.optimizer, list(other.q_function.network.network)[::2]) == 1
    obs = torch.randn(5, O_DIM)
    assert torch.equal(algo.q_function(obs), other.q_function(obs))


def test_group_signature_refuses_differing_quantiles_and_mixes():
    from rl_replicas_b200.algorithms import LearnerGroup
    from rl_replicas_b200.replay_buffer import PrioritizedReplayBuffer
    from test_c51 import make_c51
    from test_dqn import make_dqn
    g = LearnerGroup()
    g.add(make_qr(seed=0))
    g.add(make_qr(seed=1))
    with pytest.raises(ValueError, match="network|n_quantiles"):
        g.add(make_qr(seed=2, n_quantiles=16))
    for other in (make_dqn(seed=2), make_c51(seed=2)):
        with pytest.raises(ValueError, match="class"):
            g.add(other)
    with pytest.raises(ValueError, match="target_update_interval"):
        g.add(make_qr(seed=2, target_update_interval=7))
    with pytest.raises(ValueError, match="n_step"):
        g.add(make_qr(seed=2, n_step=3))
    with pytest.raises(ValueError, match="prioritized replay"):
        g.add(make_qr(seed=2, replay_buffer=PrioritizedReplayBuffer(1000)))
    p = LearnerGroup()  # prioritized n-step members, each with its own buffer
    for k in range(2):
        p.add(make_qr(seed=k, n_step=3, replay_buffer=PrioritizedReplayBuffer(1000)))
    assert len(p) == 2


class OracleQR:
    """QRDQN.train with the float32 oracle in place of the engine: the same host random stream for the indices, the
    oracle's networks written back into the learner's."""

    @staticmethod
    def patch(algo):
        q = algo.q_function
        oracle = OQ.QrDqnOracle(q.network, algo.target_q_function.network, q.optimizer, n_quantiles=q.n_quantiles,
                                gamma=algo.gamma, target_update_interval=algo.target_update_interval,
                                double_q=algo.double_q)

        def train(replay_buffer, num_train_steps, minibatch_size):
            S, B = num_train_steps, minibatch_size
            idx = np.stack([replay_buffer.sample_indices(B) for _ in range(S)])
            oracle.train([replay_buffer.gather(idx[s]) for s in range(S)])
            algo.q_function.network.load_state_dict(oracle.q.state_dict())
            algo.target_q_function.network.load_state_dict(oracle.q_targ.state_dict())
        algo.train = train
        return oracle


def test_oracle_driven_learn_loop_solves_the_choice_task(tmp_path):
    """The bar the GPU learn() loop must clear (tests/test_gpu_qr.py) is one the oracle reaches with the same seeds."""
    np.random.seed(0)
    algo = make_qr(**QR_KW)
    OracleQR.patch(algo)
    before = evaluation_return(algo)
    algo.learn(output_dir=str(tmp_path), **LEARN)
    after = evaluation_return(algo)
    print(f"oracle-driven learn: evaluation return {before:.3f} -> {after:.3f}")
    assert before < 0.6 and after > RETURN_BAR, (before, after)
