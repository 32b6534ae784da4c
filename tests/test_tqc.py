"""CPU: TQC's host side -- ContinuousQuantileQFunction, the truncated pooled target against a brute-force selection,
the closed-form critic and policy gradients against autograd, the float32 oracle against the float64 reference, the
TQC constructor's refusals, the checkpoint round trip, the LearnerGroup signature, and the oracle-driven learn() loop
that sets the bar for the GPU end-to-end test (tests/test_gpu_tqc.py)."""
import math

import numpy as np
import pytest
import torch

from oracle import tqc as OT
from oracle.qr import taus
from test_sac import A_DIM, LEARN, O_DIM, RETURN_BAR, BanditEnv, evaluation_return

M_DEFAULT = 25


def make_tqc(hidden=64, seed=0, n_quantiles=M_DEFAULT, n_quantiles_2=None, act=torch.nn.ReLU, replay_buffer=None,
             q_opt=torch.optim.Adam, **kw):
    from rl_replicas_b200.algorithms import TQC
    from rl_replicas_b200.critics import ContinuousQuantileQFunction
    from rl_replicas_b200.evaluator import Evaluator
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import RandomPolicy, SquashedGaussianPolicy
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    from rl_replicas_b200.samplers import BatchSampler
    torch.manual_seed(seed)
    env = BanditEnv()
    M2 = n_quantiles if n_quantiles_2 is None else n_quantiles_2
    pnet = MLP([O_DIM, hidden, hidden, 2 * A_DIM], act)
    q1, q2 = MLP([O_DIM + A_DIM, hidden, hidden, n_quantiles], act), MLP([O_DIM + A_DIM, hidden, hidden, M2], act)
    policy = SquashedGaussianPolicy(pnet, torch.optim.Adam(pnet.parameters(), lr=1e-3))
    return TQC(policy, RandomPolicy(env.action_space),
               ContinuousQuantileQFunction(q1, q_opt(q1.parameters(), lr=1e-3), n_quantiles=n_quantiles),
               ContinuousQuantileQFunction(q2, torch.optim.Adam(q2.parameters(), lr=1e-3), n_quantiles=M2), env,
               BatchSampler(env, seed=0), replay_buffer if replay_buffer is not None else ReplayBuffer(100000),
               Evaluator(seed=0), **kw)


def oracle_for(algo, **kw):
    return OT.TqcOracle(algo.policy.network, algo.q_function_1.network, algo.q_function_2.network,
                        n_quantiles=algo.q_function_1.n_quantiles, n_drop=algo.top_quantiles_to_drop_per_net,
                        gamma=algo.gamma, rho=algo.polyak_rho, alpha=algo.alpha, learn_alpha=algo.learn_alpha,
                        target_entropy=algo.target_entropy, limit=algo.policy.action_limit, **kw)


def random_minibatch(B, rng, O=O_DIM, A=A_DIM):
    return dict(observations=rng.uniform(-1, 1, (B, O)).astype(np.float32),
                actions=rng.uniform(-1, 1, (B, A)).astype(np.float32),
                rewards=rng.uniform(-3, 0, B).astype(np.float32),
                next_observations=rng.uniform(-1, 1, (B, O)).astype(np.float32),
                dones=rng.random(B) < 0.2)


def test_continuous_quantile_q_function_taus_and_mean():
    from rl_replicas_b200.critics import ContinuousQuantileQFunction, QuantileQFunction
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.q_function import ContinuousQuantileQFunction as Reexported
    assert Reexported is ContinuousQuantileQFunction
    net = MLP([O_DIM + A_DIM, 16, 7], torch.nn.ReLU)
    q = ContinuousQuantileQFunction(net, torch.optim.Adam(net.parameters()), n_quantiles=7)
    qr = QuantileQFunction(MLP([O_DIM, 16, 7], torch.nn.ReLU), None, n_quantiles=7)
    assert torch.equal(q.taus, qr.taus) and torch.equal(q.taus, taus(7))
    assert q.MAX_QUANTILES == 256
    o, a = torch.rand(5, O_DIM), torch.rand(5, A_DIM)
    z = q.quantiles(o, a)
    assert z.shape == (5, 7)
    torch.testing.assert_close(z, net(torch.cat([o, a], -1)))
    torch.testing.assert_close(q(o, a), z.sum(-1) / 7, rtol=0, atol=0)
    for bad in (0, 257, 2.5, True):
        with pytest.raises(ValueError, match="n_quantiles"):
            ContinuousQuantileQFunction(net, None, n_quantiles=bad)


@pytest.mark.parametrize("M,d", [(1, 0), (5, 1), (25, 2), (25, 24), (8, 0)])
def test_truncated_target_matches_a_brute_force_selection(M, d):
    """The kept atoms against repeated selection in float64, on random rows, rows full of ties and rows with NaNs."""
    kN = 2 * (M - d)
    rng = np.random.default_rng(M * 31 + d)
    rows = [rng.standard_normal((2, M)), rng.integers(-2, 3, (2, M)).astype(np.float64), np.zeros((2, M))]
    nan_row = rng.standard_normal((2, M))
    nan_row[0, rng.integers(0, M)] = np.nan
    nan_row[1, rng.integers(0, M)] = np.nan
    rows.append(nan_row)
    for r in rows:
        z1, z2 = torch.as_tensor(r[0:1]), torch.as_tensor(r[1:2])
        got = OT.truncated_atoms(z1, z2, kN)[0].numpy()
        want = np.asarray(OT.truncated_atoms_loop(r[0], r[1], kN))
        np.testing.assert_array_equal(got, want)
        assert len(got) == kN


def test_closed_form_gradients_match_autograd():
    """The critic head's -(sum_i k clamp(u)) / (kN M) / B and the policy head's -1 / (2 M B) against autograd."""
    rng = np.random.default_rng(3)
    B, M, kN = 16, 9, 14
    theta = torch.as_tensor(rng.standard_normal((B, M)) * 2, dtype=torch.float64).requires_grad_(True)
    y = torch.as_tensor(np.sort(rng.standard_normal((B, kN)) * 2, -1), dtype=torch.float64)
    tau = taus(M, torch.float64)
    OT.row_losses(theta, y, tau).mean().backward()
    torch.testing.assert_close(theta.grad, OT.critic_grad_closed_form(theta.detach(), y, tau), rtol=1e-12, atol=1e-15)
    z1 = torch.as_tensor(rng.standard_normal((B, M)), dtype=torch.float64).requires_grad_(True)
    z2 = torch.as_tensor(rng.standard_normal((B, M)), dtype=torch.float64).requires_grad_(True)
    logp = torch.as_tensor(rng.standard_normal(B), dtype=torch.float64)
    (0.2 * logp - torch.cat([z1, z2], -1).mean(-1)).mean().backward()
    for g in (z1.grad, z2.grad):
        torch.testing.assert_close(g, torch.full((B, M), -1.0 / (2 * M * B), dtype=torch.float64), rtol=1e-15, atol=0)


@pytest.mark.parametrize("learn_alpha", [False, True])
@pytest.mark.parametrize("M,d", [(25, 2), (5, 0), (5, 4), (1, 0)])
def test_float32_oracle_agrees_with_the_float64_reference(M, d, learn_alpha):
    """One TqcOracle step against oracle/tqc.py's float64 stages: target atoms, critic losses, Q-values and gradients
    (Adam's first moment over 1 - beta1 after one step), the policy loss, its gradient and mean log pi."""
    algo = make_tqc(seed=1, n_quantiles=M, top_quantiles_to_drop_per_net=d, learn_alpha=learn_alpha)
    oracle = oracle_for(algo)
    rng = np.random.default_rng(5)
    B = 64
    mb = random_minibatch(B, rng)
    noise = rng.standard_normal((1, 2, B, A_DIM)).astype(np.float32)
    flat = lambda m: torch.nn.utils.parameters_to_vector(m.parameters()).detach().double().numpy()
    nets = dict(policy=flat(oracle.pi), q1=flat(oracle.q1), q2=flat(oracle.q2), target_q1=flat(oracle.q1_targ),
                target_q2=flat(oracle.q2_targ))
    psz, qsz = [O_DIM, 64, 64, 2 * A_DIM], [O_DIM + A_DIM, 64, 64, M]
    logs = oracle.train([mb], noise)
    c = OT.critic_stage_f64(nets, mb, noise[0, 0], 0.2, psz, qsz, M, d)
    rel = lambda a, b: float(np.max(np.abs(np.asarray(a, np.float64) - b)) / max(np.max(np.abs(b)), 1e-30))
    assert rel(logs["targets"][0], c["y"]) < 1e-5
    for k, opt in ((1, oracle.q1_opt), (2, oracle.q2_opt)):
        assert rel(logs[f"q{k}_values"][0], c[f"q{k}_values"]) < 1e-5
        assert rel(logs[f"q{k}_losses"][0], c[f"q{k}_loss"]) < 1e-5
        m1 = torch.cat([opt.state[p]["exp_avg"].reshape(-1) for p in opt.param_groups[0]["params"]]).double().numpy()
        assert rel(m1 / 0.1, c[f"q{k}_grad"]) < 1e-4
    p = OT.policy_stage_f64(nets["policy"], flat(oracle.q1), flat(oracle.q2), mb["observations"], noise[0, 1], 0.2,
                            psz, qsz)
    assert rel(logs["policy_losses"][0], p["loss"]) < 1e-5
    assert rel(logs["log_prob_means"][0], p["logp_mean"]) < 1e-5
    m1 = torch.cat([oracle.pi_opt.state[q]["exp_avg"].reshape(-1) for q in oracle.pi_opt.param_groups[0]["params"]])
    assert rel(m1.double().numpy() / 0.1, p["grad"]) < 1e-4


def test_constructor_refusals():
    from rl_replicas_b200.algorithms import TQC
    from rl_replicas_b200.critics import ContinuousQuantileQFunction
    from rl_replicas_b200.networks import MLP, NoisyMLP
    from rl_replicas_b200.policies import DeterministicPolicy, RandomPolicy, SquashedGaussianPolicy
    from rl_replicas_b200.q_function import QFunction
    from rl_replicas_b200.replay_buffer import PrioritizedReplayBuffer
    make_tqc()
    with pytest.raises(ValueError, match="same n_quantiles"):
        make_tqc(n_quantiles=5, n_quantiles_2=7)
    for d in (-1, 25, 1.5, True):
        with pytest.raises(ValueError, match="top_quantiles_to_drop_per_net"):
            make_tqc(top_quantiles_to_drop_per_net=d)
    make_tqc(n_quantiles=1, top_quantiles_to_drop_per_net=0)
    with pytest.raises(ValueError, match="PrioritizedReplayBuffer"):
        make_tqc(replay_buffer=PrioritizedReplayBuffer(1000))
    with pytest.raises(NotImplementedError, match="Adam"):
        make_tqc(q_opt=torch.optim.SGD)
    env = BanditEnv()
    pnet = MLP([O_DIM, 16, 2 * A_DIM], torch.nn.ReLU)
    pol = SquashedGaussianPolicy(pnet, torch.optim.Adam(pnet.parameters()))

    def critic(sizes, cls=ContinuousQuantileQFunction, net_cls=MLP, **kw):
        net = net_cls(sizes, torch.nn.ReLU)
        return cls(net, torch.optim.Adam(net.parameters()), **kw)

    good = lambda: critic([O_DIM + A_DIM, 16, 5], n_quantiles=5)
    with pytest.raises(TypeError, match="ContinuousQuantileQFunction"):
        TQC(pol, RandomPolicy(env.action_space), critic([O_DIM + A_DIM, 16, 1], QFunction), good(), env, None, None,
            None)
    with pytest.raises(ValueError, match="Q network must map"):
        TQC(pol, RandomPolicy(env.action_space), critic([O_DIM + A_DIM, 16, 6], n_quantiles=5), good(), env, None,
            None, None, top_quantiles_to_drop_per_net=1)
    with pytest.raises(ValueError, match="Q network must map"):
        TQC(pol, RandomPolicy(env.action_space), critic([O_DIM + 2 * A_DIM, 16, 5], n_quantiles=5), good(), env,
            None, None, None, top_quantiles_to_drop_per_net=1)
    with pytest.raises(NotImplementedError, match="noisy"):
        TQC(pol, RandomPolicy(env.action_space), critic([O_DIM + A_DIM, 16, 5], net_cls=NoisyMLP, n_quantiles=5),
            good(), env, None, None, None, top_quantiles_to_drop_per_net=1)
    dnet = MLP([O_DIM, 16, A_DIM], torch.nn.ReLU)
    with pytest.raises(TypeError, match="SquashedGaussianPolicy"):
        TQC(DeterministicPolicy(dnet, torch.optim.Adam(dnet.parameters())), RandomPolicy(env.action_space), good(),
            good(), env, None, None, None, top_quantiles_to_drop_per_net=1)


def test_dueling_and_iqn_networks_are_refused():
    from rl_replicas_b200.algorithms import TQC
    from rl_replicas_b200.critics import ContinuousQuantileQFunction
    from rl_replicas_b200.networks import MLP, DuelingMLP, ImplicitQuantileMLP
    from rl_replicas_b200.policies import RandomPolicy, SquashedGaussianPolicy
    env = BanditEnv()
    pnet = MLP([O_DIM, 16, 2 * A_DIM], torch.nn.ReLU)
    pol = SquashedGaussianPolicy(pnet, torch.optim.Adam(pnet.parameters()))
    good = MLP([O_DIM + A_DIM, 16, 5], torch.nn.ReLU)
    for net in (DuelingMLP([O_DIM + A_DIM, 16, 16], 1, 5), ImplicitQuantileMLP([O_DIM + A_DIM, 16, 16], 5)):
        with pytest.raises(NotImplementedError, match="dueling and IQN"):
            TQC(pol, RandomPolicy(env.action_space),
                ContinuousQuantileQFunction(net, torch.optim.Adam(net.parameters()), n_quantiles=5),
                ContinuousQuantileQFunction(good, torch.optim.Adam(good.parameters()), n_quantiles=5), env, None,
                None, None, top_quantiles_to_drop_per_net=1)


def test_save_and_load_round_trip(tmp_path):
    """SAC's checkpoint keys: networks, Adam states, targets and the temperature come back exactly."""
    algo = make_tqc(seed=2, learn_alpha=True)
    oracle = oracle_for(algo)
    rng = np.random.default_rng(1)
    oracle.train([random_minibatch(32, rng)], rng.standard_normal((1, 2, 32, A_DIM)).astype(np.float32))
    for src, dst in ((oracle.pi, algo.policy.network), (oracle.q1, algo.q_function_1.network),
                     (oracle.q2, algo.q_function_2.network)):
        dst.load_state_dict(src.state_dict())
    for m in (algo.policy, algo.q_function_1, algo.q_function_2):
        m.optimizer.zero_grad()
        m.network(torch.rand(4, m.network.network[0].in_features)).pow(2).sum().backward()
        m.optimizer.step()
    algo.alpha_optimizer.zero_grad()
    (algo.log_alpha * 2.0).backward()
    algo.alpha_optimizer.step()
    algo.current_total_steps = 77
    path = str(tmp_path / "model.pt")
    algo.save_model(4, path)
    keys = set(torch.load(path, weights_only=True).keys())
    assert "target_q_function_2_state_dict" in keys and "log_alpha" in keys and "target_policy_state_dict" not in keys
    other = make_tqc(seed=9, learn_alpha=True)
    assert other.load_model(path) == 4 and other.current_total_steps == 77
    flat = lambda m: torch.nn.utils.parameters_to_vector(m.parameters()).detach()
    for a, b in ((algo.policy, other.policy), (algo.q_function_1, other.q_function_1),
                 (algo.q_function_2, other.q_function_2), (algo.target_q_function_1, other.target_q_function_1),
                 (algo.target_q_function_2, other.target_q_function_2)):
        assert torch.equal(flat(a.network), flat(b.network))
    sa, sb = algo.q_function_2.optimizer.state_dict()["state"], other.q_function_2.optimizer.state_dict()["state"]
    assert sa.keys() == sb.keys() and all(torch.equal(sa[k]["exp_avg"], sb[k]["exp_avg"]) for k in sa)
    assert torch.equal(algo.log_alpha.detach(), other.log_alpha.detach())


def test_group_signature():
    from rl_replicas_b200.algorithms import LearnerGroup
    from test_sac import make_sac
    g = LearnerGroup()
    g.add(make_tqc(seed=0))
    g.add(make_tqc(seed=1))
    for other, what in ((make_tqc(seed=2, n_quantiles=21), "network"),
                        (make_tqc(seed=2, top_quantiles_to_drop_per_net=3), "top_quantiles_to_drop_per_net"),
                        (make_tqc(seed=2, learn_alpha=True), "learn_alpha"),
                        (make_sac(), "class")):
        with pytest.raises(ValueError, match=what):
            g.add(other)


class OracleTQC:
    """TQC.train with the oracle in place of the engine: SAC's host random streams (indices from numpy, then the
    [S, 2, B, A] noise from torch), the oracle's parameters written back into the learner's networks."""

    @staticmethod
    def patch(algo):
        from rl_replicas_b200.algorithms._onpolicy import describe_mlp, flat_params, write_flat
        oracle = oracle_for(algo)

        def train(replay_buffer, num_train_steps, minibatch_size):
            S, B = num_train_steps, minibatch_size
            idx = np.stack([replay_buffer.sample_indices(B) for _ in range(S)])
            noise = algo._noise(S, B)
            oracle.train([replay_buffer.gather(idx[s]) for s in range(S)], noise)
            for src, dst in ((oracle.pi, algo.policy.network), (oracle.q1, algo.q_function_1.network),
                             (oracle.q2, algo.q_function_2.network)):
                write_flat(describe_mlp(dst)[3], flat_params(describe_mlp(src)[3]))
        algo.train = train
        return oracle


def test_oracle_driven_learn_loop_solves_the_bandit(tmp_path):
    """The bar the GPU learn() loop must clear (tests/test_gpu_tqc.py) is one the oracle reaches with the same seeds."""
    np.random.seed(0)
    algo = make_tqc(learn_alpha=True)
    OracleTQC.patch(algo)
    before = evaluation_return(algo)
    algo.learn(output_dir=str(tmp_path), **LEARN)
    after = evaluation_return(algo)
    print(f"oracle-driven learn: evaluation return {before:.3f} -> {after:.3f}")
    assert before < -0.3 and after > RETURN_BAR, (before, after)
    assert not math.isnan(after)
