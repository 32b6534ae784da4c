"""CPU: IQL's host side -- the float32 oracle against the float64 stages, the heads' closed-form gradients (clamped
log-std rows and capped weights included), beta = 0 as behaviour cloning, tau = 0.5 as half the MSE, the constructor's
refusals, the checkpoint round trip, the group signature, and an oracle-driven learn_offline run on a mixed-quality
bandit dataset that sets the bar for the GPU run (tests/test_gpu_iql.py)."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import iql as OI
from test_cql import OFFLINE, bandit_dataset
from test_sac import A_DIM, LEARN, O_DIM, BanditEnv, evaluation_return

GAP_MARGIN = 0.05  # IQL (beta = 3, tau = 0.7) beats behaviour cloning's evaluation return by at least this much (the
                  # oracle: -0.002 against -0.121)
ONLINE_BAR = -0.1  # IQL.learn's evaluation return after LEARN's online epochs from scratch, at least (the oracle: -0.019;
                   # a uniform random policy scores about -0.85)


def mixed_dataset(n=20000, seed=0):
    """Half near-expert rows, a = clip(f(s) + N(0, 0.05^2), -1, 1), and half uniform actions on [-1, 1]^A (rewards
    recomputed for them): behaviour cloning's mean is pulled toward 0."""
    d = bandit_dataset(n, seed=seed, noise=0.05)
    rng = np.random.default_rng(seed + 1)
    half = np.arange(n) % 2 == 1
    d["actions"][half] = rng.uniform(-1, 1, (int(half.sum()), A_DIM)).astype(np.float32)
    f = 0.8 * np.tanh(d["observations"] @ BanditEnv.M.T)
    d["rewards"] = -np.sum((d["actions"].astype(np.float64) - f) ** 2, axis=1)
    return d


def make_iql(hidden=64, seed=0, dataset=None, v_lr=1e-3, v_betas=(0.9, 0.999), q2_lr=1e-3, online=False, **kw):
    """An IQL learner on BanditEnv: offline on ``dataset`` (the mixed one by default), or ``online`` with a sampler,
    a uniform exploration policy and an empty replay buffer."""
    from rl_replicas_b200.algorithms import IQL
    from rl_replicas_b200.critics import ValueFunction
    from rl_replicas_b200.evaluator import Evaluator
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import TanhMeanGaussianPolicy
    from rl_replicas_b200.q_function import QFunction
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    torch.manual_seed(seed)
    env = BanditEnv()
    pnet = MLP([O_DIM, hidden, hidden, 2 * A_DIM], torch.nn.ReLU)
    q1, q2 = (MLP([O_DIM + A_DIM, hidden, hidden, 1], torch.nn.ReLU) for _ in range(2))
    vnet = MLP([O_DIM, hidden, hidden, 1], torch.nn.ReLU)
    policy = TanhMeanGaussianPolicy(pnet, torch.optim.Adam(pnet.parameters(), lr=1e-3))
    if online:
        from rl_replicas_b200.policies import RandomPolicy
        from rl_replicas_b200.samplers import BatchSampler
        rb, explore, sampler = ReplayBuffer(buffer_size=100000), RandomPolicy(env.action_space), BatchSampler(env, seed=0)
    else:
        rb, explore, sampler = ReplayBuffer.from_dataset(mixed_dataset() if dataset is None else dataset), None, None
    return IQL(policy, explore, QFunction(q1, torch.optim.Adam(q1.parameters(), lr=1e-3)),
               QFunction(q2, torch.optim.Adam(q2.parameters(), lr=q2_lr)),
               ValueFunction(vnet, torch.optim.Adam(vnet.parameters(), lr=v_lr, betas=v_betas)), env, sampler, rb,
               Evaluator(seed=0), **kw)


def oracle_of(algo):
    """The oracle of ``algo`` with each network's own Adam settings (the policy's and critics' betas and eps are Adam's
    defaults in every test)."""
    g = lambda m: m.optimizer.param_groups[0]
    v = g(algo.value_function)
    return OI.IqlOracle(algo.policy.network, algo.q_function_1.network, algo.q_function_2.network,
                        algo.value_function.network, pi_lr=g(algo.policy)["lr"], q_lr=g(algo.q_function_1)["lr"],
                        q2_lr=g(algo.q_function_2)["lr"], v_lr=v["lr"], v_betas=v["betas"], v_eps=v["eps"],
                        gamma=algo.gamma, rho=algo.polyak_rho, expectile=algo.expectile, beta=algo.beta,
                        max_weight=algo.max_weight, limit=algo.policy.action_limit,
                        log_std_min=algo.policy.log_std_min, log_std_max=algo.policy.log_std_max)


class OracleIQL:
    """IQL.train with the oracle in place of the engine, on the learner's host index draws."""

    @staticmethod
    def patch(algo):
        from rl_replicas_b200.algorithms._onpolicy import describe_mlp, flat_params, write_flat
        oracle = oracle_of(algo)

        def train(replay_buffer, num_train_steps, minibatch_size):
            S, B = num_train_steps, minibatch_size
            idx = np.stack([replay_buffer.sample_indices(B) for _ in range(S)])
            oracle.train([replay_buffer.gather(idx[s]) for s in range(S)])
            for src, dst in ((oracle.pi, algo.policy.network), (oracle.q1, algo.q_function_1.network),
                             (oracle.q2, algo.q_function_2.network), (oracle.v, algo.value_function.network)):
                write_flat(describe_mlp(dst)[3], flat_params(describe_mlp(src)[3]))
        algo.train = train
        return oracle


def _random_nets(sizes, seed):
    rng = np.random.default_rng(seed)
    size = lambda s: sum(s[i + 1] * (s[i] + 1) for i in range(len(s) - 1))
    return {k: rng.standard_normal(size(s)) * 0.3 for k, s in sizes.items()}


def _module(flat, sizes, act=torch.nn.ReLU):
    from rl_replicas_b200.networks import MLP
    m = MLP(sizes, act)
    torch.nn.utils.vector_to_parameters(torch.as_tensor(flat, dtype=torch.float32), m.parameters())
    return m


def _adam_grad(opt):
    return torch.cat([opt.state[p]["exp_avg"].reshape(-1) for p in opt.param_groups[0]["params"]]).numpy() / 0.1


@pytest.mark.parametrize("tau,beta,W", [(0.7, 3.0, 100.0), (0.9, 0.0, 100.0), (0.5, 10.0, 2.0)])
def test_float32_oracle_agrees_with_the_float64_stages(tau, beta, W):
    """One oracle step's value, policy and critic gradients (Adam's first moment / 0.1), losses and logged values
    against the float64 stages at the same parameters (the policy and critic stages read V' from the value stage)."""
    O, A, H, B = 4, 2, 16, 32
    sizes = dict(policy=[O, H, H, 2 * A], q1=[O + A, H, H, 1], q2=[O + A, H, H, 1], target_q1=[O + A, H, H, 1],
                 target_q2=[O + A, H, H, 1], v=[O, H, H, 1])
    nets = _random_nets(sizes, 3)
    mods = {k: _module(v, sizes[k]) for k, v in nets.items()}
    rng = np.random.default_rng(4)
    f32 = lambda x: np.asarray(x, np.float32)
    mb = dict(observations=f32(rng.standard_normal((B, O))), actions=f32(rng.uniform(-1, 1, (B, A))),
              rewards=f32(rng.standard_normal(B)), next_observations=f32(rng.standard_normal((B, O))),
              dones=rng.random(B) < 0.3)
    oracle = OI.IqlOracle(mods["policy"], mods["q1"], mods["q2"], mods["v"], expectile=tau, beta=beta, max_weight=W)
    with torch.no_grad():
        for k in ("q1", "q2"):
            torch.nn.utils.vector_to_parameters(torch.as_tensor(nets["target_" + k], dtype=torch.float32),
                                                getattr(oracle, k + "_targ").parameters())
    logs = oracle.train([mb])
    rel = lambda a, b: float(np.max(np.abs(np.asarray(a, np.float64) - b)) / max(np.max(np.abs(b)), 1e-12))
    vs = OI.value_stage_f64(nets, mb, sizes["q1"], sizes["v"], tau)
    assert rel(_adam_grad(oracle.v_opt), vs["grad"]) < 1e-4
    assert rel(logs["value_losses"][0], vs["loss"]) < 1e-5
    assert rel(logs["value_means"][0], vs["v"].mean()) < 1e-5
    v_new = oracle.v(torch.as_tensor(mb["observations"])).detach().double().numpy()[:, 0]
    v_next = oracle.v(torch.as_tensor(mb["next_observations"])).detach().double().numpy()[:, 0]
    ps = OI.policy_stage_f64(nets["policy"], mb["observations"], mb["actions"], vs["q_hat"], v_new, sizes["policy"],
                             beta, W)
    assert rel(_adam_grad(oracle.pi_opt), ps["grad"]) < 1e-4
    assert rel(logs["policy_losses"][0], ps["loss"]) < 1e-5
    assert rel(logs["weight_means"][0], ps["weights"].mean()) < 1e-5
    cs = OI.critic_stage_f64(nets, mb, v_next, sizes["q1"])
    for k, opt in ((1, oracle.q1_opt), (2, oracle.q2_opt)):
        assert rel(_adam_grad(opt), cs[f"q{k}_grad"]) < 1e-4
        assert rel(logs[f"q{k}_losses"][0], cs[f"q{k}_loss"]) < 1e-5
        assert rel(logs[f"q{k}_values"][0], cs[f"q{k}_values"]) < 1e-5


def test_closed_form_expectile_gradient_matches_autograd():
    rng = np.random.default_rng(0)
    q = torch.tensor(rng.standard_normal(64))
    for tau in (0.5, 0.7, 0.95):
        v = torch.tensor(rng.standard_normal(64), requires_grad=True)
        OI.expectile_loss(q, v, tau).backward()
        np.testing.assert_allclose(v.grad.numpy(), OI.expectile_grad_closed_form(q, v.detach(), tau).numpy(),
                                   rtol=1e-12, atol=1e-15)


def test_closed_form_awr_gradient_matches_autograd_with_clamped_rows_and_capped_weights():
    """Rows whose log-std leaves the clamp on either side get a zero log-std gradient (torch.clamp's rule), and rows
    whose weight is capped at W carry W."""
    rng = np.random.default_rng(1)
    B, A, L, lmin, lmax, beta, W = 40, 3, 2.0, -5.0, 2.0, 3.0, 5.0
    out = torch.tensor(rng.standard_normal((B, 2 * A)), requires_grad=True)
    with torch.no_grad():
        out[:5, A:] = 3.0    # above log_std_max
        out[5:10, A:] = -6.0  # below log_std_min
    act = torch.tensor(rng.uniform(-L, L, (B, A)))
    q, v = torch.tensor(rng.standard_normal(B)), torch.tensor(rng.standard_normal(B))
    q[10:20] += 3.0  # exp(beta (q - v)) above W
    e = OI.awr_weights(q, v, beta, W)
    assert (e == W).sum() >= 5 and (e < W).sum() >= 5
    (-(e * OI.log_prob(out, act, L, lmin, lmax)).mean()).backward()
    g = OI.awr_grad_closed_form(out.detach(), act, e, L, lmin, lmax)
    np.testing.assert_allclose(out.grad.numpy(), g.numpy(), rtol=1e-10, atol=1e-14)
    assert (g[:10, A:] == 0).all()


def test_beta_zero_is_the_behaviour_cloning_gradient():
    rng = np.random.default_rng(2)
    B, A, L = 32, 2, 1.0
    out = torch.tensor(rng.standard_normal((B, 2 * A)), requires_grad=True)
    act = torch.tensor(rng.uniform(-L, L, (B, A)))
    q, v = torch.tensor(rng.standard_normal(B) * 5), torch.tensor(rng.standard_normal(B))
    e = OI.awr_weights(q, v, 0.0, 100.0)
    assert (e == 1).all()
    (-OI.log_prob(out, act, L, -5.0, 2.0).mean()).backward()
    np.testing.assert_allclose(OI.awr_grad_closed_form(out.detach(), act, e, L, -5.0, 2.0).numpy(), out.grad.numpy(),
                               rtol=1e-10, atol=1e-14)


def test_expectile_one_half_is_half_the_mse():
    rng = np.random.default_rng(3)
    q, v = torch.tensor(rng.standard_normal(50)), torch.tensor(rng.standard_normal(50))
    assert float(OI.expectile_loss(q, v, 0.5)) == pytest.approx(0.5 * float(((q - v) ** 2).mean()), rel=1e-14)


def test_tanh_mean_gaussian_policy():
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import SquashedGaussianPolicy, TanhMeanGaussianPolicy
    torch.manual_seed(0)
    net = MLP([O_DIM, 16, 2 * A_DIM], torch.nn.ReLU)
    pol = TanhMeanGaussianPolicy(net, torch.optim.Adam(net.parameters()), action_limit=2.0)
    assert (pol.log_std_min, pol.log_std_max) == (-5.0, 2.0)
    obs = torch.randn(200, O_DIM)
    a = pol.get_action_tensor(obs)
    assert a.shape == (200, A_DIM) and a.abs().max() <= 2.0
    sac_eval = SquashedGaussianPolicy(net, torch.optim.Adam(net.parameters()), action_limit=2.0).deterministic()
    assert torch.equal(pol.deterministic().get_action_tensor(obs), sac_eval.get_action_tensor(obs))
    edge = torch.full((200, A_DIM), 2.0)  # a dataset action on the bound: finite, no atanh
    lp = pol.log_prob(obs, edge)
    assert torch.isfinite(lp).all()
    out = net(obs)
    np.testing.assert_allclose(lp.detach().numpy(), OI.log_prob(out, edge, 2.0, -5.0, 2.0).detach().numpy(), rtol=1e-6)


def test_constructor_refusals():
    from rl_replicas_b200.algorithms import IQL
    from rl_replicas_b200.critics import ContinuousQuantileQFunction, ValueFunction
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import SquashedGaussianPolicy
    from rl_replicas_b200.replay_buffer import PrioritizedReplayBuffer
    for kw, match in ((dict(expectile=0.0), "expectile"), (dict(expectile=1.0), "expectile"),
                      (dict(beta=-1.0), "beta"), (dict(max_weight=0.0), "max_weight"),
                      (dict(beta=math.inf), "finite"), (dict(expectile=math.nan), "finite"),
                      (dict(max_weight=math.inf), "finite")):
        with pytest.raises(ValueError, match=match):
            make_iql(dataset=bandit_dataset(100), **kw)
    a = make_iql(dataset=bandit_dataset(100))
    args = lambda **o: [o.get(k, getattr(a, k)) for k in ("policy", "exploration_policy", "q_function_1",
                                                           "q_function_2", "value_function", "env", "sampler",
                                                           "replay_buffer", "evaluator")]
    sq = SquashedGaussianPolicy(a.policy.network, a.policy.optimizer)
    with pytest.raises(TypeError, match="IQL needs a TanhMeanGaussianPolicy"):
        IQL(*args(policy=sq))
    qn = MLP([O_DIM + A_DIM, 8, 5], torch.nn.ReLU)
    with pytest.raises(TypeError, match="IQL: q_function_1"):
        IQL(*args(q_function_1=ContinuousQuantileQFunction(qn, torch.optim.Adam(qn.parameters()), n_quantiles=5)))
    with pytest.raises(ValueError, match="IQL does not train on a PrioritizedReplayBuffer"):
        IQL(*args(replay_buffer=PrioritizedReplayBuffer()))
    vn = MLP([O_DIM, 8, 1], torch.nn.ReLU)
    with pytest.raises(NotImplementedError, match="IQL value-function optimizer"):
        IQL(*args(value_function=ValueFunction(vn, torch.optim.SGD(vn.parameters(), lr=0.1))))
    vn2 = MLP([O_DIM, 8, 2], torch.nn.ReLU)
    with pytest.raises(ValueError, match="IQL: the value network"):
        IQL(*args(value_function=ValueFunction(vn2, torch.optim.Adam(vn2.parameters()))))
    with pytest.raises(ValueError, match="learn_offline"):
        a.learn(num_epochs=1)


def test_save_and_load_round_trip(tmp_path):
    algo = make_iql(dataset=bandit_dataset(100))
    with torch.no_grad():
        for p in algo.value_function.network.parameters():
            p.add_(0.25)
    path = os.path.join(tmp_path, "model.pt")
    algo.save_model(2, path)
    other = make_iql(seed=5, dataset=bandit_dataset(100))
    assert other.load_model(path) == 2
    for a, b in ((algo.q_function_1, other.q_function_1), (algo.policy, other.policy),
                 (algo.value_function, other.value_function)):
        for x, y in zip(a.network.parameters(), b.network.parameters()):
            assert torch.equal(x, y)
    keys = set(torch.load(path).keys())
    assert {"value_function_state_dict", "value_function_optimizer_state_dict", "policy_state_dict"} <= keys
    assert "log_alpha" not in keys


def test_group_signature():
    from rl_replicas_b200.algorithms import LearnerGroup
    d = bandit_dataset(100)
    g = LearnerGroup()
    g.add(make_iql(dataset=d))
    g.add(make_iql(seed=1, dataset=d))
    for kw in (dict(beta=1.0), dict(expectile=0.9), dict(max_weight=10.0), dict(v_lr=3e-4), dict(hidden=32)):
        with pytest.raises(ValueError, match="differs"):
            g.add(make_iql(seed=2, dataset=d, **kw))


def _offline_run(tmp_path, beta):
    np.random.seed(0)
    torch.manual_seed(0)
    algo = make_iql(beta=beta, expectile=0.7)
    OracleIQL.patch(algo)
    algo.learn_offline(output_dir=str(tmp_path), **OFFLINE)
    return algo


def test_oracle_driven_learn_offline_beats_behaviour_cloning(tmp_path):
    """The bar test_gpu_iql.py's learn_offline run must clear, reached here by the oracle with the same seeds: on the
    mixed-quality dataset IQL (beta = 3, tau = 0.7) beats the same learner at beta = 0 (behaviour cloning) by
    GAP_MARGIN."""
    iql = _offline_run(tmp_path / "iql", 3.0)
    bc = _offline_run(tmp_path / "bc", 0.0)
    ret, ret_bc = evaluation_return(iql), evaluation_return(bc)
    print(f"IQL return {ret:.3f}, behaviour cloning {ret_bc:.3f}")
    assert ret > ret_bc + GAP_MARGIN
    assert os.path.exists(tmp_path / "iql" / "model.pt")


def test_each_network_keeps_its_own_adam_settings():
    """The engine's critic rows take each critic's own optimizer, never the value function's: V's learning rate and
    betas go to set_iql alone."""
    algo = make_iql(dataset=bandit_dataset(100), v_lr=5e-5, v_betas=(0.8, 0.99), q2_lr=3e-4)
    hp = algo._hparams(False, 1)
    assert (hp.q1_lr, hp.q2_lr) == (1e-3, 3e-4)
    assert (hp.q_beta1, hp.q_beta2) == (0.9, 0.999)
    ip = algo.iql_hparams()
    assert (ip["v_lr"], ip["v_betas"]) == (5e-5, (0.8, 0.99))


def test_oracle_driven_online_learn_solves_the_bandit(tmp_path):
    """IQL.learn (online: the sampler explores uniformly, then samples the policy) with the oracle in place of the
    engine, from scratch on BanditEnv with the SAC tests' schedule: the bar test_gpu_iql.py's learn run must clear."""
    np.random.seed(0)
    algo = make_iql(online=True)
    OracleIQL.patch(algo)
    before = evaluation_return(algo)
    algo.learn(output_dir=str(tmp_path), **LEARN)
    after = evaluation_return(algo)
    print(f"oracle-driven IQL.learn: evaluation return {before:.3f} -> {after:.3f}")
    assert before < -0.3 and after > ONLINE_BAR, (before, after)
