"""CPU: SAC's host side -- the oracle's squashed-Gaussian log-probability, SquashedGaussianPolicy, the SAC constructor's
validation, its checkpoint round trip, and the oracle-driven learn() loop that sets the bar for the GPU end-to-end
test (tests/test_gpu_sac.py)."""
import types

import numpy as np
import pytest
import torch

from oracle import sac as OS

O_DIM, A_DIM = 3, 2


class BanditEnv:
    """One-step contextual bandit (gymnasium protocol): obs ~ U[-1, 1]^3, reward = -||a - f(obs)||^2 with
    f(obs) = 0.8 tanh(M obs); every episode ends after its single step."""
    M = np.asarray([[1.0, -1.0, 0.5], [0.5, 1.0, -1.0]], np.float32)

    def __init__(self, limit=1.0):
        self.rng = np.random.default_rng(0)
        hi = np.full(A_DIM, limit, np.float32)
        self.action_space = types.SimpleNamespace(high=hi, low=-hi, shape=(A_DIM,),
                                                  sample=lambda: self.rng.uniform(-limit, limit, A_DIM).astype(np.float32))
        self.observation_space = types.SimpleNamespace(shape=(O_DIM,))
        self.spec = types.SimpleNamespace(id="SacBandit-v0")

    def reset(self, seed=None):
        if seed is not None:
            self.rng = np.random.default_rng(seed)
        self.obs = self.rng.uniform(-1, 1, O_DIM).astype(np.float32)
        return self.obs, {}

    def step(self, action):
        target = 0.8 * np.tanh(self.M @ self.obs)
        reward = -float(np.sum((np.asarray(action, np.float64).reshape(-1) - target) ** 2))
        obs, _ = self.reset()
        return obs, reward, True, False, {}


def make_sac(hidden=64, limit=1.0, act=torch.nn.ReLU, seed=0, **kw):
    from rl_replicas_b200.algorithms import SAC
    from rl_replicas_b200.evaluator import Evaluator
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import RandomPolicy, SquashedGaussianPolicy
    from rl_replicas_b200.q_function import QFunction
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    from rl_replicas_b200.samplers import BatchSampler
    torch.manual_seed(seed)
    env = BanditEnv(limit)
    pnet = MLP([O_DIM, hidden, hidden, 2 * A_DIM], act)
    q1, q2 = MLP([O_DIM + A_DIM, hidden, hidden, 1], act), MLP([O_DIM + A_DIM, hidden, hidden, 1], act)
    policy = SquashedGaussianPolicy(pnet, torch.optim.Adam(pnet.parameters(), lr=1e-3), action_limit=limit)
    return SAC(policy, RandomPolicy(env.action_space), QFunction(q1, torch.optim.Adam(q1.parameters(), lr=1e-3)),
               QFunction(q2, torch.optim.Adam(q2.parameters(), lr=1e-3)), env, BatchSampler(env, seed=0),
               ReplayBuffer(buffer_size=100000), Evaluator(seed=0), **kw)


def test_oracle_log_prob_matches_the_tanh_transformed_normal_in_float64():
    from torch.distributions import Normal, TanhTransform, TransformedDistribution
    g = torch.Generator().manual_seed(0)
    B, A, L = 4096, 3, 2.0
    # |u| stays below ~10: beyond that tanh(u) rounds to 1 even in float64 and the reference's atanh is infinite
    out = torch.randn(B, 2 * A, generator=g, dtype=torch.float64) * torch.tensor([1.0] * A + [0.5] * A, dtype=torch.float64)
    eps = torch.randn(B, A, generator=g, dtype=torch.float64)
    act, logp = OS.squash(out, eps, L)
    mu, std = out[:, :A], torch.exp(torch.clamp(out[:, A:], -20, 2))
    ref = TransformedDistribution(Normal(mu, std), TanhTransform()).log_prob(act / L).sum(-1)
    assert act.abs().max() <= L
    assert torch.allclose(logp, ref, rtol=0, atol=1e-6), float((logp - ref).abs().max())


def test_squashed_gaussian_policy_bounds_and_views():
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import SquashedGaussianPolicy
    torch.manual_seed(1)
    net = MLP([O_DIM, 32, 32, 2 * A_DIM], torch.nn.ReLU)
    with torch.no_grad():
        net.network[-2].bias[:A_DIM] = 3.0    # mean far into the tanh saturation
        net.network[-2].bias[A_DIM:] = 40.0   # log_std far above the clamp
    pol = SquashedGaussianPolicy(net, torch.optim.Adam(net.parameters()), action_limit=2.0)
    obs = torch.rand(256, O_DIM) * 2 - 1
    a, logp = pol(obs)
    assert a.shape == (256, A_DIM) and logp.shape == (256,) and a.abs().max() <= 2.0
    assert torch.isfinite(logp).all()
    out = net(obs)
    mu = out[:, :A_DIM]
    a_det, lp_det = pol(obs, deterministic=True)
    torch.testing.assert_close(a_det, 2.0 * torch.tanh(mu))
    # the clamp: log_std = 40 acts as log_std_max = 2, at u = mu the Gaussian term is -A (2 + log sqrt(2 pi))
    clamped = torch.cat([mu, torch.full_like(mu, 2.0)], -1)
    torch.testing.assert_close(lp_det, OS.squash(clamped, torch.zeros(256, A_DIM), 2.0)[1])
    corr = (2 * (np.log(2) - mu - torch.nn.functional.softplus(-2 * mu))).sum(-1)
    torch.testing.assert_close(lp_det, -A_DIM * (2.0 + 0.5 * np.log(2 * np.pi)) - corr)
    view = pol.deterministic()
    np.testing.assert_allclose(view.get_action_numpy(obs[0].numpy()), (2.0 * torch.tanh(mu[0])).detach().numpy(), rtol=1e-6)
    sampled = pol.get_action_numpy(obs[0].numpy())
    assert sampled.shape == (A_DIM,) and np.abs(sampled).max() <= 2.0


def test_sac_constructor_rejects_bad_networks_and_optimizers():
    from rl_replicas_b200.algorithms import SAC
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import RandomPolicy, SquashedGaussianPolicy
    from rl_replicas_b200.q_function import QFunction
    env = BanditEnv()

    def build(p_out=2 * A_DIM, q_in=O_DIM + A_DIM, opt=torch.optim.Adam):
        pnet = MLP([O_DIM, 16, 16, p_out], torch.nn.ReLU)
        q1, q2 = MLP([q_in, 16, 16, 1], torch.nn.ReLU), MLP([O_DIM + A_DIM, 16, 16, 1], torch.nn.ReLU)
        return SAC(SquashedGaussianPolicy(pnet, opt(pnet.parameters(), lr=1e-3)), RandomPolicy(env.action_space),
                   QFunction(q1, torch.optim.Adam(q1.parameters())), QFunction(q2, torch.optim.Adam(q2.parameters())),
                   env, None, None, None)

    build()
    with pytest.raises(ValueError, match="mean \\| log_std"):
        build(p_out=A_DIM)
    with pytest.raises(ValueError, match="Q network"):
        build(q_in=O_DIM + 2 * A_DIM)
    with pytest.raises(NotImplementedError, match="Adam"):
        build(opt=torch.optim.SGD)


def test_save_and_load_restore_networks_adam_states_and_the_temperature(tmp_path):
    algo = make_sac(learn_alpha=True)
    # one optimizer step everywhere so that every Adam state exists
    obs = torch.rand(8, O_DIM)
    for m, x in ((algo.policy, obs), (algo.q_function_1, torch.rand(8, O_DIM + A_DIM)),
                 (algo.q_function_2, torch.rand(8, O_DIM + A_DIM))):
        m.optimizer.zero_grad()
        m.network(x).pow(2).sum().backward()
        m.optimizer.step()
    algo.alpha_optimizer.zero_grad()
    (algo.log_alpha * 3.0).backward()
    algo.alpha_optimizer.step()
    with torch.no_grad():
        for p in algo.target_q_function_1.network.parameters():
            p.add_(0.25)
    algo.current_total_steps = 123
    path = str(tmp_path / "model.pt")
    algo.save_model(7, path)
    other = make_sac(seed=5, learn_alpha=True)
    assert other.load_model(path) == 7 and other.current_total_steps == 123
    flat = lambda m: torch.nn.utils.parameters_to_vector(m.parameters()).detach()
    for a, b in ((algo.policy, other.policy), (algo.q_function_1, other.q_function_1),
                 (algo.q_function_2, other.q_function_2), (algo.target_q_function_1, other.target_q_function_1),
                 (algo.target_q_function_2, other.target_q_function_2)):
        assert torch.equal(flat(a.network), flat(b.network))
    for a, b in ((algo.policy.optimizer, other.policy.optimizer), (algo.q_function_1.optimizer, other.q_function_1.optimizer),
                 (algo.alpha_optimizer, other.alpha_optimizer)):
        sa, sb = a.state_dict()["state"], b.state_dict()["state"]
        assert sa.keys() == sb.keys() and len(sa) > 0
        for k in sa:
            for key in ("step", "exp_avg", "exp_avg_sq"):
                assert torch.equal(sa[k][key], sb[k][key])
    assert torch.equal(algo.log_alpha.detach(), other.log_alpha.detach())
    assert float(other.log_alpha.detach()) != float(np.log(0.2))


class OracleSAC:
    """SAC.train with the oracle in place of the engine: the same host random streams (indices from numpy, then the
    [S, 2, B, A] noise from torch), the oracle's parameters written back into the learner's networks."""

    @staticmethod
    def patch(algo, **oracle_kw):
        from rl_replicas_b200.algorithms._onpolicy import describe_mlp, flat_params, write_flat
        oracle = OS.SacOracle(algo.policy.network, algo.q_function_1.network, algo.q_function_2.network,
                              gamma=algo.gamma, rho=algo.polyak_rho, alpha=algo.alpha, learn_alpha=algo.learn_alpha,
                              target_entropy=algo.target_entropy, limit=algo.policy.action_limit, **oracle_kw)

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


LEARN = dict(num_epochs=50, batch_size=50, minibatch_size=64, num_start_steps=500, num_steps_before_update=500,
             num_train_steps=50, num_evaluation_episodes=10, evaluation_interval=500, model_saving_interval=500)
RETURN_BAR = -0.1  # a uniform random policy scores about -0.85 on BanditEnv


def evaluation_return(algo):
    from rl_replicas_b200.evaluator import Evaluator
    returns, _ = Evaluator(seed=123).evaluate(algo.evaluation_policy, BanditEnv(), 200)
    return float(np.mean(returns))


def test_oracle_driven_learn_loop_solves_the_bandit(tmp_path):
    """The bar the GPU learn() loop must clear (tests/test_gpu_sac.py) is one the oracle reaches with the same seeds."""
    np.random.seed(0)
    algo = make_sac(learn_alpha=True)
    OracleSAC.patch(algo)
    before = evaluation_return(algo)
    algo.learn(output_dir=str(tmp_path), **LEARN)
    after = evaluation_return(algo)
    print(f"oracle-driven learn: evaluation return {before:.3f} -> {after:.3f}")
    assert before < -0.3 and after > RETURN_BAR, (before, after)
