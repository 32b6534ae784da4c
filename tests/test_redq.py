"""CPU: REDQ's host side -- the autograd oracle against float64 stages, the policy-delay schedule, the constructor's
refusals, the checkpoint round trip, the group signature, and the oracle-driven learn() loop that sets the bar for the
GPU end-to-end test (tests/test_gpu_redq.py)."""
import math

import numpy as np
import pytest
import torch

from oracle import redq as OR
from test_sac import LEARN, RETURN_BAR, A_DIM, O_DIM, BanditEnv, evaluation_return, make_sac


def make_redq(n=5, hidden=64, limit=1.0, act=torch.nn.ReLU, seed=0, q_sizes=None, lrs=None, **kw):
    from rl_replicas_b200.algorithms import REDQ
    from rl_replicas_b200.evaluator import Evaluator
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import RandomPolicy, SquashedGaussianPolicy
    from rl_replicas_b200.q_function import QFunction
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    from rl_replicas_b200.samplers import BatchSampler
    torch.manual_seed(seed)
    env = BanditEnv(limit)
    pnet = MLP([O_DIM, hidden, hidden, 2 * A_DIM], act)
    qs = []
    for i in range(n):
        net = MLP((q_sizes or {}).get(i, [O_DIM + A_DIM, hidden, hidden, 1]), act)
        qs.append(QFunction(net, torch.optim.Adam(net.parameters(), lr=(lrs or {}).get(i, 1e-3))))
    policy = SquashedGaussianPolicy(pnet, torch.optim.Adam(pnet.parameters(), lr=1e-3), action_limit=limit)
    return REDQ(policy, RandomPolicy(env.action_space), qs, env, BatchSampler(env, seed=0),
                ReplayBuffer(buffer_size=100000), Evaluator(seed=0), **kw)


def flat(m):
    return torch.nn.utils.parameters_to_vector(m.parameters()).detach().numpy()


def test_policy_delay_schedule():
    for S, G in ((1, 20), (5, 20), (20, 20), (45, 20), (1000, 20), (7, 1), (10, 3)):
        steps = OR.policy_steps(S, G)
        assert len(steps) == math.ceil(S / G), (S, G)
        assert steps[-1] == S - 1 and all((st + 1) % G == 0 for st in steps[:-1])


def test_oracle_agrees_with_float64_stages():
    """One oracle step against the float64 critic and policy stages at the same parameters and draws."""
    torch.manual_seed(3)
    rng = np.random.default_rng(3)
    N, M, B, H = 6, 3, 32, 32
    pi = torch.nn.Sequential(torch.nn.Linear(O_DIM, H), torch.nn.ReLU(), torch.nn.Linear(H, 2 * A_DIM))
    qs = [torch.nn.Sequential(torch.nn.Linear(O_DIM + A_DIM, H), torch.nn.ReLU(), torch.nn.Linear(H, 1))
          for _ in range(N)]
    oracle = OR.RedqOracle(pi, qs, alpha=0.3, policy_delay=1)
    for qt in oracle.q_targs:  # targets apart from the critics, so the subset matters
        with torch.no_grad():
            for p in qt.parameters():
                p.add_(0.1 * torch.randn_like(p))
    mb = dict(observations=rng.standard_normal((B, O_DIM)).astype(np.float32),
              actions=rng.uniform(-1, 1, (B, A_DIM)).astype(np.float32),
              rewards=rng.standard_normal(B).astype(np.float32),
              next_observations=rng.standard_normal((B, O_DIM)).astype(np.float32),
              dones=rng.random(B) < 0.2)
    noise = rng.standard_normal((1, 2, B, A_DIM)).astype(np.float32)
    subsets = np.array([[4, 0, 2]], np.int32)
    fl = lambda m: torch.nn.utils.parameters_to_vector(m.parameters()).detach().double().numpy()
    nets = dict(policy=fl(oracle.pi), q=[fl(q) for q in oracle.qs], target_q=[fl(q) for q in oracle.q_targs])
    psz, qsz = [O_DIM, H, 2 * A_DIM], [O_DIM + A_DIM, H, 1]
    c = OR.critic_stage_f64(nets, mb, noise[0, 0], subsets[0], 0.3, psz, qsz)
    logs = oracle.train([mb], noise, subsets)
    for k in range(N):
        np.testing.assert_allclose(logs["q_values"][k][0], c["values"][k], rtol=1e-5, atol=1e-5)
        assert abs(logs["q_losses"][k][0] - c["losses"][k]) < 1e-5 * max(1.0, abs(c["losses"][k]))
    p = OR.policy_stage_f64(nets["policy"], [fl(q) for q in oracle.qs], mb["observations"], noise[0, 1], 0.3, psz, qsz)
    assert abs(logs["policy_losses"][0] - p["loss"]) < 1e-5 * max(1.0, abs(p["loss"]))
    assert abs(logs["log_prob_means"][0] - p["logp_mean"]) < 1e-5 * max(1.0, abs(p["logp_mean"]))
    # the subset decides the target: M = N with the same draws gives a smaller (or equal) target everywhere
    c_all = OR.critic_stage_f64(nets, mb, noise[0, 0], range(N), 0.3, psz, qsz)
    assert (c_all["y"] <= c["y"] + 1e-12).all() and (c_all["y"] < c["y"]).any()


def test_redq_constructor_refusals():
    from rl_replicas_b200.replay_buffer import PrioritizedReplayBuffer
    make_redq(n=3, n_min=3, policy_delay=1)
    with pytest.raises(ValueError, match="at least 2 critics"):
        make_redq(n=1, n_min=1)
    with pytest.raises(ValueError, match="n_min"):
        make_redq(n=3, n_min=4)
    with pytest.raises(ValueError, match="n_min"):
        make_redq(n=3, n_min=0)
    with pytest.raises(ValueError, match="policy_delay"):
        make_redq(n=3, policy_delay=0)
    with pytest.raises(ValueError, match="same shape"):
        make_redq(n=3, q_sizes={2: [O_DIM + A_DIM, 32, 64, 1]})
    with pytest.raises(NotImplementedError, match="Adam"):
        make_redq(n=3, lrs={1: 3e-4})
    algo = make_redq(n=3)
    with pytest.raises(ValueError, match="PrioritizedReplayBuffer"):
        type(algo)(algo.policy, algo.exploration_policy, algo.q_functions, algo.env, None,
                   PrioritizedReplayBuffer(buffer_size=100), None)


def test_checkpoint_round_trip_and_sac_keys_at_two_critics(tmp_path):
    algo = make_redq(n=4, learn_alpha=True)
    obs = torch.rand(8, O_DIM)
    for m, x in [(algo.policy, obs)] + [(q, torch.rand(8, O_DIM + A_DIM)) for q in algo.q_functions]:
        m.optimizer.zero_grad()
        m.network(x).pow(2).sum().backward()
        m.optimizer.step()
    with torch.no_grad():
        for p in algo.target_q_functions[3].network.parameters():
            p.add_(0.25)
    algo.current_total_steps = 77
    path = str(tmp_path / "model.pt")
    algo.save_model(5, path)
    other = make_redq(n=4, seed=9, learn_alpha=True)
    assert other.load_model(path) == 5 and other.current_total_steps == 77
    for a, b in zip([algo.policy] + algo.q_functions + algo.target_q_functions,
                    [other.policy] + other.q_functions + other.target_q_functions):
        assert np.array_equal(flat(a.network), flat(b.network))
    for a, b in zip(algo.q_functions, other.q_functions):
        sa, sb = a.optimizer.state_dict()["state"], b.optimizer.state_dict()["state"]
        assert sa.keys() == sb.keys() and len(sa) > 0
        for k in sa:
            assert torch.equal(sa[k]["exp_avg_sq"], sb[k]["exp_avg_sq"])
    # at N = 2 the checkpoint holds exactly SAC's keys
    two, sac = make_redq(n=2), make_sac()
    two.save_model(1, str(tmp_path / "redq.pt"))
    sac.save_model(1, str(tmp_path / "sac.pt"))
    assert torch.load(str(tmp_path / "redq.pt")).keys() == torch.load(str(tmp_path / "sac.pt")).keys()


def test_group_signature():
    from rl_replicas_b200.algorithms.group import _signature
    sig = dict(_signature(make_redq(n=4, n_min=2, policy_delay=5)))
    assert sig["class"] == "REDQ" and sig["(n_critics, n_min)"] == (4, 2) and sig["policy_delay"] == 5
    assert "q_function_4 network" in sig and "log_std bounds" in sig
    base = _signature(make_redq(n=4, n_min=2, policy_delay=5))
    for other in (make_redq(n=4, n_min=3, policy_delay=5), make_redq(n=4, n_min=2, policy_delay=4),
                  make_redq(n=4, n_min=2, policy_delay=5, lrs={i: 3e-4 for i in range(4)})):
        assert _signature(other) != base
    assert len(_signature(make_redq(n=5))) > len(_signature(make_redq(n=4)))


class OracleREDQ:
    """REDQ.train with the oracle in place of the engine: the same host random streams (indices from numpy, then the
    subsets from numpy, then the noise from torch), the oracle's parameters written back into the learner."""

    @staticmethod
    def patch(algo):
        from rl_replicas_b200.algorithms._onpolicy import describe_mlp, flat_params, write_flat
        oracle = OR.RedqOracle(algo.policy.network, [q.network for q in algo.q_functions], gamma=algo.gamma,
                               rho=algo.polyak_rho, alpha=algo.alpha, learn_alpha=algo.learn_alpha,
                               target_entropy=algo.target_entropy, limit=algo.policy.action_limit,
                               policy_delay=algo.policy_delay)

        def train(replay_buffer, num_train_steps, minibatch_size):
            S, B = num_train_steps, minibatch_size
            idx = np.stack([replay_buffer.sample_indices(B) for _ in range(S)])
            noise, subsets = algo._noise(S, B)
            oracle.train([replay_buffer.gather(idx[s]) for s in range(S)], noise, subsets)
            for src, dst in [(oracle.pi, algo.policy.network)] + list(zip(oracle.qs, [q.network for q in algo.q_functions])):
                write_flat(describe_mlp(dst)[3], flat_params(describe_mlp(src)[3]))
        algo.train = train
        return oracle


# REDQ's regime: many critic updates per environment step (an update-to-data ratio of 5 here), the policy every 5
REDQ_LEARN = dict(LEARN, num_epochs=30, num_train_steps=250)


def test_oracle_driven_learn_loop_solves_the_bandit(tmp_path):
    """The bar the GPU learn() loop must clear (tests/test_gpu_redq.py) is one the oracle reaches with the same seeds."""
    np.random.seed(0)
    algo = make_redq(n=5, n_min=2, policy_delay=5, learn_alpha=True)
    OracleREDQ.patch(algo)
    before = evaluation_return(algo)
    algo.learn(output_dir=str(tmp_path), **REDQ_LEARN)
    after = evaluation_return(algo)
    print(f"oracle-driven REDQ learn: evaluation return {before:.3f} -> {after:.3f}")
    assert before < -0.3 and after > RETURN_BAR, (before, after)
