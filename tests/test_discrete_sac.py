"""CPU: discrete SAC's host side -- the float32 oracle (oracle/discrete_sac.py) against the float64 reference, the
closed-form logit gradient against autograd, the DiscreteSAC constructor's refusals, its checkpoint round trip, the
LearnerGroup signature for DiscreteSAC members, and the oracle-driven learn() loop that sets the bar for the GPU
end-to-end test (tests/test_gpu_discrete_sac.py)."""
import math
import types

import numpy as np
import pytest
import torch

from oracle import discrete_sac as OD
from test_dqn import ChooseEnv, N_ACT, O_DIM, random_minibatch

LR = 1e-3


def make_dsac(hidden=64, seed=0, n=N_ACT, O=O_DIM, env=None, replay_buffer=None, **kw):
    from rl_replicas_b200.algorithms import DiscreteSAC
    from rl_replicas_b200.critics import DiscreteQFunction
    from rl_replicas_b200.evaluator import Evaluator
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import CategoricalPolicy, RandomPolicy
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    from rl_replicas_b200.samplers import BatchSampler
    torch.manual_seed(seed)
    env = ChooseEnv() if env is None else env
    pnet = MLP([O, hidden, hidden, n], torch.nn.ReLU)
    q1, q2 = MLP([O, hidden, hidden, n], torch.nn.ReLU), MLP([O, hidden, hidden, n], torch.nn.ReLU)
    return DiscreteSAC(CategoricalPolicy(pnet, torch.optim.Adam(pnet.parameters(), lr=LR)),
                       RandomPolicy(env.action_space), DiscreteQFunction(q1, torch.optim.Adam(q1.parameters(), lr=LR)),
                       DiscreteQFunction(q2, torch.optim.Adam(q2.parameters(), lr=LR)), env,
                       BatchSampler(env, seed=0) if hasattr(env, "reset") else None,
                       ReplayBuffer(buffer_size=100000) if replay_buffer is None else replay_buffer, Evaluator(seed=0),
                       **kw)


def flat(m):
    return torch.nn.utils.parameters_to_vector(m.parameters()).detach().numpy().astype(np.float64)


def adam_m(opt, params):
    return torch.cat([opt.state[p]["exp_avg"].reshape(-1) for p in params]).numpy().astype(np.float64)


def rel(x, r):
    x, r = np.asarray(x, np.float64), np.asarray(r, np.float64)
    return float(np.max(np.abs(x - r)) / max(np.max(np.abs(r)), 1e-30))


@pytest.mark.parametrize("learn_alpha", [False, True])
def test_float32_oracle_agrees_with_the_float64_reference(learn_alpha):
    """One step: Q-values, losses, both critics' gradients, the policy's gradient and loss, mean E and the temperature
    gradient (gradients read from Adam's first moment, beta1 = 0.9) of the float32 oracle within 1e-5 of float64."""
    from rl_replicas_b200.networks import MLP
    torch.manual_seed(3)
    O, n, H = 4, 5, 32
    sizes = [O, H, H, n]
    pi, q1, q2 = (MLP(sizes, torch.nn.ReLU) for _ in range(3))
    mb = random_minibatch(np.random.default_rng(0), 64, n=n, O=O)
    o = OD.DiscreteSacOracle(pi, q1, q2, gamma=0.99, alpha=0.3, learn_alpha=learn_alpha)
    la0 = float(o.log_alpha.detach())
    p0, q10, q20 = flat(o.pi), flat(o.q1), flat(o.q2)
    logs = o.train([mb])
    alpha = math.exp(la0) if learn_alpha else 0.3
    c = OD.critic_stage_f64(q10, q20, q10, q20, p0, sizes, sizes, mb["observations"], mb["actions"], mb["rewards"],
                            mb["next_observations"], mb["dones"], alpha, 0.99)
    for k, opt, net in ((1, o.q1_opt, o.q1), (2, o.q2_opt, o.q2)):
        assert rel(logs[f"q{k}_values"][0], c[f"q{k}_values"]) < 1e-5
        assert abs(logs[f"q{k}_losses"][0] - c[f"q{k}_loss"]) <= 1e-5 * abs(c[f"q{k}_loss"])
        assert rel(adam_m(opt, list(net.parameters())) / 0.1, c[f"q{k}_grad"]) < 1e-5
    p = OD.policy_stage_f64(p0, flat(o.q1), flat(o.q2), sizes, sizes, mb["observations"], alpha, o.target_entropy,
                            log_alpha=la0)
    assert abs(logs["policy_losses"][0] - p["loss"]) <= 1e-5 * abs(p["loss"])
    assert abs(logs["log_prob_means"][0] - p["ent_mean"]) <= 1e-5 * abs(p["ent_mean"])
    assert rel(adam_m(o.pi_opt, list(o.pi.parameters())) / 0.1, p["grad"]) < 1e-5
    assert logs["alphas"][0] == pytest.approx(alpha, rel=1e-6)
    if learn_alpha:
        assert float(o.alpha_opt.state[o.log_alpha]["exp_avg"]) / 0.1 == pytest.approx(p["alpha_grad"], rel=1e-5)
    assert o.target_entropy == pytest.approx(0.98 * math.log(n), rel=1e-12)


def test_closed_form_logit_gradient_and_entropy_term_match_autograd():
    """pi_k (c_k - sum_a pi_a c_a) / B and E = sum_a pi_a log pi_a against autograd in float64, including rows whose
    probabilities vanish (log_softmax keeps pi log pi at 0, never NaN) and ties of the two critics."""
    g = torch.Generator().manual_seed(0)
    B, n = 257, 18
    x = torch.randn(B, n, generator=g, dtype=torch.float64) * 3
    x[0, 0] = 800.0  # every other probability underflows to 0
    x[1] = 0.0       # uniform
    q1 = torch.randn(B, n, generator=g, dtype=torch.float64)
    q2 = torch.randn(B, n, generator=g, dtype=torch.float64)
    q2[2] = q1[2]    # ties
    for alpha in (0.0, 0.2, 5.0):
        xr = x.clone().requires_grad_(True)
        L, E = OD.policy_terms(xr, q1, q2, alpha)
        L.mean().backward()
        cf = OD.closed_form_logit_grad(x, q1, q2, alpha)
        assert torch.isfinite(cf).all() and torch.isfinite(E).all() and torch.isfinite(L).all()
        torch.testing.assert_close(cf, xr.grad, rtol=1e-12, atol=1e-15)
        p = torch.softmax(x, -1)
        want_e = torch.where(p > 0, p * torch.log(p), torch.zeros_like(p)).sum(-1)
        torch.testing.assert_close(E, want_e, rtol=1e-12, atol=1e-15)
        E = E.detach()
        assert float(E[0]) == 0.0 and float(E[1]) == pytest.approx(-math.log(n), rel=1e-14)
    # the soft value of a uniform policy is the mean of min(q1t, q2t) plus alpha log n
    v = OD.soft_value(torch.zeros(1, n, dtype=torch.float64), q1[:1], q2[:1], 0.5)
    assert float(v) == pytest.approx(float(torch.min(q1[:1], q2[:1]).mean()) + 0.5 * math.log(n), rel=1e-12)


def test_constructor_refusals():
    from rl_replicas_b200.algorithms import DiscreteSAC
    from rl_replicas_b200.critics import CategoricalQFunction, DiscreteQFunction
    from rl_replicas_b200.networks import MLP, DuelingMLP, NoisyMLP
    from rl_replicas_b200.policies import CategoricalPolicy, GaussianPolicy
    from rl_replicas_b200.replay_buffer import PrioritizedReplayBuffer
    env = ChooseEnv()
    mk = lambda sizes: MLP(sizes, torch.nn.ReLU)
    adam = lambda m: torch.optim.Adam(m.parameters())
    pn, qn1, qn2 = mk([O_DIM, 16, N_ACT]), mk([O_DIM, 16, N_ACT]), mk([O_DIM, 16, N_ACT])
    pol, q1, q2 = CategoricalPolicy(pn, adam(pn)), DiscreteQFunction(qn1, adam(qn1)), DiscreteQFunction(qn2, adam(qn2))
    build = lambda *a, **kw: DiscreteSAC(*a, **kw)
    build(pol, None, q1, q2, env, None, None, None)
    cont = types.SimpleNamespace(action_space=types.SimpleNamespace(shape=(2,), high=np.ones(2)),
                                 observation_space=env.observation_space, spec=env.spec)
    with pytest.raises(ValueError, match="discrete action space"):
        build(pol, None, q1, q2, cont, None, None, None)
    one = types.SimpleNamespace(action_space=types.SimpleNamespace(n=1, shape=()), observation_space=env.observation_space,
                                spec=env.spec)
    with pytest.raises(ValueError, match="at least 2 actions"):
        build(pol, None, q1, q2, one, None, None, None)
    gp = GaussianPolicy(pn, adam(pn), torch.nn.Parameter(torch.zeros(N_ACT)))
    with pytest.raises(TypeError, match="CategoricalPolicy"):
        build(gp, None, q1, q2, env, None, None, None)
    wide = mk([O_DIM, 16, N_ACT + 1])
    with pytest.raises(ValueError, match="policy network must map obs 2 -> 3 logits"):
        build(CategoricalPolicy(wide, adam(wide)), None, q1, q2, env, None, None, None)
    with pytest.raises(ValueError, match="Q network must map obs 2 -> 3 values"):
        build(pol, None, q1, DiscreteQFunction(wide, adam(wide)), env, None, None, None)
    noisy = NoisyMLP([O_DIM, 16, N_ACT], torch.nn.ReLU)
    with pytest.raises(NotImplementedError, match="noisy layers"):
        build(pol, None, DiscreteQFunction(noisy, adam(noisy)), q2, env, None, None, None)
    duel = DuelingMLP([O_DIM, 16, 16], N_ACT)
    with pytest.raises(NotImplementedError, match="dueling and IQN networks are not implemented"):
        build(pol, None, DiscreteQFunction(duel, adam(duel)), q2, env, None, None, None)
    cat = mk([O_DIM, 16, N_ACT * 5])
    with pytest.raises(TypeError, match="DiscreteQFunction"):
        build(pol, None, CategoricalQFunction(cat, adam(cat), n_atoms=5), q2, env, None, None, None)
    with pytest.raises(ValueError, match="PrioritizedReplayBuffer"):
        build(pol, None, q1, q2, env, None, PrioritizedReplayBuffer(), None)
    with pytest.raises(NotImplementedError, match="Adam"):
        build(CategoricalPolicy(pn, torch.optim.SGD(pn.parameters(), lr=0.1)), None, q1, q2, env, None, None, None)
    with pytest.raises(ValueError, match="alpha must be > 0"):
        build(pol, None, q1, q2, env, None, None, None, alpha=0.0)
    a = build(pol, None, q1, q2, env, None, None, None)
    assert a.target_entropy == pytest.approx(0.98 * math.log(N_ACT)) and not a.learn_alpha and a.alpha == 0.2
    assert build(pol, None, q1, q2, env, None, None, None, target_entropy=0.5).target_entropy == 0.5


def test_save_and_load_restore_networks_adam_states_and_the_temperature(tmp_path):
    algo = make_dsac(learn_alpha=True)
    obs = torch.rand(8, O_DIM)
    for m in (algo.policy, algo.q_function_1, algo.q_function_2):
        m.optimizer.zero_grad()
        m.network(obs).pow(2).sum().backward()
        m.optimizer.step()
    algo.alpha_optimizer.zero_grad()
    (algo.log_alpha * 3.0).backward()
    algo.alpha_optimizer.step()
    with torch.no_grad():
        for p in algo.target_q_function_2.network.parameters():
            p.add_(0.25)
    algo.current_total_steps = 321
    path = str(tmp_path / "model.pt")
    algo.save_model(9, path)
    ckpt = torch.load(path, weights_only=True)
    assert set(ckpt) == {"epoch", "total_steps", "policy_state_dict", "policy_optimizer_state_dict",
                         "q_function_1_state_dict", "q_function_1_optimizer_state_dict",
                         "target_q_function_1_state_dict", "q_function_2_state_dict",
                         "q_function_2_optimizer_state_dict", "target_q_function_2_state_dict", "log_alpha",
                         "alpha_optimizer_state_dict"}
    other = make_dsac(seed=5, learn_alpha=True)
    assert other.load_model(path) == 9 and other.current_total_steps == 321
    for a, b in ((algo.policy, other.policy), (algo.q_function_1, other.q_function_1),
                 (algo.q_function_2, other.q_function_2), (algo.target_q_function_1, other.target_q_function_1),
                 (algo.target_q_function_2, other.target_q_function_2)):
        assert (flat(a.network) == flat(b.network)).all()
    for a, b in ((algo.policy.optimizer, other.policy.optimizer), (algo.q_function_2.optimizer, other.q_function_2.optimizer),
                 (algo.alpha_optimizer, other.alpha_optimizer)):
        sa, sb = a.state_dict()["state"], b.state_dict()["state"]
        assert sa.keys() == sb.keys() and len(sa) > 0
        for k in sa:
            for key in ("step", "exp_avg", "exp_avg_sq"):
                assert torch.equal(sa[k][key], sb[k][key])
    assert torch.equal(algo.log_alpha.detach(), other.log_alpha.detach())
    assert float(other.log_alpha.detach()) != float(np.log(0.2))
    assert other._alpha_state() == algo._alpha_state()


def test_group_signature():
    from rl_replicas_b200.algorithms import LearnerGroup
    from test_dqn import make_dqn
    from test_sac import make_sac
    g = LearnerGroup()
    g.add(make_dsac(seed=0, learn_alpha=True))
    g.add(make_dsac(seed=1, learn_alpha=True))
    with pytest.raises(ValueError, match="learn_alpha"):
        g.add(make_dsac(seed=2, learn_alpha=False))
    with pytest.raises(ValueError, match="target_entropy"):
        g.add(make_dsac(seed=2, learn_alpha=True, target_entropy=0.1))
    with pytest.raises(ValueError, match="policy network"):
        g.add(make_dsac(seed=2, learn_alpha=True, hidden=32))
    with pytest.raises(ValueError, match="class"):
        g.add(make_dqn(seed=2))
    with pytest.raises(ValueError, match="class"):
        g.add(make_sac(seed=2))
    s = LearnerGroup()
    s.add(make_sac(seed=0))
    with pytest.raises(ValueError, match="class"):
        s.add(make_dsac(seed=0))
    with pytest.raises(ValueError, match="DiscreteSAC"):
        s.add(object())


class OracleDSAC:
    """DiscreteSAC.train with the float32 oracle in place of the engine: the same host random stream for the indices,
    the oracle's parameters written back into the learner's networks."""

    @staticmethod
    def patch(algo):
        oracle = OD.DiscreteSacOracle(algo.policy.network, algo.q_function_1.network, algo.q_function_2.network,
                                      pi_lr=LR, q_lr=LR, gamma=algo.gamma, rho=algo.polyak_rho, alpha=algo.alpha,
                                      learn_alpha=algo.learn_alpha, target_entropy=algo.target_entropy)

        def train(replay_buffer, num_train_steps, minibatch_size):
            S, B = num_train_steps, minibatch_size
            idx = np.stack([replay_buffer.sample_indices(B) for _ in range(S)])
            oracle.train([replay_buffer.gather(idx[s]) for s in range(S)])
            for src, dst in ((oracle.pi, algo.policy.network), (oracle.q1, algo.q_function_1.network),
                             (oracle.q2, algo.q_function_2.network)):
                dst.load_state_dict(src.state_dict())
        algo.train = train
        return oracle


LEARN = dict(num_epochs=40, batch_size=50, minibatch_size=64, num_start_steps=500, num_steps_before_update=500,
             num_train_steps=50, num_evaluation_episodes=10, evaluation_interval=500, model_saving_interval=500)
RETURN_BAR = 0.85  # a uniform random policy scores 1/3 on ChooseEnv


def evaluation_return(algo):
    from rl_replicas_b200.evaluator import Evaluator
    returns, _ = Evaluator(seed=123).evaluate(algo.evaluation_policy, ChooseEnv(), 400)
    return float(np.mean(returns))


def test_oracle_driven_learn_loop_solves_the_choice_task(tmp_path):
    """The bar the GPU learn() loop must clear (tests/test_gpu_discrete_sac.py) is one the oracle reaches with the
    same seeds, on tests/test_dqn.py's one-step choice task."""
    np.random.seed(0)
    algo = make_dsac(learn_alpha=True)
    OracleDSAC.patch(algo)
    before = evaluation_return(algo)
    algo.learn(output_dir=str(tmp_path), **LEARN)
    after = evaluation_return(algo)
    print(f"oracle-driven learn: evaluation return {before:.3f} -> {after:.3f}")
    assert before < 0.6 and after > RETURN_BAR, (before, after)
