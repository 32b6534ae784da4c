"""CPU: EDAC's host side -- the float32 autograd oracle against float64 stages, the float64 diversity gradient against
finite differences, the hand-derived decomposition the CUDA pass runs against autograd's double backward, the closed
form for identical critics, the exact zeros of the diversity term's bias and obs-column gradients, eta = 0 as REDQ with
M = N, the constructor's refusals, the checkpoint round trip, the group signature, the host draws, and the
oracle-driven learn_offline run that sets the bars for the GPU end-to-end test (tests/test_gpu_edac.py)."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import edac as OE
from oracle import redq as OR
from test_cql import OFFLINE
from test_iql import mixed_dataset
from test_sac import A_DIM, O_DIM, BanditEnv, evaluation_return

# EDAC.learn_offline on the mixed dataset (OFFLINE's epochs, N = 5, eta = 5), at least; the oracle reaches the value
# printed by test_oracle_driven_learn_offline (-0.010 when this was written; a uniform random policy scores about -0.85)
OFFLINE_BAR = -0.1
OFFLINE_ETA, OFFLINE_N = 5.0, 5


def make_edac(n=5, hidden=64, act=torch.nn.ReLU, seed=0, q_sizes=None, lrs=None, dataset=None, online=False, **kw):
    """An EDAC learner on BanditEnv: offline on ``dataset`` (tests/test_iql.py's mixed one by default), or ``online``
    with a sampler, a uniform exploration policy and an empty replay buffer."""
    from rl_replicas_b200.algorithms import EDAC
    from rl_replicas_b200.evaluator import Evaluator
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import RandomPolicy, SquashedGaussianPolicy
    from rl_replicas_b200.q_function import QFunction
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    from rl_replicas_b200.samplers import BatchSampler
    torch.manual_seed(seed)
    env = BanditEnv()
    pnet = MLP([O_DIM, hidden, hidden, 2 * A_DIM], torch.nn.ReLU)
    qs = []
    for i in range(n):
        net = MLP((q_sizes or {}).get(i, [O_DIM + A_DIM, hidden, hidden, 1]), act)
        qs.append(QFunction(net, torch.optim.Adam(net.parameters(), lr=(lrs or {}).get(i, 1e-3))))
    policy = SquashedGaussianPolicy(pnet, torch.optim.Adam(pnet.parameters(), lr=1e-3))
    if online:
        rb, explore, sampler = ReplayBuffer(buffer_size=100000), RandomPolicy(env.action_space), BatchSampler(env, seed=0)
    else:
        rb, explore, sampler = ReplayBuffer.from_dataset(mixed_dataset() if dataset is None else dataset), None, None
    return EDAC(policy, explore, qs, env, sampler, rb, Evaluator(seed=0), **kw)


def flat(m):
    return torch.nn.utils.parameters_to_vector(m.parameters()).detach().numpy()


def _mlp(sizes, act=torch.nn.ReLU, dtype=torch.float32):
    layers = []
    for i, (a, b) in enumerate(zip(sizes[:-1], sizes[1:])):
        layers.append(torch.nn.Linear(a, b))
        if i < len(sizes) - 2:
            layers.append(act())
    return torch.nn.Sequential(*layers).to(dtype)


def _minibatch(rng, B):
    return dict(observations=rng.standard_normal((B, O_DIM)).astype(np.float32),
                actions=rng.uniform(-1, 1, (B, A_DIM)).astype(np.float32),
                rewards=rng.standard_normal(B).astype(np.float32),
                next_observations=rng.standard_normal((B, O_DIM)).astype(np.float32),
                dones=rng.random(B) < 0.2)


def _adam_grads(opt):
    return [p.grad.detach().double().numpy().ravel() for g in opt.param_groups for p in g["params"]]


@pytest.mark.parametrize("eta", [0.0, 1.0, 5.0])
def test_oracle_agrees_with_float64_stages(eta):
    """One oracle step against the float64 critic and policy stages at the same parameters and draws."""
    torch.manual_seed(3)
    rng = np.random.default_rng(3)
    N, B, H = 4, 32, 32
    pi = _mlp([O_DIM, H, 2 * A_DIM])
    qs = [_mlp([O_DIM + A_DIM, H, H, 1]) for _ in range(N)]
    oracle = OE.EdacOracle(pi, qs, alpha=0.3, eta=eta)
    for qt in oracle.q_targs:
        with torch.no_grad():
            for p in qt.parameters():
                p.add_(0.1 * torch.randn_like(p))
    mb = _minibatch(rng, B)
    noise = rng.standard_normal((1, 2, B, A_DIM)).astype(np.float32)
    fl = lambda m: torch.nn.utils.parameters_to_vector(m.parameters()).detach().double().numpy()
    nets = dict(policy=fl(oracle.pi), q=[fl(q) for q in oracle.qs], target_q=[fl(q) for q in oracle.q_targs])
    psz, qsz = [O_DIM, H, 2 * A_DIM], [O_DIM + A_DIM, H, H, 1]
    c = OE.critic_stage_f64(nets, mb, noise[0, 0], 0.3, eta, psz, qsz)
    assert c["margin"].min() > 1e-6
    logs = oracle.train([mb], noise)
    for k in range(N):
        np.testing.assert_allclose(logs["q_values"][k][0], c["values"][k], rtol=1e-5, atol=1e-5)
        assert abs(logs["q_losses"][k][0] - c["losses"][k]) < 1e-5 * max(1.0, abs(c["losses"][k]))
        g = np.concatenate(_adam_grads(oracle.q_opts[k]))
        np.testing.assert_allclose(g, c["grads"][k], rtol=1e-4, atol=1e-5 * np.abs(c["grads"][k]).max())
    if eta > 0:
        assert abs(logs["diversity"][0] - c["diversity"]) < 1e-5 * max(1.0, abs(c["diversity"]))
        assert max(np.abs(g).max() for g in c["div_grads"]) > 1e-3  # the penalty moves the critics
    p = OE.policy_stage_f64(nets["policy"], [fl(q) for q in oracle.qs], mb["observations"], noise[0, 1], 0.3, psz, qsz)
    assert p["min_gap"].min() > 1e-5
    assert abs(logs["policy_losses"][0] - p["loss"]) < 1e-5 * max(1.0, abs(p["loss"]))
    assert abs(logs["log_prob_means"][0] - p["logp_mean"]) < 1e-5 * max(1.0, abs(p["logp_mean"]))
    g = np.concatenate(_adam_grads(oracle.pi_opt))
    np.testing.assert_allclose(g, p["grad"], rtol=1e-4, atol=1e-5 * np.abs(p["grad"]).max())


def _f64_critics(N, sizes, seed):
    torch.manual_seed(seed)
    return [_mlp(sizes, dtype=torch.float64) for _ in range(N)]


def _flats(nets):
    return [torch.nn.utils.parameters_to_vector(n.parameters()).detach().clone().requires_grad_(True) for n in nets]


def test_diversity_gradient_against_finite_differences():
    """torch.autograd.gradcheck of eta D with respect to every critic's flat parameters, at a point whose ReLU margins
    keep every unit on one side of its kink under the finite-difference steps."""
    N, B, sizes = 3, 8, [O_DIM + A_DIM, 8, 8, 1]
    rng = np.random.default_rng(5)
    obs = torch.as_tensor(rng.standard_normal((B, O_DIM)))
    act = torch.as_tensor(rng.uniform(-1, 1, (B, A_DIM)))
    ps = _flats(_f64_critics(N, sizes, 5))
    _, _, margin = OE.diversity_f64(ps, sizes, obs, act)
    assert margin.min() > 1e-4, margin.min()
    f = lambda *p: 2.5 * OE.diversity_f64(p, sizes, obs, act)[0]
    assert torch.autograd.gradcheck(f, tuple(ps), eps=1e-7, atol=1e-6, rtol=1e-5)


def _hand_derived(nets, obs, act, eta):
    """The diversity pass as the CUDA path computes it (b200rl.h, "EDAC"): a ones-backward for g, the head's u, a
    tangent forward of u through the ReLU masks and the weight gradients; returns (D, [[dW, db] per layer] per critic)."""
    O = obs.shape[1]
    x = torch.cat([obs, act], -1)
    per = []
    for net in nets:
        lins = [m for m in net if isinstance(m, torch.nn.Linear)]
        hs = [x]
        for i, lin in enumerate(lins):
            z = hs[-1] @ lin.weight.T + lin.bias
            hs.append(torch.relu(z) if i < len(lins) - 1 else z)
        e = [None] * (len(lins) + 1)  # e[l]: the ungated input gradient of sum_b Q at hs[l]
        e[len(lins)] = torch.ones(x.shape[0], 1, dtype=x.dtype)
        for l in range(len(lins) - 1, -1, -1):
            gate = (hs[l + 1] > 0).to(x.dtype) if l < len(lins) - 1 else 1.0
            e[l] = (e[l + 1] * gate) @ lins[l].weight
        per.append((lins, hs, e, e[0][:, O:]))
    G = torch.stack([p[3] for p in per])
    n = G.norm(dim=2, keepdim=True)
    gh = G / (n + OE.NORM_EPS)
    B, N = G.shape[1], G.shape[0]
    v = 2 * eta * (gh.sum(0, keepdim=True) - gh) / (B * (N - 1))
    corr = torch.where(n > 0, (G * v).sum(2, keepdim=True) / (n * (n + OE.NORM_EPS) ** 2), torch.zeros_like(n))
    U = v / (n + OE.NORM_EPS) - G * corr
    out = []
    for k, (lins, hs, e, _) in enumerate(per):
        L = len(lins)
        t = [None] * (L + 1)
        t[0] = torch.cat([torch.zeros_like(obs), U[k]], -1)
        for l in range(L - 1):
            t[l + 1] = (hs[l + 1] > 0).to(x.dtype) * (t[l] @ lins[l].weight.T)
        grads = []
        for l in range(L):
            gate = (hs[l + 1] > 0).to(x.dtype) if l < L - 1 else 1.0
            grads += [(e[l + 1] * gate).T @ t[l], torch.zeros_like(lins[l].bias)]
        out.append(grads)
    return OE.diversity(G), out


@pytest.mark.parametrize("sizes", [[O_DIM + A_DIM, 16, 16, 1], [O_DIM + A_DIM, 24, 16, 8, 1]])
def test_hand_derived_pass_matches_double_backward(sizes):
    """The CUDA path's decomposition of the diversity gradient (ones-backward, head, tangent forward, weight
    gradients) against autograd's double backward in float64, at two and three hidden layers."""
    N, B, eta = 4, 32, 2.0
    nets = _f64_critics(N, sizes, 7)
    rng = np.random.default_rng(7)
    obs = torch.as_tensor(rng.standard_normal((B, O_DIM)))
    act = torch.as_tensor(rng.uniform(-1, 1, (B, A_DIM)))
    at = act.clone().requires_grad_(True)
    grads = []
    for net in nets:
        (g,) = torch.autograd.grad(net(torch.cat([obs, at], -1)).sum(), at, create_graph=True)
        grads.append(g)
    d_auto = OE.diversity(torch.stack(grads))
    params = [p for net in nets for p in net.parameters()]
    ref = torch.autograd.grad(eta * d_auto, params, allow_unused=True)
    ref = [torch.zeros_like(p) if r is None else r for p, r in zip(params, ref)]
    with torch.no_grad():
        d_hand, hand = _hand_derived(nets, obs, act, eta)
    hand = [g for per in hand for g in per]
    assert abs(float(d_hand) - float(d_auto.detach())) < 1e-12
    for r, h in zip(ref, hand):
        assert float((r - h).abs().max()) <= 1e-12 * max(1.0, float(r.abs().max()))


def test_identical_critics_closed_form():
    """N identical critics with nonzero action gradients: every gh_i is the same unit vector (up to the 1e-10), so
    D = N (n / (n + 1e-10))^2 averaged over the rows, i.e. D ~= N."""
    N, B = 6, 16
    torch.manual_seed(0)
    one = _mlp([O_DIM + A_DIM, 16, 16, 1], dtype=torch.float64)
    ps = _flats([one] * N)
    rng = np.random.default_rng(0)
    obs = torch.as_tensor(rng.standard_normal((B, O_DIM)))
    act = torch.as_tensor(rng.uniform(-1, 1, (B, A_DIM)))
    d, _, _ = OE.diversity_f64(ps, [O_DIM + A_DIM, 16, 16, 1], obs, act)
    at = act.clone().requires_grad_(True)
    (g,) = torch.autograd.grad(one(torch.cat([obs, at], -1)).sum(), at)
    n = g.norm(dim=1)
    assert (n > 1e-3).all()
    expected = float((N * (n / (n + 1e-10)) ** 2).mean())
    d = float(d.detach())
    assert abs(d - expected) < 1e-12 and abs(d - N) < 1e-6


def test_diversity_bias_and_obs_column_gradients_are_exactly_zero():
    """The CUDA path never writes these entries of the diversity gradient (its block is zeroed at create): autograd's
    double backward must give exactly 0 there."""
    N, B, sizes = 4, 32, [O_DIM + A_DIM, 16, 16, 16, 1]
    nets = _f64_critics(N, sizes, 11)
    rng = np.random.default_rng(11)
    obs = torch.as_tensor(rng.standard_normal((B, O_DIM)))
    act = torch.as_tensor(rng.uniform(-1, 1, (B, A_DIM)))
    at = act.clone().requires_grad_(True)
    gs = [torch.autograd.grad(n(torch.cat([obs, at], -1)).sum(), at, create_graph=True)[0] for n in nets]
    d = OE.diversity(torch.stack(gs))
    lins = [[m for m in net if isinstance(m, torch.nn.Linear)] for net in nets]
    flat_grads = torch.autograd.grad(d, [p for ls in lins for l in ls for p in (l.weight, l.bias)], allow_unused=True)
    per = 2 * len(lins[0])
    for k in range(N):
        grads = flat_grads[k * per:(k + 1) * per]
        for i, g in enumerate(grads):
            if i % 2 == 1 or i == 0:  # every bias; the first weight's obs columns
                gz = torch.zeros(1, dtype=torch.float64) if g is None else (g[:, :O_DIM] if i == 0 else g)
                assert torch.count_nonzero(gz) == 0, i
        assert grads[0] is not None and torch.count_nonzero(grads[0][:, O_DIM:]) > 0


def test_eta_zero_critic_step_is_redq_with_every_target_critic():
    """At eta = 0 (SAC-N) the critic step is REDQ's with M = N."""
    torch.manual_seed(4)
    rng = np.random.default_rng(4)
    N, B, H = 5, 32, 32
    pi = _mlp([O_DIM, H, 2 * A_DIM])
    qs = [_mlp([O_DIM + A_DIM, H, H, 1]) for _ in range(N)]
    e = OE.EdacOracle(pi, qs, alpha=0.3, learn_alpha=False, eta=0.0)
    r = OR.RedqOracle(pi, qs, alpha=0.3, learn_alpha=False, policy_delay=1)
    for a, b in zip(e.q_targs, r.q_targs):
        with torch.no_grad():
            for pa, pb in zip(a.parameters(), b.parameters()):
                pa.add_(0.1 * torch.randn_like(pa))
                pb.copy_(pa)
    mb, noise = _minibatch(rng, B), rng.standard_normal((1, 2, B, A_DIM)).astype(np.float32)
    le, lr = e.train([mb], noise), r.train([mb], noise, np.arange(N, dtype=np.int32)[None])
    for k in range(N):
        np.testing.assert_array_equal(le["q_values"][k][0], lr["q_values"][k][0])
        np.testing.assert_allclose(flat(e.qs[k]), flat(r.qs[k]), rtol=0, atol=1e-7)


def test_edac_constructor_refusals():
    from rl_replicas_b200.replay_buffer import PrioritizedReplayBuffer
    make_edac(n=3, eta=0.0)
    make_edac(n=3, eta=0.0, act=torch.nn.Tanh)  # SAC-N takes any activation
    with pytest.raises(ValueError, match="EDAC needs at least 2 critics"):
        make_edac(n=1)
    with pytest.raises(ValueError, match="at most 32"):
        make_edac(n=33, hidden=4)
    for eta in (-1.0, math.inf, math.nan):
        with pytest.raises(ValueError, match="eta"):
            make_edac(n=3, eta=eta)
    with pytest.raises(NotImplementedError, match="ReLU"):
        make_edac(n=3, eta=1.0, act=torch.nn.Tanh)
    with pytest.raises(ValueError, match="same shape"):
        make_edac(n=3, q_sizes={2: [O_DIM + A_DIM, 32, 64, 1]})
    with pytest.raises(NotImplementedError, match="Adam"):
        make_edac(n=3, lrs={1: 3e-4})
    algo = make_edac(n=3)
    with pytest.raises(ValueError, match="PrioritizedReplayBuffer"):
        type(algo)(algo.policy, algo.exploration_policy, algo.q_functions, algo.env, None,
                   PrioritizedReplayBuffer(buffer_size=100), None)


def test_checkpoint_round_trip(tmp_path):
    algo = make_edac(n=4)
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
    assert {f"target_q_function_{i}_state_dict" for i in range(1, 5)} <= set(torch.load(path).keys())
    other = make_edac(n=4, seed=9)
    assert other.load_model(path) == 5 and other.current_total_steps == 77
    for a, b in zip([algo.policy] + algo.q_functions + algo.target_q_functions,
                    [other.policy] + other.q_functions + other.target_q_functions):
        assert np.array_equal(flat(a.network), flat(b.network))


def test_group_signature():
    from rl_replicas_b200.algorithms.group import _signature
    sig = dict(_signature(make_edac(n=4, eta=2.0)))
    assert sig["class"] == "EDAC" and sig["(n_critics, eta)"] == (4, 2.0) and "q_function_4 network" in sig
    base = _signature(make_edac(n=4, eta=2.0))
    for other in (make_edac(n=4, eta=1.0), make_edac(n=5, eta=2.0), make_edac(n=4, eta=2.0, learn_alpha=False)):
        assert _signature(other) != base


def test_host_draws_are_sacs():
    """The indices come from numpy, then per step torch.randn(B, A) for s' and then for s; nothing else is drawn."""
    from rl_replicas_b200.algorithms.sac import SAC
    algo = make_edac(n=3)
    torch.manual_seed(1)
    np.random.seed(1)
    state = np.random.get_state()
    noise = algo._noise(4, 8)
    assert np.random.get_state()[1].tolist() == state[1].tolist()  # no subsets
    torch.manual_seed(1)
    ref = SAC._noise(algo, 4, 8)
    torch.manual_seed(1)
    manual = np.stack([np.stack([torch.randn(8, A_DIM).numpy(), torch.randn(8, A_DIM).numpy()]) for _ in range(4)])
    assert np.array_equal(noise, ref) and np.array_equal(noise, manual)


class OracleEDAC:
    """EDAC.train with the oracle in place of the engine: the same host random streams (indices from numpy, then the
    noise from torch), the oracle's parameters written back into the learner."""

    @staticmethod
    def patch(algo):
        from rl_replicas_b200.algorithms._onpolicy import describe_mlp, flat_params, write_flat
        oracle = OE.EdacOracle(algo.policy.network, [q.network for q in algo.q_functions], gamma=algo.gamma,
                               rho=algo.polyak_rho, alpha=algo.alpha, learn_alpha=algo.learn_alpha,
                               target_entropy=algo.target_entropy, limit=algo.policy.action_limit, eta=algo.eta)

        def train(replay_buffer, num_train_steps, minibatch_size):
            S, B = num_train_steps, minibatch_size
            idx = np.stack([replay_buffer.sample_indices(B) for _ in range(S)])
            oracle.train([replay_buffer.gather(idx[s]) for s in range(S)], algo._noise(S, B))
            for src, dst in [(oracle.pi, algo.policy.network)] + list(zip(oracle.qs, [q.network for q in algo.q_functions])):
                write_flat(describe_mlp(dst)[3], flat_params(describe_mlp(src)[3]))
        algo.train = train
        return oracle


def test_oracle_driven_learn_offline(tmp_path):
    """The bar the GPU learn_offline run must clear (tests/test_gpu_edac.py) is one the oracle reaches with the same
    seeds."""
    np.random.seed(0)
    torch.manual_seed(0)
    algo = make_edac(n=OFFLINE_N, eta=OFFLINE_ETA)
    OracleEDAC.patch(algo)
    algo.learn_offline(output_dir=str(tmp_path), **OFFLINE)
    ret = evaluation_return(algo)
    print(f"oracle-driven EDAC learn_offline: evaluation return {ret:.3f}")
    assert ret > OFFLINE_BAR
    assert os.path.exists(tmp_path / "model.pt")
