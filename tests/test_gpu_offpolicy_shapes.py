"""GPU: one step of the off-policy engine (OffPolicyEngine, C ABI underneath) at edge shapes against the float64
reference oracle/offpolicy_f64.py, the SAC head at its edges, and bit-identical execution paths at shapes whose GEMMs
need more than one prefetch round.

Every probe starts from zeroed Adam state and runs ONE step (S = 1) on a host-staged minibatch, so each quantity is
compared from the engine's own inputs to its stage:
* gradients are read from Adam: after one step from zero, exp_avg = fl((1 - b1) g) (adam.cu), so exp_avg / (1 - b1)
  is the kernel's gradient to within one rounding; sqrt(exp_avg_sq / (1 - b2)) is a second, independent readout of |g|;
* the policy stage takes the critics' post-step parameters read back from the engine (td3.py:309; SAC the same);
* post-step parameters are restated in float32 from the kernel's own moments, the polyak targets from its post-step
  parameters.  Both restatements follow the kernels' operation order including nvcc's FMA contraction (see
  offpolicy_f64.fma_f32), and the square root and divisions are correctly rounded on both sides, so both must match
  bit for bit.
The bar for everything compared with the float64 reference is the project's 1e-5 normwise error (conftest.rel_err).

ReLU kinks: a float32 kernel and the float64 reference may gate a ReLU differently when its pre-activation is within
rounding of 0, which is not a kernel error.  Minibatch rows are therefore drawn from a pool and kept only if every ReLU
pre-activation of the passes that depend on the step's inputs alone has |z| >= 1e-6 (sum_k |x_k w_k| + |b|); the one
pass that depends on the update (the critics on [s | pi(s)]) reports its smallest margin in the assertion message.  Seeds
are fixed; a case that fails with a margin below 1e-6 gets another seed (say so at the case), never a looser bar."""
import os
from dataclasses import dataclass

import numpy as np
import pytest
import torch

from conftest import rel_err
from oracle import offpolicy_f64 as R
from oracle import onpolicy as O
from oracle import sac as OS

pytestmark = pytest.mark.gpu

BAR = 1e-5
KINK = 1e-6
GAMMA, RHO, LR, ALPHA_LR, B1, B2, EPS = 0.99, 0.995, 1e-3, 3e-3, 0.9, 0.999, 1e-8
LOG_STD_MIN, LOG_STD_MAX = -20.0, 2.0


@dataclass
class Case:
    algo: str  # "td3", "ddpg" or "sac"
    policy: list
    q: list
    B: int
    hidden: str
    limit: float = 1.0
    noise: float = 0.2
    clip: float = 0.5
    learn_alpha: bool = False
    seed: int = 0

    @property
    def n_q(self):
        return 1 if self.algo == "ddpg" else 2

    @property
    def O(self):
        return self.policy[0]

    @property
    def A(self):
        return self.q[0] - self.policy[0]


# The GEMM tile fetches 8 k-tiles (K = 256) per prefetch round; B is the K of the weight-gradient products.
CASES = {
    # K = 400: two rounds; N = 300 ragged; B ragged
    "td3_paper": Case("td3", [17, 400, 300, 6], [23, 400, 300, 1], 100, "relu"),
    # first-layer K = 376 / 393 with the [s | a] split at column 376, inside the second round; A = 17
    "humanoid": Case("td3", [376, 256, 256, 17], [393, 256, 256, 1], 256, "relu"),
    # one row, A = 1, one critic
    "pendulum": Case("ddpg", [3, 64, 64, 1], [4, 64, 64, 1], 1, "relu"),
    # widths one off a tile, the split at k = 5, the clamp to the action limit binds
    "odd": Case("td3", [5, 33, 31, 2], [7, 33, 31, 1], 33, "tanh", limit=0.5, noise=0.4, clip=0.3),
    # 4 layers (no side-stream dW), dW K = 257: the bias column sums cross a prefetch round
    "deep": Case("td3", [11, 64, 48, 40, 3], [14, 96, 64, 32, 1], 257, "tanh"),
    # policy and critics of different depth: the target critic has more hidden layers than the target policy
    "mixed_depth": Case("ddpg", [8, 300, 2], [10, 40, 70, 50, 1], 64, "relu"),
    # dW K in four rounds; the single-CTA loss over 1000 rows
    "big_batch": Case("td3", [11, 256, 256, 3], [14, 256, 256, 1], 1000, "tanh"),
    "sac_paper": Case("sac", [17, 400, 300, 12], [23, 400, 300, 1], 100, "relu", learn_alpha=True),
    "sac_pendulum": Case("sac", [3, 64, 64, 2], [4, 64, 64, 1], 1, "tanh"),
    "sac_humanoid": Case("sac", [376, 256, 256, 34], [393, 256, 256, 1], 256, "tanh", learn_alpha=True),
}


# ---- problem set-up ------------------------------------------------------------------------------------------------
def init_nets(case, rng):
    def mk(sizes, sac_head=False):
        layers = [(rng.standard_normal((o, i)).astype(np.float32) / np.float32(np.sqrt(i)),
                   0.1 * rng.standard_normal(o).astype(np.float32)) for i, o in zip(sizes[:-1], sizes[1:])]
        if sac_head:  # log_std well inside [LOG_STD_MIN, LOG_STD_MAX]: the clamp's edges have tests of their own
            w, b = layers[-1]
            w[case.A:] *= 0.3
            b[case.A:] = -0.5 + 0.1 * rng.standard_normal(case.A).astype(np.float32)
        return O.flatten_layers(layers)

    nets = {"policy": mk(case.policy, case.algo == "sac"), "q1": mk(case.q)}
    if case.n_q == 2:
        nets["q2"] = mk(case.q)
    for k in list(nets):
        if k == "policy" and case.algo == "sac":
            continue  # SAC has no target policy
        nets["target_" + k] = (nets[k] + 0.02 * rng.standard_normal(nets[k].size)).astype(np.float32)
    return nets


def draw_rows(case, rng, n):
    mb = {"observations": rng.standard_normal((n, case.O)).astype(np.float32),
          "actions": rng.uniform(-case.limit, case.limit, (n, case.A)).astype(np.float32),
          "rewards": rng.standard_normal(n).astype(np.float32),
          "next_observations": rng.standard_normal((n, case.O)).astype(np.float32),
          "dones": (rng.random(n) < 0.1).astype(np.float32)}
    if case.algo == "td3":
        noise = rng.standard_normal((n, case.A)).astype(np.float32)
    elif case.algo == "sac":
        noise = rng.standard_normal((2, n, case.A)).astype(np.float32)
    else:
        noise = None
    return mb, noise


def take(mb, noise, rows):
    mb = {k: v[rows] for k, v in mb.items()}
    if noise is not None:
        noise = noise[rows] if noise.ndim == 2 else noise[:, rows]
    return mb, noise


def sac_alpha0(case):
    return float(np.float32(np.log(0.2)))


def alpha_of(case):
    return float(np.exp(np.float32(sac_alpha0(case)))) if case.learn_alpha else 0.2


def critic_stage(case, nets, mb, noise):
    if case.algo == "sac":
        return R.sac_critic_stage(nets, mb, noise[0], alpha_of(case), case.policy, case.q, case.hidden, GAMMA,
                                  case.limit, LOG_STD_MIN, LOG_STD_MAX)
    return R.td3_critic_stage(nets, mb, noise, case.policy, case.q, case.hidden, case.hidden, GAMMA, case.noise,
                              case.clip, case.limit)


def policy_stage(case, policy, q1, q2, mb, noise):
    if case.algo == "sac":
        return R.sac_policy_stage(policy, q1, q2, mb["observations"], noise[1], alpha_of(case), case.policy, case.q,
                                  case.hidden, case.limit, LOG_STD_MIN, LOG_STD_MAX, target_entropy=-case.A)
    return R.td3_policy_stage(policy, q1, mb["observations"], case.policy, case.q, case.hidden, case.hidden)


def minibatch(case, nets, rng):
    """B rows of a pool whose ReLU pre-activations, in every pass that depends on the step's inputs only, are at least
    KINK (relative) away from 0."""
    mb, noise = draw_rows(case, rng, 2 * case.B + 16)
    margin = critic_stage(case, nets, mb, noise)["margin"]
    margin = np.minimum(margin, policy_stage(case, nets["policy"], nets["q1"], nets.get("q2"), mb, noise)["margin_pi"])
    keep = np.flatnonzero(margin >= KINK)[:case.B]
    assert keep.size == case.B, f"only {keep.size} of {margin.size} pool rows clear the ReLU margin"
    return take(mb, noise, keep)


# ---- the engine ----------------------------------------------------------------------------------------------------
def hparams(case, delay=1):
    from rl_replicas_b200._lib import OffPolicyHparams
    hp = OffPolicyHparams()
    hp.gamma, hp.polyak_rho = GAMMA, RHO
    td3 = case.algo == "td3"
    hp.target_noise_scale, hp.target_noise_clip = (case.noise, case.clip) if td3 else (0.0, 0.0)
    hp.action_limit = case.limit
    hp.policy_delay, hp.use_target_noise = int(delay), int(td3)
    hp.policy_lr, hp.policy_beta1, hp.policy_beta2, hp.policy_eps = LR, B1, B2, EPS
    hp.q1_lr, hp.q2_lr, hp.q_beta1, hp.q_beta2, hp.q_eps = LR, LR, B1, B2, EPS
    return hp


def sac_hparams(case):
    from rl_replicas_b200._lib import SacHparams
    sp = SacHparams()
    sp.alpha, sp.learn_alpha, sp.target_entropy = 0.2, int(case.learn_alpha), -float(case.A)
    sp.alpha_lr, sp.alpha_beta1, sp.alpha_beta2, sp.alpha_eps = ALPHA_LR, B1, B2, EPS
    sp.log_std_min, sp.log_std_max = LOG_STD_MIN, LOG_STD_MAX
    return sp


def make_engine(case, nets, max_minibatch, max_steps):
    from rl_replicas_b200.engine import OffPolicyEngine as E
    sac = case.algo == "sac"
    e = E(case.policy, case.q, case.n_q, max_minibatch, max_steps, (case.hidden, "identity" if sac else "tanh"),
          (case.hidden, "identity"), algo=E.SAC if sac else E.TD3)
    for name, i in E.NETS.items():
        if name in nets:
            e.set_params(i, nets[name])
    for i in range(1 + case.n_q):
        e.set_adam(i, None, None, 0)
    if sac:
        e.set_sac(sac_hparams(case))
        e.set_alpha(sac_alpha0(case))
    return e


def stacked(mb, noise, S=1):
    """[B, ...] -> [S, B, ...] (the same minibatch for every step; noise of SAC [2, B, A] -> [S, 2, B, A])"""
    cols = [np.ascontiguousarray(np.broadcast_to(mb[k], (S,) + mb[k].shape)) for k in
            ("observations", "actions", "rewards", "next_observations", "dones")]
    nz = None if noise is None else np.ascontiguousarray(np.broadcast_to(noise, (S,) + noise.shape))
    return cols, nz


def ulps(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return np.abs(ia - ib)


def grad_readout(m, v):
    """(g, |g|) from Adam's moments after one step from zero."""
    g = m.astype(np.float64) / np.float64(np.float32(1.0 - B1))
    return g, np.sqrt(v.astype(np.float64) / np.float64(np.float32(1.0 - B2)))


def check_elementwise(case, e, nets):
    """Post-step parameters from the kernel's moments and polyak targets from its parameters, bit for bit."""
    names = ["policy", "q1", "q2"][:1 + case.n_q]
    post = {}
    for i, name in enumerate(names):
        m, v, step = e.get_adam(i)
        assert step == 1, (name, step)
        post[name] = e.get_params(i)
        d = ulps(post[name], R.adam_update_f32(nets[name], m, v, 1, LR, B1, B2, EPS))
        assert d.max() == 0, (name, f"{int((d > 0).sum())} parameters differ by up to {int(d.max())} ulp")
    from rl_replicas_b200.engine import OffPolicyEngine as E
    for name in names:
        t = "target_" + name
        if t in nets:
            np.testing.assert_array_equal(e.get_params(E.NETS[t]), R.polyak_f32(nets[t], post[name], RHO), err_msg=t)
    return post


def run_probe(case, nets, mb, noise, label):
    """One engine step against the reference; returns the errors (asserted below BAR by the caller)."""
    cols, nz = stacked(mb, noise)
    e = make_engine(case, nets, case.B, 1)
    out = e.train(hparams(case), *cols, nz)
    errs = {}
    crit = critic_stage(case, nets, mb, noise)
    for i in range(case.n_q):
        errs[f"q{i + 1}_values"] = rel_err(out[f"q{i + 1}_values"][0], crit["q_values"][i])
        errs[f"q{i + 1}_loss"] = rel_err(out[f"q{i + 1}_losses"][0], crit["losses"][i])
        g, ga = grad_readout(*e.get_adam(1 + i)[:2])
        errs[f"q{i + 1}.grad"] = rel_err(g, crit["grads"][i])
        errs[f"q{i + 1}.|grad|"] = rel_err(ga, np.abs(crit["grads"][i]))
    post = check_elementwise(case, e, nets)
    pol = policy_stage(case, nets["policy"], post["q1"], post.get("q2"), mb, noise)
    errs["policy_loss"] = rel_err(out["policy_losses"][0], pol["loss"])
    g, ga = grad_readout(*e.get_adam(0)[:2])
    errs["policy.grad"] = rel_err(g, pol["grad"])
    errs["policy.|grad|"] = rel_err(ga, np.abs(pol["grad"]))
    if case.algo == "sac":
        errs["log_prob_mean"] = rel_err(out["log_prob_means"][0], pol["logp_mean"])
        errs["alpha"] = rel_err(out["alphas"][0], alpha_of(case))
        la, am, av, astep = e.get_alpha()
        if case.learn_alpha:
            assert astep == 1
            errs["log_alpha.grad"] = rel_err(am / np.float64(np.float32(1.0 - B1)), pol["alpha_grad"])
            d = ulps(la, R.adam_update_f32(np.float32(sac_alpha0(case)), am, av, 1, ALPHA_LR, B1, B2, EPS))
            assert d.max() == 0, ("log_alpha", la)
        else:
            assert la == np.float32(sac_alpha0(case)) and astep == 0
    e.close()
    margin_q = float(np.min(pol["margin_q"]))
    print(f"\n{label}: " + ", ".join(f"{k} {v:.1e}" for k, v in errs.items()) +
          f"; smallest ReLU margin after the critic update {margin_q:.1e}")
    for k, v in errs.items():
        assert v < BAR, (label, k, v, f"smallest ReLU margin on [s | pi(s)] after the critic update: {margin_q:.1e}")
    return errs


@pytest.mark.parametrize("name", list(CASES))
def test_one_step_matches_the_float64_reference(name):
    case = CASES[name]
    rng = np.random.default_rng(case.seed)
    nets = init_nets(case, rng)
    mb, noise = minibatch(case, nets, rng)
    run_probe(case, nets, mb, noise, name)


# ---- the SAC head at its edges -------------------------------------------------------------------------------------
# Which reference for what:
# * gradients: float64.  The kernel's d log_std = g_u sigma eps - c is the exact derivative; float32 autograd picks up a
#   spurious (u - mu) cancellation term at extreme sigma.
# * log pi (and the policy loss and temperature gradient built from it) at sigma = exp(log_std_min): sigma eps is below
#   one ulp of mu, so u - mu rounds to 0 and the float32 semantics of oracle/sac.py ARE the specification.
# The critics' targets are kept free of log pi(a' | s') by done = 1 on every row.
HEAD = Case("sac", [5, 32, 32, 8], [9, 32, 32, 1], 64, "tanh")


def head_nets(rng, mu_bias, mu_scale, log_std_bias, log_std_scale):
    nets = init_nets(HEAD, rng)
    layers = O.unflatten_layers(nets["policy"], HEAD.policy)
    w, b = layers[-1]
    A = HEAD.A
    w[:A] *= np.float32(mu_scale)[:, None]
    w[A:] *= np.float32(log_std_scale)
    b[:A] = np.where(np.isnan(mu_bias), b[:A], mu_bias).astype(np.float32)
    b[A:] = np.asarray(log_std_bias, np.float32)
    nets["policy"] = O.flatten_layers(layers)
    return nets


def f32_module(flat, sizes):
    m = torch.nn.Sequential(*[x for i, o in zip(sizes[:-1], sizes[1:]) for x in (torch.nn.Linear(i, o), torch.nn.Tanh())][:-1])
    torch.nn.utils.vector_to_parameters(torch.as_tensor(flat), m.parameters())
    return m


@pytest.mark.parametrize("edge", ["clamp_bounds", "saturated_tanh"])
def test_sac_head_edges(edge):
    rng = np.random.default_rng(5)
    up, down = np.nextafter(np.float32(LOG_STD_MAX), np.float32(np.inf)), np.nextafter(np.float32(LOG_STD_MIN),
                                                                                      np.float32(-np.inf))
    if edge == "clamp_bounds":
        # log_std exactly on each bound (the clamp's gradient mask is inclusive) and one float32 step outside each;
        # the means paired with the log_std_min columns are exactly 0.75 and -0.6, so u == mu there
        nets = head_nets(rng, np.array([np.nan, 0.75, np.nan, -0.6]), np.array([1, 0, 1, 0]),
                         [LOG_STD_MAX, LOG_STD_MIN, up, down], 0.0)
    else:
        # |u| > 10: tanh saturates in float32 (1 - t^2 == 0), softplus(-2u) takes its x > 20 branch where u < -10
        nets = head_nets(rng, np.array([12.0, -12.0, 13.0, -14.0]), np.full(4, 0.01), [-1.0, -1.2, -0.8, -1.0], 0.1)
    mb, noise = draw_rows(HEAD, rng, HEAD.B)
    noise = np.clip(noise, -3.5, 3.5)  # keeps |u| > 10 in the saturated case
    mb["dones"][:] = 1.0
    cols, nz = stacked(mb, noise)
    e = make_engine(HEAD, nets, HEAD.B, 1)
    out = e.train(hparams(HEAD), *cols, nz)
    errs = {}
    crit = critic_stage(HEAD, nets, mb, noise)
    for i in range(2):
        errs[f"q{i + 1}_loss"] = rel_err(out[f"q{i + 1}_losses"][0], crit["losses"][i])
        errs[f"q{i + 1}.grad"] = rel_err(grad_readout(*e.get_adam(1 + i)[:2])[0], crit["grads"][i])
    post = check_elementwise(HEAD, e, nets)
    pol = policy_stage(HEAD, nets["policy"], post["q1"], post["q2"], mb, noise)
    g = grad_readout(*e.get_adam(0)[:2])[0]
    errs["policy.grad"] = rel_err(g, pol["grad"])
    # the output layer's log_std rows: the gradient the clamp mask lets through (or stops)
    A, H = HEAD.A, HEAD.policy[-2]
    off = sum(o * i + o for i, o in zip(HEAD.policy[:-2], HEAD.policy[1:-1]))
    w_ls = lambda x: x[off + A * H:off + 2 * A * H].reshape(A, H)
    errs["policy.grad[log_std rows]"] = rel_err(w_ls(g), w_ls(pol["grad"]))
    if edge == "clamp_bounds":
        assert (w_ls(g)[2:] == 0).all()  # outside the bounds: no gradient
        assert (np.abs(w_ls(g)[:2]).max(axis=1) > 0).all()  # on the bounds: the gradient passes
        with torch.no_grad():  # log pi with float32 semantics
            o = f32_module(nets["policy"], HEAD.policy)(torch.as_tensor(mb["observations"]))
            a, logp = OS.squash(o, torch.as_tensor(noise[1]), HEAD.limit, LOG_STD_MIN, LOG_STD_MAX)
            x = torch.cat([torch.as_tensor(mb["observations"]), a], -1)
            q = torch.minimum(f32_module(post["q1"], HEAD.q)(x)[:, 0], f32_module(post["q2"], HEAD.q)(x)[:, 0])
            want_lp, want_loss = float(logp.mean()), float((0.2 * logp - q).mean())
    else:
        want_lp, want_loss = pol["logp_mean"], pol["loss"]
    errs["log_prob_mean"] = rel_err(out["log_prob_means"][0], want_lp)
    errs["policy_loss"] = rel_err(out["policy_losses"][0], want_loss)
    e.close()
    print(f"\nsac head {edge}: " + ", ".join(f"{k} {v:.1e}" for k, v in errs.items()))
    for k, v in errs.items():
        assert v < BAR, (edge, k, v)


# ---- execution paths ---------------------------------------------------------------------------------------------
PATHS = {  # name: (B200RL_OFFPOLICY_GRAPH, device gather)
    "graph": ("1", False), "gather": ("1", True), "gather_plain": ("0", True)}


def run_path(case, nets, delay, graph, gather, data, S, calls=2):
    os.environ["B200RL_OFFPOLICY_GRAPH"] = graph
    e = make_engine(case, nets, case.B, S)
    hp = hparams(case, delay)
    outs = []
    for c in range(calls):  # the second call replays the captured graph
        table, idx, noise = data[c]
        if gather:
            dev = [torch.as_tensor(table[k], device="cuda") for k in
                   ("observations", "actions", "rewards", "next_observations", "dones")]
            outs.append(e.train_gather(hp, dev, len(table["rewards"]), idx, noise))
        else:
            cols = [np.ascontiguousarray(table[k][idx]) for k in
                    ("observations", "actions", "rewards", "next_observations", "dones")]
            outs.append(e.train(hp, *cols, noise))
    blob, steps = e.get_state()
    e.close()
    return outs, blob.copy(), steps


@pytest.mark.parametrize("delay", [2, 3])
@pytest.mark.parametrize("name", ["td3_paper", "deep", "mixed_depth"])
def test_execution_paths_are_bit_identical(name, delay):
    """Host-staged plain launches, the CUDA graph and the device gather give identical outputs and networks over S = 5
    steps with a delayed policy step, at shapes whose GEMMs need several prefetch rounds (K = 400, B = 257) and with
    4-layer / mixed-depth networks."""
    case = CASES[name]
    S = 5
    rng = np.random.default_rng(11)
    nets = init_nets(case, rng)
    data = []
    for _ in range(2):
        table, _ = draw_rows(case, rng, S * case.B + 7)
        idx = rng.integers(0, S * case.B + 7, (S, case.B))
        noise = rng.standard_normal((S, case.B, case.A)).astype(np.float32) if case.algo == "td3" else None
        data.append((table, idx, noise))
    try:
        ref_outs, ref_blob, ref_steps = run_path(case, nets, delay, "0", False, data, S)
        assert len(ref_outs[0]["policy_losses"]) == (S + delay - 1) // delay
        for path, (graph, gather) in PATHS.items():
            outs, blob, steps = run_path(case, nets, delay, graph, gather, data, S)
            for c, (a, b) in enumerate(zip(outs, ref_outs)):
                assert a.keys() == b.keys()
                for k in a:
                    np.testing.assert_array_equal(a[k], b[k], err_msg=f"{name} delay={delay} {path} call {c}: {k}")
            assert steps == ref_steps
            np.testing.assert_array_equal(blob, ref_blob, err_msg=f"{name} delay={delay} {path}: networks / Adam")
    finally:
        os.environ.pop("B200RL_OFFPOLICY_GRAPH", None)


@pytest.mark.parametrize("graph", ["0", "1"])
def test_shape_change_on_a_live_engine_matches_a_fresh_engine(graph):
    """An engine keeps its workspace across calls while max_minibatch >= B, and recaptures its graph when B changes:
    B = 256, then 100, then 256 again on one engine gives, call by call, what a fresh engine of exactly that B gives
    from the same state.  With plain launches and with the graph."""
    case = CASES["td3_paper"]
    S = 3
    rng = np.random.default_rng(13)
    nets = init_nets(case, rng)
    try:
        os.environ["B200RL_OFFPOLICY_GRAPH"] = graph
        live = make_engine(case, nets, 256, S)
        hp = hparams(case, 2)
        for B in (256, 100, 256):
            table, _ = draw_rows(case, rng, S * B)
            cols = [table[k].reshape((S, B) + table[k].shape[1:]) for k in
                    ("observations", "actions", "rewards", "next_observations", "dones")]
            noise = rng.standard_normal((S, B, case.A)).astype(np.float32)
            blob, steps = live.get_state()
            blob = blob.copy()
            got = live.train(hp, *cols, noise)
            got_blob = live.get_state()[0].copy()
            fresh = make_engine(case, nets, B, S)
            fresh.set_state(blob, steps)
            want = fresh.train(hp, *cols, noise)
            for k in want:
                np.testing.assert_array_equal(got[k], want[k], err_msg=f"B={B} graph={graph}: {k}")
            np.testing.assert_array_equal(got_blob, fresh.get_state()[0], err_msg=f"B={B} graph={graph}: state")
            fresh.close()
        live.close()
    finally:
        os.environ.pop("B200RL_OFFPOLICY_GRAPH", None)
