"""float64 one-step reference of the off-policy engine (TD3 / DDPG and SAC).  TEST INFRASTRUCTURE ONLY -- see
oracle/__init__.py.

torch autograd in float64 on the CPU.  One train step is split into stages, and every stage takes its inputs as
arguments, so a test can feed each stage the engine's own inputs to it (the policy stage takes the critics' post-step
parameters read back from the engine): errors of one stage never reach the next, and nothing compounds over Adam steps.
A float64 reference does not share the kernels' float32 rounding, so a kernel error a float32 oracle would reproduce or
blur shows up here.

* ``td3_critic_stage`` / ``td3_policy_stage``: TD3 (ref: algorithms/td3.py:214-358) and DDPG (``twin=False``, no noise).
* ``sac_critic_stage`` / ``sac_policy_stage``: SAC as oracle/sac.py states it (``squash`` below).
* ``adam_update_f32`` / ``polyak_f32``: the elementwise steps restated in float32 with the kernels' operation order,
  including the multiply-adds nvcc contracts into one FMA (adam.cu adam_step_kernel, offpolicy.cu polyak_kernel).

Networks are flat float32 vectors in torch's parameters_to_vector order (W0 [out, in], b0, W1, b1, ...).  Every forward
pass also returns, per row, the smallest relative ReLU margin |z| / (sum_k |x_k w_k| + |b|) over its ReLU units: a row
whose margin is at rounding level may be gated differently by a float32 kernel, which is not an error of the kernel.
"""
from __future__ import annotations

import math
from typing import Dict, Sequence

import numpy as np
import torch
import torch.nn.functional as F

D = torch.float64
F32 = np.float32
_ACT = {"identity": lambda z: z, "tanh": torch.tanh, "relu": torch.relu}


def _t(x, grad=False):
    t = torch.as_tensor(np.asarray(x, dtype=np.float64))
    return t.clone().requires_grad_(True) if grad else t


def mlp(flat: torch.Tensor, sizes: Sequence[int], x: torch.Tensor, hidden: str, out: str):
    """(output, per-row smallest relative ReLU margin; +inf without ReLU units)"""
    L, o, h = len(sizes) - 1, 0, x
    margin = torch.full((x.shape[0],), math.inf, dtype=D)
    for l in range(L):
        n_in, n_out = sizes[l], sizes[l + 1]
        W = flat[o:o + n_out * n_in].view(n_out, n_in)
        o += n_out * n_in
        b = flat[o:o + n_out]
        o += n_out
        z = h @ W.T + b
        kind = out if l == L - 1 else hidden
        if kind == "relu":
            with torch.no_grad():
                scale = h.detach().abs() @ W.detach().abs().T + b.detach().abs()
                margin = torch.minimum(margin, (z.detach().abs() / scale.clamp_min(1e-300)).min(dim=1).values)
        h = _ACT[kind](z)
    assert o == flat.numel()
    return h, margin


def squash(out: torch.Tensor, eps: torch.Tensor, limit: float, log_std_min: float, log_std_max: float):
    """(limit * tanh(u), log pi) of oracle/sac.py's squash, u = mu + sigma eps, with Normal(mu, sigma).log_prob(u)
    written as -eps^2 / 2 - log sigma - log sqrt(2 pi): the same function, since (u - mu) / sigma = eps.  Autograd of
    the textbook form subtracts mu from u and divides by sigma^2, which at sigma = exp(-20) turns rounding of u into
    gradient terms of order 1e9 even in float64."""
    A = out.shape[-1] // 2
    mu, log_std = out[..., :A], torch.clamp(out[..., A:], log_std_min, log_std_max)
    u = mu + eps * torch.exp(log_std)
    logp = (-0.5 * eps ** 2 - log_std - 0.5 * math.log(2 * math.pi)).sum(-1)
    logp = logp - (2 * (math.log(2) - u - F.softplus(-2 * u))).sum(-1)
    return limit * torch.tanh(u), logp


def _grad(loss, flat):
    (g,) = torch.autograd.grad(loss, flat)
    return g.numpy()


def _critic_step(q_flats, q_sizes, q_hidden, obs, act, y):
    """MSE of each critic on [s | a] against y (F.mse_loss) and its gradient."""
    out = dict(q_values=[], losses=[], grads=[])
    margin = torch.full((obs.shape[0],), math.inf, dtype=D)
    for qf in q_flats:
        p = _t(qf, grad=True)
        q, m = mlp(p, q_sizes, torch.cat([obs, act], -1), q_hidden, "identity")
        margin = torch.minimum(margin, m)
        loss = ((q[:, 0] - y) ** 2).mean()
        out["q_values"].append(q[:, 0].detach().numpy())
        out["losses"].append(float(loss.detach()))
        out["grads"].append(_grad(loss, p))
    return out, margin


def td3_critic_stage(nets: Dict[str, np.ndarray], mb: Dict[str, np.ndarray], noise, policy_sizes, q_sizes,
                     p_hidden="relu", q_hidden="relu", gamma=0.99, noise_scale=0.2, noise_clip=0.5, action_limit=1.0):
    """The critic step of TD3 (critics q1, q2) or DDPG (q1 only; noise None): the smoothed and clamped target action,
    y = r + gamma (1 - d) min(Q1targ, Q2targ)(s', a'), each critic's Q-values on [s | a], loss and gradient.
    ``margin``: per row, over every forward pass of the stage (all depend only on the step's inputs)."""
    twin = "q2" in nets
    obs, act, rew = _t(mb["observations"]), _t(mb["actions"]), _t(mb["rewards"])
    nobs, done = _t(mb["next_observations"]), _t(np.asarray(mb["dones"], dtype=np.float64))
    a2, margin = mlp(_t(nets["target_policy"]), policy_sizes, nobs, p_hidden, "tanh")
    if noise is not None:
        eps = torch.clamp(noise_scale * _t(noise), -noise_clip, noise_clip)
        a2 = torch.clamp(a2 + eps, -action_limit, action_limit)
    tq = None
    for name in ["target_q1"] + (["target_q2"] if twin else []):
        q, m = mlp(_t(nets[name]), q_sizes, torch.cat([nobs, a2], -1), q_hidden, "identity")
        margin = torch.minimum(margin, m)
        tq = q[:, 0] if tq is None else torch.minimum(tq, q[:, 0])
    y = rew + gamma * (1 - done) * tq
    out, m = _critic_step([nets["q1"]] + ([nets["q2"]] if twin else []), q_sizes, q_hidden, obs, act, y)
    out.update(target_action=a2.numpy(), y=y.numpy(), margin=torch.minimum(margin, m).numpy())
    return out


def td3_policy_stage(policy: np.ndarray, q1: np.ndarray, obs, policy_sizes, q_sizes, p_hidden="relu", q_hidden="relu"):
    """-mean(Q1(s, pi(s))) with the critic's parameters frozen, and its gradient w.r.t. the policy.  ``q1`` is the
    critic AFTER this step's critic update (td3.py:309).  margin_pi: the policy pass (depends on the step's inputs
    only); margin_q: the critic pass on [s | pi(s)] (depends on the critic update)."""
    obs = _t(obs)
    p = _t(policy, grad=True)
    a, margin_pi = mlp(p, policy_sizes, obs, p_hidden, "tanh")
    q, margin_q = mlp(_t(q1), q_sizes, torch.cat([obs, a], -1), q_hidden, "identity")
    loss = -q[:, 0].mean()
    return dict(loss=float(loss.detach()), grad=_grad(loss, p), margin_pi=margin_pi.numpy(), margin_q=margin_q.numpy())


def sac_critic_stage(nets: Dict[str, np.ndarray], mb: Dict[str, np.ndarray], eps_next, alpha: float, policy_sizes,
                     q_sizes, hidden="relu", gamma=0.99, action_limit=1.0, log_std_min=-20.0, log_std_max=2.0):
    """The SAC critic step: a', log pi(a' | s') from the current policy and the draw ``eps_next``,
    y = r + gamma (1 - d) (min(Q1targ, Q2targ)(s', a') - alpha log pi(a' | s')), each critic's Q-values, loss and
    gradient.  ``margin``: per row, over every forward pass of the stage."""
    obs, act, rew = _t(mb["observations"]), _t(mb["actions"]), _t(mb["rewards"])
    nobs, done = _t(mb["next_observations"]), _t(np.asarray(mb["dones"], dtype=np.float64))
    out2, margin = mlp(_t(nets["policy"]), policy_sizes, nobs, hidden, "identity")
    a2, logp2 = squash(out2, _t(eps_next), action_limit, log_std_min, log_std_max)
    tq = None
    for name in ("target_q1", "target_q2"):
        q, m = mlp(_t(nets[name]), q_sizes, torch.cat([nobs, a2], -1), hidden, "identity")
        margin = torch.minimum(margin, m)
        tq = q[:, 0] if tq is None else torch.minimum(tq, q[:, 0])
    y = rew + gamma * (1 - done) * (tq - alpha * logp2)
    out, m = _critic_step([nets["q1"], nets["q2"]], q_sizes, hidden, obs, act, y)
    out.update(y=y.numpy(), logp_next=logp2.numpy(), margin=torch.minimum(margin, m).numpy())
    return out


def sac_policy_stage(policy: np.ndarray, q1: np.ndarray, q2: np.ndarray, obs, eps_cur, alpha: float, policy_sizes,
                     q_sizes, hidden="relu", action_limit=1.0, log_std_min=-20.0, log_std_max=2.0, target_entropy=None):
    """mean(alpha log pi - min(Q1, Q2)(s, a_pi)) with the critics AFTER this step's update, frozen; its gradient
    w.r.t. the policy; mean log pi; and the temperature's gradient -mean(log pi + target_entropy) w.r.t. log_alpha."""
    obs = _t(obs)
    p = _t(policy, grad=True)
    out, margin_pi = mlp(p, policy_sizes, obs, hidden, "identity")
    a, logp = squash(out, _t(eps_cur), action_limit, log_std_min, log_std_max)
    margin_q = torch.full((obs.shape[0],), math.inf, dtype=D)
    qs = []
    for qf in (q1, q2):
        q, m = mlp(_t(qf), q_sizes, torch.cat([obs, a], -1), hidden, "identity")
        qs.append(q[:, 0])
        margin_q = torch.minimum(margin_q, m.detach())
    loss = (alpha * logp - torch.minimum(qs[0], qs[1])).mean()
    te = -float(a.shape[-1]) if target_entropy is None else float(target_entropy)
    return dict(loss=float(loss.detach()), grad=_grad(loss, p), logp_mean=float(logp.detach().mean()),
                alpha_grad=float(-(logp.detach() + te).mean()), logp=logp.detach().numpy(),
                margin_pi=margin_pi.numpy(), margin_q=margin_q.numpy())


# ---- elementwise steps, float32 --------------------------------------------------------------------------------------
def fma_f32(a, b, c) -> np.ndarray:
    """a * b + c rounded once to float32 (a CUDA FFMA).  a * b of two float32 values is exact in float64; the sum is
    rounded to float64 and then to float32, which can only err when the float64 sum lands exactly halfway between two
    float32 values: those elements are rounded towards the exact sum's side, known from the sum's exact error term."""
    a, b, c = (np.asarray(x, dtype=F32).astype(np.float64) for x in (a, b, c))
    p = a * b
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)  # s + err == p + c exactly (TwoSum)
    r = s.astype(F32)
    rd = r.astype(np.float64)
    diff = s - rd
    nb = np.nextafter(r, np.where(diff > 0, np.inf, -np.inf).astype(F32)).astype(np.float64)
    fix = (diff != 0) & (2 * diff == nb - rd) & (err != 0) & (np.sign(err) == np.sign(diff))
    return np.where(fix, nb.astype(F32), r)


def adam_scalars(step: int, lr: float, beta1: float, beta2: float):
    """{lr / (1 - beta1^t), sqrt(1 - beta2^t)} in float32, as adam.cu's adam_scalars casts torch's host arithmetic."""
    return F32(lr / (1.0 - beta1 ** step)), F32(math.sqrt(1.0 - beta2 ** step))


def adam_moments_f32(g, m, v, beta1=0.9, beta2=0.999):
    """exp_avg = fma(g - m, 1 - b1, m); exp_avg_sq = fma(v, b2, (1 - b2) * (g * g))."""
    g, m, v = (np.asarray(x, dtype=F32) for x in (g, m, v))
    return fma_f32(g - m, F32(1.0 - beta1), m), fma_f32(v, F32(beta2), F32(1.0 - beta2) * (g * g))


def adam_update_f32(p, m, v, step: int, lr: float, beta1=0.9, beta2=0.999, eps=1e-8):
    """The parameter update from the NEW moments: p - step_size * (m / (sqrt(v) / bc2_sqrt + eps)), the last
    multiply-subtract one FMA."""
    step_size, bc2 = adam_scalars(step, lr, beta1, beta2)
    m, v = np.asarray(m, dtype=F32), np.asarray(v, dtype=F32)
    denom = np.sqrt(v) / bc2 + F32(eps)
    return fma_f32(m / denom, -step_size, p)


def polyak_f32(target, param, rho: float):
    """rho * target + (1 - rho) * param as polyak_kernel computes it: fma(rho, target, (1 - rho) * param)."""
    return fma_f32(F32(rho), target, F32(1.0 - rho) * np.asarray(param, dtype=F32))
