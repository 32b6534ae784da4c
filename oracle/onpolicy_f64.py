"""float64 one-step reference of the on-policy kernels (PPO / VPG / TRPO losses, value MSE, evaluation, forward-only
passes with the true KL, and the Fisher-vector product).  TEST INFRASTRUCTURE ONLY -- see oracle/__init__.py.

torch autograd in float64 on the CPU, shaped like oracle/offpolicy_f64.py.  Every function takes its inputs as
arguments -- old log-probs, raw advantages with their statistics, returns -- so a test can hand it the engine's own
inputs, and every gradient comes back split into its W and b tensors.  A float64 reference does not share the kernels'
float32 rounding (oracle/onpolicy.py does), so a kernel error that a float32 oracle would reproduce or blur shows here.

* ``policy_loss``: PPO clip (ref: algorithms/ppo.py:237-257, written with torch.min / torch.clamp like the reference, so
  torch's tie and boundary rules apply), VPG (vpg.py:200-203), TRPO surrogate (trpo.py:154-165), and evaluation
  (per-row log pi; sums of entropy, log pi, log pi^2).  Gaussian policies with a state-independent log_std, optionally
  trained (its gradient is returned separately), and categorical policies.
* ``value_loss``: F.mse_loss of the value head (ppo.py:282-287).
* ``forward_kl``: raw outputs and the true KL(old || new) per row (trpo.py:167-175).
* ``fvp``: the Fisher-vector product the way the reference forms it: double backprop of the mean KL(old || new) with the
  old distribution detached (conjugate_gradient_optimizer.py:133-167), at damping 0.
* ``gae_scan``: returns and GAE advantages before their float32 cast, with their conditioning scales (numpy / scipy).

Every gradient also comes with its scale: per entry, the sum over rows of the magnitudes of the rows' contributions.
Where those contributions cancel, a float32 sum over rows is only accurate to ~2^-24 of that scale, not of the result,
so a kernel's gradient error is measured against it (the way a loss sum is measured against the sum of |term|).

Advantages are normalised exactly as the kernels read them (utils.py:90-92): mean and UNBIASED std from
``adv_stats`` = [sum, sum of squares, count], no epsilon.  Networks are flat float32 vectors in torch's
parameters_to_vector order (W0 [out, in], b0, W1, b1, ...); ``mlp`` also reports the smallest relative ReLU margin per
row (see offpolicy_f64.mlp).
"""
from __future__ import annotations

import math
from typing import Dict, List, Sequence

import numpy as np
import torch
from torch.distributions import Categorical, Normal, kl_divergence

from oracle.offpolicy_f64 import _ACT, _t, mlp

LOSSES = ("eval", "ppo_clip", "vpg", "trpo_surrogate")


def tensor_names(sizes: Sequence[int]) -> List[str]:
    return [f"{k}{l}" for l in range(len(sizes) - 1) for k in ("W", "b")]


def split(flat, sizes: Sequence[int]) -> Dict[str, np.ndarray]:
    """flat parameter-order vector -> {"W0": [out, in], "b0": [out], ...}"""
    flat = np.asarray(flat)
    out, o = {}, 0
    for l in range(len(sizes) - 1):
        n_in, n_out = sizes[l], sizes[l + 1]
        out[f"W{l}"] = flat[o:o + n_out * n_in].reshape(n_out, n_in)
        o += n_out * n_in
        out[f"b{l}"] = flat[o:o + n_out]
        o += n_out
    assert o == flat.size, (o, flat.size)
    return out


def _forward(p: torch.Tensor, sizes: Sequence[int], x: torch.Tensor, hidden: str):
    """offpolicy_f64.mlp with an identity output that also returns every layer's (pre-activation z, input h), so the
    per-row contributions to each gradient entry can be formed from dLoss/dz."""
    L, o, h = len(sizes) - 1, 0, x
    margin = torch.full((x.shape[0],), math.inf, dtype=torch.float64)
    layers = []
    for l in range(L):
        n_in, n_out = sizes[l], sizes[l + 1]
        W = p[o:o + n_out * n_in].view(n_out, n_in)
        o += n_out * n_in
        b = p[o:o + n_out]
        o += n_out
        z = h @ W.T + b
        layers.append((z, h))
        kind = "identity" if l == L - 1 else hidden
        if kind == "relu":
            with torch.no_grad():
                scale = h.detach().abs() @ W.detach().abs().T + b.detach().abs()
                margin = torch.minimum(margin, (z.detach().abs() / scale.clamp_min(1e-300)).min(dim=1).values)
        h = _ACT[kind](z)
    assert o == p.numel()
    return h, margin, layers


def _grad_scales(dzs, layers, sizes) -> np.ndarray:
    """Per gradient entry, the sum over rows of the magnitudes of the rows' contributions: |dz|^T |h| for W, sum |dz|
    for b (flat parameter order).  A float32 sum over rows cannot be trusted to better than ~2^-24 of this, however
    much the contributions cancel, so it is the scale a kernel's gradient error is measured against."""
    out = []
    for dz, (_, h) in zip(dzs, layers):
        out += [(dz.abs().T @ h.detach().abs()).reshape(-1), dz.abs().sum(0)]
    return torch.cat(out).numpy()


def normalized_advantages(adv_raw, adv_stats) -> torch.Tensor:
    """(adv - mean) / std with mean = s1 / n and the unbiased std sqrt((s2 - n mean^2) / (n - 1)); adv_stats None: the
    raw advantages as they are."""
    a = _t(adv_raw)
    if adv_stats is None:
        return a
    s1, s2, n = (float(x) for x in adv_stats)
    mean = s1 / n
    return (a - mean) / math.sqrt((s2 - n * mean * mean) / (n - 1.0))


def _dist(kind: str, out: torch.Tensor, log_std: torch.Tensor | None):
    if kind == "gaussian":
        return Normal(out, torch.exp(log_std).expand_as(out))
    return Categorical(logits=out)


def _log_prob(kind, d, act):
    if kind == "gaussian":
        return d.log_prob(_t(act)).sum(-1)
    return d.log_prob(torch.as_tensor(np.asarray(act)).long())


def _entropy(kind, d):
    return d.entropy().sum(-1) if kind == "gaussian" else d.entropy()


def policy_loss(flat, sizes, obs, act, dist: str, loss: str, log_std=None, adv_raw=None, adv_stats=None,
                old_logp=None, clip: float = 0.2, hidden: str = "tanh", n_global: int | None = None):
    """One policy launch.  Returns dict with
    grad (flat), grads ({"W0": ..}), scales ({"W0": ..}: per entry the sum over rows of |contribution|, see
    _grad_scales), grad_log_std and scale_log_std ([A], Gaussian), logp (per row), ratio (PPO / TRPO), margin (ReLU),
    and the kernels' scalar sums: loss_sum (sum of the per-row loss terms; the loss is loss_sum / n_global), kl_sum
    (sum of old_logp - logp), entropy_sum, logp_sum, logp2_sum; loss_abs_sum and logp_abs_sum (sums of |term| and
    |logp|, the scale of a float32 kernel's rounding in loss_sum, kl_sum and logp_sum)."""
    p = _t(flat, grad=True)
    ls = _t(log_std, grad=True) if dist == "gaussian" else None
    x = _t(obs)
    out, margin, layers = _forward(p, sizes, x, hidden)
    lsr = ls.expand(out.shape) if ls is not None else None  # one row of log_std per row: per-row contributions
    d = _dist(dist, out, lsr)
    logp = _log_prob(dist, d, act)
    n = x.shape[0] if n_global is None else n_global
    res = dict(margin=margin.numpy())
    if loss == "eval":
        terms = torch.zeros_like(logp)
    else:
        adv = normalized_advantages(adv_raw, adv_stats)
        if loss == "vpg":
            terms = -(logp * adv)
        else:
            ratio = torch.exp(logp - _t(old_logp))
            res["ratio"] = ratio.detach().numpy()
            if loss == "ppo_clip":  # ppo.py:245-255
                terms = -torch.min(ratio * adv, torch.clamp(ratio, 1.0 - clip, 1.0 + clip) * adv)
            elif loss == "trpo_surrogate":
                terms = -(ratio * adv)
            else:
                raise ValueError(loss)
        zs = [z for z, _ in layers]
        g = torch.autograd.grad(terms.sum() / n, [p] + zs + ([ls, lsr] if ls is not None else []))
        res["grad"] = g[0].numpy()
        res["grads"] = split(res["grad"], sizes)
        res["scales"] = split(_grad_scales(g[1:1 + len(zs)], layers, sizes), sizes)
        if ls is not None:
            res["grad_log_std"] = g[-2].numpy()
            res["scale_log_std"] = g[-1].abs().sum(0).numpy()
    logp = logp.detach()
    terms = terms.detach()
    res.update(logp=logp.numpy(), loss_sum=float(terms.sum()), entropy_sum=float(_entropy(dist, d).detach().sum()),
               logp_sum=float(logp.sum()), logp2_sum=float((logp ** 2).sum()),
               # the scale of each sum's float32 rounding: the sums of the magnitudes of their terms
               loss_abs_sum=float(terms.abs().sum()), logp_abs_sum=float(logp.abs().sum()))
    if old_logp is not None:
        res["kl_sum"] = float((_t(old_logp) - logp).sum())
    return res


def value_loss(flat, sizes, obs, ret, hidden: str = "tanh", n_global: int | None = None):
    """mean((V(s) - ret)^2) and its gradient: dict(grad, grads, scales (as policy_loss), values, loss_sum = sum of
    squared errors, margin)."""
    p = _t(flat, grad=True)
    out, margin, layers = _forward(p, sizes, _t(obs), hidden)
    v = out[:, 0]
    n = v.shape[0] if n_global is None else n_global
    sq = (v - _t(ret)) ** 2
    g = torch.autograd.grad(sq.sum() / n, [p] + [z for z, _ in layers])
    return dict(grad=g[0].numpy(), grads=split(g[0].numpy(), sizes), scales=split(_grad_scales(g[1:], layers, sizes), sizes),
                values=v.detach().numpy(), loss_sum=float(sq.detach().sum()), margin=margin.numpy())


def values(flat, sizes, obs, hidden: str = "tanh"):
    """V(s) per row (the EVAL launch of a value head)."""
    with torch.no_grad():
        return mlp(_t(flat), sizes, _t(obs), hidden, "identity")[0][:, 0].numpy()


def forward_kl(flat, sizes, obs, dist: str, old_out, log_std=None, hidden: str = "tanh"):
    """Raw outputs of the network and kl_divergence(old_dist, dist) per row (Gaussian: the same log_std for both)."""
    with torch.no_grad():
        out = mlp(_t(flat), sizes, _t(obs), hidden, "identity")[0]
        ls = _t(log_std) if dist == "gaussian" else None
        kl = kl_divergence(_dist(dist, _t(old_out), ls), _dist(dist, out, ls))
        if dist == "gaussian":
            kl = kl.sum(-1)
    return dict(out=out.numpy(), kl=kl.numpy())


def fvp(flat, sizes, obs, dist: str, v, log_std=None, hidden: str = "tanh"):
    """F v at damping 0: the gradient of (grad mean KL(old || new)) . v, old = the network at ``flat``, detached.
    Returns dict(fvp (flat), tensors ({"W0": ..}))."""
    p = _t(flat, grad=True)
    x = _t(obs)
    out = mlp(p, sizes, x, hidden, "identity")[0]
    ls = _t(log_std) if dist == "gaussian" else None
    kl = kl_divergence(_dist(dist, out.detach(), ls), _dist(dist, out, ls))
    if dist == "gaussian":
        kl = kl.sum(-1)
    (g,) = torch.autograd.grad(kl.mean(), p, create_graph=True)
    (hv,) = torch.autograd.grad((g * _t(v)).sum(), p)
    hv = hv.numpy()
    return dict(fvp=hv, tensors=split(hv, sizes))


def fvp_explicit(flat, sizes, obs, dist: str, v, log_std=None, hidden: str = "tanh") -> np.ndarray:
    """(1/N) sum_i J_i^T M_i J_i v with the Jacobian of every row's outputs formed explicitly and the metric written
    out (Gaussian: diag(1 / var); categorical: diag(p) - p p^T).  Independent of double backprop; tiny networks only."""
    x = _t(obs)
    p0 = _t(flat)
    f = lambda q: mlp(q, sizes, x, hidden, "identity")[0]
    out = f(p0)
    J = torch.autograd.functional.jacobian(f, p0)  # [N, A, P]
    N, A = out.shape
    if dist == "gaussian":
        M = torch.diag_embed((1.0 / torch.exp(2 * _t(log_std))).expand(N, A))
    else:
        pr = torch.softmax(out, -1)
        M = torch.diag_embed(pr) - pr[:, :, None] * pr[:, None, :]
    Jv = J @ _t(v)
    return (torch.einsum("nap,nab,nb->p", J, M, Jv) / N).numpy()


def clip_margin(ratio, clip: float = 0.2) -> np.ndarray:
    """Per row, the distance of the PPO ratio from the nearer clip bound, relative to that bound: rows within float32
    rounding of a bound may be clipped differently by a float32 kernel, which is not an error of the kernel."""
    r = np.asarray(ratio, dtype=np.float64)
    return np.minimum(np.abs(r - (1.0 - clip)) / (1.0 - clip), np.abs(r - (1.0 + clip)) / (1.0 + clip))


def _segmented_reverse_scan(x: np.ndarray, off: np.ndarray, lens: np.ndarray, a: float) -> np.ndarray:
    """y_i = x_i + a * y_{i+1} inside every episode, y = 0 past its end, in float64 (lfilter, ref: utils.py:28).
    Episodes of one length run as one [episodes, length] block, so a batch of millions of items takes seconds."""
    from scipy.signal import lfilter
    y = np.empty_like(x)
    order = np.argsort(lens, kind="stable")
    for grp in np.split(order, np.flatnonzero(np.diff(lens[order])) + 1):
        L = int(lens[grp[0]])
        idx = off[grp][:, None] + np.arange(L)[None, :]
        y[idx] = lfilter([1.0], [1.0, -a], x[idx][:, ::-1], axis=1)[:, ::-1]
    return y


def gae_scan(rewards, values, last_values, ep_offsets, ep_done, gamma: float, lam: float):
    """Returns and GAE advantages of a packed batch, UNROUNDED float64 (oracle/onpolicy.py's gae_and_returns before its
    final cast), with a conditioning scale per output.  The two float32 details of the reference are kept:
      delta_i = (r_i + f32(f32(gamma) * v_{i+1})) - v_i,  with v_L = V(last_obs) on the last step even when done;
      the return of the last step adds gamma * V(last_obs), in float64, only when the episode is not done.
    The scales S_adv / S_ret run the same recurrences over the magnitudes of every term (|r| + |f32 product| + |v| and
    |r| + |gamma * V_L|, coefficients |gamma * lam| and |gamma|): float64 reassociation of a scan is accurate to a few
    ulp of S, not of the result.  Returns (adv64, ret64, S_adv, S_ret), each [N] float64."""
    off = np.asarray(ep_offsets, dtype=np.int64)
    lens = np.diff(off)
    n = int(off[-1])
    r = np.asarray(rewards, dtype=np.float64)
    v = np.asarray(values, dtype=np.float32)
    lv = np.asarray(last_values, dtype=np.float32)
    last = off[1:] - 1
    vnext = np.empty(n, dtype=np.float32)
    vnext[:-1] = v[1:]
    vnext[last] = lv
    prod = (np.float32(gamma) * vnext).astype(np.float64)  # float32 product, exactly rounded
    delta = (r + prod) - v.astype(np.float64)
    boot = np.where(np.asarray(ep_done, dtype=bool), 0.0, gamma * lv.astype(np.float64))
    rb = r.copy()
    rb[last] += boot
    rb_abs = np.abs(r)
    rb_abs[last] += np.abs(boot)
    gl = gamma * lam
    adv = _segmented_reverse_scan(delta, off, lens, gl)
    ret = _segmented_reverse_scan(rb, off, lens, gamma)
    s_adv = _segmented_reverse_scan(np.abs(r) + np.abs(prod) + np.abs(v.astype(np.float64)), off, lens, abs(gl))
    s_ret = _segmented_reverse_scan(rb_abs, off, lens, abs(gamma))
    return adv, ret, s_adv, s_ret
