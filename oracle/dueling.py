"""float64 one-step references of dueling DQN, C51 and QR-DQN.  TEST INFRASTRUCTURE ONLY -- see oracle/__init__.py.

* ``dueling_mlp``: the dueling Q network (include/b200rl.h, "Dueling Q networks") in float64 from a flat parameter
  vector in parameters_to_vector order (trunk, value hidden, value out, advantage hidden, advantage out, each [W, b]),
  returning, like oracle/offpolicy_f64.mlp, the per-row smallest relative ReLU margin over its ReLU units.
* ``dqn_step_f64`` / ``c51_step_f64`` / ``qr_step_f64``: the steps of oracle/dqn.py, oracle/c51.py and oracle/qr.py
  with this network in place of the plain MLP: the same heads (td_values, project, quantile_huber), the same returned
  fields, and per-entry gradient scales (per row, vmapped) that cover the five layers.

The float32 oracles (DqnOracle, C51Oracle, QrDqnOracle) take a DuelingMLP as they are: they deep-copy the torch module.
"""
from __future__ import annotations

import math
from typing import Dict, Sequence

import numpy as np
import torch
import torch.nn.functional as F

from .c51 import _log_dist, project, support
from .dqn import huber_f64, td_values
from .offpolicy_f64 import _ACT, D, _t
from .qr import _quantiles, quantile_huber, taus


def _dueling_layers(flat: torch.Tensor, sizes: Sequence[int], k: int):
    """[(W, b)] of trunk, value hidden, value out, advantage hidden, advantage out; sizes = [obs, h1, h2, n k]."""
    O, h1, h2, nk = sizes
    out, o = [], 0
    for n_in, n_out in ((O, h1), (h1, h2), (h2, k), (h1, h2), (h2, nk)):
        W = flat[o:o + n_out * n_in].view(n_out, n_in)
        o += n_out * n_in
        out.append((W, flat[o:o + n_out]))
        o += n_out
    assert o == flat.numel()
    return out


def _relu_margin(h, W, b, z):
    scale = h.detach().abs() @ W.detach().abs().T + b.detach().abs()
    return (z.detach().abs() / scale.clamp_min(1e-300)).min(dim=1).values


def dueling_mlp(flat: torch.Tensor, sizes: Sequence[int], k: int, x: torch.Tensor, hidden: str = "relu",
                margins: bool = True):
    """(Q [B, n k], per-row smallest relative ReLU margin; +inf without ReLU units): h = act(x W1^T + b1),
    V = act(h Wv^T + bv) Vo^T + vo, A = act(h Wa^T + ba) Ao^T + ao, Q[a, i] = V[i] + (A[a, i] - mean_b A[b, i])."""
    (W1, b1), (Wv, bv), (Vo, vo), (Wa, ba), (Ao, ao) = _dueling_layers(flat, sizes, k)
    act = _ACT[hidden]
    margin = torch.full((x.shape[0],), math.inf, dtype=D)
    z1 = x @ W1.T + b1
    h = act(z1)
    zv, za = h @ Wv.T + bv, h @ Wa.T + ba
    if margins and hidden == "relu":
        with torch.no_grad():
            for inp, W, b, z in ((x, W1, b1, z1), (h, Wv, bv, zv), (h, Wa, ba, za)):
                margin = torch.minimum(margin, _relu_margin(inp, W, b, z))
    v = (act(zv) @ Vo.T + vo).unflatten(-1, (1, k))
    a = (act(za) @ Ao.T + ao).unflatten(-1, (-1, k))
    return (v + (a - a.mean(dim=-2, keepdim=True))).flatten(-2), margin


def _per_row_scale(p, obs, sizes, k, hidden, row_fn, *aux):
    """Per entry, the sum over rows of |that row's gradient contribution|; row_fn(q_row [n k], *aux_row) is the row's
    share of the loss."""
    def one(flat_p, o, *a):
        q, _ = dueling_mlp(flat_p, sizes, k, o[None], hidden, margins=False)
        return row_fn(q[0], *a)
    per_row = torch.func.vmap(torch.func.grad(one), in_dims=(None, 0) + (0,) * len(aux))(p.detach(), obs, *aux)
    return per_row.abs().sum(0)


def _inputs(mb):
    obs, act, rew = _t(mb["observations"]), np.asarray(mb["actions"]).reshape(-1), _t(mb["rewards"])
    nobs, done = _t(mb["next_observations"]), _t(np.asarray(mb["dones"], dtype=np.float64))
    return obs, torch.as_tensor(act.astype(np.int64)), rew, nobs, done


def _gap(values):
    """Per row, the two largest values apart (+inf for one column)."""
    if values.shape[1] < 2:
        return torch.full((values.shape[0],), math.inf, dtype=D)
    top2 = values.topk(2, dim=1).values
    return top2[:, 0] - top2[:, 1]


def dqn_step_f64(q_flat, targ_flat, mb: Dict[str, np.ndarray], sizes: Sequence[int], hidden="relu", gamma=0.99,
                 double_q=False):
    """oracle/dqn.dqn_step_f64 with a dueling network (k = 1): dict(q_values, loss, grad, scale, y, margin, gap, delta)."""
    obs, a, rew, nobs, done = _inputs(mb)
    B, n = obs.shape[0], sizes[-1]
    with torch.no_grad():
        qt, margin = dueling_mlp(_t(targ_flat), sizes, 1, nobs, hidden)
        gap, qn = torch.full((B,), math.inf, dtype=D), None
        if double_q:
            qn, m2 = dueling_mlp(_t(q_flat), sizes, 1, nobs, hidden)
            margin, gap = torch.minimum(margin, m2), _gap(qn)
        y = rew + gamma * (1 - done) * td_values(qt, qn, double_q)
    p = _t(q_flat, grad=True)
    q, m3 = dueling_mlp(p, sizes, 1, obs, hidden)
    q_sa = q.gather(1, a[:, None]).squeeze(1)
    delta = q_sa - y
    loss = huber_f64(delta).mean()
    (grad,) = torch.autograd.grad(loss, p)
    scale = _per_row_scale(p, obs, sizes, 1, hidden, lambda qr, ai, yi: huber_f64((qr * ai).sum() - yi) / B,
                           F.one_hot(a, n).to(D), y)
    return dict(q_values=q_sa.detach().numpy(), loss=float(loss.detach()), grad=grad.numpy(), scale=scale.numpy(),
                y=y.numpy(), margin=torch.minimum(margin, m3).numpy(), gap=gap.numpy(), delta=delta.detach().numpy())


def c51_step_f64(q_flat, targ_flat, mb: Dict[str, np.ndarray], sizes: Sequence[int], n_atoms: int, v_min: float,
                 v_max: float, hidden="relu", gamma=0.99, double_q=False):
    """oracle/c51.c51_step_f64 with a dueling network (k = n_atoms, aggregated on the logits): dict(q_values, loss,
    grad, scale, m, margin, gap)."""
    obs, a, rew, nobs, done = _inputs(mb)
    B, N = obs.shape[0], int(n_atoms)
    z = _t(support(N, v_min, v_max))
    rows = torch.arange(B)
    with torch.no_grad():
        qt, margin = dueling_mlp(_t(targ_flat), sizes, N, nobs, hidden)
        pt = _log_dist(qt, N).exp()
        pick = pt
        if double_q:
            qn, m2 = dueling_mlp(_t(q_flat), sizes, N, nobs, hidden)
            margin = torch.minimum(margin, m2)
            pick = _log_dist(qn, N).exp()
        ev = (pick * z).sum(-1)
        m = project(pt[rows, ev.argmax(1)], rew, done, z, v_min, v_max, (v_max - v_min) / (N - 1), gamma)
    p = _t(q_flat, grad=True)
    q, m3 = dueling_mlp(p, sizes, N, obs, hidden)
    logp = _log_dist(q, N)[rows, a]
    loss = -(m * logp).sum(-1).mean()
    (grad,) = torch.autograd.grad(loss, p)
    scale = _per_row_scale(p, obs, sizes, N, hidden,
                           lambda qr, ai, mi: -((ai[:, None] * _log_dist(qr, N)) * mi[None]).sum() / B,
                           F.one_hot(a, sizes[-1] // N).to(D), m)
    return dict(q_values=(logp.detach().exp() * z).sum(-1).numpy(), loss=float(loss.detach()), grad=grad.numpy(),
                scale=scale.numpy(), m=m.numpy(), margin=torch.minimum(margin, m3).numpy(), gap=_gap(ev).numpy())


def qr_step_f64(q_flat, targ_flat, mb: Dict[str, np.ndarray], sizes: Sequence[int], n_quantiles: int, hidden="relu",
                gamma=0.99, double_q=False):
    """oracle/qr.qr_step_f64 with a dueling network (k = n_quantiles, aggregated on the quantile locations); ``gamma``
    may be a float64 tensor [B] of per-row discounts: dict(q_values, loss, row_loss, grad, scale, target, margin, gap,
    u_min)."""
    obs, a, rew, nobs, done = _inputs(mb)
    B, N = obs.shape[0], int(n_quantiles)
    tau = taus(N, D)
    rows = torch.arange(B)
    with torch.no_grad():
        qt, margin = dueling_mlp(_t(targ_flat), sizes, N, nobs, hidden)
        tq = _quantiles(qt, N)
        pick = tq
        if double_q:
            qn, m2 = dueling_mlp(_t(q_flat), sizes, N, nobs, hidden)
            margin = torch.minimum(margin, m2)
            pick = _quantiles(qn, N)
        means = pick.sum(-1) / N
        g = gamma if torch.is_tensor(gamma) else torch.tensor(gamma, dtype=D)
        target = rew[:, None] + (g * (1 - done))[..., None] * tq[rows, means.argmax(1)]
    p = _t(q_flat, grad=True)
    q, m3 = dueling_mlp(p, sizes, N, obs, hidden)
    theta = _quantiles(q, N)[rows, a]
    row_loss = quantile_huber(theta, target, tau)
    loss = row_loss.mean()
    (grad,) = torch.autograd.grad(loss, p)
    with torch.no_grad():
        u = (target[:, None, :] - theta[:, :, None]).abs().reshape(B, -1)
        u_min = torch.minimum((u - 1).abs().min(1).values, u.min(1).values)
    scale = _per_row_scale(p, obs, sizes, N, hidden,
                           lambda qr, ai, ti: quantile_huber((_quantiles(qr, N) * ai[:, None]).sum(0)[None], ti[None],
                                                             tau)[0] / B,
                           F.one_hot(a, sizes[-1] // N).to(D), target)
    return dict(q_values=(theta.detach().sum(-1) / N).numpy(), loss=float(loss.detach()),
                row_loss=row_loss.detach().numpy(), grad=grad.numpy(), scale=scale.numpy(), target=target.numpy(),
                margin=torch.minimum(margin, m3).numpy(), gap=_gap(means).numpy(), u_min=u_min.numpy())
