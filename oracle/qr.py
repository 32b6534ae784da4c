"""torch-CPU oracles of QRDQN.train.  TEST INFRASTRUCTURE ONLY -- see oracle/__init__.py.

* ``QrDqnOracle``: float32, torch autograd and torch.optim.Adam, the QR-DQN update exactly as the project states it
  (include/b200rl.h): tau_i = (2i + 1) / (2N) in float32, a* = argmax of the quantile means, the target quantiles
  r + (g (1 - d)) theta_j(s', a*) from Q_targ, the quantile Huber loss (kappa = 1), DQN's target copies.  Given the
  drawn leaves' priorities and each step's beta it is the prioritized variant (importance weights, new priorities
  (L_b + eps)^alpha); a minibatch with a ``discounts`` key (oracle/nstep.py) is discounted per row.  It shares nothing
  with the CUDA kernel's hand-derived gradient.
* ``qr_step_f64``: one step in float64 from given flat parameters, with per-entry gradient scales, ReLU margins and the
  gap between the two largest quantile means of Q(s') of the net that picks a*.
* ``rho_loop_f64``: one row's loss as the paper writes it, an explicit double loop over i and j in float64, written
  independently of the tensor forms above so that both can be held against it.
"""
from __future__ import annotations

import math
from typing import Dict, List, Sequence

import numpy as np
import torch

from .dqn import DqnOracle, _layers
from .offpolicy_f64 import _ACT, D, _t, mlp


def taus(N: int, dtype=torch.float32) -> torch.Tensor:
    """tau_i = (2i + 1) / (2N): one division in ``dtype`` (float32: the engine's bits)."""
    return torch.arange(1, 2 * N, 2, dtype=dtype) / torch.tensor(2 * N, dtype=dtype)


def quantile_huber(theta: torch.Tensor, target: torch.Tensor, tau: torch.Tensor) -> torch.Tensor:
    """Per-row L [B] = (1/N) sum_i sum_j |tau_i - 1{u_ij < 0}| h(u_ij), u_ij = target_j - theta_i, h the Huber loss with
    kappa = 1; theta and target [B, N].  Autograd differentiates h only (the indicator is a constant)."""
    u = target[:, None, :] - theta[:, :, None]  # [B, i, j]
    k = (tau[None, :, None] - (u.detach() < 0).to(u.dtype)).abs()
    h = torch.where(u.abs() < 1, 0.5 * u * u, u.abs() - 0.5)
    return (k * h).sum(2).sum(1) / theta.shape[1]


def rho_loop_f64(theta, target) -> float:
    """One row's L with explicit loops: for each i, j: u = T_j - theta_i, rho = |tau_i - [u < 0]| * (u^2 / 2 if |u| < 1
    else |u| - 1/2); L = sum / N."""
    theta, target = [float(x) for x in theta], [float(x) for x in target]
    N = len(theta)
    total = 0.0
    for i in range(N):
        tau = (2 * i + 1) / (2 * N)
        for j in range(N):
            u = target[j] - theta[i]
            weight = abs(tau - (1.0 if u < 0 else 0.0))
            total += weight * (u * u / 2 if abs(u) < 1 else abs(u) - 0.5)
    return total / N


def _quantiles(x: torch.Tensor, N: int) -> torch.Tensor:
    return x.unflatten(-1, (-1, N))


class QrDqnOracle(DqnOracle):
    """DqnOracle with the quantile Huber head: ``train`` runs one QRDQN.train call; with ``leaf_priorities`` and
    ``betas`` (as oracle/per.PerDqnOracle takes them) the prioritized one."""

    def __init__(self, q, q_targ, optimizer, n_quantiles=200, alpha: float = 0.6, eps: float = 1e-6, **kw):
        super().__init__(q, q_targ, optimizer, **kw)
        self.N, self.tau = int(n_quantiles), taus(int(n_quantiles))
        self.alpha, self.eps = float(alpha), float(eps)

    def train(self, minibatches: List[dict], leaf_priorities: Sequence[np.ndarray] = None,
              betas: Sequence[float] = None) -> Dict[str, list]:
        logs = dict(q1_values=[], q1_losses=[], copied=[], row_losses=[], weights=[], priorities=[])
        t = lambda x: torch.as_tensor(np.asarray(x, dtype=np.float32))
        N = self.N
        for k, mb in enumerate(minibatches):
            o, a, r = t(mb["observations"]), t(mb["actions"]).reshape(-1).long(), t(mb["rewards"])
            o2, d = t(mb["next_observations"]), t(np.asarray(mb["dones"]).astype(np.int32))
            g = t(mb["discounts"]) if "discounts" in mb else torch.tensor(self.gamma, dtype=torch.float32)
            rows = torch.arange(o.shape[0])
            with torch.no_grad():
                tq = _quantiles(self.q_targ(o2), N)
                pick = _quantiles(self.q(o2), N) if self.double_q else tq
                a_star = (pick.sum(-1) / N).argmax(1)
                target = r[:, None] + (g * (1 - d))[..., None] * tq[rows, a_star]
            theta = _quantiles(self.q(o), N)[rows, a]
            L = quantile_huber(theta, target, self.tau)
            if leaf_priorities is not None:
                p = np.asarray(leaf_priorities[k], np.float64)
                w64 = (p.min() / p) ** float(betas[k])
                loss = (torch.as_tensor(w64.astype(np.float32)) * L).mean()
                logs["weights"].append(w64)
                logs["priorities"].append((L.detach().double().numpy() + self.eps) ** self.alpha)
            else:
                loss = L.mean()
            logs["row_losses"].append(L.detach().numpy().copy())
            self.opt.zero_grad()
            loss.backward()
            self.opt.step()
            logs["q1_values"].append((theta.detach().sum(-1) / N).numpy().copy())
            logs["q1_losses"].append(float(loss.detach()))
            copy_now = self.step_count() % self.interval == 0
            if copy_now:
                self.q_targ.load_state_dict(self.q.state_dict())
            logs["copied"].append(copy_now)
        return logs


def qr_step_f64(q_flat, targ_flat, mb: Dict[str, np.ndarray], sizes: Sequence[int], n_quantiles: int, hidden="relu",
                gamma=0.99, double_q=False):
    """One QR-DQN step's loss, logged Q(s, a) and gradient w.r.t. the Q network in float64 (tau in float64).  ``gamma``
    may be a float64 tensor [B] of per-row discounts.  Returns dict(q_values, loss, row_loss, grad (flat), scale (flat:
    per entry the sum over rows of |that row's contribution|), target [B, N], margin (per row, over every forward pass),
    gap (per row: the two largest quantile means of Q(s') of the net that picks a* apart; +inf for one action), u_min
    (per row: the smallest ||u_ij| - 1| and |u_ij|, the distance to a kink of the loss))."""
    obs, act, rew = _t(mb["observations"]), np.asarray(mb["actions"]).reshape(-1), _t(mb["rewards"])
    nobs, done = _t(mb["next_observations"]), _t(np.asarray(mb["dones"], dtype=np.float64))
    B, N = obs.shape[0], int(n_quantiles)
    tau = taus(N, D)
    rows = torch.arange(B)
    with torch.no_grad():
        qt, margin = mlp(_t(targ_flat), sizes, nobs, hidden, "identity")
        tq = _quantiles(qt, N)
        pick = tq
        if double_q:
            qn, m2 = mlp(_t(q_flat), sizes, nobs, hidden, "identity")
            margin = torch.minimum(margin, m2)
            pick = _quantiles(qn, N)
        means = pick.sum(-1) / N
        gap = torch.full((B,), math.inf, dtype=D)
        if means.shape[1] > 1:
            top2 = means.topk(2, dim=1).values
            gap = top2[:, 0] - top2[:, 1]
        g = gamma if torch.is_tensor(gamma) else torch.tensor(gamma, dtype=D)
        target = rew[:, None] + (g * (1 - done))[..., None] * tq[rows, means.argmax(1)]
    p = _t(q_flat, grad=True)
    q, m3 = mlp(p, sizes, obs, hidden, "identity")
    margin = torch.minimum(margin, m3)
    a = torch.as_tensor(act.astype(np.int64))
    theta = _quantiles(q, N)[rows, a]
    row_loss = quantile_huber(theta, target, tau)
    loss = row_loss.mean()
    (grad,) = torch.autograd.grad(loss, p)
    with torch.no_grad():
        u = (target[:, None, :] - theta[:, :, None]).abs().reshape(B, -1)
        u_min = torch.minimum((u - 1).abs().min(1).values, u.min(1).values)

    def row_fn(flat_p, o, ai, ti):  # ai: the row's action one-hot [n], ti: its target quantiles [N]
        h = o[None]
        for l, (W, b) in enumerate(_layers(flat_p, sizes)):
            h = h @ W.T + b
            if l < len(sizes) - 2:
                h = _ACT[hidden](h)
        th = (_quantiles(h[0], N) * ai[:, None]).sum(0)
        return quantile_huber(th[None], ti[None], tau)[0] / B
    onehot = torch.nn.functional.one_hot(a, sizes[-1] // N).to(D)
    per_row = torch.func.vmap(torch.func.grad(row_fn), in_dims=(None, 0, 0, 0))(p.detach(), obs, onehot, target)
    scale = per_row.abs().sum(0)
    return dict(q_values=(theta.detach().sum(-1) / N).numpy(), loss=float(loss.detach()),
                row_loss=row_loss.detach().numpy(), grad=grad.numpy(), scale=scale.numpy(), target=target.numpy(),
                margin=margin.numpy(), gap=gap.numpy(), u_min=u_min.numpy())
