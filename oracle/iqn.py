"""torch-CPU oracles of IQN.train.  TEST INFRASTRUCTURE ONLY -- see oracle/__init__.py.

* ``iqn_taus``: the device's fraction draws (b200rl.h, "IQN"), bit for bit, from the host Philox of oracle/per.py.
* ``IqnOracle``: float32, torch autograd and torch.optim.Adam, the IQN update exactly as the project states it, driven
  by the engine's fractions: a* = argmax of the K argmax samples' means, the target samples r + (g (1 - d))
  Z_targ(s', tau'_j, a*), the sampled-fraction quantile Huber loss (kappa = 1, 1/N'), DQN's target copies.  Given the
  drawn leaves' priorities and each step's beta it is the prioritized variant; a minibatch with a ``discounts`` key
  (oracle/nstep.py) is discounted per row.  It shares nothing with the CUDA kernels' hand-derived gradient.
* ``iqn_step_f64``: one step in float64 from given flat parameters and fractions, with per-entry gradient scales, ReLU
  margins and the gap between the two largest argmax means.
* ``rho_loop_f64``: one row's loss as the paper writes it, an explicit double loop over i < N and j < N' in float64,
  written independently of the tensor forms above so that both can be held against it.
"""
from __future__ import annotations

import math
from typing import Dict, List, Sequence

import numpy as np
import torch

from .dqn import DqnOracle
from .offpolicy_f64 import _ACT, D, _t
from .per import philox4x32_10


def iqn_taus(seed: int, call: int, st: int, B: int, Mt: int) -> np.ndarray:
    """The fractions [B, Mt] of step ``st``: draw t = b Mt + j is word t % 4 of Philox4x32-10(counter (t / 4, st, call,
    0xB00), key seed) = r, tau = (2 (r >> 9) + 1) 2^-24 (float32, exact)."""
    seed, call = int(seed) & (2 ** 64 - 1), int(call) & (2 ** 64 - 1)
    t = np.arange(B * Mt, dtype=np.uint64)
    r = np.stack(philox4x32_10(t >> np.uint64(2), st, call & 0xFFFFFFFF, 0xB00, seed & 0xFFFFFFFF, seed >> 32))
    r = r[(t & np.uint64(3)).astype(np.int64), np.arange(t.size)]
    return ((np.uint64(2) * (r >> np.uint64(9)) + np.uint64(1)).astype(np.float32) * np.float32(2.0 ** -24)).reshape(B, Mt)


def sampled_quantile_huber(theta: torch.Tensor, target: torch.Tensor, tau: torch.Tensor) -> torch.Tensor:
    """Per-row L [B] = (1/N') sum_i sum_j |tau_i - 1{u_ij < 0}| h(u_ij), u_ij = target_j - theta_i, h the Huber loss
    with kappa = 1; theta and tau [B, N], target [B, N'].  Autograd differentiates h only (the indicator is a
    constant)."""
    u = target[:, None, :] - theta[:, :, None]  # [B, i, j]
    k = (tau[:, :, None] - (u.detach() < 0).to(u.dtype)).abs()
    h = torch.where(u.abs() < 1, 0.5 * u * u, u.abs() - 0.5)
    return (k * h).sum(2).sum(1) / target.shape[1]


def rho_loop_f64(theta, target, tau) -> float:
    """One row's L with explicit loops: for each i < N, j < N': u = T_j - theta_i, rho = |tau_i - [u < 0]| * (u^2 / 2 if
    |u| < 1 else |u| - 1/2); L = sum / N'."""
    theta, target, tau = [float(x) for x in theta], [float(x) for x in target], [float(x) for x in tau]
    total = 0.0
    for i in range(len(theta)):
        for j in range(len(target)):
            u = target[j] - theta[i]
            weight = abs(tau[i] - (1.0 if u < 0 else 0.0))
            total += weight * (u * u / 2 if abs(u) < 1 else abs(u) - 0.5)
    return total / len(target)


class IqnOracle(DqnOracle):
    """DqnOracle over ImplicitQuantileMLP copies with IQN's head: ``train`` runs one IQN.train call on the engine's
    fractions (one [B, N + N' + K] array per step); with ``leaf_priorities`` and ``betas`` (as oracle/per.PerDqnOracle
    takes them) the prioritized one."""

    def __init__(self, q, q_targ, optimizer, n_quantiles=64, n_target_quantiles=64, n_policy_quantiles=32,
                 alpha: float = 0.6, eps: float = 1e-6, **kw):
        super().__init__(q, q_targ, optimizer, **kw)
        self.N, self.Nt, self.K = int(n_quantiles), int(n_target_quantiles), int(n_policy_quantiles)
        self.alpha, self.eps = float(alpha), float(eps)

    def train(self, minibatches: List[dict], taus: Sequence[np.ndarray], leaf_priorities: Sequence[np.ndarray] = None,
              betas: Sequence[float] = None) -> Dict[str, list]:
        logs = dict(q1_values=[], q1_losses=[], copied=[], row_losses=[], weights=[], priorities=[])
        t = lambda x: torch.as_tensor(np.asarray(x, dtype=np.float32))
        N, Nt, K = self.N, self.Nt, self.K
        for k, mb in enumerate(minibatches):
            o, a, r = t(mb["observations"]), t(mb["actions"]).reshape(-1).long(), t(mb["rewards"])
            o2, d = t(mb["next_observations"]), t(np.asarray(mb["dones"]).astype(np.int32))
            g = t(mb["discounts"]) if "discounts" in mb else torch.tensor(self.gamma, dtype=torch.float32)
            tau = t(taus[k])
            rows = torch.arange(o.shape[0])
            with torch.no_grad():
                zt = self.q_targ(o2, tau[:, N:])  # [B, N' + K, n]: the target samples, then the argmax samples
                pick = self.q(o2, tau[:, N + Nt:]) if self.double_q else zt[:, Nt:]
                a_star = (pick.sum(1) / K).argmax(1)
                target = r[:, None] + (g * (1 - d))[..., None] * zt[rows, :Nt, a_star]
            theta = self.q(o, tau[:, :N])[rows, :, a]
            L = sampled_quantile_huber(theta, target, tau[:, :N])
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


def _iqn_params(flat: torch.Tensor, sizes: Sequence[int], n_cos: int):
    """(W, b) of psi, phi, head hidden and head out from the flat vector (W_psi, b_psi, W_phi, b_phi, W_h, b_h, W_out,
    b_out)."""
    O, d, h, n = sizes
    out, o = [], 0
    for rows, cols in ((d, O), (d, n_cos), (h, d), (n, h)):
        out.append((flat[o:o + rows * cols].view(rows, cols), flat[o + rows * cols:o + rows * cols + rows]))
        o += rows * cols + rows
    assert o == flat.numel()
    return out


def _features_f64(tau: torch.Tensor, n_cos: int) -> torch.Tensor:
    """cos(pi x) in float64 of x = float32(i tau), the engine's argument."""
    x = tau.float()[..., None] * torch.arange(n_cos, dtype=torch.float32)
    return torch.cos(math.pi * x.double())


def iqn_net_f64(flat: torch.Tensor, sizes: Sequence[int], n_cos: int, obs: torch.Tensor, tau: torch.Tensor,
                hidden: str):
    """(Z [B, M, n], per-row smallest relative ReLU margin over psi, phi and the head's hidden layer; +inf without
    ReLU) of obs [B, O] at the fractions tau [B, M], in float64."""
    (Wp, bp), (Wc, bc), (Wh, bh), (Wo, bo) = _iqn_params(flat, sizes, n_cos)
    x = _features_f64(tau, n_cos)
    margin = torch.full((obs.shape[0],), math.inf, dtype=D)

    def layer(inp, W, b):
        nonlocal margin
        z = inp @ W.T + b
        if hidden == "relu":
            with torch.no_grad():
                scale = inp.detach().abs() @ W.detach().abs().T + b.detach().abs()
                m = (z.detach().abs() / scale.clamp_min(1e-300))
                margin = torch.minimum(margin, m.reshape(obs.shape[0], -1).min(dim=1).values)
        return _ACT[hidden](z)
    psi, phi = layer(obs, Wp, bp), layer(x, Wc, bc)
    hh = layer(psi[:, None, :] * phi, Wh, bh)
    return hh @ Wo.T + bo, margin


def iqn_step_f64(q_flat, targ_flat, mb: Dict[str, np.ndarray], taus: np.ndarray, sizes: Sequence[int], n_cos: int,
                 N: int, Nt: int, K: int, hidden="relu", gamma=0.99, double_q=False):
    """One IQN step's loss, logged Q(s, a) and gradient w.r.t. the Q network in float64 on the engine's fractions
    ``taus`` [B, N + N' + K] (float32 values).  ``sizes`` = [obs, d, h, n_actions].  Returns dict(q_values, loss,
    row_loss, grad (flat), scale (flat: per entry the sum over rows of |that row's contribution|), target [B, N'],
    margin (per row, over every forward pass), gap (per row: the two largest argmax means apart; +inf for one action),
    u_min (per row: the distance of the nearest u_ij to a kink of the loss))."""
    obs, act, rew = _t(mb["observations"]), np.asarray(mb["actions"]).reshape(-1), _t(mb["rewards"])
    nobs, done = _t(mb["next_observations"]), _t(np.asarray(mb["dones"], dtype=np.float64))
    tau = torch.as_tensor(np.asarray(taus, np.float32))
    tau_on = tau[:, :N].double()
    B = obs.shape[0]
    rows = torch.arange(B)
    with torch.no_grad():
        zt, margin = iqn_net_f64(_t(targ_flat), sizes, n_cos, nobs, tau[:, N:], hidden)
        pick = zt[:, Nt:]
        if double_q:
            pick, m2 = iqn_net_f64(_t(q_flat), sizes, n_cos, nobs, tau[:, N + Nt:], hidden)
            margin = torch.minimum(margin, m2)
        means = pick.sum(1) / K
        gap = torch.full((B,), math.inf, dtype=D)
        if means.shape[1] > 1:
            top2 = means.topk(2, dim=1).values
            gap = top2[:, 0] - top2[:, 1]
        g = gamma if torch.is_tensor(gamma) else torch.tensor(gamma, dtype=D)
        target = rew[:, None] + (g * (1 - done))[..., None] * zt[rows, :Nt, means.argmax(1)]
    p = _t(q_flat, grad=True)
    z, m3 = iqn_net_f64(p, sizes, n_cos, obs, tau[:, :N], hidden)
    margin = torch.minimum(margin, m3)
    a = torch.as_tensor(act.astype(np.int64))
    theta = z[rows, :, a]
    row_loss = sampled_quantile_huber(theta, target, tau_on)
    loss = row_loss.mean()
    (grad,) = torch.autograd.grad(loss, p)
    with torch.no_grad():
        u = (target[:, None, :] - theta[:, :, None]).abs().reshape(B, -1)
        u_min = torch.minimum((u - 1).abs().min(1).values, u.min(1).values)

    def row_fn(flat_p, o, ai, ti, tu):  # ai: the row's action one-hot [n], ti: its targets [N'], tu: its fractions [N]
        zr, _ = iqn_net_f64(flat_p, sizes, n_cos, o[None], tu[None].float(), hidden)
        th = (zr[0] * ai).sum(-1)
        return sampled_quantile_huber(th[None], ti[None], tu[None])[0] / B
    onehot = torch.nn.functional.one_hot(a, sizes[-1]).to(D)
    per_row = torch.func.vmap(torch.func.grad(row_fn), in_dims=(None, 0, 0, 0, 0))(p.detach(), obs, onehot, target,
                                                                                   tau_on)
    scale = per_row.abs().sum(0)
    return dict(q_values=(theta.detach().sum(-1) / N).numpy(), loss=float(loss.detach()),
                row_loss=row_loss.detach().numpy(), grad=grad.numpy(), scale=scale.numpy(), target=target.numpy(),
                margin=margin.numpy(), gap=gap.numpy(), u_min=u_min.numpy())
