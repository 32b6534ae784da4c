"""torch-CPU oracles of TQC.train.  TEST INFRASTRUCTURE ONLY -- see oracle/__init__.py.

* ``TqcOracle``: float32, torch autograd and torch.optim.Adam, the TQC update exactly as the project states it
  (include/b200rl.h, "TQC"): SAC's squashed-Gaussian head (oracle/sac.py), the 2M target atoms of both target critics
  pooled, sorted with ``torch.sort`` and truncated to the smallest kN, the quantile Huber loss of oracle/qr.py scaled
  by 1 / (kN M), and a policy loss on the mean of both critics' quantiles.  It shares nothing with the CUDA kernels'
  hand-derived gradients.
* ``critic_stage_f64`` / ``policy_stage_f64``: one step's stages in float64 from given flat parameters, with the
  per-row ReLU margins of every forward pass.
* ``truncated_atoms_loop``: one row's kept atoms by an explicit selection in float64, written independently of
  ``torch.sort``, NaN last.
"""
from __future__ import annotations

import math
from typing import Dict, List

import numpy as np
import torch

from .offpolicy_f64 import D, _grad, _t, mlp
from .offpolicy_f64 import squash as squash_f64
from .qr import quantile_huber, taus
from .sac import SacOracle


def truncated_atoms(z1: torch.Tensor, z2: torch.Tensor, kN: int) -> torch.Tensor:
    """The smallest kN of the 2M pooled atoms [B, M] + [B, M], ascending (torch.sort: NaN last) -> [B, kN]."""
    return torch.sort(torch.cat([z1, z2], dim=-1), dim=-1).values[:, :kN]


def truncated_atoms_loop(z1, z2, kN: int) -> List[float]:
    """One row's kept atoms by repeated selection of the smallest remaining value, NaN after every number."""
    pool = [float(x) for x in list(z1) + list(z2)]
    key = lambda v: (1, 0.0) if math.isnan(v) else (0, v)
    out = []
    for _ in range(kN):
        k = min(range(len(pool)), key=lambda i: key(pool[i]))
        out.append(pool.pop(k))
    return out


def row_losses(theta: torch.Tensor, y: torch.Tensor, tau: torch.Tensor) -> torch.Tensor:
    """L [B] = (1 / (kN M)) sum_m sum_i |tau_m - 1{u_mi < 0}| h(u_mi), u_mi = y_i - theta_m; theta [B, M], y [B, kN]."""
    return quantile_huber(theta, y, tau) / y.shape[1]


def critic_grad_closed_form(theta: torch.Tensor, y: torch.Tensor, tau: torch.Tensor) -> torch.Tensor:
    """d mean_B(L) / d theta [B, M] as the engine's head writes it: -(sum_i |tau_m - 1{u < 0}| clamp(u, -1, 1)) /
    (kN M) / B."""
    B, M, kN = theta.shape[0], theta.shape[1], y.shape[1]
    u = y[:, None, :] - theta[:, :, None]
    k = (tau[None, :, None] - (u < 0).to(u.dtype)).abs()
    return -(k * u.clamp(-1, 1)).sum(2) / (kN * M) / B


class TqcOracle(SacOracle):
    """SacOracle with quantile critics: q1, q2 map [s | a] to M quantiles; ``train`` runs one TQC.train call."""

    def __init__(self, pi, q1, q2, n_quantiles: int = 25, n_drop: int = 2, **kw):
        super().__init__(pi, q1, q2, **kw)
        self.M, self.kN = int(n_quantiles), 2 * (int(n_quantiles) - int(n_drop))
        self.tau = taus(self.M)

    def _z(self, q, o, a):
        return q(torch.cat([o, a], dim=-1))

    def train(self, minibatches: List[dict], noise: np.ndarray) -> Dict[str, list]:
        """minibatches: S dicts of the replay buffer's columns; noise [S, 2, B, A] (the draw for s', then for s)."""
        logs = dict(q1_values=[], q2_values=[], q1_losses=[], q2_losses=[], policy_losses=[], log_prob_means=[],
                    alphas=[], targets=[])
        t = lambda x: torch.as_tensor(np.asarray(x, dtype=np.float32))
        M = self.M
        for st, mb in enumerate(minibatches):
            o, a, r = t(mb["observations"]), t(mb["actions"]), t(mb["rewards"])
            o2, d = t(mb["next_observations"]), t(np.asarray(mb["dones"]).astype(np.int32))
            alpha = self.log_alpha.detach().exp() if self.learn_alpha else torch.tensor(self.alpha, dtype=torch.float32)
            logs["alphas"].append(float(alpha))
            with torch.no_grad():
                a2, logp_a2 = self._head(o2, t(noise[st, 0]))
                z = truncated_atoms(self._z(self.q1_targ, o2, a2), self._z(self.q2_targ, o2, a2), self.kN)
                y = r[:, None] + (self.gamma * (1 - d))[:, None] * (z - alpha * logp_a2[:, None])
            logs["targets"].append(y.numpy().copy())
            for i, (q, opt) in enumerate(((self.q1, self.q1_opt), (self.q2, self.q2_opt)), 1):
                theta = self._z(q, o, a)
                loss_q = row_losses(theta, y, self.tau).mean()
                opt.zero_grad()
                loss_q.backward()
                opt.step()
                logs[f"q{i}_values"].append((theta.detach().sum(-1) / M).numpy().copy())
                logs[f"q{i}_losses"].append(float(loss_q.detach()))
            for p in list(self.q1.parameters()) + list(self.q2.parameters()):
                p.requires_grad = False
            a_pi, logp_pi = self._head(o, t(noise[st, 1]))
            q_pi = torch.cat([self._z(self.q1, o, a_pi), self._z(self.q2, o, a_pi)], -1).sum(-1) / (2 * M)
            loss_pi = (alpha * logp_pi - q_pi).mean()
            self.pi_opt.zero_grad()
            loss_pi.backward()
            self.pi_opt.step()
            for p in list(self.q1.parameters()) + list(self.q2.parameters()):
                p.requires_grad = True
            logs["policy_losses"].append(float(loss_pi.detach()))
            logs["log_prob_means"].append(float(logp_pi.detach().mean()))
            if self.learn_alpha:
                loss_alpha = -(self.log_alpha * (logp_pi.detach() + self.target_entropy)).mean()
                self.alpha_opt.zero_grad()
                loss_alpha.backward()
                self.alpha_opt.step()
            with torch.no_grad():
                for q, qt in ((self.q1, self.q1_targ), (self.q2, self.q2_targ)):
                    for p, p_targ in zip(q.parameters(), qt.parameters()):
                        p_targ.data.mul_(self.rho)
                        p_targ.data.add_((1 - self.rho) * p.data)
        return logs


# ---- float64 one-step reference ----------------------------------------------------------------------------------
def critic_stage_f64(nets: Dict[str, np.ndarray], mb: Dict[str, np.ndarray], eps_next, alpha: float, policy_sizes,
                     q_sizes, n_quantiles: int, n_drop: int, hidden="relu", gamma=0.99, action_limit=1.0,
                     log_std_min=-20.0, log_std_max=2.0) -> Dict[str, np.ndarray]:
    """The TQC critic step at the given flat parameters: a', log pi' from the policy and ``eps_next``, the kept target
    atoms y [B, kN], and each critic's logged Q-values (quantile means), loss and gradient.  ``margin``: per row, over
    every forward pass of the stage."""
    M, kN = int(n_quantiles), 2 * (int(n_quantiles) - int(n_drop))
    obs, act, rew = _t(mb["observations"]), _t(mb["actions"]), _t(mb["rewards"])
    nobs, done = _t(mb["next_observations"]), _t(np.asarray(mb["dones"], dtype=np.float64))
    out2, margin = mlp(_t(nets["policy"]), policy_sizes, nobs, hidden, "identity")
    a2, logp2 = squash_f64(out2, _t(eps_next), action_limit, log_std_min, log_std_max)
    zs = []
    for name in ("target_q1", "target_q2"):
        z, m = mlp(_t(nets[name]), q_sizes, torch.cat([nobs, a2], -1), hidden, "identity")
        zs.append(z)
        margin = torch.minimum(margin, m)
    y = rew[:, None] + (gamma * (1 - done))[:, None] * (truncated_atoms(zs[0], zs[1], kN) - alpha * logp2[:, None])
    tau = taus(M, D)
    out = dict(y=y.detach().numpy(), logp_next=logp2.detach().numpy())
    for k, name in ((1, "q1"), (2, "q2")):
        p = _t(nets[name], grad=True)
        theta, m = mlp(p, q_sizes, torch.cat([obs, act], -1), hidden, "identity")
        margin = torch.minimum(margin, m)
        loss = row_losses(theta, y.detach(), tau).mean()
        out[f"q{k}_values"] = (theta.detach().sum(-1) / M).numpy()
        out[f"q{k}_loss"], out[f"q{k}_grad"] = float(loss.detach()), _grad(loss, p)
    out["margin"] = margin.numpy()
    return out


def policy_stage_f64(policy: np.ndarray, q1: np.ndarray, q2: np.ndarray, obs, eps_cur, alpha: float, policy_sizes,
                     q_sizes, hidden="relu", action_limit=1.0, log_std_min=-20.0, log_std_max=2.0,
                     target_entropy=None) -> Dict[str, np.ndarray]:
    """mean(alpha log pi - mean of both critics' quantiles at (s, a_pi)) with the critics AFTER this step's update,
    frozen; its gradient w.r.t. the policy; mean log pi; and the temperature's gradient -mean(log pi + target_entropy)
    w.r.t. log_alpha."""
    obs = _t(obs)
    p = _t(policy, grad=True)
    out, margin_pi = mlp(p, policy_sizes, obs, hidden, "identity")
    a, logp = squash_f64(out, _t(eps_cur), action_limit, log_std_min, log_std_max)
    margin_q = torch.full((obs.shape[0],), math.inf, dtype=D)
    zs = []
    for qf in (q1, q2):
        z, m = mlp(_t(qf), q_sizes, torch.cat([obs, a], -1), hidden, "identity")
        zs.append(z)
        margin_q = torch.minimum(margin_q, m.detach())
    loss = (alpha * logp - torch.cat(zs, -1).mean(-1)).mean()
    te = -float(a.shape[-1]) if target_entropy is None else float(target_entropy)
    return dict(loss=float(loss.detach()), grad=_grad(loss, p), logp_mean=float(logp.detach().mean()),
                alpha_grad=float(-(logp.detach() + te).mean()), margin_pi=margin_pi.numpy(),
                margin_q=margin_q.numpy())

