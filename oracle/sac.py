"""torch-CPU oracle of SAC.train.  TEST INFRASTRUCTURE ONLY -- see oracle/__init__.py.

A float32 restatement of Spinning Up's SAC update (sac/core.py SquashedGaussianMLPActor / MLPQFunction, sac/sac.py
compute_loss_q / compute_loss_pi / update) with the optional learned temperature of the SAC paper (Haarnoja et al.
2018, "Soft Actor-Critic Algorithms and Applications", eq. 18).  It consumes given minibatches and noise draws; every
gradient comes from autograd and every optimizer is torch.optim.Adam, so it shares nothing with the CUDA kernels'
hand-derived backward pass.  The policy network's last Linear is Spinning Up's mu_layer and log_std_layer stacked:
network(obs) = [mu | log_std].
"""
from __future__ import annotations

import copy
from typing import Dict, List

import numpy as np
import torch
import torch.nn.functional as F
from torch.distributions import Normal


def squash(out: torch.Tensor, eps: torch.Tensor, limit: float, log_std_min: float = -20.0, log_std_max: float = 2.0):
    """(limit * tanh(u), log pi) with u = mu + exp(clamp(log_std)) * eps, the rsample of SquashedGaussianMLPActor."""
    A = out.shape[-1] // 2
    mu, log_std = out[..., :A], torch.clamp(out[..., A:], log_std_min, log_std_max)
    std = torch.exp(log_std)
    dist = Normal(mu, std)
    u = mu + eps * std
    logp = dist.log_prob(u).sum(axis=-1)
    logp = logp - (2 * (np.log(2) - u - F.softplus(-2 * u))).sum(axis=-1)
    return limit * torch.tanh(u), logp


class SacOracle:
    """Holds pi, q1, q2 (deep copies of the given modules), their targets, torch Adams and log_alpha; ``train`` runs
    one SAC.train call."""

    def __init__(self, pi: torch.nn.Module, q1: torch.nn.Module, q2: torch.nn.Module, pi_lr=1e-3, q_lr=1e-3,
                 gamma=0.99, rho=0.995, alpha=0.2, learn_alpha=False, target_entropy=None, alpha_lr=3e-4,
                 limit=1.0, log_std_min=-20.0, log_std_max=2.0):
        self.pi, self.q1, self.q2 = copy.deepcopy(pi), copy.deepcopy(q1), copy.deepcopy(q2)
        self.q1_targ, self.q2_targ = copy.deepcopy(q1), copy.deepcopy(q2)
        for p in list(self.q1_targ.parameters()) + list(self.q2_targ.parameters()):
            p.requires_grad = False
        self.pi_opt = torch.optim.Adam(self.pi.parameters(), lr=pi_lr)
        self.q1_opt = torch.optim.Adam(self.q1.parameters(), lr=q_lr)
        self.q2_opt = torch.optim.Adam(self.q2.parameters(), lr=q_lr)
        A = [m for m in self.pi.modules() if isinstance(m, torch.nn.Linear)][-1].out_features // 2
        self.gamma, self.rho, self.alpha, self.learn_alpha = gamma, rho, alpha, learn_alpha
        self.target_entropy = float(-A if target_entropy is None else target_entropy)
        self.log_alpha = torch.nn.Parameter(torch.tensor(float(np.log(alpha)), dtype=torch.float32))
        self.alpha_opt = torch.optim.Adam([self.log_alpha], lr=alpha_lr)
        self.limit, self.log_std_min, self.log_std_max = limit, log_std_min, log_std_max

    def _q(self, q, o, a):
        return q(torch.cat([o, a], dim=-1)).squeeze(-1)

    def _head(self, o, eps):
        return squash(self.pi(o), eps, self.limit, self.log_std_min, self.log_std_max)

    def train(self, minibatches: List[dict], noise: np.ndarray) -> Dict[str, list]:
        """minibatches: S dicts of the replay buffer's columns; noise [S, 2, B, A] (the draw for s', then for s)."""
        logs = dict(q1_values=[], q2_values=[], q1_losses=[], q2_losses=[], policy_losses=[], log_prob_means=[],
                    alphas=[])
        t = lambda x: torch.as_tensor(np.asarray(x, dtype=np.float32))
        for st, mb in enumerate(minibatches):
            o, a, r = t(mb["observations"]), t(mb["actions"]), t(mb["rewards"])
            o2, d = t(mb["next_observations"]), t(np.asarray(mb["dones"]).astype(np.int32))
            alpha = self.log_alpha.detach().exp() if self.learn_alpha else torch.tensor(self.alpha, dtype=torch.float32)
            logs["alphas"].append(float(alpha))
            # compute_loss_q
            with torch.no_grad():
                a2, logp_a2 = self._head(o2, t(noise[st, 0]))
                q_pi_targ = torch.min(self._q(self.q1_targ, o2, a2), self._q(self.q2_targ, o2, a2))
                backup = r + self.gamma * (1 - d) * (q_pi_targ - alpha * logp_a2)
            for i, (q, opt) in enumerate(((self.q1, self.q1_opt), (self.q2, self.q2_opt)), 1):
                qv = self._q(q, o, a)
                loss_q = ((qv - backup) ** 2).mean()
                opt.zero_grad()
                loss_q.backward()
                opt.step()
                logs[f"q{i}_values"].append(qv.detach().numpy().copy())
                logs[f"q{i}_losses"].append(float(loss_q.detach()))
            # compute_loss_pi with the critics just updated, their parameters frozen
            for p in list(self.q1.parameters()) + list(self.q2.parameters()):
                p.requires_grad = False
            a_pi, logp_pi = self._head(o, t(noise[st, 1]))
            q_pi = torch.min(self._q(self.q1, o, a_pi), self._q(self.q2, o, a_pi))
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
