"""torch-CPU oracles of CQL.train.  TEST INFRASTRUCTURE ONLY -- see oracle/__init__.py.

* ``CqlOracle``: float32, torch autograd and torch.optim.Adam, the CQL(H) update exactly as the project states it
  (include/b200rl.h, "CQL"): SAC's squashed-Gaussian head (oracle/sac.py) for every policy sample, the 3N sampled
  values of each critic at s, ``torch.logsumexp`` for the penalty, and the optional Lagrange step on log alpha'.  It
  consumes the host draw order (``CQL._noise``) and shares nothing with the CUDA kernels' hand-derived gradients.
* ``critic_stage_f64``: one step's critic stage in float64 from given flat parameters and draws, with the per-row
  ReLU margins of every forward pass.
* ``penalty_grad_closed_form``: d loss / d Q of the penalty as the engine's head writes it.
"""
from __future__ import annotations

import math
from typing import Dict, List

import numpy as np
import torch

from .offpolicy_f64 import _grad, _t, mlp
from .offpolicy_f64 import squash as squash_f64
from .sac import SacOracle, squash

MAX_ALPHA_PRIME = 1e6


def sampled_actions(squash_fn, out_next, out_cur, draws, limit: float, *squash_args):
    """([B, 3N, A] actions, [B, 3N] log densities) in the penalty's block order: uniform, pi(.|s'), pi(.|s).
    ``draws`` [3, B, N, A] = (x, eps at s, eps at s'); ``out_*`` [B, 2A] the policy outputs."""
    x, eps_s, eps_n = draws[0], draws[1], draws[2]
    B, N, A = x.shape
    u = limit * (2 * x - 1)
    lu = -A * math.log(2 * limit)
    a_n, lp_n = squash_fn(out_next[:, None, :].expand(B, N, 2 * A), eps_n, limit, *squash_args)
    a_s, lp_s = squash_fn(out_cur[:, None, :].expand(B, N, 2 * A), eps_s, limit, *squash_args)
    acts = torch.cat([u, a_n, a_s], 1)
    logd = torch.cat([torch.full((B, N), lu, dtype=x.dtype), lp_n, lp_s], 1)
    return acts, logd


def penalty(q_samples: torch.Tensor, logd: torch.Tensor, q_data: torch.Tensor, temperature: float):
    """gap = mean_i T logsumexp_j((q_ij - logd_ij) / T) - mean_i q_data_i."""
    P = temperature * torch.logsumexp((q_samples - logd) / temperature, dim=1)
    return P.mean() - q_data.mean()


def penalty_grad_closed_form(q_samples, logd, w_eff: float, temperature: float):
    """(d w_eff gap / d q_samples [B, 3N], d w_eff gap / d q_data [B]) as cql_penalty_kernel writes them."""
    B = q_samples.shape[0]
    sm = torch.softmax((q_samples - logd) / temperature, dim=1)
    return w_eff * sm / B, torch.full((B,), -w_eff / B, dtype=q_samples.dtype)


class CqlOracle(SacOracle):
    """SacOracle with CQL's penalty; ``train`` runs one CQL.train call on minibatches and (SAC's noise, CQL's draws)."""

    def __init__(self, pi, q1, q2, cql_weight=5.0, cql_n_actions=10, cql_temperature=1.0, cql_target_action_gap=None,
                 cql_alpha_lr=3e-4, backup_entropy=False, **kw):
        super().__init__(pi, q1, q2, **kw)
        self.w, self.N, self.T = float(cql_weight), int(cql_n_actions), float(cql_temperature)
        self.tau = cql_target_action_gap
        self.backup_entropy = bool(backup_entropy)
        self.log_alpha_prime = torch.nn.Parameter(torch.tensor(0.0, dtype=torch.float32))
        self.alpha_prime_opt = torch.optim.Adam([self.log_alpha_prime], lr=cql_alpha_lr)

    def train(self, minibatches: List[dict], noise) -> Dict[str, list]:
        sac_noise, draws = noise
        logs = dict(q1_values=[], q2_values=[], q1_losses=[], q2_losses=[], policy_losses=[], log_prob_means=[],
                    alphas=[], cql_gap_1=[], cql_gap_2=[], alpha_primes=[])
        t = lambda x: torch.as_tensor(np.asarray(x, dtype=np.float32))
        lag = self.tau is not None
        for st, mb in enumerate(minibatches):
            o, a, r = t(mb["observations"]), t(mb["actions"]), t(mb["rewards"])
            o2, d = t(mb["next_observations"]), t(np.asarray(mb["dones"]).astype(np.int32))
            B = o.shape[0]
            alpha = self.log_alpha.detach().exp() if self.learn_alpha else torch.tensor(self.alpha, dtype=torch.float32)
            logs["alphas"].append(float(alpha))
            ap = torch.clamp(self.log_alpha_prime.exp(), 0.0, MAX_ALPHA_PRIME)
            logs["alpha_primes"].append(float(ap.detach()) if lag else 1.0)
            w_eff = ap.detach() * self.w if lag else self.w
            with torch.no_grad():
                a2, logp_a2 = self._head(o2, t(sac_noise[st, 0]))
                q_pi_targ = torch.min(self._q(self.q1_targ, o2, a2), self._q(self.q2_targ, o2, a2))
                soft = q_pi_targ - alpha * logp_a2 if self.backup_entropy else q_pi_targ
                backup = r + self.gamma * (1 - d) * soft
                acts, logd = sampled_actions(squash, self.pi(o2), self.pi(o), t(draws[st]), self.limit,
                                             self.log_std_min, self.log_std_max)
            o_rep = o[:, None, :].expand(B, acts.shape[1], o.shape[1])
            gaps = []
            for i, (q, opt) in enumerate(((self.q1, self.q1_opt), (self.q2, self.q2_opt)), 1):
                qv = self._q(q, o, a)
                qs = self._q(q, o_rep, acts)
                gap = penalty(qs, logd, qv, self.T)
                loss_q = ((qv - backup) ** 2).mean() + w_eff * gap
                if lag:
                    loss_q = loss_q - ap.detach() * self.tau
                opt.zero_grad()
                loss_q.backward()
                opt.step()
                gaps.append(gap.detach())
                logs[f"q{i}_values"].append(qv.detach().numpy().copy())
                logs[f"q{i}_losses"].append(float(loss_q.detach()))
                logs[f"cql_gap_{i}"].append(float(gap.detach()))
            if lag:
                loss_ap = -0.5 * (ap * (self.w * gaps[0] - self.tau) + ap * (self.w * gaps[1] - self.tau))
                self.alpha_prime_opt.zero_grad()
                loss_ap.backward()
                self.alpha_prime_opt.step()
            for p in list(self.q1.parameters()) + list(self.q2.parameters()):
                p.requires_grad = False
            a_pi, logp_pi = self._head(o, t(sac_noise[st, 1]))
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


# ---- float64 one-step reference ----------------------------------------------------------------------------------
def critic_stage_f64(nets: Dict[str, np.ndarray], mb: Dict[str, np.ndarray], eps_next, draws, alpha: float,
                     policy_sizes, q_sizes, cql_weight: float, cql_temperature: float, alpha_prime: float = 1.0,
                     target_action_gap=None, backup_entropy=False, hidden="relu", gamma=0.99, action_limit=1.0,
                     log_std_min=-20.0, log_std_max=2.0) -> Dict[str, np.ndarray]:
    """The CQL critic stage at the given flat parameters: SAC's target (with or without the entropy term), each critic's
    logged Q-values, gap, loss and gradient, and the Lagrange gradient w.r.t. log alpha' (``alpha_prime`` the clamped
    alpha' of the step).  ``draws`` [3, B, N, A] as ``CQL._noise`` draws them; ``margin``: per row, over every forward
    pass of the stage."""
    obs, act, rew = _t(mb["observations"]), _t(mb["actions"]), _t(mb["rewards"])
    nobs, done = _t(mb["next_observations"]), _t(np.asarray(mb["dones"], dtype=np.float64))
    B = obs.shape[0]
    out2, margin = mlp(_t(nets["policy"]), policy_sizes, nobs, hidden, "identity")
    out1, m1 = mlp(_t(nets["policy"]), policy_sizes, obs, hidden, "identity")
    margin = torch.minimum(margin, m1)
    a2, logp2 = squash_f64(out2, _t(eps_next), action_limit, log_std_min, log_std_max)
    qt = []
    for name in ("target_q1", "target_q2"):
        z, m = mlp(_t(nets[name]), q_sizes, torch.cat([nobs, a2], -1), hidden, "identity")
        qt.append(z[:, 0])
        margin = torch.minimum(margin, m)
    soft = torch.minimum(qt[0], qt[1]) - (alpha * logp2 if backup_entropy else 0.0)
    y = rew + gamma * (1 - done) * soft
    acts, logd = sampled_actions(squash_f64, out2, out1, _t(draws), action_limit, log_std_min, log_std_max)
    n3 = acts.shape[1]
    x_s = torch.cat([obs[:, None, :].expand(B, n3, obs.shape[1]), acts], -1).reshape(B * n3, -1)
    lag = target_action_gap is not None
    w_eff = alpha_prime * cql_weight if lag else cql_weight
    out = dict(y=y.detach().numpy())
    gaps = []
    for k, name in ((1, "q1"), (2, "q2")):
        p = _t(nets[name], grad=True)
        q, m = mlp(p, q_sizes, torch.cat([obs, act], -1), hidden, "identity")
        qs, ms = mlp(p, q_sizes, x_s, hidden, "identity")
        margin = torch.minimum(margin, torch.minimum(m, ms.view(B, n3).min(1).values))
        gap = penalty(qs.view(B, n3), logd.detach(), q[:, 0], cql_temperature)
        loss = ((q[:, 0] - y.detach()) ** 2).mean() + w_eff * gap - (alpha_prime * target_action_gap if lag else 0.0)
        gaps.append(float(gap.detach()))
        out[f"q{k}_values"] = q.detach()[:, 0].numpy()
        out[f"q{k}_gap"] = gaps[-1]
        out[f"q{k}_loss"], out[f"q{k}_grad"] = float(loss.detach()), _grad(loss, p)
    if lag:
        e = alpha_prime  # exp(log alpha') inside the clamp
        out["alpha_prime_grad"] = -0.5 * sum(cql_weight * g - target_action_gap for g in gaps) * e
    out["margin"] = margin.numpy()
    return out
