"""torch-CPU oracles of IQL.train.  TEST INFRASTRUCTURE ONLY -- see oracle/__init__.py.

* ``IqlOracle``: float32, torch autograd and torch.optim.Adam, the IQL update exactly as the project states it
  (include/b200rl.h, "IQL"), in the order of the authors' reference implementation: ``update_v``, the AWR actor step
  with the new V, ``update_q`` with the new V, then the target critics.  It shares nothing with the CUDA kernels'
  hand-derived gradients.
* ``value_stage_f64`` / ``policy_stage_f64`` / ``critic_stage_f64``: each step's stages in float64 from given flat
  parameters, with the per-row ReLU margins of every forward pass.
* ``expectile_grad_closed_form`` / ``awr_grad_closed_form``: the output gradients as the engine's heads write them.
"""
from __future__ import annotations

import copy
from typing import Dict, List

import numpy as np
import torch
from torch.distributions import Independent, Normal

from .offpolicy_f64 import _grad, _t, mlp


def expectile_loss(q_hat: torch.Tensor, v: torch.Tensor, tau: float) -> torch.Tensor:
    """mean_i |tau - 1{u_i < 0}| u_i^2, u = q_hat - v (w = tau where u > 0)."""
    u = q_hat - v
    w = torch.where(u > 0, torch.full_like(u, tau), torch.full_like(u, 1 - tau))
    return (w * u ** 2).mean()


def awr_weights(q_hat: torch.Tensor, v: torch.Tensor, beta: float, max_weight: float) -> torch.Tensor:
    """min(exp(beta (q_hat - v)), W), a constant of the policy step."""
    return torch.clamp(torch.exp(beta * (q_hat - v)), max=max_weight).detach()


def log_prob(out: torch.Tensor, act: torch.Tensor, limit: float, log_std_min: float, log_std_max: float):
    """sum_j Normal(limit tanh(m_j), exp(clamp(l_j))).log_prob(act_j), out = [m | l]."""
    A = out.shape[-1] // 2
    mu = limit * torch.tanh(out[..., :A])
    log_std = torch.clamp(out[..., A:], log_std_min, log_std_max)
    return Independent(Normal(mu, torch.exp(log_std)), 1).log_prob(act)


def expectile_grad_closed_form(q_hat, v, tau: float):
    """d mean(w u^2) / d v = -2 w u / B, as iql_value_loss_kernel writes it."""
    u = q_hat - v
    w = torch.where(u > 0, torch.full_like(u, tau), torch.full_like(u, 1 - tau))
    return -2 * w * u / u.shape[0]


def awr_grad_closed_form(out, act, e, limit: float, log_std_min: float, log_std_max: float):
    """d (-mean(e log pi)) / d [m | l] [B, 2A], as iql_policy_loss_kernel writes it."""
    B, A = act.shape
    m, raw = out[:, :A], out[:, A:]
    t = torch.tanh(m)
    var = torch.exp(2 * torch.clamp(raw, log_std_min, log_std_max))
    d = act - limit * t
    c = (e / B)[:, None]
    dm = -c * (d / var) * limit * (1 - t * t)
    inside = (raw >= log_std_min) & (raw <= log_std_max)
    dl = torch.where(inside, -c * (d * d / var - 1), torch.zeros_like(raw))
    return torch.cat([dm, dl], 1)


class IqlOracle:
    """Holds pi, q1, q2, v (deep copies of the given modules), the critics' targets and torch Adams; ``train`` runs one
    IQL.train call on the given minibatches."""

    def __init__(self, pi: torch.nn.Module, q1: torch.nn.Module, q2: torch.nn.Module, v: torch.nn.Module, pi_lr=1e-3,
                 q_lr=1e-3, v_lr=1e-3, gamma=0.99, rho=0.995, expectile=0.7, beta=3.0, max_weight=100.0, limit=1.0,
                 log_std_min=-5.0, log_std_max=2.0, q2_lr=None, v_betas=(0.9, 0.999), v_eps=1e-8):
        self.pi, self.q1, self.q2, self.v = (copy.deepcopy(m) for m in (pi, q1, q2, v))
        self.q1_targ, self.q2_targ = copy.deepcopy(q1), copy.deepcopy(q2)
        for p in list(self.q1_targ.parameters()) + list(self.q2_targ.parameters()):
            p.requires_grad = False
        self.pi_opt = torch.optim.Adam(self.pi.parameters(), lr=pi_lr)
        self.q1_opt = torch.optim.Adam(self.q1.parameters(), lr=q_lr)
        self.q2_opt = torch.optim.Adam(self.q2.parameters(), lr=q_lr if q2_lr is None else q2_lr)
        self.v_opt = torch.optim.Adam(self.v.parameters(), lr=v_lr, betas=v_betas, eps=v_eps)
        self.gamma, self.rho = gamma, rho
        self.tau, self.beta, self.max_weight = float(expectile), float(beta), float(max_weight)
        self.limit, self.log_std_min, self.log_std_max = limit, log_std_min, log_std_max

    @staticmethod
    def _q(q, o, a):
        return q(torch.cat([o, a], dim=-1)).squeeze(-1)

    def train(self, minibatches: List[dict]) -> Dict[str, list]:
        logs = dict(q1_values=[], q2_values=[], q1_losses=[], q2_losses=[], policy_losses=[], value_losses=[],
                    value_means=[], weight_means=[])
        t = lambda x: torch.as_tensor(np.asarray(x, dtype=np.float32))
        for mb in minibatches:
            o, a, r = t(mb["observations"]), t(mb["actions"]), t(mb["rewards"])
            o2, d = t(mb["next_observations"]), t(np.asarray(mb["dones"]).astype(np.int32))
            with torch.no_grad():
                q_hat = torch.min(self._q(self.q1_targ, o, a), self._q(self.q2_targ, o, a))
            # value step
            v = self.v(o).squeeze(-1)
            loss_v = expectile_loss(q_hat, v, self.tau)
            self.v_opt.zero_grad()
            loss_v.backward()
            self.v_opt.step()
            logs["value_losses"].append(float(loss_v.detach()))
            logs["value_means"].append(float(v.detach().mean()))
            # policy step with the new V
            with torch.no_grad():
                v_new = self.v(o).squeeze(-1)
                v_next = self.v(o2).squeeze(-1)
            e = awr_weights(q_hat, v_new, self.beta, self.max_weight)
            loss_pi = -(e * log_prob(self.pi(o), a, self.limit, self.log_std_min, self.log_std_max)).mean()
            self.pi_opt.zero_grad()
            loss_pi.backward()
            self.pi_opt.step()
            logs["policy_losses"].append(float(loss_pi.detach()))
            logs["weight_means"].append(float(e.mean()))
            # critic step with the new V
            y = r + self.gamma * (1 - d) * v_next
            for i, (q, opt) in enumerate(((self.q1, self.q1_opt), (self.q2, self.q2_opt)), 1):
                qv = self._q(q, o, a)
                loss_q = ((qv - y) ** 2).mean()
                opt.zero_grad()
                loss_q.backward()
                opt.step()
                logs[f"q{i}_values"].append(qv.detach().numpy().copy())
                logs[f"q{i}_losses"].append(float(loss_q.detach()))
            with torch.no_grad():
                for q, qt in ((self.q1, self.q1_targ), (self.q2, self.q2_targ)):
                    for p, p_targ in zip(q.parameters(), qt.parameters()):
                        p_targ.data.mul_(self.rho)
                        p_targ.data.add_((1 - self.rho) * p.data)
        return logs


# ---- float64 one-step references ---------------------------------------------------------------------------------
def _batch(mb):
    return (_t(mb["observations"]), _t(mb["actions"]), _t(mb["rewards"]), _t(mb["next_observations"]),
            _t(np.asarray(mb["dones"], dtype=np.float64)))


def value_stage_f64(nets: Dict[str, np.ndarray], mb, q_sizes, v_sizes, expectile: float, hidden="relu"):
    """q_hat, V(s), the value loss and its gradient w.r.t. V's flat parameters; ``margin`` per row."""
    obs, act = _batch(mb)[:2]
    x = torch.cat([obs, act], -1)
    z1, m1 = mlp(_t(nets["target_q1"]), q_sizes, x, hidden, "identity")
    z2, m2 = mlp(_t(nets["target_q2"]), q_sizes, x, hidden, "identity")
    q_hat = torch.minimum(z1[:, 0], z2[:, 0])
    p = _t(nets["v"], grad=True)
    v, mv = mlp(p, v_sizes, obs, hidden, "identity")
    loss = expectile_loss(q_hat, v[:, 0], expectile)
    return dict(q_hat=q_hat.numpy(), v=v.detach()[:, 0].numpy(), loss=float(loss.detach()), grad=_grad(loss, p),
                margin=torch.minimum(torch.minimum(m1, m2), mv).numpy())


def policy_stage_f64(policy: np.ndarray, obs, act, q_hat, v_new, policy_sizes, beta: float, max_weight: float,
                     limit=1.0, log_std_min=-5.0, log_std_max=2.0, hidden="relu"):
    """The AWR step at the given flat policy: its loss, weights and gradient w.r.t. the policy's flat parameters."""
    p = _t(policy, grad=True)
    out, margin = mlp(p, policy_sizes, _t(obs), hidden, "identity")
    e = awr_weights(_t(q_hat), _t(v_new), beta, max_weight)
    loss = -(e * log_prob(out, _t(act), limit, log_std_min, log_std_max)).mean()
    return dict(loss=float(loss.detach()), weights=e.numpy(), grad=_grad(loss, p), margin=margin.numpy())


def critic_stage_f64(nets: Dict[str, np.ndarray], mb, v_next, q_sizes, gamma=0.99, hidden="relu"):
    """y = r + gamma (1 - d) V'(s') and each critic's logged Q-values, loss and gradient."""
    obs, act, rew, _, done = _batch(mb)
    y = rew + gamma * (1 - done) * _t(v_next)
    out, margin = dict(y=y.numpy()), None
    for k, name in ((1, "q1"), (2, "q2")):
        p = _t(nets[name], grad=True)
        q, m = mlp(p, q_sizes, torch.cat([obs, act], -1), hidden, "identity")
        loss = ((q[:, 0] - y) ** 2).mean()
        margin = m if margin is None else torch.minimum(margin, m)
        out[f"q{k}_values"] = q.detach()[:, 0].numpy()
        out[f"q{k}_loss"], out[f"q{k}_grad"] = float(loss.detach()), _grad(loss, p)
    out["margin"] = margin.numpy()
    return out
