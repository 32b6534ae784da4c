"""torch-CPU oracles of EDAC.train (SAC-N at eta = 0).  TEST INFRASTRUCTURE ONLY -- see oracle/__init__.py.

* ``EdacOracle``: float32, torch autograd and torch.optim.Adam, the EDAC update as the project states it
  (include/b200rl.h, "EDAC"; An, Moon, Kim & Song 2021): SAC's squashed-Gaussian head (oracle/sac.py), a target that
  takes ``torch.fmin`` over all N target critics, one Adam step per critic on its MSE plus eta times the diversity
  penalty -- the action gradients taken with ``torch.autograd.grad(..., create_graph=True)`` as the authors' code takes
  them -- and a policy loss on the per-row min of the critics just updated.  It shares nothing with the CUDA path's
  hand-derived diversity gradient.
* ``diversity``: the penalty D of stacked action gradients [N, B, A] (the authors' ``grad_loss`` without eta).
* ``critic_stage_f64`` / ``policy_stage_f64``: one step's stages in float64 from given flat parameters, with the
  per-row ReLU margins of every forward pass.
"""
from __future__ import annotations

import copy
import math
from typing import Dict, List, Sequence

import numpy as np
import torch

from .offpolicy_f64 import D, _t, mlp
from .offpolicy_f64 import squash as squash_f64
from .redq import fmin_all
from .sac import squash

NORM_EPS = 1e-10


def diversity(g: torch.Tensor) -> torch.Tensor:
    """D = sum_b sum_{i != j} gh_i(b) . gh_j(b) / (B (N - 1)), gh = g / (|g|_2 + 1e-10), for g [N, B, A]."""
    N, B = g.shape[0], g.shape[1]
    gh = g / (g.norm(dim=2, keepdim=True) + NORM_EPS)
    cos = torch.einsum("ibk,jbk->bij", gh, gh) * (1 - torch.eye(N, dtype=g.dtype))
    return cos.sum() / (B * (N - 1))


def first_argmin(vals: torch.Tensor) -> torch.Tensor:
    """Per column of vals [N, B]: the first row that attains the min, a NaN losing to a number (fminf's min)."""
    v = torch.where(torch.isnan(vals), torch.full_like(vals, math.inf), vals).detach()
    return (v == v.min(0, keepdim=True).values).to(torch.int64).argmax(0)  # argmax: the first maximal index


def action_gradients(qs, o: torch.Tensor, a: torch.Tensor, create_graph: bool):
    """(values [N, B], action gradients [N, B, A]) of the critics at [o | a]."""
    at = a.detach().clone().requires_grad_(True)
    vals, grads = [], []
    for q in qs:
        v = q(torch.cat([o, at], dim=-1)).squeeze(-1)
        (g,) = torch.autograd.grad(v.sum(), at, create_graph=create_graph, retain_graph=True)
        vals.append(v)
        grads.append(g)
    return torch.stack(vals), torch.stack(grads)


class EdacOracle:
    """Holds pi, the N critics (deep copies), their targets, torch Adams and log_alpha; ``train`` runs one EDAC.train
    call on given minibatches and noise."""

    def __init__(self, pi: torch.nn.Module, qs: Sequence[torch.nn.Module], pi_lr=1e-3, q_lr=1e-3, gamma=0.99,
                 rho=0.995, alpha=0.2, learn_alpha=True, target_entropy=None, alpha_lr=3e-4, limit=1.0,
                 log_std_min=-20.0, log_std_max=2.0, eta=1.0):
        self.pi = copy.deepcopy(pi)
        self.qs = [copy.deepcopy(q) for q in qs]
        self.q_targs = [copy.deepcopy(q) for q in qs]
        for qt in self.q_targs:
            for p in qt.parameters():
                p.requires_grad = False
        self.pi_opt = torch.optim.Adam(self.pi.parameters(), lr=pi_lr)
        self.q_opts = [torch.optim.Adam(q.parameters(), lr=q_lr) for q in self.qs]
        A = [m for m in self.pi.modules() if isinstance(m, torch.nn.Linear)][-1].out_features // 2
        self.gamma, self.rho, self.alpha, self.learn_alpha = gamma, rho, alpha, learn_alpha
        self.target_entropy = float(-A if target_entropy is None else target_entropy)
        self.log_alpha = torch.nn.Parameter(torch.tensor(float(np.log(alpha)), dtype=torch.float32))
        self.alpha_opt = torch.optim.Adam([self.log_alpha], lr=alpha_lr)
        self.limit, self.log_std_min, self.log_std_max = limit, log_std_min, log_std_max
        self.eta = float(eta)

    def _q(self, q, o, a):
        return q(torch.cat([o, a], dim=-1)).squeeze(-1)

    def _head(self, o, eps):
        return squash(self.pi(o), eps, self.limit, self.log_std_min, self.log_std_max)

    def train(self, minibatches: List[dict], noise: np.ndarray) -> Dict[str, list]:
        """minibatches: S dicts of the replay buffer's columns; noise [S, 2, B, A] (the draw for s', then for s)."""
        N = len(self.qs)
        logs = dict(q_values=[[] for _ in range(N)], q_losses=[[] for _ in range(N)], diversity=[], policy_losses=[],
                    log_prob_means=[], alphas=[])
        t = lambda x: torch.as_tensor(np.asarray(x, dtype=np.float32))
        for st, mb in enumerate(minibatches):
            o, a, r = t(mb["observations"]), t(mb["actions"]), t(mb["rewards"])
            o2, d = t(mb["next_observations"]), t(np.asarray(mb["dones"]).astype(np.int32))
            alpha = self.log_alpha.detach().exp() if self.learn_alpha else torch.tensor(self.alpha, dtype=torch.float32)
            logs["alphas"].append(float(alpha))
            with torch.no_grad():
                a2, logp_a2 = self._head(o2, t(noise[st, 0]))
                q_targ = fmin_all([self._q(qt, o2, a2) for qt in self.q_targs])
                backup = r + self.gamma * (1 - d) * (q_targ - alpha * logp_a2)
            vals, grads = action_gradients(self.qs, o, a, create_graph=self.eta > 0)
            losses = ((vals - backup) ** 2).mean(1)
            div = diversity(grads)
            loss = losses.sum() + (self.eta * div if self.eta > 0 else 0.0)
            for opt in self.q_opts:
                opt.zero_grad()
            loss.backward()
            for opt in self.q_opts:
                opt.step()
            for i in range(N):
                logs["q_values"][i].append(vals[i].detach().numpy().copy())
                logs["q_losses"][i].append(float(losses[i].detach()))
            logs["diversity"].append(float(div.detach()) if self.eta > 0 else 0.0)
            # the policy loss on the per-row min of the critics just updated, their parameters frozen
            for q in self.qs:
                for p in q.parameters():
                    p.requires_grad = False
            a_pi, logp_pi = self._head(o, t(noise[st, 1]))
            q_all = torch.stack([self._q(q, o, a_pi) for q in self.qs])
            q_pi = q_all.gather(0, first_argmin(q_all)[None])[0]
            loss_pi = (alpha * logp_pi - q_pi).mean()
            self.pi_opt.zero_grad()
            loss_pi.backward()
            self.pi_opt.step()
            for q in self.qs:
                for p in q.parameters():
                    p.requires_grad = True
            logs["policy_losses"].append(float(loss_pi.detach()))
            logs["log_prob_means"].append(float(logp_pi.detach().mean()))
            if self.learn_alpha:
                loss_alpha = -(self.log_alpha * (logp_pi.detach() + self.target_entropy)).mean()
                self.alpha_opt.zero_grad()
                loss_alpha.backward()
                self.alpha_opt.step()
            with torch.no_grad():
                for q, qt in zip(self.qs, self.q_targs):
                    for p, p_targ in zip(q.parameters(), qt.parameters()):
                        p_targ.data.mul_(self.rho)
                        p_targ.data.add_((1 - self.rho) * p.data)
        return logs


# ---- float64 one-step reference ----------------------------------------------------------------------------------
def diversity_f64(q_flats: Sequence[torch.Tensor], q_sizes, obs: torch.Tensor, act: torch.Tensor, hidden="relu"):
    """(D, values [N, B], per-row ReLU margin) of the critics with flat float64 parameters ``q_flats`` at [obs | act],
    differentiable w.r.t. the parameters (the action gradients are taken with create_graph=True)."""
    at = act.detach().clone().requires_grad_(True)
    margin = torch.full((obs.shape[0],), math.inf, dtype=D)
    vals, grads = [], []
    for p in q_flats:
        v, m = mlp(p, q_sizes, torch.cat([obs, at], -1), hidden, "identity")
        (g,) = torch.autograd.grad(v.sum(), at, create_graph=True)
        vals.append(v[:, 0])
        grads.append(g)
        margin = torch.minimum(margin, m)
    return diversity(torch.stack(grads)), torch.stack(vals), margin


def critic_stage_f64(nets: Dict[str, np.ndarray], mb: Dict[str, np.ndarray], eps_next, alpha: float, eta: float,
                     policy_sizes, q_sizes, hidden="relu", gamma=0.99, action_limit=1.0, log_std_min=-20.0,
                     log_std_max=2.0) -> Dict[str, np.ndarray]:
    """The EDAC critic step at the given flat parameters (``nets``: "policy", "q" [N flat vectors], "target_q" [N]):
    a', log pi', the target y over all target critics, every critic's logged values and TD loss, D, and every critic's
    gradient of its TD loss ("td_grads") and of eta D ("div_grads").  ``margin``: per row, over every forward pass."""
    obs, act, rew = _t(mb["observations"]), _t(mb["actions"]), _t(mb["rewards"])
    nobs, done = _t(mb["next_observations"]), _t(np.asarray(mb["dones"], dtype=np.float64))
    out2, margin = mlp(_t(nets["policy"]), policy_sizes, nobs, hidden, "identity")
    a2, logp2 = squash_f64(out2, _t(eps_next), action_limit, log_std_min, log_std_max)
    zs = []
    for qt in nets["target_q"]:
        z, m = mlp(_t(qt), q_sizes, torch.cat([nobs, a2], -1), hidden, "identity")
        zs.append(z[:, 0])
        margin = torch.minimum(margin, m)
    y = (rew + gamma * (1 - done) * (fmin_all(zs) - alpha * logp2)).detach()
    ps = [_t(qf, grad=True) for qf in nets["q"]]
    div, vals, m = diversity_f64(ps, q_sizes, obs, act, hidden)
    margin = torch.minimum(margin, m)
    losses = ((vals - y) ** 2).mean(1)
    td = [g.numpy() for g in torch.autograd.grad(losses.sum(), ps, retain_graph=True)]
    dv = [g.numpy() for g in torch.autograd.grad(eta * div, ps)] if eta > 0 else [np.zeros_like(x) for x in td]
    return dict(y=y.numpy(), values=[v.detach().numpy() for v in vals], losses=[float(x) for x in losses.detach()],
                diversity=float(div.detach()), td_grads=td, div_grads=dv, grads=[a + b for a, b in zip(td, dv)],
                margin=margin.numpy())


def policy_stage_f64(policy: np.ndarray, qs: Sequence[np.ndarray], obs, eps_cur, alpha: float, policy_sizes, q_sizes,
                     hidden="relu", action_limit=1.0, log_std_min=-20.0, log_std_max=2.0,
                     target_entropy=None) -> Dict[str, np.ndarray]:
    """mean(alpha log pi - min_k Q_k(s, a_pi)) with the critics after this step's update, frozen; its gradient w.r.t.
    the policy; mean log pi; the temperature's gradient; the margins; and ``min_gap``, per row the distance between the
    smallest and the second smallest critic value (a gap near 0 makes the argmin critic a matter of rounding)."""
    obs = _t(obs)
    p = _t(policy, grad=True)
    out, margin_pi = mlp(p, policy_sizes, obs, hidden, "identity")
    a, logp = squash_f64(out, _t(eps_cur), action_limit, log_std_min, log_std_max)
    margin_q = torch.full((obs.shape[0],), math.inf, dtype=D)
    vals = []
    for qf in qs:
        z, m = mlp(_t(qf), q_sizes, torch.cat([obs, a], -1), hidden, "identity")
        vals.append(z[:, 0])
        margin_q = torch.minimum(margin_q, m.detach())
    v = torch.stack(vals)
    q_min = v.gather(0, first_argmin(v)[None])[0]
    loss = (alpha * logp - q_min).mean()
    te = -float(a.shape[-1]) if target_entropy is None else float(target_entropy)
    srt = v.detach().sort(0).values
    (g,) = torch.autograd.grad(loss, p)
    return dict(loss=float(loss.detach()), grad=g.numpy(), logp_mean=float(logp.detach().mean()),
                alpha_grad=float(-(logp.detach() + te).mean()), margin_pi=margin_pi.numpy(),
                margin_q=margin_q.numpy(), min_gap=(srt[1] - srt[0]).numpy())
