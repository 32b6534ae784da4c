"""torch-CPU oracles of REDQ.train.  TEST INFRASTRUCTURE ONLY -- see oracle/__init__.py.

* ``RedqOracle``: float32, torch autograd and torch.optim.Adam, the REDQ update exactly as the project states it
  (include/b200rl.h, "REDQ"; Chen, Wang, Zhou & Ross 2021, Algorithm 1): SAC's squashed-Gaussian head (oracle/sac.py),
  a target that takes ``torch.fmin`` over the step's M drawn target critics, one Adam step per critic on its own MSE,
  and on policy steps a policy loss on the mean of all N critics just updated.  It shares nothing with the CUDA kernels'
  hand-derived gradients.
* ``critic_stage_f64`` / ``policy_stage_f64``: one step's stages in float64 from given flat parameters, with the
  per-row ReLU margins of every forward pass.
* ``policy_steps``: the steps of a call that run the policy step.
"""
from __future__ import annotations

import copy
import math
from typing import Dict, List, Sequence

import numpy as np
import torch

from .offpolicy_f64 import D, _grad, _t, mlp
from .offpolicy_f64 import squash as squash_f64
from .sac import squash


def policy_steps(S: int, G: int) -> List[int]:
    """The steps st of an S-step call that take a policy step: (st + 1) % G == 0, and the last step."""
    return [st for st in range(S) if (st + 1) % G == 0 or st == S - 1]


def fmin_all(qs: Sequence[torch.Tensor]) -> torch.Tensor:
    """torch.fmin over the list in order: a NaN loses to a number."""
    out = qs[0]
    for q in qs[1:]:
        out = torch.fmin(out, q)
    return out


class RedqOracle:
    """Holds pi, the N critics (deep copies), their targets, torch Adams and log_alpha; ``train`` runs one REDQ.train
    call on given minibatches, noise and subsets."""

    def __init__(self, pi: torch.nn.Module, qs: Sequence[torch.nn.Module], pi_lr=1e-3, q_lr=1e-3, gamma=0.99,
                 rho=0.995, alpha=0.2, learn_alpha=False, target_entropy=None, alpha_lr=3e-4, limit=1.0,
                 log_std_min=-20.0, log_std_max=2.0, policy_delay=1):
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
        self.G = int(policy_delay)

    def _q(self, q, o, a):
        return q(torch.cat([o, a], dim=-1)).squeeze(-1)

    def _head(self, o, eps):
        return squash(self.pi(o), eps, self.limit, self.log_std_min, self.log_std_max)

    def train(self, minibatches: List[dict], noise: np.ndarray, subsets: np.ndarray) -> Dict[str, list]:
        """minibatches: S dicts of the replay buffer's columns; noise [S, 2, B, A] (the draw for s', then for s; slot
        1 is read on policy steps only); subsets [S, M] the target critics of each step."""
        N = len(self.qs)
        logs = dict(q_values=[[] for _ in range(N)], q_losses=[[] for _ in range(N)], policy_losses=[],
                    log_prob_means=[], alphas=[])
        t = lambda x: torch.as_tensor(np.asarray(x, dtype=np.float32))
        S = len(minibatches)
        pol = set(policy_steps(S, self.G))
        for st, mb in enumerate(minibatches):
            o, a, r = t(mb["observations"]), t(mb["actions"]), t(mb["rewards"])
            o2, d = t(mb["next_observations"]), t(np.asarray(mb["dones"]).astype(np.int32))
            alpha = self.log_alpha.detach().exp() if self.learn_alpha else torch.tensor(self.alpha, dtype=torch.float32)
            logs["alphas"].append(float(alpha))
            with torch.no_grad():
                a2, logp_a2 = self._head(o2, t(noise[st, 0]))
                q_targ = fmin_all([self._q(self.q_targs[int(k)], o2, a2) for k in subsets[st]])
                backup = r + self.gamma * (1 - d) * (q_targ - alpha * logp_a2)
            for i, (q, opt) in enumerate(zip(self.qs, self.q_opts)):
                qv = self._q(q, o, a)
                loss_q = ((qv - backup) ** 2).mean()
                opt.zero_grad()
                loss_q.backward()
                opt.step()
                logs["q_values"][i].append(qv.detach().numpy().copy())
                logs["q_losses"][i].append(float(loss_q.detach()))
            if st in pol:  # the policy loss on the mean of the critics just updated, their parameters frozen
                for q in self.qs:
                    for p in q.parameters():
                        p.requires_grad = False
                a_pi, logp_pi = self._head(o, t(noise[st, 1]))
                q_pi = torch.stack([self._q(q, o, a_pi) for q in self.qs]).mean(0)
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
def critic_stage_f64(nets: Dict[str, np.ndarray], mb: Dict[str, np.ndarray], eps_next, subset, alpha: float,
                     policy_sizes, q_sizes, hidden="relu", gamma=0.99, action_limit=1.0, log_std_min=-20.0,
                     log_std_max=2.0) -> Dict[str, np.ndarray]:
    """The REDQ critic step at the given flat parameters (``nets``: "policy", "q" [N flat vectors], "target_q" [N]):
    a', log pi', the target y over the ``subset``'s target critics, and every critic's logged values, loss and
    gradient.  ``margin``: per row, over every forward pass of the stage."""
    obs, act, rew = _t(mb["observations"]), _t(mb["actions"]), _t(mb["rewards"])
    nobs, done = _t(mb["next_observations"]), _t(np.asarray(mb["dones"], dtype=np.float64))
    out2, margin = mlp(_t(nets["policy"]), policy_sizes, nobs, hidden, "identity")
    a2, logp2 = squash_f64(out2, _t(eps_next), action_limit, log_std_min, log_std_max)
    zs = []
    for k in subset:
        z, m = mlp(_t(nets["target_q"][int(k)]), q_sizes, torch.cat([nobs, a2], -1), hidden, "identity")
        zs.append(z[:, 0])
        margin = torch.minimum(margin, m)
    y = rew + gamma * (1 - done) * (fmin_all(zs) - alpha * logp2)
    out = dict(y=y.detach().numpy(), values=[], losses=[], grads=[])
    for qf in nets["q"]:
        p = _t(qf, grad=True)
        qv, m = mlp(p, q_sizes, torch.cat([obs, act], -1), hidden, "identity")
        margin = torch.minimum(margin, m)
        loss = ((qv[:, 0] - y.detach()) ** 2).mean()
        out["values"].append(qv.detach()[:, 0].numpy())
        out["losses"].append(float(loss.detach()))
        out["grads"].append(_grad(loss, p))
    out["margin"] = margin.numpy()
    return out


def policy_stage_f64(policy: np.ndarray, qs: Sequence[np.ndarray], obs, eps_cur, alpha: float, policy_sizes, q_sizes,
                     hidden="relu", action_limit=1.0, log_std_min=-20.0, log_std_max=2.0,
                     target_entropy=None) -> Dict[str, np.ndarray]:
    """mean(alpha log pi - mean_k Q_k(s, a_pi)) with the critics after this step's update, frozen; its gradient w.r.t.
    the policy; mean log pi; and the temperature's gradient -mean(log pi + target_entropy) w.r.t. log_alpha."""
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
    loss = (alpha * logp - torch.stack(vals).mean(0)).mean()
    te = -float(a.shape[-1]) if target_entropy is None else float(target_entropy)
    return dict(loss=float(loss.detach()), grad=_grad(loss, p), logp_mean=float(logp.detach().mean()),
                alpha_grad=float(-(logp.detach() + te).mean()), margin_pi=margin_pi.numpy(),
                margin_q=margin_q.numpy())
