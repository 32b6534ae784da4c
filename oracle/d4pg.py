"""torch-CPU oracles of D4PG.train.  TEST INFRASTRUCTURE ONLY -- see oracle/__init__.py.

* ``D4pgOracle``: float32, torch autograd and torch.optim.Adam, the D4PG update exactly as the project states it
  (include/b200rl.h, "D4PG"): a' = mu_targ(s'), the triangular projection (oracle/c51.project) of the target critic's
  p(s', a'), the critic's (weighted) cross-entropy against log_softmax, the policy's -mean Q(s, mu(s)) through the critic
  just updated, Polyak averaging.  With prioritized replay it takes each step's drawn leaf priorities and beta and
  returns the importance weights (oracle/per.PerDqnOracle's rule) and the new priorities (KL + eps)^alpha.  It shares
  nothing with the CUDA kernels' hand-derived logit gradients.
* ``d4pg_step_f64``: one critic step and one actor step in float64 from given flat parameters, with the gradients, their
  per-entry scales (the sum over rows of |that row's contribution|) and the per-row ReLU margins of every forward pass,
  as oracle/c51.c51_step_f64 returns them.
"""
from __future__ import annotations

import copy
from typing import Dict, List, Sequence

import numpy as np
import torch

from .c51 import project, support
from .dqn import _layers
from .offpolicy_f64 import _ACT, D, _t, mlp


def per_weights(leaf_priorities, beta: float) -> np.ndarray:
    """w = (min p / p)^beta in float64 (oracle/per.PerDqnOracle's rule; the engine rounds it to float32)."""
    p = np.asarray(leaf_priorities, np.float64)
    return (p.min() / p) ** float(beta)


class D4pgOracle:
    """Deep copies of the policy, the critic and their targets, torch Adams over the copies carrying the given
    optimizers' states; ``train`` runs one D4PG.train call on given minibatches (a minibatch's ``discounts`` [B], when
    present, takes the place of gamma: n-step returns)."""

    def __init__(self, policy, critic, target_policy, target_critic, policy_optimizer, critic_optimizer, n_atoms=51,
                 v_min=-10.0, v_max=10.0, gamma=0.99, rho=0.995, alpha=0.6, eps=1e-6):
        self.pi, self.q = copy.deepcopy(policy), copy.deepcopy(critic)
        self.pi_t, self.q_t = copy.deepcopy(target_policy), copy.deepcopy(target_critic)
        for p in list(self.pi_t.parameters()) + list(self.q_t.parameters()):
            p.requires_grad = False
        self.opt_pi, self.opt_q = (self._adam(net, opt) for net, opt in ((self.pi, policy_optimizer),
                                                                          (self.q, critic_optimizer)))
        self.N, self.v_min, self.v_max = int(n_atoms), float(v_min), float(v_max)
        self.z = torch.from_numpy(support(self.N, self.v_min, self.v_max))
        self.dz = np.float32((self.v_max - self.v_min) / (self.N - 1))
        self.gamma, self.rho, self.alpha, self.eps = gamma, float(rho), float(alpha), float(eps)

    @staticmethod
    def _adam(net, optimizer):
        g = optimizer.param_groups[0]
        opt = torch.optim.Adam(net.parameters(), lr=g["lr"], betas=g["betas"], eps=g["eps"])
        opt.load_state_dict(copy.deepcopy(optimizer.state_dict()))
        return opt

    def train(self, minibatches: List[dict], leaf_priorities: Sequence[np.ndarray] = None,
              betas: Sequence[float] = None) -> Dict[str, list]:
        logs = dict(q1_values=[], q1_losses=[], policy_losses=[], kl=[], weights=[], priorities=[])
        t = lambda x: torch.as_tensor(np.asarray(x, dtype=np.float32))
        z = self.z
        for k, mb in enumerate(minibatches):
            o, a, r = t(mb["observations"]), t(mb["actions"]), t(mb["rewards"])
            o2, d = t(mb["next_observations"]), t(np.asarray(mb["dones"]).astype(np.int32)).float()
            gamma = np.asarray(mb["discounts"], np.float32)[:, None] if "discounts" in mb else np.float32(self.gamma)
            w = None
            if leaf_priorities is not None:
                w64 = per_weights(leaf_priorities[k], betas[k])
                w = torch.as_tensor(w64.astype(np.float32))
                logs["weights"].append(w64)
            with torch.no_grad():
                pt = torch.softmax(self.q_t(torch.cat((o2, self.pi_t(o2)), -1)), -1)
                m = project(pt, r, d, z, np.float32(self.v_min), np.float32(self.v_max), self.dz, gamma)
            logp = torch.log_softmax(self.q(torch.cat((o, a), -1)), -1)
            ce = -(m * logp).sum(-1)
            loss = (ce if w is None else w * ce).mean()
            self.opt_q.zero_grad()
            loss.backward()
            self.opt_q.step()
            kl = (ce.detach() + torch.where(m > 0, m * torch.log(m), torch.zeros_like(m)).sum(-1)).numpy()
            logs["q1_values"].append((logp.detach().exp() * z).sum(-1).numpy().copy())
            logs["q1_losses"].append(float(loss.detach()))
            logs["kl"].append(kl.copy())
            logs["priorities"].append((np.maximum(kl.astype(np.float64), 0.0) + self.eps) ** self.alpha)
            q_pi = (torch.softmax(self.q(torch.cat((o, self.pi(o)), -1)), -1) * z).sum(-1)
            ploss = -q_pi.mean()
            self.opt_pi.zero_grad()
            ploss.backward()
            self.opt_pi.step()
            logs["policy_losses"].append(float(ploss.detach()))
            with torch.no_grad():
                for src, dst in ((self.pi, self.pi_t), (self.q, self.q_t)):
                    for ps, pd in zip(src.parameters(), dst.parameters()):
                        pd.mul_(self.rho).add_((1.0 - self.rho) * ps)
        return logs


def _net(flat, sizes, x, hidden, out):
    h = x
    for l, (W, b) in enumerate(_layers(flat, sizes)):
        h = h @ W.T + b
        h = _ACT[hidden if l < len(sizes) - 2 else out](h)
    return h


def d4pg_step_f64(nets: Dict[str, np.ndarray], mb: Dict[str, np.ndarray], policy_sizes: Sequence[int],
                  q_sizes: Sequence[int], n_atoms: int, v_min: float, v_max: float, hidden="relu", gamma=0.99,
                  q_after=None, weights=None):
    """One D4PG step in float64 from flat parameters ``nets`` (policy, q1, target_policy, target_q1); the support is
    the float32 one the engine uses.  The actor step runs through ``q_after`` (the critic after this step's update;
    default nets["q1"]).  ``gamma`` may be a per-row discount [B]; ``weights`` [B] the importance weights.  Returns
    dict(q_values, loss, kl, m, grad_q, scale_q, policy_loss, grad_pi, scale_pi, margin (critic stage), margin_pi
    (the policy pass), margin_q (the critic pass on [s | mu(s)]))."""
    obs, act, rew = _t(mb["observations"]), _t(mb["actions"]), _t(mb["rewards"])
    nobs, done = _t(mb["next_observations"]), _t(np.asarray(mb["dones"], dtype=np.float64))
    B, N = obs.shape[0], int(n_atoms)
    z = _t(support(N, v_min, v_max))
    w = torch.ones(B, dtype=D) if weights is None else _t(weights)
    g = np.asarray(gamma, np.float64)[:, None] if np.ndim(gamma) else gamma
    with torch.no_grad():
        a2, margin = mlp(_t(nets["target_policy"]), policy_sizes, nobs, hidden, "tanh")
        qt, m2 = mlp(_t(nets["target_q1"]), q_sizes, torch.cat([nobs, a2], -1), hidden, "identity")
        margin = torch.minimum(margin, m2)
        m = project(torch.softmax(qt, -1), rew, done, z, v_min, v_max, (v_max - v_min) / (N - 1), g)
    p = _t(nets["q1"], grad=True)
    q, m3 = mlp(p, q_sizes, torch.cat([obs, act], -1), hidden, "identity")
    margin = torch.minimum(margin, m3)
    logp = torch.log_softmax(q, -1)
    ce = -(m * logp).sum(-1)
    loss = (w * ce).mean()
    (grad_q,) = torch.autograd.grad(loss, p)
    kl = ce.detach() + torch.where(m > 0, m * torch.log(torch.where(m > 0, m, torch.ones_like(m))),
                                   torch.zeros_like(m)).sum(-1)

    def critic_row(flat_p, x, mi, wi):
        return -wi * (mi * torch.log_softmax(_net(flat_p, q_sizes, x[None], hidden, "identity")[0], -1)).sum() / B
    per_row = torch.func.vmap(torch.func.grad(critic_row), in_dims=(None, 0, 0, 0))(
        p.detach(), torch.cat([obs, act], -1), m, w)
    scale_q = per_row.abs().sum(0)

    qa = _t(nets["q1"] if q_after is None else q_after)
    pp = _t(nets["policy"], grad=True)
    a, margin_pi = mlp(pp, policy_sizes, obs, hidden, "tanh")
    qpi, margin_q = mlp(qa, q_sizes, torch.cat([obs, a], -1), hidden, "identity")
    ploss = -(torch.softmax(qpi, -1) * z).sum(-1).mean()
    (grad_pi,) = torch.autograd.grad(ploss, pp)

    def policy_row(flat_p, o):
        ai = _net(flat_p, policy_sizes, o[None], hidden, "tanh")
        x = _net(qa, q_sizes, torch.cat([o[None], ai], -1), hidden, "identity")[0]
        return -(torch.softmax(x, -1) * z).sum() / B
    scale_pi = torch.func.vmap(torch.func.grad(policy_row), in_dims=(None, 0))(pp.detach(), obs).abs().sum(0)
    return dict(q_values=(logp.detach().exp() * z).sum(-1).numpy(), loss=float(loss.detach()), kl=kl.numpy(),
                m=m.numpy(), grad_q=grad_q.numpy(), scale_q=scale_q.numpy(), policy_loss=float(ploss.detach()),
                grad_pi=grad_pi.numpy(), scale_pi=scale_pi.numpy(), margin=margin.numpy(),
                margin_pi=margin_pi.numpy(), margin_q=margin_q.numpy())

