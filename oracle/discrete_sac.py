"""torch-CPU oracle of DiscreteSAC.train.  TEST INFRASTRUCTURE ONLY -- see oracle/__init__.py.

A float32 restatement of discrete SAC (Christodoulou 2019, "Soft Actor-Critic for Discrete Action Settings") in the
order of oracle/sac.py: one critic step, one policy step with the critics just updated, the optional temperature step,
polyak.  With log pi = log_softmax of the policy's logits (x - max - log(sum exp(x - max)), never log(softmax)) and
alpha = exp(log_alpha) at the start of the step:

  critics     V(s') = sum_a' pi'(a') (min(Q1targ, Q2targ)(s', a') - alpha log pi'(a')), pi' the policy at s',
              y = r + gamma (1 - d) V(s'); one Adam step each on mean_B (Qk(s)[a] - y)^2
  policy      one Adam step on mean_B sum_a pi(a) (alpha log pi(a) - min(Q1, Q2)(s, a)), no gradient into the critics
  alpha       learn_alpha: one Adam step on -mean_B(log_alpha (E + target_entropy)), E = sum_a pi(a) log pi(a);
              target_entropy defaults to 0.98 log(n)
  polyak      both target critics

Every gradient comes from autograd and every optimizer is torch.optim.Adam, so the oracle shares nothing with the CUDA
kernels' closed-form head gradients.  ``critic_stage_f64`` / ``policy_stage_f64`` are the float64 one-step reference
in the style of oracle/offpolicy_f64.py: each stage takes its inputs as arguments (flat parameter vectors) and returns
the losses, logged values and gradients in float64.
"""
from __future__ import annotations

import copy
import math
from typing import Dict, List, Sequence

import numpy as np
import torch

from .offpolicy_f64 import D, _t, mlp


def default_target_entropy(n: int) -> float:
    """0.98 log(n), the paper's choice."""
    return 0.98 * math.log(n)


def soft_value(logits: torch.Tensor, q1t: torch.Tensor, q2t: torch.Tensor, alpha) -> torch.Tensor:
    """V(s') = sum_a pi(a) (min(q1t, q2t)(a) - alpha log pi(a)) per row."""
    logp = torch.log_softmax(logits, dim=-1)
    return (logp.exp() * (torch.min(q1t, q2t) - alpha * logp)).sum(-1)


def policy_terms(logits: torch.Tensor, q1: torch.Tensor, q2: torch.Tensor, alpha):
    """(L [B] = sum_a pi (alpha log pi - min(q1, q2)), E [B] = sum_a pi log pi)."""
    logp = torch.log_softmax(logits, dim=-1)
    p = logp.exp()
    return (p * (alpha * logp - torch.min(q1, q2))).sum(-1), (p * logp).sum(-1)


def closed_form_logit_grad(logits: torch.Tensor, q1: torch.Tensor, q2: torch.Tensor, alpha) -> torch.Tensor:
    """The engine's head gradient d(mean_B L)/d logits = pi_k (c_k - sum_a pi_a c_a) / B, c = alpha log pi - min(q1, q2)
    (the tests check it against autograd)."""
    logp = torch.log_softmax(logits, dim=-1)
    p = logp.exp()
    c = alpha * logp - torch.min(q1, q2)
    return p * (c - (p * c).sum(-1, keepdim=True)) / logits.shape[0]


class DiscreteSacOracle:
    """Holds pi, q1, q2 (deep copies of the given modules), their targets, torch Adams and log_alpha; ``train`` runs
    one DiscreteSAC.train call."""

    def __init__(self, pi: torch.nn.Module, q1: torch.nn.Module, q2: torch.nn.Module, pi_lr=1e-3, q_lr=1e-3,
                 gamma=0.99, rho=0.995, alpha=0.2, learn_alpha=False, target_entropy=None, alpha_lr=3e-4):
        self.pi, self.q1, self.q2 = copy.deepcopy(pi), copy.deepcopy(q1), copy.deepcopy(q2)
        self.q1_targ, self.q2_targ = copy.deepcopy(q1), copy.deepcopy(q2)
        for p in list(self.q1_targ.parameters()) + list(self.q2_targ.parameters()):
            p.requires_grad = False
        self.pi_opt = torch.optim.Adam(self.pi.parameters(), lr=pi_lr)
        self.q1_opt = torch.optim.Adam(self.q1.parameters(), lr=q_lr)
        self.q2_opt = torch.optim.Adam(self.q2.parameters(), lr=q_lr)
        n = [m for m in self.pi.modules() if isinstance(m, torch.nn.Linear)][-1].out_features
        self.gamma, self.rho, self.alpha, self.learn_alpha = gamma, rho, alpha, learn_alpha
        self.target_entropy = float(default_target_entropy(n) if target_entropy is None else target_entropy)
        self.log_alpha = torch.nn.Parameter(torch.tensor(float(np.log(alpha)), dtype=torch.float32))
        self.alpha_opt = torch.optim.Adam([self.log_alpha], lr=alpha_lr)

    def train(self, minibatches: List[dict]) -> Dict[str, list]:
        """minibatches: S dicts of the replay buffer's columns, actions as indices [B] (or [B, 1])."""
        logs = dict(q1_values=[], q2_values=[], q1_losses=[], q2_losses=[], policy_losses=[], log_prob_means=[],
                    alphas=[])
        t = lambda x: torch.as_tensor(np.asarray(x, dtype=np.float32))
        for mb in minibatches:
            o, r = t(mb["observations"]), t(mb["rewards"])
            a = torch.as_tensor(np.asarray(mb["actions"]).reshape(-1).astype(np.int64))
            o2, d = t(mb["next_observations"]), t(np.asarray(mb["dones"]).astype(np.int32))
            alpha = self.log_alpha.detach().exp() if self.learn_alpha else torch.tensor(self.alpha, dtype=torch.float32)
            logs["alphas"].append(float(alpha))
            with torch.no_grad():
                v = soft_value(self.pi(o2), self.q1_targ(o2), self.q2_targ(o2), alpha)
                backup = r + self.gamma * (1 - d) * v
            for i, (q, opt) in enumerate(((self.q1, self.q1_opt), (self.q2, self.q2_opt)), 1):
                qv = q(o).gather(1, a[:, None]).squeeze(1)
                loss_q = ((qv - backup) ** 2).mean()
                opt.zero_grad()
                loss_q.backward()
                opt.step()
                logs[f"q{i}_values"].append(qv.detach().numpy().copy())
                logs[f"q{i}_losses"].append(float(loss_q.detach()))
            with torch.no_grad():  # the critics just updated, no gradient into them
                q1v, q2v = self.q1(o), self.q2(o)
            L, E = policy_terms(self.pi(o), q1v, q2v, alpha)
            loss_pi = L.mean()
            self.pi_opt.zero_grad()
            loss_pi.backward()
            self.pi_opt.step()
            logs["policy_losses"].append(float(loss_pi.detach()))
            logs["log_prob_means"].append(float(E.detach().mean()))
            if self.learn_alpha:
                loss_alpha = -(self.log_alpha * (E.detach() + self.target_entropy)).mean()
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
def critic_stage_f64(q1, q2, q1t, q2t, pi, q_sizes: Sequence[int], pi_sizes: Sequence[int], obs, act, rew, next_obs,
                     done, alpha: float, gamma: float, hidden: str = "relu") -> Dict[str, np.ndarray]:
    """The critic step at the given flat parameters: y, each critic's logged Q(s)[a], loss and gradient."""
    a = torch.as_tensor(np.asarray(act).reshape(-1).astype(np.int64))
    o, o2 = _t(obs), _t(next_obs)
    with torch.no_grad():
        logits2, _ = mlp(_t(pi), pi_sizes, o2, hidden, "identity")
        t1, _ = mlp(_t(q1t), q_sizes, o2, hidden, "identity")
        t2, _ = mlp(_t(q2t), q_sizes, o2, hidden, "identity")
        y = _t(rew) + gamma * (1.0 - _t(done)) * soft_value(logits2, t1, t2, alpha)
    out = dict(y=y.numpy())
    for k, flat in ((1, q1), (2, q2)):
        w = _t(flat, grad=True)
        qv, margin = mlp(w, q_sizes, o, hidden, "identity")
        qa = qv.gather(1, a[:, None]).squeeze(1)
        loss = ((qa - y) ** 2).mean()
        loss.backward()
        out[f"q{k}_values"], out[f"q{k}_loss"] = qa.detach().numpy(), float(loss.detach())
        out[f"q{k}_grad"], out[f"q{k}_margin"] = w.grad.numpy(), margin.numpy()
    return out


def policy_stage_f64(pi, q1, q2, q_sizes: Sequence[int], pi_sizes: Sequence[int], obs, alpha: float,
                     target_entropy: float, log_alpha: float = 0.0, hidden: str = "relu") -> Dict[str, np.ndarray]:
    """The policy step at the given flat parameters (q1, q2: the critics after their step): the loss, mean E, the
    policy gradient, and the temperature loss's gradient w.r.t. log_alpha."""
    o = _t(obs)
    with torch.no_grad():
        a1, _ = mlp(_t(q1), q_sizes, o, hidden, "identity")
        a2, _ = mlp(_t(q2), q_sizes, o, hidden, "identity")
    w = _t(pi, grad=True)
    logits, margin = mlp(w, pi_sizes, o, hidden, "identity")
    L, E = policy_terms(logits, a1, a2, alpha)
    L.mean().backward()
    la = torch.tensor(float(log_alpha), dtype=D, requires_grad=True)
    (-(la * (E.detach() + target_entropy)).mean()).backward()
    return dict(loss=float(L.detach().mean()), ent_mean=float(E.detach().mean()), grad=w.grad.numpy(),
                alpha_grad=float(la.grad), margin=margin.numpy())
