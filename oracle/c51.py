"""torch-CPU oracles of C51.train.  TEST INFRASTRUCTURE ONLY -- see oracle/__init__.py.

* ``C51Oracle``: float32, torch autograd and torch.optim.Adam, the C51 update exactly as the project states it
  (include/b200rl.h): the support z_i = float32(v_min + i dz), a* = argmax of the expected values, the triangular
  projection of Q_targ's p(s', a*), the cross-entropy against log_softmax(Q(s)), DQN's target copies.  It shares
  nothing with the CUDA kernel's hand-derived gradient.
* ``c51_step_f64``: one step in float64 from given flat parameters, with per-entry gradient scales, ReLU margins and the
  gap between the two largest expected Q(s') values of the net that picks a*.
* ``project_f64``: Bellemare et al.'s Algorithm 1 (floor / ceil, the l == u case), written independently of the
  triangular form the engine and the oracles use, so that the two can be held against each other.
"""
from __future__ import annotations

import math
from typing import Dict, List, Sequence

import numpy as np
import torch

from .dqn import DqnOracle, _layers
from .offpolicy_f64 import _ACT, D, _t, mlp


def support(n_atoms: int, v_min: float, v_max: float) -> np.ndarray:
    """z_i = float32(v_min + i dz), dz = (v_max - v_min) / (N - 1), evaluated in double (not linspace)."""
    dz = (v_max - v_min) / (n_atoms - 1)
    return np.asarray([v_min + i * dz for i in range(n_atoms)], np.float64).astype(np.float32)


def project(p_next: torch.Tensor, rew: torch.Tensor, done: torch.Tensor, z: torch.Tensor, v_min, v_max, dz,
            gamma) -> torch.Tensor:
    """m [B, N] = sum_j max(0, 1 - |b_j - i|) p_j with b_j = (clamp(r + gamma (1 - d) z_j, v_min, v_max) - v_min) / dz
    (Dopamine's triangular form), in the dtype of its tensor arguments (the scalars are cast to it)."""
    dt = p_next.dtype
    v_min, v_max, dz, gamma = (torch.tensor(x, dtype=dt) for x in (v_min, v_max, dz, gamma))
    tz = (rew[:, None] + gamma * (1 - done[:, None]) * z[None]).clamp(v_min, v_max)
    b = (tz - v_min) / dz
    i = torch.arange(z.numel(), dtype=dt)
    w = (1 - (b[:, :, None] - i[None, None, :]).abs()).clamp(min=0)  # [B, j, i]
    return (w * p_next[:, :, None]).sum(1)


def project_f64(p_next, rew, done, z, v_min: float, v_max: float, gamma: float) -> np.ndarray:
    """Bellemare, Dabney & Munos (2017), Algorithm 1, in float64: each atom's mass goes to its floor and ceiling
    neighbours in proportion to the distances, all of it to l when l == u."""
    p_next, z = np.asarray(p_next, np.float64), np.asarray(z, np.float64)
    B, N = p_next.shape
    dz = (v_max - v_min) / (N - 1)
    m = np.zeros((B, N))
    for r in range(B):
        for j in range(N):
            tz = min(max(float(rew[r]) + gamma * (1.0 - float(done[r])) * z[j], v_min), v_max)
            b = (tz - v_min) / dz
            l, u = min(math.floor(b), N - 1), min(math.ceil(b), N - 1)
            if l == u:
                m[r, l] += p_next[r, j]
            else:
                m[r, l] += p_next[r, j] * (u - b)
                m[r, u] += p_next[r, j] * (b - l)
    return m


def _log_dist(logits: torch.Tensor, N: int) -> torch.Tensor:
    return torch.log_softmax(logits.unflatten(-1, (-1, N)), dim=-1)


class C51Oracle(DqnOracle):
    """DqnOracle with the categorical head: ``train`` runs one C51.train call."""

    def __init__(self, q, q_targ, optimizer, n_atoms=51, v_min=-10.0, v_max=10.0, **kw):
        super().__init__(q, q_targ, optimizer, **kw)
        self.N, self.v_min, self.v_max = int(n_atoms), float(v_min), float(v_max)
        self.z = torch.from_numpy(support(self.N, self.v_min, self.v_max))
        self.dz = np.float32((self.v_max - self.v_min) / (self.N - 1))

    def train(self, minibatches: List[dict]) -> Dict[str, list]:
        logs = dict(q1_values=[], q1_losses=[], copied=[])
        t = lambda x: torch.as_tensor(np.asarray(x, dtype=np.float32))
        N, z = self.N, self.z
        for mb in minibatches:
            o, a, r = t(mb["observations"]), t(mb["actions"]).reshape(-1).long(), t(mb["rewards"])
            o2, d = t(mb["next_observations"]), t(np.asarray(mb["dones"]).astype(np.int32))
            rows = torch.arange(o.shape[0])
            with torch.no_grad():
                pt = _log_dist(self.q_targ(o2), N).exp()
                pick = _log_dist(self.q(o2), N).exp() if self.double_q else pt
                a_star = (pick * z).sum(-1).argmax(1)
                m = project(pt[rows, a_star], r, d.float(), z, np.float32(self.v_min), np.float32(self.v_max),
                            self.dz, np.float32(self.gamma))
            logp = _log_dist(self.q(o), N)[rows, a]
            loss = -(m * logp).sum(-1).mean()
            self.opt.zero_grad()
            loss.backward()
            self.opt.step()
            logs["q1_values"].append((logp.detach().exp() * z).sum(-1).numpy().copy())
            logs["q1_losses"].append(float(loss.detach()))
            copy_now = self.step_count() % self.interval == 0
            if copy_now:
                self.q_targ.load_state_dict(self.q.state_dict())
            logs["copied"].append(copy_now)
        return logs


def c51_step_f64(q_flat, targ_flat, mb: Dict[str, np.ndarray], sizes: Sequence[int], n_atoms: int, v_min: float,
                 v_max: float, hidden="relu", gamma=0.99, double_q=False):
    """One C51 step's loss, logged Q(s, a) and gradient w.r.t. the Q network in float64 (the support is the float32
    one the engine uses).  Returns dict(q_values, loss, grad (flat), scale (flat: per entry the sum over rows of |that
    row's contribution|), m (the projected targets [B, N]), margin (per row, over every forward pass), gap (per row: the
    two largest expected Q(s') values of the net that picks a* apart; +inf for one action))."""
    obs, act, rew = _t(mb["observations"]), np.asarray(mb["actions"]).reshape(-1), _t(mb["rewards"])
    nobs, done = _t(mb["next_observations"]), _t(np.asarray(mb["dones"], dtype=np.float64))
    B, N = obs.shape[0], int(n_atoms)
    z = _t(support(N, v_min, v_max))
    rows = torch.arange(B)
    with torch.no_grad():
        qt, margin = mlp(_t(targ_flat), sizes, nobs, hidden, "identity")
        pt = _log_dist(qt, N).exp()
        pick = pt
        if double_q:
            qn, m2 = mlp(_t(q_flat), sizes, nobs, hidden, "identity")
            margin = torch.minimum(margin, m2)
            pick = _log_dist(qn, N).exp()
        ev = (pick * z).sum(-1)
        gap = torch.full((B,), math.inf, dtype=D)
        if ev.shape[1] > 1:
            top2 = ev.topk(2, dim=1).values
            gap = top2[:, 0] - top2[:, 1]
        m = project(pt[rows, ev.argmax(1)], rew, done, z, v_min, v_max, (v_max - v_min) / (N - 1), gamma)
    p = _t(q_flat, grad=True)
    q, m3 = mlp(p, sizes, obs, hidden, "identity")
    margin = torch.minimum(margin, m3)
    a = torch.as_tensor(act.astype(np.int64))
    logp = _log_dist(q, N)[rows, a]
    loss = -(m * logp).sum(-1).mean()
    (grad,) = torch.autograd.grad(loss, p)

    def row_loss(flat_p, o, ai, mi):  # ai: the row's action one-hot [n], mi: its target [N]
        h = o[None]
        for l, (W, b) in enumerate(_layers(flat_p, sizes)):
            h = h @ W.T + b
            if l < len(sizes) - 2:
                h = _ACT[hidden](h)
        lp = _log_dist(h[0], N)
        return -((ai[:, None] * lp) * mi[None]).sum() / B
    onehot = torch.nn.functional.one_hot(a, sizes[-1] // N).to(D)
    per_row = torch.func.vmap(torch.func.grad(row_loss), in_dims=(None, 0, 0, 0))(p.detach(), obs, onehot, m)
    scale = per_row.abs().sum(0)
    return dict(q_values=(logp.detach().exp() * z).sum(-1).numpy(), loss=float(loss.detach()), grad=grad.numpy(),
                scale=scale.numpy(), m=m.numpy(), margin=margin.numpy(), gap=gap.numpy())
