"""torch-CPU oracles of DQN.train.  TEST INFRASTRUCTURE ONLY -- see oracle/__init__.py.

* ``DqnOracle``: float32, torch autograd and torch.optim.Adam, the DQN / Double DQN update exactly as the project
  states it (F.smooth_l1_loss against y = r + gamma (1 - d) v, an exact target copy whenever the Q optimizer's step
  count reaches a multiple of the interval).  It shares nothing with the CUDA kernels' hand-derived backward pass.
* ``dqn_step_f64``: one step in float64 from given flat parameters, with per-entry gradient scales (the sum over rows
  of the magnitudes of each row's contribution, as in oracle/onpolicy_f64.py), the per-row ReLU margins of every
  forward pass (oracle/offpolicy_f64.mlp) and, for Double DQN, the per-row gap between the two largest Q(s') values.
"""
from __future__ import annotations

import copy
import math
from typing import Dict, List, Sequence

import numpy as np
import torch
import torch.nn.functional as F

from .offpolicy_f64 import _ACT, D, _t, mlp


def _layers(flat: torch.Tensor, sizes: Sequence[int]):
    """[(W [out, in], b)] views of a flat parameter vector in parameters_to_vector order."""
    out, o = [], 0
    for n_in, n_out in zip(sizes[:-1], sizes[1:]):
        W = flat[o:o + n_out * n_in].view(n_out, n_in)
        o += n_out * n_in
        out.append((W, flat[o:o + n_out]))
        o += n_out
    return out


def td_values(q_next_targ: torch.Tensor, q_next_online, double_q: bool) -> torch.Tensor:
    """v per row: Q_targ(s')[argmax Q(s')] (Double DQN) or max Q_targ(s') -- torch's max / argmax (NaN wins, ties go to
    the first index)."""
    if double_q:
        a_star = q_next_online.argmax(1)
        return q_next_targ.gather(1, a_star[:, None]).squeeze(1)
    return q_next_targ.max(1).values


class DqnOracle:
    """Deep copies of the Q network and its target, a torch Adam over the copy carrying the given optimizer's state
    (so the step count, and with it the copy schedule, continues from there); ``train`` runs one DQN.train call."""

    def __init__(self, q: torch.nn.Module, q_targ: torch.nn.Module, optimizer: torch.optim.Optimizer, gamma=0.99,
                 target_update_interval=1000, double_q=False):
        self.q, self.q_targ = copy.deepcopy(q), copy.deepcopy(q_targ)
        for p in self.q_targ.parameters():
            p.requires_grad = False
        g = optimizer.param_groups[0]
        self.opt = torch.optim.Adam(self.q.parameters(), lr=g["lr"], betas=g["betas"], eps=g["eps"])
        self.opt.load_state_dict(copy.deepcopy(optimizer.state_dict()))
        self.gamma, self.interval, self.double_q = gamma, int(target_update_interval), bool(double_q)

    def step_count(self) -> int:
        st = self.opt.state.get(next(iter(self.q.parameters())), {})
        return int(float(st["step"])) if "step" in st else 0

    def train(self, minibatches: List[dict]) -> Dict[str, list]:
        logs = dict(q1_values=[], q1_losses=[], copied=[])
        t = lambda x: torch.as_tensor(np.asarray(x, dtype=np.float32))
        for mb in minibatches:
            o, a, r = t(mb["observations"]), t(mb["actions"]).reshape(-1), t(mb["rewards"])
            o2, d = t(mb["next_observations"]), t(np.asarray(mb["dones"]).astype(np.int32))
            with torch.no_grad():
                v = td_values(self.q_targ(o2), self.q(o2) if self.double_q else None, self.double_q)
                y = r + self.gamma * (1 - d) * v
            q_sa = self.q(o).gather(1, a.long()[:, None]).squeeze(1)
            loss = F.smooth_l1_loss(q_sa, y)
            self.opt.zero_grad()
            loss.backward()
            self.opt.step()
            logs["q1_values"].append(q_sa.detach().numpy().copy())
            logs["q1_losses"].append(float(loss.detach()))
            copy_now = self.step_count() % self.interval == 0
            if copy_now:
                self.q_targ.load_state_dict(self.q.state_dict())
            logs["copied"].append(copy_now)
        return logs


def huber_f64(delta: torch.Tensor) -> torch.Tensor:
    """Per-row Huber loss (beta = 1) in float64; its autograd gradient is clamp(delta, -1, 1)."""
    ad = delta.abs()
    return torch.where(ad < 1, 0.5 * delta * delta, ad - 0.5)


def dqn_step_f64(q_flat, targ_flat, mb: Dict[str, np.ndarray], sizes: Sequence[int], hidden="relu", gamma=0.99,
                 double_q=False):
    """One DQN step's loss, logged Q(s, a) and gradient w.r.t. the Q network in float64.  Returns dict(q_values, loss,
    grad (flat), scale (flat: per entry the sum over rows of |that row's contribution|), y, margin (per row, over every
    forward pass), gap (per row: the two largest Q(s') values apart, Double DQN; +inf otherwise), delta)."""
    obs, act, rew = _t(mb["observations"]), np.asarray(mb["actions"]).reshape(-1), _t(mb["rewards"])
    nobs, done = _t(mb["next_observations"]), _t(np.asarray(mb["dones"], dtype=np.float64))
    B, n = obs.shape[0], sizes[-1]
    with torch.no_grad():
        qt, margin = mlp(_t(targ_flat), sizes, nobs, hidden, "identity")
        gap = torch.full((B,), math.inf, dtype=D)
        qn = None
        if double_q:
            qn, m2 = mlp(_t(q_flat), sizes, nobs, hidden, "identity")
            margin = torch.minimum(margin, m2)
            if n > 1:
                top2 = qn.topk(2, dim=1).values
                gap = top2[:, 0] - top2[:, 1]
        y = rew + gamma * (1 - done) * td_values(qt, qn, double_q)
    p = _t(q_flat, grad=True)
    q, m3 = mlp(p, sizes, obs, hidden, "identity")
    margin = torch.minimum(margin, m3)
    a = torch.as_tensor(act.astype(np.int64))
    q_sa = q.gather(1, a[:, None]).squeeze(1)
    delta = q_sa - y
    rows = huber_f64(delta)
    loss = rows.mean()
    (grad,) = torch.autograd.grad(loss, p, retain_graph=True)
    # per-row gradients (vmapped over rows) for the scale: |d row_i / d theta| summed over rows
    def row_loss(flat_p, o, ai, yi):
        h = o[None]
        for l, (W, b) in enumerate(_layers(flat_p, sizes)):
            h = h @ W.T + b
            if l < len(sizes) - 2:
                h = _ACT[hidden](h)
        return huber_f64((h[0] * ai).sum() - yi) / B  # ai: the row's action one-hot
    onehot = F.one_hot(a, n).to(D)
    per_row = torch.func.vmap(torch.func.grad(row_loss), in_dims=(None, 0, 0, 0))(p.detach(), obs, onehot, y)
    scale = per_row.abs().sum(0)
    return dict(q_values=q_sa.detach().numpy(), loss=float(loss.detach()), grad=grad.numpy(), scale=scale.numpy(),
                y=y.numpy(), margin=margin.numpy(), gap=gap.numpy(), delta=delta.detach().numpy())
