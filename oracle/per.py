"""NumPy / torch-CPU oracles of prioritized experience replay for DQN.  TEST INFRASTRUCTURE ONLY -- see oracle/__init__.py.

* ``philox4x32_10`` and ``per_uniforms``: the device's counter-based generator and the U_j of a prioritized draw, bit
  for bit, so the device's draws can be reproduced.
* ``tree_levels`` / ``tree_offsets`` / ``root_f32``: the sum tree's levels (32 children per node) in float64, the float
  layout of b200rl.h, and the root as the device computes it (float32, children added in index order).
* ``SumTree``: a float64 proportional sampler over leaf priorities, and ``stratified_draw``: one step's stratified draw
  with the distance of each u_j to the nearest cumulative boundary.
* ``PerDqnOracle``: ``DqnOracle`` with importance weights: it takes the drawn minibatches, the priorities of the drawn
  leaves and each step's beta, and returns delta, the weights and the new priorities with the usual logs.
"""
from __future__ import annotations

from typing import Dict, List, Sequence

import numpy as np
import torch
import torch.nn.functional as F

from .dqn import DqnOracle, td_values

FAN = 32
_M32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 on uint32 arrays (any broadcastable shapes); returns the four output words as uint64 arrays."""
    c = [np.asarray(x, np.uint64) & _M32 for x in (c0, c1, c2, c3)]
    k0, k1 = np.uint64(k0) & _M32, np.uint64(k1) & _M32
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c[0]
        p1 = np.uint64(0xCD9E8D57) * c[2]
        c = [((p1 >> np.uint64(32)) ^ c[1] ^ k0) & _M32, p1 & _M32, ((p0 >> np.uint64(32)) ^ c[3] ^ k1) & _M32,
             p0 & _M32]
        k0 = (k0 + np.uint64(0x9E3779B9)) & _M32
        k1 = (k1 + np.uint64(0xBB67AE85)) & _M32
    return c


def per_uniforms(seed: int, call: int, st: int, B: int) -> np.ndarray:
    """U_j, j < B, of step ``st`` of the call keyed by (seed, call): the top 24 bits of the first Philox word of counter
    (j, st, call, 0x9E5), times 2^-24 (float32, exact)."""
    seed, call = int(seed) & (2 ** 64 - 1), int(call) & (2 ** 64 - 1)
    r = philox4x32_10(np.arange(B, dtype=np.uint64), st, call & 0xFFFFFFFF, 0x9E5, seed & 0xFFFFFFFF, seed >> 32)
    return (r[0] >> np.uint64(8)).astype(np.float32) * np.float32(2.0 ** -24)


def tree_levels(leaves: np.ndarray) -> List[np.ndarray]:
    """[level 0 (the leaves), level 1, ..., root level] in float64: node i of level k + 1 = the sum of nodes
    32 i .. 32 i + 31 of level k; at least one level above the leaves."""
    levels = [np.asarray(leaves, np.float64)]
    while True:
        c = levels[-1]
        pad = np.zeros(-len(c) % FAN)
        levels.append(np.concatenate([c, pad]).reshape(-1, FAN).sum(1))
        if len(levels[-1]) == 1:
            return levels


def tree_offsets(n: int):
    """(offset of every level, total floats) of a tree over n leaves in b200rl.h's layout."""
    offs, c = [0], n
    while True:
        offs.append(offs[-1] + -(-c // FAN) * FAN)
        c = -(-c // FAN)
        if c == 1:
            return offs, offs[-1] + FAN


def root_f32(leaves: np.ndarray) -> np.float32:
    """The root as the device computes it: float32 sums of 32 children, added in index order, level by level."""
    c = np.asarray(leaves, np.float32)
    while True:
        c = np.concatenate([c, np.zeros(-len(c) % FAN, np.float32)]).reshape(-1, FAN)
        s = np.zeros(len(c), np.float32)
        for i in range(FAN):
            s = (s + c[:, i]).astype(np.float32)
        c = s
        if len(c) == 1:
            return c[0]


class SumTree:
    """Float64 proportional sampling over leaf priorities: ``find(u)`` = the leaf whose cumulative interval
    [c_{i-1}, c_i) holds u; a leaf of priority 0 is never returned, and u at or past the total maps to the last leaf
    with a nonzero priority."""

    def __init__(self, leaves: np.ndarray):
        self.p = np.asarray(leaves, np.float64)
        self.c = np.cumsum(self.p)
        self.total = float(self.c[-1])
        nz = np.flatnonzero(self.p > 0)
        self.last = int(nz[-1]) if len(nz) else 0

    def find(self, u: np.ndarray) -> np.ndarray:
        i = np.searchsorted(self.c, u, side="right")
        return np.where(i >= len(self.p), self.last, np.minimum(i, len(self.p) - 1))

    def boundary_distance(self, u: np.ndarray) -> np.ndarray:
        """|u - nearest cumulative boundary| (0 and every c_i count as boundaries)."""
        b = np.concatenate([[0.0], self.c])
        i = np.clip(np.searchsorted(b, u), 1, len(b) - 1)
        return np.minimum(np.abs(u - b[i - 1]), np.abs(b[i] - u))


def stratified_draw(leaves: np.ndarray, seed: int, call: int, st: int, B: int):
    """One step's draw: (leaf indices [B], distance of each u_j to its nearest boundary / the total).  u_j is computed
    as the device computes it, (float32(j) + U_j) * (M / B) in float32 with M = the float32 root, and located in the
    float64 tree."""
    U = per_uniforms(seed, call, st, B)
    M = root_f32(leaves)
    step = np.float32(M / np.float32(B))
    u = ((np.arange(B, dtype=np.float32) + U).astype(np.float32) * step).astype(np.float32).astype(np.float64)
    tree = SumTree(leaves)
    return tree.find(u), tree.boundary_distance(u) / tree.total


def beta_schedule(t, beta_start: float, beta_anneal_steps: int):
    """beta of a step taken at Q optimizer count t (before the step)."""
    return np.minimum(1.0, beta_start + (1.0 - beta_start) * np.asarray(t, np.float64) / beta_anneal_steps)


class PerDqnOracle(DqnOracle):
    """``DqnOracle`` with importance weights (float32, torch autograd): loss = mean(w * smooth_l1(Q(s, a), y)).  Per step
    it takes the drawn minibatch, the priorities p of the drawn leaves and beta; w = (min p / p)^beta (float64, then
    float32), new priorities (|delta| + eps)^alpha (float64 of the float32 delta, computed before the Adam step)."""

    def __init__(self, *args, alpha: float = 0.6, eps: float = 1e-6, **kw):
        super().__init__(*args, **kw)
        self.alpha, self.eps = float(alpha), float(eps)

    def train(self, minibatches: List[dict], leaf_priorities: Sequence[np.ndarray] = None,
              betas: Sequence[float] = None) -> Dict[str, list]:
        logs = dict(q1_values=[], q1_losses=[], copied=[], delta=[], weights=[], priorities=[])
        t = lambda x: torch.as_tensor(np.asarray(x, dtype=np.float32))
        for mb, p, beta in zip(minibatches, leaf_priorities, betas):
            p = np.asarray(p, np.float64)
            w64 = (p.min() / p) ** float(beta)
            w = torch.as_tensor(w64.astype(np.float32))
            o, a, r = t(mb["observations"]), t(mb["actions"]).reshape(-1), t(mb["rewards"])
            o2, d = t(mb["next_observations"]), t(np.asarray(mb["dones"]).astype(np.int32))
            with torch.no_grad():
                v = td_values(self.q_targ(o2), self.q(o2) if self.double_q else None, self.double_q)
                y = r + self.gamma * (1 - d) * v
            q_sa = self.q(o).gather(1, a.long()[:, None]).squeeze(1)
            delta = (q_sa - y).detach().numpy().copy()
            loss = (w * F.smooth_l1_loss(q_sa, y, reduction="none")).mean()
            self.opt.zero_grad()
            loss.backward()
            self.opt.step()
            logs["q1_values"].append(q_sa.detach().numpy().copy())
            logs["q1_losses"].append(float(loss.detach()))
            logs["delta"].append(delta)
            logs["weights"].append(w64)
            logs["priorities"].append((np.abs(delta.astype(np.float64)) + self.eps) ** self.alpha)
            copy_now = self.step_count() % self.interval == 0
            if copy_now:
                self.q_targ.load_state_dict(self.q.state_dict())
            logs["copied"].append(copy_now)
        return logs


def apply_priorities(leaves: np.ndarray, idx: np.ndarray, new_p: np.ndarray) -> np.ndarray:
    """The leaves after one step's update: rows in order, a later row on the same leaf wins, rows whose new priority is
    not finite leave their leaf alone."""
    out = np.array(leaves, np.float64)
    for i, p in zip(np.asarray(idx), np.asarray(new_p, np.float64)):
        if np.isfinite(p):
            out[i] = p
    return out
