"""n-step returns for the DQN / C51 oracles.  TEST INFRASTRUCTURE ONLY -- see oracle/__init__.py.

* ``walk_f32``: the window walk exactly as include/b200rl.h states it, in NumPy float32 over the physical rows of a
  replay ring (every product and sum rounded on its own, as the device rounds them), so the device's returns and
  discounts can be held to it bit for bit.
* ``episode_returns_f64``: an independent float64 form that works from the episode lists the experiences held, not from
  the ring: per transition, the rows up to n - 1 further on in its episode, stopping at a done row.
* ``nstep_minibatch``: ``sample_minibatch``'s dict at given physical rows with the n-step columns, plus ``discounts``.
* ``NStepDqnOracle`` / ``NStepC51Oracle`` / ``NStepPerDqnOracle``: the oracles of oracle/dqn.py, oracle/c51.py and
  oracle/per.py with each minibatch's per-row discount (its ``discounts`` key) in place of gamma; a minibatch without
  the key uses gamma, exactly as the one-step oracles do.  ``dqn_step_f64`` and ``c51_step_f64`` take a per-row discount
  as gamma (a float64 tensor [B] and an array [B, 1]); ``project_f64`` below is Algorithm 1 with one discount per row.
"""
from __future__ import annotations

from typing import Dict, List, Sequence

import numpy as np
import torch

from . import c51 as OC
from .dqn import DqnOracle
from .per import PerDqnOracle


def walk_f32(rew, done, ends, p0, n: int, gamma: float):
    """(last rows, R, discounts) of the windows that start at physical rows ``p0`` over a ring of len(rew) rows:
    R = rew[p0] + g rew[p0 + 1] + ..., g = gamma^k, in float32 with every operation rounded on its own."""
    rew = np.asarray(rew, np.float32)
    done, ends = np.asarray(done) != 0, np.asarray(ends) != 0
    rows = len(rew)
    gamma = np.float32(gamma)
    p = np.array(p0, np.int64).reshape(-1)
    R, g = rew[p].copy(), np.full(p.shape, gamma, np.float32)
    live = np.ones(p.shape, bool)
    for _ in range(1, n):
        live &= ~(done[p] | ends[p])
        nxt = np.where(live, (p + 1) % rows, p)
        R = np.where(live, (R + (g * rew[nxt]).astype(np.float32)).astype(np.float32), R)
        g = np.where(live, (g * gamma).astype(np.float32), g)
        p = nxt
    shape = np.shape(p0)
    return p.reshape(shape), R.reshape(shape), g.reshape(shape)


def episode_returns_f64(episodes: Sequence, n: int, gamma: float):
    """``episodes``: (rewards, dones) of every episode in the order they were appended.  Returns per transition, in
    that order: (flat index of its window's last transition, R, discount gamma^k) in float64."""
    last, R, disc = [], [], []
    base = 0
    for rewards, dones in episodes:
        rewards, dones = np.asarray(rewards, np.float64), np.asarray(dones, bool)
        L = len(rewards)
        for t in range(L):
            end = min(t + n - 1, L - 1)
            stop = np.flatnonzero(dones[t:end])  # a done row ends the window there
            end = t + int(stop[0]) if len(stop) else end
            k = end - t + 1
            R.append(float(np.sum(rewards[t:end + 1] * gamma ** np.arange(k))))
            disc.append(gamma ** k)
            last.append(base + end)
        base += L
    return np.asarray(last, np.int64), np.asarray(R), np.asarray(disc)


def nstep_minibatch(rb, phys_idx, n: int, gamma: float) -> Dict[str, np.ndarray]:
    """The n-step minibatch at physical rows ``phys_idx`` of ReplayBuffer ``rb``: observations and actions of the start
    rows, rewards := R, next_observations and dones of the last rows, discounts := gamma^k (float32 walk)."""
    c = rb._cols
    p0 = np.asarray(phys_idx, np.int64)
    last, R, g = walk_f32(c["rewards"].astype(np.float32), c["dones"], rb._ends, p0, n, gamma)
    return dict(observations=c["observations"][p0], actions=c["actions"][p0], rewards=R,
                next_observations=c["next_observations"][last], dones=c["dones"][last], discounts=g)


class _PerRowDiscount:
    """Runs the one-step oracle's ``train`` one minibatch at a time with gamma set to that minibatch's discounts."""

    @staticmethod
    def _gamma_of(disc: np.ndarray):
        return torch.as_tensor(np.asarray(disc, np.float32))

    def train(self, minibatches: List[dict], *per_step) -> Dict[str, list]:
        logs: Dict[str, list] = {}
        base = self.gamma
        try:
            for k, mb in enumerate(minibatches):
                self.gamma = self._gamma_of(mb["discounts"]) if "discounts" in mb else base
                out = super().train([mb], *([x[k]] for x in per_step))
                for key, v in out.items():
                    logs.setdefault(key, []).extend(v)
        finally:
            self.gamma = base
        return logs


class NStepDqnOracle(_PerRowDiscount, DqnOracle):
    pass


class NStepPerDqnOracle(_PerRowDiscount, PerDqnOracle):
    pass


class NStepC51Oracle(_PerRowDiscount, OC.C51Oracle):
    @staticmethod
    def _gamma_of(disc: np.ndarray):
        return np.asarray(disc, np.float32)[:, None]  # project() broadcasts it over the atoms


def project_f64(p_next, rew, done, z, v_min: float, v_max: float, discounts) -> np.ndarray:
    """oracle/c51.project_f64 (Bellemare et al.'s Algorithm 1) with row r discounted by discounts[r]."""
    return np.concatenate([OC.project_f64(p_next[r:r + 1], rew[r:r + 1], done[r:r + 1], z, v_min, v_max,
                                          float(discounts[r])) for r in range(len(rew))])
