"""The implicit quantile network of IQN (Dabney, Ostrovski, Silver & Munos 2018): Z(s, tau) for any fraction tau."""
from __future__ import annotations

import math
from typing import Sequence, Type

import torch
from torch import Tensor, nn


def cosine_features(taus: Tensor, n_cos: int) -> Tensor:
    """x_i = cos(pi * i * tau) for i = 0 .. n_cos - 1 [..., M, n_cos] of float32 fractions [..., M], as the engine
    computes them: i * tau rounded to float32 once, then the cosine of pi times it evaluated in float64 and rounded to
    float32 (the engine's cospif is within one ulp of that)."""
    i = torch.arange(n_cos, dtype=torch.float32)
    x = taus.float()[..., None] * i
    return torch.cos(math.pi * x.double()).float()


class ImplicitQuantileMLP(nn.Module):
    """Z(s, tau) [..., M, n_actions] = head(psi(s)[..., None, :] * phi(tau)) with

        embedding      psi = act(s W_psi^T + b_psi)                    [obs -> d]
        tau_embedding  phi = act(x W_phi^T + b_phi), x = cosine_features(tau, n_cos)   [n_cos -> d]
        head           Linear(d, h), act, Linear(h, n_actions)

    ``sizes`` = [obs, d, h].  The submodules are registered in this order, so ``parameters()`` (and the engine's flat
    vector) is W_psi, b_psi, W_phi, b_phi, W_h, b_h, W_out, b_out."""

    def __init__(self, sizes: Sequence[int], n_actions: int, n_cos: int = 64,
                 activation_function: Type[nn.Module] = nn.ReLU) -> None:
        super().__init__()
        sizes = [int(x) for x in sizes]
        if len(sizes) != 3 or min(sizes) < 1:
            raise ValueError(f"ImplicitQuantileMLP takes sizes = [obs, d, h], got {sizes}")
        if int(n_actions) < 1 or int(n_cos) < 1:
            raise ValueError(f"n_actions and n_cos must be >= 1, got {n_actions} and {n_cos}")
        obs, d, h = sizes
        self.sizes, self.n_actions, self.n_cos = sizes, int(n_actions), int(n_cos)
        self.embedding = nn.Sequential(nn.Linear(obs, d), activation_function())
        self.tau_embedding = nn.Sequential(nn.Linear(self.n_cos, d), activation_function())
        self.head = nn.Sequential(nn.Linear(d, h), activation_function(), nn.Linear(h, self.n_actions))

    def forward(self, observation: Tensor, taus: Tensor) -> Tensor:
        psi = self.embedding(observation)
        phi = self.tau_embedding(cosine_features(taus, self.n_cos))
        return self.head(psi[..., None, :] * phi)
