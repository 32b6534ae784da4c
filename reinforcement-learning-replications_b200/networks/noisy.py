"""Noisy networks (Fortunato et al. 2018, "Noisy Networks for Exploration") with factorized Gaussian noise.  A
``NoisyLinear`` layer registers ``weight_mu``, ``weight_sigma``, ``bias_mu`` and ``bias_sigma`` in that order: the
checkpoint keys and the update engine's flat parameter layout (include/b200rl.h, "Noisy networks").  Its noise
(``eps_in``, ``eps_out``) is a pair of non-persistent buffers that ``reset_noise`` redraws from torch's CPU generator;
the engine draws its own on the device at every train step."""
import math
from typing import List, Sequence, Type

import torch
from torch import Tensor, nn


def _f(x: Tensor) -> Tensor:
    """f(x) = copysign(sqrt(|x|), x), the paper's factorization of the noise."""
    return torch.copysign(x.abs().sqrt(), x)


class NoisyLinear(nn.Module):
    """y = x W^T + b with W = W_mu + W_sigma * e, e_ij = f(eps_out_i) f(eps_in_j), b = b_mu + b_sigma * f(eps_out) in
    train mode, and W_mu, b_mu in eval mode.  Initialization: mu ~ U(-1/sqrt(in), 1/sqrt(in)), sigma = sigma_0 /
    sqrt(in).  Not an ``nn.Linear``: code that needs a plain layer refuses it."""

    def __init__(self, in_features: int, out_features: int, sigma_0: float = 0.5) -> None:
        super().__init__()
        self.in_features, self.out_features, self.sigma_0 = int(in_features), int(out_features), float(sigma_0)
        if self.in_features < 1 or self.out_features < 1:
            raise ValueError(f"NoisyLinear needs positive widths, got {in_features} -> {out_features}")
        self.weight_mu = nn.Parameter(torch.empty(self.out_features, self.in_features))
        self.weight_sigma = nn.Parameter(torch.empty(self.out_features, self.in_features))
        self.bias_mu = nn.Parameter(torch.empty(self.out_features))
        self.bias_sigma = nn.Parameter(torch.empty(self.out_features))
        self.register_buffer("eps_in", torch.zeros(self.in_features), persistent=False)
        self.register_buffer("eps_out", torch.zeros(self.out_features), persistent=False)
        bound = 1.0 / math.sqrt(self.in_features)
        with torch.no_grad():
            self.weight_mu.uniform_(-bound, bound)
            self.bias_mu.uniform_(-bound, bound)
            self.weight_sigma.fill_(self.sigma_0 * bound)
            self.bias_sigma.fill_(self.sigma_0 * bound)

    def reset_noise(self) -> None:
        """New eps_in, eps_out ~ N(0, 1) from torch's default CPU generator."""
        self.eps_in.copy_(torch.randn(self.in_features))
        self.eps_out.copy_(torch.randn(self.out_features))

    def composed(self):
        """(W, b) of the current noise, each product and sum rounded on its own as the engine rounds them."""
        fo = _f(self.eps_out)
        return self.weight_mu + self.weight_sigma * torch.outer(fo, _f(self.eps_in)), self.bias_mu + self.bias_sigma * fo

    def forward(self, input: Tensor) -> Tensor:
        if not self.training:
            return nn.functional.linear(input, self.weight_mu, self.bias_mu)
        return nn.functional.linear(input, *self.composed())

    def extra_repr(self) -> str:
        return f"in_features={self.in_features}, out_features={self.out_features}, sigma_0={self.sigma_0}"


class NoisyMLP(nn.Module):
    """``MLP``'s layout (``network`` = Sequential with the layers at the even indices, Identity after the last) with
    every layer a ``NoisyLinear``."""

    def __init__(self, sizes: Sequence[int], activation_function: Type[nn.Module] = nn.ReLU,
                 sigma_0: float = 0.5) -> None:
        super().__init__()
        self.sizes: List[int] = [int(w) for w in sizes]
        if len(self.sizes) < 2:
            raise ValueError("NoisyMLP needs at least an input and an output width")
        stack: List[nn.Module] = []
        for fan_in, fan_out in zip(self.sizes, self.sizes[1:]):
            stack += [NoisyLinear(fan_in, fan_out, sigma_0), activation_function()]
        stack[-1] = nn.Identity()
        self.network: nn.Module = nn.Sequential(*stack)

    def forward(self, input: Tensor) -> Tensor:
        return self.network(input)


def reset_noise(module: nn.Module) -> None:
    """``reset_noise`` of every NoisyLinear in ``module``, in module order."""
    for m in module.modules():
        if isinstance(m, NoisyLinear):
            m.reset_noise()


def has_noisy_layers(module: nn.Module) -> bool:
    return any(isinstance(m, NoisyLinear) for m in module.modules())
