"""Policy classes with the reference's public surface (ref: policies/*.py).

Action SAMPLING stays on the host through torch CPU ops, exactly like the reference
(ref: policies/stochastic_policy.py:26-41): a GPU Philox stream cannot reproduce torch's CPU mt19937 draws, and
BASELINE.json asks for bit-exact sampled action indices.  The device copy of the parameters is written back into
these host modules after every train().
"""
from abc import ABC, abstractmethod

import numpy as np
import torch
from torch import Tensor, nn
from torch.distributions import Categorical, Distribution, Independent, Normal
from torch.optim import Optimizer

from ..networks.noisy import reset_noise


class Policy(nn.Module, ABC):
    """ref: policies/policy.py:8-30"""

    @abstractmethod
    def get_action_tensor(self, observation: Tensor) -> Tensor:
        raise NotImplementedError

    @abstractmethod
    def get_action_numpy(self, observation: np.ndarray) -> np.ndarray:
        raise NotImplementedError


class StochasticPolicy(Policy):
    """ref: policies/stochastic_policy.py:11-41"""

    @abstractmethod
    def forward(self, observation: Tensor) -> Distribution:
        raise NotImplementedError

    def get_action_tensor(self, observation: Tensor) -> Tensor:
        with torch.no_grad():
            dist = self.forward(observation)
        return dist.sample()

    def get_action_numpy(self, observation: np.ndarray) -> np.ndarray:
        action = self.get_action_tensor(torch.from_numpy(observation).float())
        return np.asarray(action.detach().numpy())


class CategoricalPolicy(StochasticPolicy):
    """ref: policies/categorical_policy.py:8-32"""

    def __init__(self, network: nn.Module, optimizer: Optimizer):
        super().__init__()
        self.network = network
        self.optimizer = optimizer

    def forward(self, observation: Tensor) -> Categorical:
        return Categorical(logits=self.network(observation))


class GaussianPolicy(StochasticPolicy):
    """ref: policies/gaussian_policy.py:9-37 -- diagonal Gaussian, mean from the network, std = exp(log_std)."""

    def __init__(self, network: nn.Module, optimizer: Optimizer, log_std: nn.Parameter):
        super().__init__()
        self.network = network
        self.optimizer = optimizer
        self.log_std = log_std

    def forward(self, observation: Tensor) -> Independent:
        return Independent(Normal(loc=self.network(observation), scale=torch.exp(self.log_std)), 1)


class SquashedGaussianPolicy(StochasticPolicy):
    """The SAC actor (Spinning Up sac/core.py SquashedGaussianMLPActor) with its mean and log_std layers stacked as the
    network's last Linear: network(obs) = [mu | log_std] (2A outputs, Identity output).  log_std is clamped to
    [log_std_min, log_std_max]; the action is action_limit * tanh(u), u ~ Normal(mu, exp(log_std))."""

    def __init__(self, network: nn.Module, optimizer: Optimizer, action_limit: float = 1.0, log_std_min: float = -20.0,
                 log_std_max: float = 2.0):
        super().__init__()
        self.network = network
        self.optimizer = optimizer
        self.action_limit, self.log_std_min, self.log_std_max = float(action_limit), float(log_std_min), float(log_std_max)

    def forward(self, observation: Tensor, deterministic: bool = False, with_logprob: bool = True):
        """(action, log pi(action | observation) or None).  deterministic: u = mu."""
        out = self.network(observation)
        A = out.shape[-1] // 2
        mu, log_std = out[..., :A], torch.clamp(out[..., A:], self.log_std_min, self.log_std_max)
        dist = Normal(mu, torch.exp(log_std))
        u = mu if deterministic else dist.rsample()
        log_prob = None
        if with_logprob:  # the tanh change of variables in its numerically stable form (Spinning Up, SAC paper eq. 21)
            log_prob = dist.log_prob(u).sum(-1) - (2 * (np.log(2) - u - nn.functional.softplus(-2 * u))).sum(-1)
        return self.action_limit * torch.tanh(u), log_prob

    def get_action_tensor(self, observation: Tensor) -> Tensor:
        with torch.no_grad():
            return self.forward(observation, with_logprob=False)[0]

    def deterministic(self) -> "Policy":
        """A view that acts with action_limit * tanh(mu) (evaluation); it shares this policy's network."""
        return _SquashedMeanPolicy(self)


class _SquashedMeanPolicy(Policy):
    def __init__(self, policy: SquashedGaussianPolicy):
        super().__init__()
        self.policy = policy

    def get_action_tensor(self, observation: Tensor) -> Tensor:
        with torch.no_grad():
            return self.policy.forward(observation, deterministic=True, with_logprob=False)[0]

    def get_action_numpy(self, observation: np.ndarray) -> np.ndarray:
        return np.asarray(self.get_action_tensor(torch.from_numpy(observation).float()).numpy())


class TanhMeanGaussianPolicy(StochasticPolicy):
    """IQL's actor: network(obs) = [m | l] (2A outputs, Identity output), a diagonal Gaussian with mean
    action_limit * tanh(m) and log std clamp(l, log_std_min, log_std_max).  Its mean is bounded by tanh, but a sample is
    not squashed: ``log_prob`` of a dataset action at +-action_limit needs no atanh.  Acting samples and clips to
    [-action_limit, action_limit]; ``deterministic()`` acts with action_limit * tanh(m), the action SAC's evaluation
    policy takes from the same network.  The default bounds are IQL's reference implementation's."""

    def __init__(self, network: nn.Module, optimizer: Optimizer, action_limit: float = 1.0, log_std_min: float = -5.0,
                 log_std_max: float = 2.0):
        super().__init__()
        self.network = network
        self.optimizer = optimizer
        self.action_limit, self.log_std_min, self.log_std_max = float(action_limit), float(log_std_min), float(log_std_max)

    def forward(self, observation: Tensor) -> Independent:
        out = self.network(observation)
        A = out.shape[-1] // 2
        mu = self.action_limit * torch.tanh(out[..., :A])
        log_std = torch.clamp(out[..., A:], self.log_std_min, self.log_std_max)
        return Independent(Normal(mu, torch.exp(log_std)), 1)

    def log_prob(self, observation: Tensor, action: Tensor) -> Tensor:
        """sum_j Normal(mu_j, sigma_j).log_prob(action_j)."""
        return self.forward(observation).log_prob(action)

    def get_action_tensor(self, observation: Tensor) -> Tensor:
        with torch.no_grad():
            return torch.clamp(self.forward(observation).sample(), -self.action_limit, self.action_limit)

    def deterministic(self) -> "Policy":
        """A view that acts with action_limit * tanh(m) (evaluation); it shares this policy's network."""
        return _TanhMeanPolicy(self)


class _TanhMeanPolicy(Policy):
    def __init__(self, policy: TanhMeanGaussianPolicy):
        super().__init__()
        self.policy = policy

    def get_action_tensor(self, observation: Tensor) -> Tensor:
        with torch.no_grad():
            return self.policy.forward(observation).mean

    def get_action_numpy(self, observation: np.ndarray) -> np.ndarray:
        return np.asarray(self.get_action_tensor(torch.from_numpy(observation).float()).numpy())


class DeterministicPolicy(Policy):
    """ref: policies/deterministic_policy.py:9-45"""

    def __init__(self, network: nn.Module, optimizer: Optimizer):
        super().__init__()
        self.network = network
        self.optimizer = optimizer

    def forward(self, observation: Tensor) -> Tensor:
        return self.network(observation)

    def get_action_tensor(self, observation: Tensor) -> Tensor:
        with torch.no_grad():
            return self.forward(observation)

    def get_action_numpy(self, observation: np.ndarray) -> np.ndarray:
        return np.asarray(self.get_action_tensor(torch.from_numpy(observation).float()).detach().numpy())


class RandomPolicy(Policy):
    """Uniform samples from the action space, for warm-up (ref: policies/random_policy.py:9-27)."""

    def __init__(self, action_space) -> None:
        super().__init__()
        self.action_space = action_space

    def get_action_tensor(self, observation: Tensor) -> Tensor:
        return torch.from_numpy(self.action_space.sample())

    def get_action_numpy(self, observation: np.ndarray) -> np.ndarray:
        return np.asarray(self.action_space.sample())


class GreedyPolicy(Policy):
    """argmax_a Q(s, a) of a DiscreteQFunction (torch.argmax: the first index among equal maxima); DQN's evaluation
    policy."""

    def __init__(self, q_function: nn.Module) -> None:
        super().__init__()
        self.q_function = q_function

    def _greedy(self, observation: Tensor) -> Tensor:
        with torch.no_grad():
            return torch.argmax(self.q_function(observation), dim=-1)

    def get_action_tensor(self, observation: Tensor) -> Tensor:
        return self._greedy(observation)

    def get_action_numpy(self, observation: np.ndarray) -> np.ndarray:
        return np.asarray(self._greedy(torch.from_numpy(np.asarray(observation, np.float32))).numpy())


class EpsilonGreedyPolicy(GreedyPolicy):
    """With probability ``epsilon`` a uniform action from ``action_space.sample()``, otherwise the greedy action.  Every
    action draws one ``np.random.random()`` (global NumPy stream), also when it then acts greedily; a batch of
    observations [N, O] draws one per row, in row order."""

    def __init__(self, q_function: nn.Module, action_space, epsilon: float) -> None:
        super().__init__(q_function)
        self.action_space = action_space
        self.epsilon = float(epsilon)

    def get_action_numpy(self, observation: np.ndarray) -> np.ndarray:
        observation = np.asarray(observation, np.float32)
        if observation.ndim == 1:
            if np.random.random() < self.epsilon:
                return np.asarray(self.action_space.sample())
            return np.asarray(self._greedy(torch.from_numpy(observation)).numpy())
        return np.stack([self.get_action_numpy(o) for o in observation])

    def get_action_tensor(self, observation: Tensor) -> Tensor:
        return torch.as_tensor(self.get_action_numpy(observation.detach().cpu().numpy()))


class NoisyGreedyPolicy(GreedyPolicy):
    """Acting with a noisy Q network (``networks.NoisyLinear``; Fortunato et al. 2018): every call first redraws the
    noise of every noisy layer (torch's default CPU generator; a batch of observations shares one sample), then acts
    greedily in train mode, on the noisy weights.  NumPy's stream is left alone.  ``deterministic()`` is the
    evaluation view: greedy on the mean weights."""

    def _greedy(self, observation: Tensor) -> Tensor:
        reset_noise(self.q_function)
        return super()._greedy(observation)

    def deterministic(self) -> "Policy":
        """A view that acts greedily with the network in eval mode (the mean weights mu), restoring the mode after."""
        return _MeanGreedyPolicy(self.q_function)


class _MeanGreedyPolicy(GreedyPolicy):
    def _greedy(self, observation: Tensor) -> Tensor:
        was = self.q_function.training
        self.q_function.eval()
        try:
            return super()._greedy(observation)
        finally:
            self.q_function.train(was)
