"""The two critic wrappers of the reference API: a torch network bundled with the optimizer that trains it.

The update engine reads ``.network`` (a 3-layer ``MLP``) and ``.optimizer`` (Adam hyper-parameters and state) from
these objects; ``forward`` is only used on the host (rollouts, evaluation, the CPU oracle)."""
import math

import torch
from torch import Tensor, nn
from torch.optim import Optimizer


class _Critic(nn.Module):
    def __init__(self, network: nn.Module, optimizer: Optimizer) -> None:
        super().__init__()
        self.network, self.optimizer = network, optimizer


class ValueFunction(_Critic):
    """V(s) (ref: value_function.py:5-28)."""

    def forward(self, observation: Tensor) -> Tensor:
        return self.network(observation)


class QFunction(_Critic):
    """Q(s, a): the network sees the concatenated pair; the trailing unit axis is dropped (ref: q_function.py:6-32)."""

    def forward(self, observation: Tensor, action: Tensor) -> Tensor:
        joint = torch.cat((observation, action), dim=-1)
        return self.network(joint).squeeze(-1)


class DiscreteQFunction(_Critic):
    """Q(s, .) for a discrete action space: the network maps an observation to one value per action, [..., n]
    (DQN's critic)."""

    def forward(self, observation: Tensor) -> Tensor:
        return self.network(observation)


class _CategoricalSupport(_Critic):
    """A critic whose network outputs logits over ``n_atoms`` fixed atoms from ``v_min`` to ``v_max`` (the support of
    C51's and D4PG's critics)."""

    MAX_ATOMS = 256  # the engine's limit (b200rl.h)

    def __init__(self, network: nn.Module, optimizer: Optimizer, n_atoms: int = 51, v_min: float = -10.0,
                 v_max: float = 10.0) -> None:
        super().__init__(network, optimizer)
        if not 2 <= int(n_atoms) <= self.MAX_ATOMS:
            raise ValueError(f"n_atoms must be 2..{self.MAX_ATOMS}, got {n_atoms}")
        v_min, v_max = float(v_min), float(v_max)
        if not (math.isfinite(v_min) and math.isfinite(v_max) and v_min < v_max):
            raise ValueError(f"the support needs finite v_min < v_max, got [{v_min}, {v_max}]")
        self.n_atoms, self.v_min, self.v_max = int(n_atoms), v_min, v_max
        # z_i = float32(v_min + i dz), evaluated in double as the engine does (torch.linspace rounds differently)
        dz = (v_max - v_min) / (self.n_atoms - 1)
        self.support = torch.tensor([v_min + i * dz for i in range(self.n_atoms)], dtype=torch.float64).float()


class CategoricalQFunction(_CategoricalSupport):
    """A return distribution per action over a fixed support (C51's critic): the network maps an observation to
    ``n_actions x n_atoms`` logits, action a owning columns a*n_atoms .. (a+1)*n_atoms - 1.  ``forward`` returns the
    expected values [..., n_actions], so greedy and epsilon-greedy policies and the evaluator use it as they use a
    ``DiscreteQFunction``."""

    def log_distribution(self, observation: Tensor) -> Tensor:
        """log p(s, a) [..., n_actions, n_atoms]."""
        logits = self.network(observation)
        return torch.log_softmax(logits.unflatten(-1, (-1, self.n_atoms)), dim=-1)

    def distribution(self, observation: Tensor) -> Tensor:
        """p(s, a) [..., n_actions, n_atoms]."""
        return self.log_distribution(observation).exp()

    def forward(self, observation: Tensor) -> Tensor:
        return (self.distribution(observation) * self.support).sum(-1)


class DistributionalQFunction(_CategoricalSupport):
    """A return distribution over a fixed support for a continuous action (D4PG's critic): the network maps the
    concatenated pair [s | a] to ``n_atoms`` logits.  ``forward`` returns the expected value Q(s, a) = sum_i z_i p_i
    with the trailing axis dropped, so host code written for a ``QFunction`` uses it unchanged."""

    def log_distribution(self, observation: Tensor, action: Tensor) -> Tensor:
        """log p(s, a) [..., n_atoms]."""
        return torch.log_softmax(self.network(torch.cat((observation, action), dim=-1)), dim=-1)

    def distribution(self, observation: Tensor, action: Tensor) -> Tensor:
        """p(s, a) [..., n_atoms]."""
        return self.log_distribution(observation, action).exp()

    def forward(self, observation: Tensor, action: Tensor) -> Tensor:
        return (self.distribution(observation, action) * self.support).sum(-1)


class _QuantileMidpoints(_Critic):
    """A critic whose network outputs ``n_quantiles`` quantile locations per action, located at the quantile midpoints
    ``taus`` (the quantiles of QR-DQN's and TQC's critics)."""

    MAX_QUANTILES = 256  # the engine's limit (b200rl.h)

    def __init__(self, network: nn.Module, optimizer: Optimizer, n_quantiles: int = 200) -> None:
        super().__init__(network, optimizer)
        if isinstance(n_quantiles, bool) or int(n_quantiles) != n_quantiles or \
                not 1 <= int(n_quantiles) <= self.MAX_QUANTILES:
            raise ValueError(f"n_quantiles must be an integer from 1 to {self.MAX_QUANTILES}, got {n_quantiles!r}")
        self.n_quantiles = int(n_quantiles)
        # tau_i = (2i + 1) / (2N), one float32 division as the engine computes it
        N = self.n_quantiles
        self.taus = torch.arange(1, 2 * N, 2, dtype=torch.float32) / torch.tensor(2 * N, dtype=torch.float32)


class QuantileQFunction(_QuantileMidpoints):
    """A return distribution per action as ``n_quantiles`` quantile locations (QR-DQN's critic): the network maps an
    observation to ``n_actions x n_quantiles`` values, action a owning columns a*n_quantiles .. (a+1)*n_quantiles - 1,
    located at the quantile midpoints ``taus``.  ``forward`` returns their means [..., n_actions], so greedy and
    epsilon-greedy policies and the evaluator use it as they use a ``DiscreteQFunction``."""

    def quantiles(self, observation: Tensor) -> Tensor:
        """theta(s, a) [..., n_actions, n_quantiles]."""
        return self.network(observation).unflatten(-1, (-1, self.n_quantiles))

    def forward(self, observation: Tensor) -> Tensor:
        return self.quantiles(observation).sum(-1) / self.n_quantiles


class ContinuousQuantileQFunction(_QuantileMidpoints):
    """A return distribution for a continuous action as ``n_quantiles`` quantile locations (TQC's critic): the network
    maps the concatenated pair [s | a] to ``n_quantiles`` values located at the quantile midpoints ``taus``.
    ``forward`` returns their mean Q(s, a) with the trailing axis dropped, so host code written for a ``QFunction`` uses
    it unchanged."""

    def __init__(self, network: nn.Module, optimizer: Optimizer, n_quantiles: int = 25) -> None:
        super().__init__(network, optimizer, n_quantiles)

    def quantiles(self, observation: Tensor, action: Tensor) -> Tensor:
        """theta(s, a) [..., n_quantiles]."""
        return self.network(torch.cat((observation, action), dim=-1))

    def forward(self, observation: Tensor, action: Tensor) -> Tensor:
        return self.quantiles(observation, action).sum(-1) / self.n_quantiles


class ImplicitQuantileQFunction(_Critic):
    """The return distribution per action as a quantile function (IQN's critic): the network (an
    ``ImplicitQuantileMLP``) maps an observation and fractions tau to Z(s, tau, a).  ``n_quantiles``,
    ``n_target_quantiles`` and ``n_policy_quantiles`` are N, N' and K of the paper: the fractions a train step samples
    per minibatch row for the online network, for the target network and for the argmax over actions.

    ``forward`` returns Q(s, a) = the mean of Z over the K fixed midpoints (2k + 1) / (2K), [..., n_actions], so greedy
    and epsilon-greedy policies and the evaluator use it as they use a ``DiscreteQFunction`` and evaluation is
    deterministic.  The paper samples the K fractions when acting; sampled-fraction and risk-sensitive acting are not
    implemented."""

    MAX_QUANTILES = 256  # the engine's limit on N, N' and K (b200rl.h)

    def __init__(self, network: nn.Module, optimizer: Optimizer, n_quantiles: int = 64, n_target_quantiles: int = 64,
                 n_policy_quantiles: int = 32) -> None:
        super().__init__(network, optimizer)
        for name, v in (("n_quantiles", n_quantiles), ("n_target_quantiles", n_target_quantiles),
                        ("n_policy_quantiles", n_policy_quantiles)):
            if isinstance(v, bool) or int(v) != v or not 1 <= int(v) <= self.MAX_QUANTILES:
                raise ValueError(f"{name} must be an integer from 1 to {self.MAX_QUANTILES}, got {v!r}")
        self.n_quantiles, self.n_target_quantiles = int(n_quantiles), int(n_target_quantiles)
        self.n_policy_quantiles = int(n_policy_quantiles)
        K = self.n_policy_quantiles
        self.policy_taus = torch.arange(1, 2 * K, 2, dtype=torch.float32) / torch.tensor(2 * K, dtype=torch.float32)

    def quantiles(self, observation: Tensor, taus: Tensor) -> Tensor:
        """Z(s, tau, a) [..., n_actions, M] at the fractions ``taus`` [..., M]."""
        return self.network(observation, taus).transpose(-1, -2)

    def forward(self, observation: Tensor) -> Tensor:
        taus = self.policy_taus.expand(*observation.shape[:-1], self.n_policy_quantiles)
        return self.quantiles(observation, taus).sum(-1) / self.n_policy_quantiles
