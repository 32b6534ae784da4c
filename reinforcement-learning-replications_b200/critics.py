"""The two critic wrappers of the reference API: a torch network bundled with the optimizer that trains it.

The update engine reads ``.network`` (a 3-layer ``MLP``) and ``.optimizer`` (Adam hyper-parameters and state) from
these objects; ``forward`` is only used on the host (rollouts, evaluation, the CPU oracle)."""
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
