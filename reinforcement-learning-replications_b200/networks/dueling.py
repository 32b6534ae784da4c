"""Dueling Q network (Wang et al. 2016): a shared trunk feeding a state-value stream and an action-advantage stream,
combined by eq. 9 of the paper per output column.  Its output has a plain Q network's ``[..., n_actions * K]`` layout,
so every critic, policy and checkpoint path that takes an ``MLP`` Q network takes it unchanged.  The submodule tree --
``trunk``, ``value``, ``advantage``, registered in that order -- is part of the checkpoint format (``trunk.0.weight``
...) and fixes the order of ``parameters()``, which is the update engine's flat parameter layout (include/b200rl.h,
"Dueling Q networks")."""
from typing import List, Sequence, Type

from torch import Tensor, nn

from .noisy import NoisyLinear


class DuelingMLP(nn.Module):
    """``sizes`` = [obs, h_trunk, h_stream]; ``outputs_per_action`` = K values per action: 1 for DQN, n_atoms logits for
    C51, n_quantiles locations for QR-DQN.  forward: h = trunk(x), V = value(h) [..., K], A = advantage(h) [..., n, K],
    Q = V + (A - mean over actions of A), flattened to [..., n K] (action a owns columns a K .. a K + K - 1).
    ``noisy`` = True makes the four stream layers ``NoisyLinear`` (initial sigma_0 / sqrt(in)) and keeps the trunk plain,
    as Rainbow does."""

    def __init__(self, sizes: Sequence[int], n_actions: int, outputs_per_action: int = 1,
                 activation_function: Type[nn.Module] = nn.ReLU, noisy: bool = False, sigma_0: float = 0.5) -> None:
        super().__init__()
        self.sizes: List[int] = [int(w) for w in sizes]
        if len(self.sizes) != 3 or min(self.sizes) < 1:
            raise ValueError(f"DuelingMLP needs sizes = [obs, h_trunk, h_stream] of positive widths, got {list(sizes)}")
        if int(n_actions) < 1 or int(outputs_per_action) < 1:
            raise ValueError(f"DuelingMLP needs n_actions >= 1 and outputs_per_action >= 1, got {n_actions} and "
                             f"{outputs_per_action}")
        self.n_actions, self.outputs_per_action = int(n_actions), int(outputs_per_action)
        O, h1, h2 = self.sizes
        K, n = self.outputs_per_action, self.n_actions
        self.trunk = nn.Sequential(nn.Linear(O, h1), activation_function())
        lin = (lambda i, o: NoisyLinear(i, o, sigma_0)) if noisy else nn.Linear
        self.value = nn.Sequential(lin(h1, h2), activation_function(), lin(h2, K))
        self.advantage = nn.Sequential(lin(h1, h2), activation_function(), lin(h2, n * K))

    def forward(self, input: Tensor) -> Tensor:
        h = self.trunk(input)
        v = self.value(h).unflatten(-1, (1, self.outputs_per_action))
        a = self.advantage(h).unflatten(-1, (self.n_actions, self.outputs_per_action))
        return (v + (a - a.mean(dim=-2, keepdim=True))).flatten(-2)
