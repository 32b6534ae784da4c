from .dueling import DuelingMLP
from .iqn import ImplicitQuantileMLP
from .mlp import MLP
from .noisy import NoisyLinear, NoisyMLP, has_noisy_layers, reset_noise

__all__ = ["DuelingMLP", "ImplicitQuantileMLP", "MLP", "NoisyLinear", "NoisyMLP", "has_noisy_layers", "reset_noise"]
