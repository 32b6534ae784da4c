from .dueling import DuelingMLP
from .mlp import MLP
from .noisy import NoisyLinear, NoisyMLP, has_noisy_layers, reset_noise

__all__ = ["DuelingMLP", "MLP", "NoisyLinear", "NoisyMLP", "has_noisy_layers", "reset_noise"]
