from .dueling import DuelingMLP
from .mlp import MLP

__all__ = ["DuelingMLP", "MLP"]
