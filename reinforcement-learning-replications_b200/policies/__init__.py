from .base import (CategoricalPolicy, DeterministicPolicy, GaussianPolicy, Policy, RandomPolicy,
                   SquashedGaussianPolicy, StochasticPolicy)

__all__ = ["Policy", "StochasticPolicy", "CategoricalPolicy", "GaussianPolicy", "SquashedGaussianPolicy",
           "DeterministicPolicy", "RandomPolicy"]
