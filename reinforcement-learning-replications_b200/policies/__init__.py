from .base import (CategoricalPolicy, DeterministicPolicy, EpsilonGreedyPolicy, GaussianPolicy, GreedyPolicy, Policy,
                   RandomPolicy, SquashedGaussianPolicy, StochasticPolicy)

__all__ = ["Policy", "StochasticPolicy", "CategoricalPolicy", "GaussianPolicy", "SquashedGaussianPolicy",
           "DeterministicPolicy", "RandomPolicy", "GreedyPolicy", "EpsilonGreedyPolicy"]
