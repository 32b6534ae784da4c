from .base import (CategoricalPolicy, DeterministicPolicy, EpsilonGreedyPolicy, GaussianPolicy, GreedyPolicy,
                   NoisyGreedyPolicy, Policy, RandomPolicy, SquashedGaussianPolicy, StochasticPolicy)

__all__ = ["Policy", "StochasticPolicy", "CategoricalPolicy", "GaussianPolicy", "SquashedGaussianPolicy",
           "DeterministicPolicy", "RandomPolicy", "GreedyPolicy", "EpsilonGreedyPolicy",
           "NoisyGreedyPolicy"]
