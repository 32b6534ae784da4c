from .base import (CategoricalPolicy, DeterministicPolicy, EpsilonGreedyPolicy, GaussianPolicy, GreedyPolicy,
                   NoisyGreedyPolicy, Policy, RandomPolicy, SquashedGaussianPolicy, StochasticPolicy,
                   TanhMeanGaussianPolicy)

__all__ = ["Policy", "StochasticPolicy", "CategoricalPolicy", "GaussianPolicy", "SquashedGaussianPolicy", "TanhMeanGaussianPolicy",
           "DeterministicPolicy", "RandomPolicy", "GreedyPolicy", "EpsilonGreedyPolicy",
           "NoisyGreedyPolicy"]
