from .critics import CategoricalQFunction, DiscreteQFunction, QFunction, QuantileQFunction  # noqa: F401  (module path of the reference API: rl_replicas.q_function)
