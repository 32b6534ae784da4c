from .critics import CategoricalQFunction, DiscreteQFunction, ImplicitQuantileQFunction, QFunction, QuantileQFunction  # noqa: F401  (module path of the reference API: rl_replicas.q_function)
