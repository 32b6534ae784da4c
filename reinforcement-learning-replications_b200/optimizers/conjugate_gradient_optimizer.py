"""ConjugateGradientOptimizer with the reference's constructor and (hyper-parameter only) state
(ref: optimizers/conjugate_gradient_optimizer.py:24-131).

In the reference, ``step(loss_fn, kl_fn)`` evaluates two torch closures many times (double backprop for every
Hessian-vector product).  ``step`` here has two routes:

* the closures ``rl_replicas_b200.algorithms.TRPO`` hands in are ``NativeClosure`` objects: the whole constrained step
  -- surrogate gradient, 11 analytic Fisher-vector products, conjugate gradient, step size, backtracking line search
  with reject / restore -- runs on the GPU (b200rl_trpo_update).  This is the product path.
* any other pair of callables (a user's own torch closures over the optimizer's parameters) cannot be turned into
  kernels; the same algorithm then runs as torch tensor operations on whatever device those parameters live on, so
  code written against ``rl_replicas.optimizers.ConjugateGradientOptimizer`` keeps working.  ``TRPO.train`` never
  takes this route.
"""
import logging
from typing import Callable, Iterable, List

import numpy as np
import torch
from torch import Tensor
from torch.optim import Optimizer

logger = logging.getLogger(__name__)

_DEFAULTS = dict(max_constraint=0.01, n_conjugate_gradients=10, max_backtracks=15, backtrack_ratio=0.8,
                 hvp_damping_coefficient=1e-5)


class ConjugateGradientOptimizer(Optimizer):
    def __init__(self, params: Iterable[Tensor], max_constraint: float = 0.01, n_conjugate_gradients: int = 10,
                 max_backtracks: int = 15, backtrack_ratio: float = 0.8, hvp_damping_coefficient: float = 1e-5):
        super().__init__(params, {})
        self.max_constraint = max_constraint
        self.n_conjugate_gradients = n_conjugate_gradients
        self.max_backtracks = max_backtracks
        self.backtrack_ratio = backtrack_ratio
        self.hvp_damping_coefficient = hvp_damping_coefficient

    def hyper_parameters(self) -> dict:
        return {k: getattr(self, k) for k in _DEFAULTS}

    @property
    def state(self) -> dict:  # only hyper-parameters are serialised, like the reference (:100-119)
        return self.hyper_parameters()

    @state.setter
    def state(self, state: dict) -> None:
        for k, default in _DEFAULTS.items():
            setattr(self, k, state.get(k, default))

    def __setstate__(self, state: dict) -> None:
        if "hvp_damping_coefficient" not in state["state"]:
            logger.warning("Resuming ConjugateGradientOptimizer with lost state.")
        self.state = state["state"]
        self.param_groups = state["param_groups"]

    def step(self, loss_function: Callable, kl_divergence_function: Callable) -> None:
        """One constrained step (ref: conjugate_gradient_optimizer.py:59-98)."""
        native = getattr(loss_function, "native_step", None)
        if native is not None and native is getattr(kl_divergence_function, "native_step", None):
            native(self)  # TRPO's own closures: everything below happens inside the engine
            return
        params = [p for group in self.param_groups for p in group["params"] if p.grad is not None]
        if not params:
            raise ValueError("ConjugateGradientOptimizer.step: no parameter has a gradient (call loss.backward() first)")
        gradient = torch.cat([p.grad.reshape(-1) for p in params])
        hvp = self._hessian_vector_product(kl_divergence_function, params)
        direction = self._solve(hvp, gradient)
        direction[direction != direction] = 0.0  # NaN entries -> 0 (:83)
        step_size = torch.sqrt(2.0 * self.max_constraint * (1.0 / (torch.dot(direction, hvp(direction)) + 1e-8)))
        if torch.isnan(step_size):  # (:92-93)
            step_size = 1.0
        self._line_search(params, step_size * direction, loss_function, kl_divergence_function)

    # ---- generic (torch-closure) route -----------------------------------------------------------------------
    def _hessian_vector_product(self, kl_function: Callable, params: List[Tensor]) -> Callable:
        """v -> H v + damping * v with H the Hessian of ``kl_function()`` in ``params``, by double backprop (:133-167)."""
        first = torch.autograd.grad(kl_function(), params, create_graph=True)
        sizes = [p.numel() for p in params]

        def product(vector: Tensor) -> Tensor:
            pieces = torch.split(vector, sizes)
            inner = sum((g * v.view_as(g)).sum() for g, v in zip(first, pieces))
            second = torch.autograd.grad(inner, params, retain_graph=True, allow_unused=True)
            flat = torch.cat([(torch.zeros_like(p) if h is None else h).reshape(-1) for h, p in zip(second, params)])
            return flat + self.hvp_damping_coefficient * vector

        return product

    def _solve(self, hvp: Callable, b: Tensor, residual_tol: float = 1e-10) -> Tensor:
        """``n_conjugate_gradients`` iterations of conjugate gradient on H x = b (:169-202)."""
        x = torch.zeros_like(b)
        residual, search = b.clone(), b.clone()
        rr = torch.dot(residual, residual)
        for _ in range(self.n_conjugate_gradients):
            z = hvp(search)
            alpha = rr / torch.dot(search, z)
            x += alpha * search
            residual -= alpha * z
            rr_next = torch.dot(residual, residual)
            search = residual + (rr_next / rr) * search
            rr = rr_next
            if rr < residual_tol:
                break
        return x

    def _line_search(self, params: List[Tensor], descent: Tensor, loss_function: Callable, kl_function: Callable) -> None:
        """Backtracking over ``backtrack_ratio ** k``; a step that ends without improving the loss inside the trust
        region is undone (:204-250)."""
        saved = [p.detach().clone() for p in params]
        sizes = [p.numel() for p in params]
        pieces = [d.view_as(p) for d, p in zip(torch.split(torch.as_tensor(descent), sizes), params)]
        before = loss_function()
        new_loss = constraint = None
        for ratio in self.backtrack_ratio ** np.arange(self.max_backtracks):
            for p, old, d in zip(params, saved, pieces):
                p.data = old - ratio * d
            new_loss, constraint = loss_function(), kl_function()
            if new_loss < before and constraint <= self.max_constraint:
                break
        if (torch.isnan(new_loss) or torch.isnan(constraint) or new_loss >= before
                or constraint >= self.max_constraint):
            logger.warning("Line search condition violated. Rejecting the step.")
            for p, old in zip(params, saved):
                p.data = old


class NativeClosure:
    """What ``TRPO.train`` passes to ``ConjugateGradientOptimizer.step`` in place of the reference's two torch closures
    (ref trpo.py:154-175): a tag that carries the native step.  Both closures of one step share ``native_step``."""

    def __init__(self, what: str, native_step: Callable):
        self.what = what
        self.native_step = native_step

    def __call__(self):
        raise NotImplementedError(
            f"the TRPO {self.what} closure of rl_replicas_b200 is evaluated inside the GPU engine; only "
            "ConjugateGradientOptimizer.step can consume it")
