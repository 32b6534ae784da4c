"""TRPO -- the reference's class surface (ref: algorithms/trpo.py:28-277) over the GPU update engine."""
from __future__ import annotations

import logging

from ..optimizers import ConjugateGradientOptimizer
from ..optimizers.conjugate_gradient_optimizer import NativeClosure
from ._onpolicy import adam_hparams
from .ppo import PPO

logger = logging.getLogger(__name__)


class TRPO(PPO):
    """Same constructor as ref algorithms/trpo.py:43-52; ``policy.optimizer`` must be a ConjugateGradientOptimizer."""

    def __init__(self, policy, value_function, env, sampler, gamma: float = 0.99, gae_lambda: float = 0.97,
                 num_value_gradients: int = 80, distributed: bool = False, process_group=None) -> None:
        """``distributed`` / ``process_group`` (not in the reference): one process per GPU, each training on its own
        block of episodes; the constrained step all-reduces every batch-derived sum (the surrogate gradient, each
        Fisher-vector product, each line-search evaluation, the value gradients), so all ranks take the same step."""
        super().__init__(policy, value_function, env, sampler, gamma=gamma, gae_lambda=gae_lambda,
                         num_policy_gradients=1, num_value_gradients=num_value_gradients, distributed=distributed,
                         process_group=process_group)
        self.last_trpo_stats = None

    def _hparams(self, engine, n_global: int):
        return engine.hparams(
            gamma=self.gamma, gae_lambda=self.gae_lambda, num_policy_gradients=1,
            num_value_gradients=self.num_value_gradients, policy_adam=(0.0, 0.9, 0.999, 1e-8),
            value_adam=adam_hparams(self.value_function.optimizer, self._vlin, "value-function optimizer"),
            n_global_rows=n_global)

    def train_packed(self, batch) -> None:
        opt = self.policy.optimizer
        if not isinstance(opt, ConjugateGradientOptimizer):
            raise NotImplementedError("TRPO needs policy.optimizer to be a ConjugateGradientOptimizer")
        engine = self._ensure_engine(batch["obs"].shape[0], batch["ep_done"].shape[0])
        want = [t for l in self._plin for t in (l.weight, l.bias)]
        have = [p for g in opt.param_groups for p in g["params"]]
        if len(have) != len(want) or any(a is not b for a, b in zip(have, want)):
            raise NotImplementedError(
                "ConjugateGradientOptimizer must hold exactly the policy network's parameters (the native constrained "
                "step covers the network; a log_std inside the conjugate-gradient optimizer is not supported)")
        self._push_state(engine, with_old=True)
        engine.load_batch(batch)
        result = {}

        def native_step(optimizer):  # runs inside optimizer.step (ref trpo.py:180-185 calls it the same way)
            result["out"] = engine.trpo_update(self._hparams(engine, self._global_rows(engine.n_rows)),
                                               process_group=self.process_group, distributed=self.distributed,
                                               **optimizer.hyper_parameters())

        opt.step(NativeClosure("surrogate loss", native_step), NativeClosure("KL divergence", native_step))
        stats, ts = result["out"]
        self._pull_state(engine, with_old=True, policy_adam=False)
        self.last_update_stats, self.last_trpo_stats = stats, ts
        if ts.rejected:
            logger.warning("Line search condition violated. Rejecting the step.")
        mm, steps = getattr(self, "metrics_manager", None), getattr(self, "current_total_steps", 0)
        if mm is not None:  # ref trpo.py:203-226
            mm.record_scalar("policy/loss", stats.policy_loss_before, steps, tensorboard=True)
            mm.record_scalar("policy/avarage_entropy", stats.entropy_before, steps, tensorboard=True)
            mm.record_scalar("policy/log_prob_std", stats.logp_std_before, steps, tensorboard=True)
            mm.record_scalar("value_function/average_loss", stats.value_loss_mean, steps, tensorboard=True)
