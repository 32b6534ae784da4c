"""EDAC and SAC-N (An, Moon, Kim & Song 2021, "Uncertainty-Based Offline Reinforcement Learning with Diversified
Q-Ensemble") over the GPU off-policy engine: SAC's squashed-Gaussian policy and temperature over an ensemble of N
critics whose target and policy head take the min over all N, plus (EDAC, ``eta`` > 0) a penalty that pushes the
critics' action gradients apart.  ``train`` is the hot path (enqueue_edac_steps in csrc/offpolicy.cu): the N critics
run as one ensemble, and the penalty's parameter gradient is a pass of its own beside the target path."""
from __future__ import annotations

import math

import numpy as np

from ..engine import OffPolicyEngine
from ._onpolicy import describe_mlp
from .redq import REDQ
from .sac import SAC
from .td3 import _learn


class EDAC(REDQ):
    """Per train step st of a call of S steps: every critic takes one Adam step on
    mean((Q_i(s, a) - y)^2) + eta D with y = r + gamma (1 - d) (min_i Q'_i(s', a') - alpha log pi(a' | s')) over all N
    target critics and D = sum_b sum_{i != j} gh_i . gh_j / (B (N - 1)), gh_i = g_i / (|g_i| + 1e-10), g_i = dQ_i / da
    at the dataset action (both terms at the parameters from before the step); then the policy takes one Adam step on
    mean(alpha log pi - min_i Q_i(s, a_pi)) with the critics just updated (the authors' code uses the critics from
    before their update), with ``learn_alpha`` the temperature takes SAC's step, and all N target critics are
    polyak-averaged.  ``eta = 0`` is SAC-N.  With ``eta`` > 0 the critics must have ReLU hidden layers and an identity
    output.

    Host random streams, per train call: SAC's -- the S minibatches' indices first (numpy), then per step
    ``torch.randn(B, A)`` for s' and then for s (torch)."""
    algo = OffPolicyEngine.EDAC

    def __init__(self, policy, exploration_policy, q_functions, env, sampler, replay_buffer, evaluator,
                 gamma: float = 0.99, polyak_rho: float = 0.995, alpha: float = 0.2, learn_alpha: bool = True,
                 target_entropy=None, alpha_lr: float = 3e-4, eta: float = 1.0) -> None:
        eta = float(eta)
        if not math.isfinite(eta) or eta < 0.0:
            raise ValueError(f"eta must be finite and >= 0, got {eta}")
        q_functions = list(q_functions)
        super().__init__(policy, exploration_policy, q_functions, env, sampler, replay_buffer, evaluator, gamma=gamma,
                         polyak_rho=polyak_rho, alpha=alpha, learn_alpha=learn_alpha, target_entropy=target_entropy,
                         alpha_lr=alpha_lr, n_min=max(len(q_functions), 1), policy_delay=1)
        _, hidden, out, lins = describe_mlp(q_functions[0].network)
        if eta > 0.0 and ((len(lins) > 1 and hidden != "relu") or out != "identity"):
            raise NotImplementedError(f"EDAC with eta > 0 needs critics with ReLU hidden layers and an identity output, "
                                      f"got {hidden} / {out} (the diversity term of other activations is not "
                                      "implemented; eta = 0, SAC-N, takes any)")
        self.eta = eta
        self.edac_config = (self.n_critics, eta)

    def _engine_extra(self) -> dict:
        return {"edac": self.edac_config}

    def _train_schedule(self):
        return True, 1

    def _noise(self, S: int, B: int):
        return SAC._noise(self, S, B)

    def learn(self, num_epochs: int = 2000, batch_size: int = 50, minibatch_size: int = 100,
              num_start_steps: int = 10000, num_steps_before_update: int = 1000, num_train_steps: int = 50,
              num_evaluation_episodes: int = 5, evaluation_interval: int = 4000, model_saving_interval: int = 4000,
              output_dir: str = ".") -> None:
        """SAC.learn: one train step per environment step by default."""
        _learn(self, num_epochs, batch_size, minibatch_size, num_start_steps, num_steps_before_update, num_train_steps,
               num_evaluation_episodes, evaluation_interval, model_saving_interval, output_dir)

    def _record_train(self, out) -> None:
        super()._record_train(out)
        mm, steps = getattr(self, "metrics_manager", None), getattr(self, "current_total_steps", 0)
        if mm is None or out is None or self.eta == 0.0:
            return
        mm.record_scalar("edac/diversity_loss", float(np.mean(out["edac_diversity"])), steps, tensorboard=True)
