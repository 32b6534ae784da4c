"""D4PG (Barth-Maron et al. 2018, "Distributed Distributional Deterministic Policy Gradients") over the GPU off-policy
engine: DDPG with a categorical critic, n-step returns and prioritized replay.  DDPG's host loop, acting, evaluation and
checkpoints; on the device DDPG's step program with C51's projected cross-entropy as the critic's head and a policy head
that differentiates the critic's expected value (enqueue_steps in csrc/offpolicy.cu)."""
from __future__ import annotations

import numpy as np

from ..critics import DistributionalQFunction
from ..engine import OffPolicyEngine
from ._onpolicy import adam_hparams, describe_mlp, refuse_noisy
from .td3 import DDPG


class D4PG(DDPG):
    """Per train step, on a minibatch (s, a, r, s', d) and the critic's support z (b200rl.h, "D4PG"):
    a' = mu_targ(s') (no target smoothing), the target distribution m = the target critic's p(s', a') projected onto z
    after Tz = clamp(r + gamma (1 - d) z, v_min, v_max), one Adam step on the critic's cross-entropy
    -sum_i m_i log p_i(s, a) (mean over the minibatch), one Adam step on the policy's -mean Q(s, mu(s)) with
    Q = sum_i z_i p_i from the critic just updated, and Polyak averaging of both targets with ``polyak_rho``.

    The constructor takes DDPG's arguments and defaults with a ``DistributionalQFunction`` critic whose network maps
    [obs | act] to its n_atoms logits.  ``n_step`` (1..32) > 1 trains on n-step returns as DQN does: R and the discount
    gamma^k of each window take the places of r and gamma.  With a ``PrioritizedReplayBuffer`` every train() call takes
    the prioritized device path (draws keyed by ``device_rng_seed``): the cross-entropy is weighted by the importance
    weights, beta follows the critic optimizer's step count, and a row's priority is (KL + eps)^alpha of the KL
    divergence of its projected target from its predicted distribution.  n_step > 1 and prioritized replay need
    ``use_device_replay = True``.

    Acting and evaluation are DDPG's: Gaussian action noise ``action_noise_scale`` after ``num_start_steps``, the
    deterministic policy for evaluation.  Metrics and checkpoint keys are DDPG's; ``q-function/average_loss`` logs the
    critic's (weighted) mean cross-entropy, the Q-value tags its expected values, and prioritized replay adds
    replay/beta."""
    algo = OffPolicyEngine.D4PG

    def __init__(self, policy, exploration_policy, q_function, env, sampler, replay_buffer, evaluator,
                 gamma: float = 0.99, polyak_rho: float = 0.995, action_noise_scale: float = 0.1,
                 n_step: int = 1) -> None:
        space = env.action_space
        if getattr(space, "n", None) is not None or getattr(space, "high", None) is None:
            raise ValueError("D4PG needs a continuous action space (one with .high)")
        if not isinstance(q_function, DistributionalQFunction):
            raise ValueError(f"D4PG needs a DistributionalQFunction critic, got {type(q_function).__name__}")
        refuse_noisy("D4PG", policy, q_function)
        psz, _, _, plins = describe_mlp(policy.network)
        qsz, _, _, qlins = describe_mlp(q_function.network)
        A = int(np.prod(space.shape))
        obs_shape = getattr(getattr(env, "observation_space", None), "shape", None)
        O = int(np.prod(obs_shape)) if obs_shape else psz[0]
        if psz[0] != O or psz[-1] != A:
            raise ValueError(f"the policy must map {O} -> {A}, got {psz[0]} -> {psz[-1]}")
        if qsz[0] != O + A or qsz[-1] != q_function.n_atoms:
            raise ValueError(f"the critic must map {O} + {A} -> {q_function.n_atoms} (the atoms' logits), got "
                             f"{qsz[0]} -> {qsz[-1]}")
        adam_hparams(policy.optimizer, plins, "policy optimizer")
        adam_hparams(q_function.optimizer, qlins, "q-function optimizer")
        if isinstance(n_step, bool) or not isinstance(n_step, (int, np.integer)) or not 1 <= n_step <= 32:
            raise ValueError(f"n_step must be an integer from 1 to 32, got {n_step!r}")
        super().__init__(policy, exploration_policy, q_function, env, sampler, replay_buffer, evaluator, gamma=gamma,
                         polyak_rho=polyak_rho, action_noise_scale=action_noise_scale)
        self.n_step = int(n_step)

    @property
    def d4pg_config(self):
        """(n_atoms, v_min, v_max): the critic's support, fixed when the engine is created."""
        q = self.q_function
        return q.n_atoms, q.v_min, q.v_max

    def _engine_extra(self) -> dict:
        return dict(d4pg=self.d4pg_config)

    def _stage_inputs(self, replay_buffer, S: int, B: int, noisy: bool):
        staged = self._stage_nstep_and_prioritized(replay_buffer, S, self.q_function.optimizer,
                                                   describe_mlp(self.q_function.network)[3])
        if staged is not None:
            return staged
        return super()._stage_inputs(replay_buffer, S, B, noisy)

    def _call_engine(self, e, hp, replay_buffer, S: int, B: int, mode, inputs):
        return self._call_nstep_and_prioritized(e, hp, replay_buffer, S, B, mode, inputs)

    def _record_train(self, out) -> None:
        super()._record_train(out)
        mm, steps = getattr(self, "metrics_manager", None), getattr(self, "current_total_steps", 0)
        if mm is not None and out is not None and getattr(self, "_last_beta", None) is not None:
            mm.record_scalar("replay/beta", self._last_beta, steps, tensorboard=True)
