"""PPO-clip with approximate-KL early stopping -- the reference's class surface (ref: algorithms/ppo.py:29-306) over
the GPU update engine.  ``learn`` / ``save_model`` keep the reference's host-side behaviour; ``train`` is the hot
path: pack -> engine (CUDA) -> write-back."""
from __future__ import annotations

import copy
import logging
import os
import time
from typing import Optional

import numpy as np
import torch

from ..experience import Experience
from ..metrics_manager import MetricsManager
from ._onpolicy import OnPolicyTrainerMixin, adam_hparams, refuse_noisy

logger = logging.getLogger(__name__)


class PPO(OnPolicyTrainerMixin):
    """Same constructor arguments and defaults as ref algorithms/ppo.py:46-59.
    ``process_group`` / ``distributed`` (new, optional) shard the batch by environment across ranks with one gradient
    all-reduce per step (SURVEY.md section 8e); every rank must then call train() collectively."""

    def __init__(self, policy, value_function, env, sampler, gamma: float = 0.99, gae_lambda: float = 0.97,
                 clip_range: float = 0.2, max_kl_divergence: float = 0.01, num_policy_gradients: int = 80,
                 num_value_gradients: int = 80, distributed: bool = False, process_group=None) -> None:
        refuse_noisy(type(self).__name__, policy, value_function)
        self.policy = policy
        self.value_function = value_function
        self.env = env
        self.sampler = sampler
        self.gamma = gamma
        self.gae_lambda = gae_lambda
        self.clip_range = clip_range
        self.max_kl_divergence = max_kl_divergence
        self.num_policy_gradients = num_policy_gradients
        self.num_value_gradients = num_value_gradients
        self.distributed = distributed
        self.process_group = process_group
        self.old_policy = copy.deepcopy(self.policy)  # ref ppo.py:70
        self.last_update_stats = None

    # ------------------------------------------------------------------------------------------------------
    def learn(self, num_epochs: int = 50, batch_size: int = 4000, model_saving_interval: int = 4000,
              output_dir: str = ".") -> None:
        """Sample -> log -> train -> maybe save, once per epoch (ref: ppo.py:72-137)."""
        started = time.time()
        self.current_total_steps = 0
        self.current_total_episodes = 0
        os.makedirs(output_dir, exist_ok=True)
        self.metrics_manager = MetricsManager(output_dir)
        mm = self.metrics_manager
        for epoch in range(1, num_epochs + 1):
            experience: Experience = self.sampler.sample(batch_size, self.policy)
            returns, lengths = experience.episode_returns, experience.episode_lengths
            self.current_total_steps += sum(lengths)
            self.current_total_episodes += sum(experience.episode_dones)
            mm.record_scalar("epoch", epoch)
            mm.record_scalar("total_steps", self.current_total_steps)
            mm.record_scalar("total_episodes", self.current_total_episodes)
            mm.record_scalar("sampling/average_episode_return", float(np.mean(returns)), self.current_total_steps,
                             tensorboard=True)
            mm.record_scalar("sampling/episode_return_std", float(np.std(returns)))
            mm.record_scalar("sampling/max_episode_return", float(np.max(returns)))
            mm.record_scalar("sampling/min_episode_return", float(np.min(returns)))
            mm.record_scalar("sampling/average_episode_length", float(np.mean(lengths)), self.current_total_steps,
                             tensorboard=True)
            self.train(experience)
            if self.current_total_steps % model_saving_interval == 0:
                self.save_model(epoch, os.path.join(output_dir, "model.pt"))
            mm.record_scalar("time", time.time() - started)
            mm.dump()
        mm.close()

    # ------------------------------------------------------------------------------------------------------
    def _hparams(self, engine, n_global: int):
        return engine.hparams(
            gamma=self.gamma, gae_lambda=self.gae_lambda, clip_range=self.clip_range,
            max_kl_divergence=self.max_kl_divergence, num_policy_gradients=self.num_policy_gradients,
            num_value_gradients=self.num_value_gradients,
            policy_adam=adam_hparams(self.policy.optimizer, self._plin, "policy optimizer", self._trainable_log_std()),
            value_adam=adam_hparams(self.value_function.optimizer, self._vlin, "value-function optimizer"),
            n_global_rows=n_global)

    def train(self, experience: Experience) -> None:
        """The per-epoch update (ref: ppo.py:139-223) on the GPU."""
        self.train_packed(self.pack(experience))

    def train_packed(self, batch) -> None:
        """Same, from an already packed batch (contiguous host arrays; see synthetic.py for the layout)."""
        engine = self._ensure_engine(batch["obs"].shape[0], batch["ep_done"].shape[0])
        self._push_state(engine, with_old=True)
        engine.load_batch(batch)
        hp = self._hparams(engine, self._global_rows(engine.n_rows))
        stats = engine.update(hp, "ppo", self.process_group, self.distributed)
        self._pull_state(engine, with_old=True)
        self.last_update_stats = stats
        if stats.policy_steps_applied < self.num_policy_gradients:
            logger.info("Early stopping at update {} due to reaching max KL divergence.".format(
                stats.policy_steps_applied - 1))
        mm, steps = getattr(self, "metrics_manager", None), getattr(self, "current_total_steps", 0)
        if mm is not None:  # ref ppo.py:194-223 (tag typos are part of the API)
            mm.record_scalar("policy/loss", stats.policy_loss_before, steps, tensorboard=True)
            mm.record_scalar("policy/avarage_entropy", stats.entropy_before, steps, tensorboard=True)
            mm.record_scalar("policy/log_prob_std", stats.logp_std_before, steps, tensorboard=True)
            mm.record_scalar("policy/kl_divergence", stats.kl_divergence, steps, tensorboard=True)
            mm.record_scalar("value_function/average_loss", stats.value_loss_mean, steps, tensorboard=True)

    # ------------------------------------------------------------------------------------------------------
    def save_model(self, epoch: int, model_path: str) -> None:
        """Checkpoint with the reference's dictionary layout (ref: ppo.py:289-306)."""
        torch.save({
            "epoch": epoch,
            "total_steps": self.current_total_steps,
            "policy_state_dict": self.policy.network.state_dict(),
            "policy_optimizer_state_dict": self.policy.optimizer.state_dict(),
            "value_function_state_dict": self.value_function.network.state_dict(),
            "value_function_optimizer_state_dict": self.value_function.optimizer.state_dict(),
        }, model_path)

    def load_model(self, model_path: str, trust_checkpoint: bool = False) -> int:
        """Resume from a checkpoint written by ``save_model`` -- or by the reference's (same dictionary layout,
        ref ppo.py:296-306; the shipped benchmarks/*/model.pt load as warm starts).  Restores both networks, both
        optimizer states (Adam moments and step counts -- the next ``train`` continues the bias correction where the run
        stopped) and ``current_total_steps``; returns the saved epoch.  The reference has no loader (SURVEY 8f-3); a
        Gaussian policy's ``log_std`` is not part of the checkpoint there either and keeps its constructor value.
        The file is read with ``weights_only=True`` (tensors, numbers and optimizer state dictionaries -- everything
        ``save_model`` writes); ``trust_checkpoint=True`` allows arbitrary pickles for legacy files you trust."""
        ckpt = torch.load(model_path, map_location="cpu", weights_only=not trust_checkpoint)
        self.policy.network.load_state_dict(ckpt["policy_state_dict"])
        self.value_function.network.load_state_dict(ckpt["value_function_state_dict"])
        for module, key in ((self.policy, "policy_optimizer_state_dict"),
                            (self.value_function, "value_function_optimizer_state_dict")):
            state = ckpt.get(key)
            if state and hasattr(module.optimizer, "load_state_dict") and state.get("state") is not None:
                try:
                    module.optimizer.load_state_dict(state)
                except (ValueError, KeyError):  # e.g. TRPO's conjugate-gradient optimizer keeps no per-parameter state
                    pass
        if hasattr(self, "old_policy"):
            self.old_policy.network.load_state_dict(self.policy.network.state_dict())  # ref ppo.py:183 invariant
        self.current_total_steps = int(ckpt.get("total_steps", 0))
        return int(ckpt.get("epoch", 0))
