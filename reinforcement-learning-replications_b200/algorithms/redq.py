"""REDQ (Chen, Wang, Zhou & Ross 2021, "Randomized Ensembled Double Q-Learning") over the GPU off-policy engine: SAC's
squashed-Gaussian policy and temperature over an ensemble of N critics, a target that takes the min over a random
subset of M target critics, and many critic updates per environment step.  ``train`` is the hot path
(enqueue_redq_steps in csrc/offpolicy.cu): the N critics run as one ensemble, one launch per layer for all of them."""
from __future__ import annotations

import copy

import numpy as np
import torch

from ..critics import ContinuousQuantileQFunction
from ..engine import OffPolicyEngine
from ..networks import ImplicitQuantileMLP
from ..replay_buffer import PrioritizedReplayBuffer
from ._onpolicy import adam_hparams, describe_mlp, refuse_noisy
from .sac import SAC
from .td3 import _learn


class REDQ(SAC):
    """Per train step st of a call of S steps: every critic takes one Adam step on mean((Q_i(s, a) - y)^2) with
    y = r + gamma (1 - d) (min_{i in M_st} Q'_i(s', a') - alpha log pi(a' | s')) over M = ``n_min`` target critics
    drawn without replacement; on steps with (st + 1) % ``policy_delay`` == 0 and on the last step the policy takes
    one Adam step on mean(alpha log pi - (1/N) sum_i Q_i(s, a_pi)) with the critics just updated (the reference code
    uses the critics from before their update), and with ``learn_alpha`` the temperature takes SAC's step; all N target
    critics are polyak-averaged every step.

    Host random streams, per train call: the S minibatches' indices first (numpy), then one
    ``np.random.choice(N, M, replace=False)`` per step (numpy), then per step ``torch.randn(B, A)`` for s' and, on
    policy steps only, one for s (torch)."""
    algo = OffPolicyEngine.REDQ

    def __init__(self, policy, exploration_policy, q_functions, env, sampler, replay_buffer, evaluator,
                 gamma: float = 0.99, polyak_rho: float = 0.995, alpha: float = 0.2, learn_alpha: bool = False,
                 target_entropy=None, alpha_lr: float = 3e-4, n_min: int = 2, policy_delay: int = 20) -> None:
        q_functions = list(q_functions)
        N, name = len(q_functions), type(self).__name__
        if N < 2:
            raise ValueError(f"{name} needs at least 2 critics, got {N}")
        if N > 32:
            raise ValueError(f"{name} supports at most 32 critics, got {N}")
        if not 1 <= int(n_min) <= N:
            raise ValueError(f"n_min must be in 1..{N} (the number of critics), got {n_min}")
        if int(policy_delay) < 1:
            raise ValueError(f"policy_delay must be >= 1, got {policy_delay}")
        if isinstance(replay_buffer, PrioritizedReplayBuffer):
            raise ValueError(f"{name} does not train on a PrioritizedReplayBuffer: prioritized replay is not "
                             "implemented for it")
        for q in q_functions:
            if isinstance(q, ContinuousQuantileQFunction) or isinstance(q.network, ImplicitQuantileMLP):
                raise TypeError(f"{name}'s critics map [obs | act] to one value, got {type(q).__name__} over "
                                f"{type(q.network).__name__}")
            if type(q.network).__name__ == "DuelingMLP":
                raise TypeError(f"{name} does not take dueling networks")
        refuse_noisy(name, policy, *q_functions)
        shapes = {(tuple(sz), hid, out) for sz, hid, out, _ in (describe_mlp(q.network) for q in q_functions)}
        if len(shapes) != 1:
            raise ValueError(f"{name}'s critics must all have the same shape, got {sorted(shapes)}")
        settings = {adam_hparams(q.optimizer, describe_mlp(q.network)[3], "q-function optimizer") for q in q_functions}
        if len(settings) != 1:
            raise NotImplementedError(f"{name}'s critics share one Adam setting (lr, betas, eps), got "
                                      f"{sorted(settings)}")
        super().__init__(policy, exploration_policy, q_functions[0], q_functions[1], env, sampler, replay_buffer,
                         evaluator, gamma=gamma, polyak_rho=polyak_rho, alpha=alpha, learn_alpha=learn_alpha,
                         target_entropy=target_entropy, alpha_lr=alpha_lr)
        for q in q_functions[2:]:  # SAC checked the first two
            qsz = describe_mlp(q.network)[0]
            O, A = describe_mlp(policy.network)[0][0], self.action_dim
            if qsz[0] != O + A or qsz[-1] != 1:
                raise ValueError(f"a Q network must map [obs {O} + act {A}] -> 1, got {qsz[0]} -> {qsz[-1]}")
        self.q_functions = q_functions
        self.target_q_functions = [self.target_q_function_1, self.target_q_function_2] + \
            [copy.deepcopy(q) for q in q_functions[2:]]
        for t in self.target_q_functions[2:]:
            for p in t.network.parameters():
                p.requires_grad = False
        self.n_critics, self.n_min, self.policy_delay = N, int(n_min), int(policy_delay)
        self.redq_config = (N, self.n_min)
        self.trainable_slots = tuple(range(1 + N))
        self.target_slots = tuple(range(1 + N, 1 + 2 * N))

    def _trainable(self):
        return [self.policy] + list(self.q_functions)

    def _nets(self):
        return self._trainable(), list(self.target_q_functions)

    def _engine_extra(self) -> dict:
        return {"redq": self.redq_config}

    def _train_schedule(self):
        return True, self.policy_delay

    def _noise(self, S: int, B: int):
        """(noise [S, 2, B, A], subsets [S, M]): the subsets from numpy (after the minibatch indices), then per step
        torch.randn(B, A) for s' and, on policy steps, for s (slot 1 of the other steps stays zero and is not read)."""
        N, M, G, A = self.n_critics, self.n_min, self.policy_delay, self.action_dim
        subsets = np.stack([np.random.choice(N, M, replace=False) for _ in range(S)]).astype(np.int32)
        out = np.zeros((S, 2, B, A), dtype=np.float32)
        for i in range(S):
            out[i, 0] = torch.randn(B, A).numpy()
            if (i + 1) % G == 0 or i == S - 1:
                out[i, 1] = torch.randn(B, A).numpy()
        return out, subsets

    def learn(self, num_epochs: int = 2000, batch_size: int = 50, minibatch_size: int = 100,
              num_start_steps: int = 10000, num_steps_before_update: int = 1000, num_train_steps: int = 1000,
              num_evaluation_episodes: int = 5, evaluation_interval: int = 4000, model_saving_interval: int = 4000,
              output_dir: str = ".") -> None:
        """SAC.learn; the default num_train_steps is 20 x batch_size: an update-to-data ratio of
        num_train_steps / batch_size = 20, the paper's G."""
        _learn(self, num_epochs, batch_size, minibatch_size, num_start_steps, num_steps_before_update, num_train_steps,
               num_evaluation_episodes, evaluation_interval, model_saving_interval, output_dir)

    def _record_train(self, out) -> None:
        mm, steps = getattr(self, "metrics_manager", None), getattr(self, "current_total_steps", 0)
        if mm is None or out is None:
            return
        mm.record_scalar("policy/average_loss", float(np.mean(out["policy_losses"])), steps, tensorboard=True)
        mm.record_scalar("policy/average_log_prob", float(np.mean(out["log_prob_means"])), steps, tensorboard=True)
        mm.record_scalar("alpha/value", float(out["alphas"][-1]), steps, tensorboard=True)
        for i in range(self.n_critics):
            q = out["redq_q_values"][i].astype(np.float64)
            mm.record_scalar(f"q-function_{i + 1}/average_loss", float(np.mean(out["redq_q_losses"][i])), steps,
                             tensorboard=True)
            mm.record_scalar(f"q-function_{i + 1}/avarage_q-value", float(np.mean(q)), steps, tensorboard=True)
            mm.record_scalar(f"q-function_{i + 1}/max_q-value", float(np.max(q)))
            mm.record_scalar(f"q-function_{i + 1}/min_q-value", float(np.min(q)))

    def save_model(self, current_epoch: int, model_path: str) -> None:
        """SAC's checkpoint keys with q_function_{i}_state_dict, q_function_{i}_optimizer_state_dict and
        target_q_function_{i}_state_dict for i = 1..N (at N = 2 exactly SAC's keys)."""
        ckpt = {"epoch": current_epoch, "total_steps": getattr(self, "current_total_steps", 0),
                "policy_state_dict": self.policy.network.state_dict(),
                "policy_optimizer_state_dict": self.policy.optimizer.state_dict()}
        for i, (q, t) in enumerate(zip(self.q_functions, self.target_q_functions), 1):
            ckpt[f"q_function_{i}_state_dict"] = q.network.state_dict()
            ckpt[f"q_function_{i}_optimizer_state_dict"] = q.optimizer.state_dict()
            ckpt[f"target_q_function_{i}_state_dict"] = t.network.state_dict()
        ckpt["log_alpha"] = self.log_alpha.detach().clone()
        ckpt["alpha_optimizer_state_dict"] = self.alpha_optimizer.state_dict()
        torch.save(ckpt, model_path)

    def load_model(self, model_path: str, trust_checkpoint: bool = False) -> int:
        """Resume from a checkpoint written by ``save_model``; returns the saved epoch."""
        ckpt = torch.load(model_path, map_location="cpu", weights_only=not trust_checkpoint)
        self.policy.network.load_state_dict(ckpt["policy_state_dict"])
        self.policy.optimizer.load_state_dict(ckpt["policy_optimizer_state_dict"])
        for i, (q, t) in enumerate(zip(self.q_functions, self.target_q_functions), 1):
            q.network.load_state_dict(ckpt[f"q_function_{i}_state_dict"])
            q.optimizer.load_state_dict(ckpt[f"q_function_{i}_optimizer_state_dict"])
            t.network.load_state_dict(ckpt[f"target_q_function_{i}_state_dict"])
        with torch.no_grad():
            self.log_alpha.copy_(ckpt["log_alpha"])
        self.alpha_optimizer.load_state_dict(ckpt["alpha_optimizer_state_dict"])
        self.current_total_steps = int(ckpt.get("total_steps", 0))
        return int(ckpt.get("epoch", 0))
