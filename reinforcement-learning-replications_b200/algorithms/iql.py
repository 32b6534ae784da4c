"""IQL (Kostrikov, Nair & Levine 2021, "Offline Reinforcement Learning with Implicit Q-Learning") over the GPU off-policy
engine: an expectile value network, an advantage-weighted policy and twin critics, none of which is evaluated at an
action outside the data.  Built for a fixed dataset (``ReplayBuffer.from_dataset`` and ``learn_offline``); ``learn``
fine-tunes online by sampling the policy.  On the device its own step program (enqueue_iql_steps in
csrc/offpolicy.cu)."""
from __future__ import annotations

import copy
import math

import numpy as np
import torch

from ..critics import ContinuousQuantileQFunction, ValueFunction
from ..engine import OffPolicyEngine
from ..networks import DuelingMLP, ImplicitQuantileMLP
from ..policies import TanhMeanGaussianPolicy
from ..replay_buffer import PrioritizedReplayBuffer
from ._onpolicy import adam_hparams, describe_mlp, refuse_noisy
from .td3 import _learn, _make_eval_env, _OffPolicyBase


class IQL(_OffPolicyBase):
    """Per train step, on a minibatch (s, a, r, s', d) (b200rl.h, "IQL"): q^ = min(Q1targ, Q2targ)(s, a); one Adam step
    on V for the expectile loss mean(|tau - 1{q^ - V(s) < 0}| (q^ - V(s))^2); one Adam step on the policy for
    -mean(e log pi(a | s)) with e = min(exp(beta (q^ - V'(s))), max_weight) from the updated V'; one Adam step on each
    critic towards r + gamma (1 - d) V'(s'); polyak averaging of both target critics.  beta = 0 is behaviour cloning.

    ``policy`` is a ``TanhMeanGaussianPolicy``, ``value_function`` a ``critics.ValueFunction`` over [obs, ..., 1], the
    critics plain ``QFunction``s over [obs + act, ..., 1]; ``sampler`` and ``exploration_policy`` may be None for
    offline training.  Metric tags are SAC's without ``alpha/value`` and ``policy/average_log_prob``, plus
    ``value-function/average_loss``, ``value-function/average_value`` and ``iql/average_weight``; the checkpoint is
    SAC's without the temperature, plus ``value_function_state_dict`` and ``value_function_optimizer_state_dict``.
    Prioritized replay, n-step returns and quantile, distributional, noisy, dueling and IQN networks are not
    implemented for IQL."""
    n_q = 2
    algo = OffPolicyEngine.IQL
    trainable_slots = (0, 1, 2, 3)  # V is engine network 3, optimizer 3
    target_slots = (4, 5)

    def __init__(self, policy, exploration_policy, q_function_1, q_function_2, value_function, env, sampler,
                 replay_buffer, evaluator, gamma: float = 0.99, polyak_rho: float = 0.995, expectile: float = 0.7,
                 beta: float = 3.0, max_weight: float = 100.0) -> None:
        if not isinstance(policy, TanhMeanGaussianPolicy):
            raise TypeError(f"IQL needs a TanhMeanGaussianPolicy, got {type(policy).__name__}")
        if not isinstance(value_function, ValueFunction):
            raise TypeError(f"IQL needs a critics.ValueFunction, got {type(value_function).__name__}")
        for what, q in (("q_function_1", q_function_1), ("q_function_2", q_function_2)):
            if isinstance(q, ContinuousQuantileQFunction) or hasattr(q, "n_atoms"):
                raise TypeError(f"IQL: {what} is a {type(q).__name__}; IQL trains plain QFunction critics (quantile "
                                "and distributional critics are not implemented for it)")
        for what, m in (("policy", policy), ("q_function_1", q_function_1), ("q_function_2", q_function_2),
                        ("value_function", value_function)):
            if isinstance(m.network, (DuelingMLP, ImplicitQuantileMLP)):
                raise NotImplementedError(f"IQL: the {what} network is a {type(m.network).__name__}: dueling and IQN "
                                          "networks are not implemented for IQL (plain MLPs only)")
        refuse_noisy("IQL", policy, q_function_1, q_function_2, value_function)
        if isinstance(replay_buffer, PrioritizedReplayBuffer):
            raise ValueError("IQL does not train on a PrioritizedReplayBuffer: prioritized replay is not implemented "
                             "for IQL")
        for name, v in (("expectile", expectile), ("beta", beta), ("max_weight", max_weight)):
            if not math.isfinite(float(v)):
                raise ValueError(f"IQL: {name} must be finite, got {v!r}")
        if not 0.0 < expectile < 1.0:
            raise ValueError(f"IQL: expectile must be in (0, 1), got {expectile}")
        if beta < 0:
            raise ValueError(f"IQL: beta must be >= 0, got {beta}")
        if max_weight <= 0:
            raise ValueError(f"IQL: max_weight must be > 0, got {max_weight}")
        A = int(np.prod(env.action_space.shape))
        psz, _, _, plin = describe_mlp(policy.network)
        O = psz[0]
        if psz[-1] != 2 * A:
            raise ValueError(f"IQL: the policy network must output [mean | log_std] = {2 * A} values, got {psz[-1]}")
        limit = float(env.action_space.high[0])
        if policy.action_limit != limit:
            raise ValueError(f"IQL: policy.action_limit {policy.action_limit} != the action space's bound {limit}")
        adam_hparams(policy.optimizer, plin, "IQL policy optimizer")
        for q in (q_function_1, q_function_2):
            qsz, _, _, qlin = describe_mlp(q.network)
            if qsz[0] != O + A or qsz[-1] != 1:
                raise ValueError(f"IQL: a Q network must map [obs {O} + act {A}] -> 1, got {qsz[0]} -> {qsz[-1]}")
            adam_hparams(q.optimizer, qlin, "IQL q-function optimizer")
        vsz, _, _, vlin = describe_mlp(value_function.network)
        if vsz[0] != O or vsz[-1] != 1:
            raise ValueError(f"IQL: the value network must map [obs {O}] -> 1, got {vsz[0]} -> {vsz[-1]}")
        adam_hparams(value_function.optimizer, vlin, "IQL value-function optimizer")
        self.policy, self.exploration_policy = policy, exploration_policy
        self.q_function_1, self.q_function_2, self.value_function = q_function_1, q_function_2, value_function
        self.env, self.sampler, self.replay_buffer, self.evaluator = env, sampler, replay_buffer, evaluator
        self.gamma, self.polyak_rho = gamma, polyak_rho
        self.expectile, self.beta, self.max_weight = float(expectile), float(beta), float(max_weight)
        self.action_dim = A
        self.noised_policy = policy  # after warm-up the policy explores by sampling
        self.evaluation_policy = policy.deterministic()
        self.evaluation_env = _make_eval_env(env)
        self.target_q_function_1, self.target_q_function_2 = [copy.deepcopy(q) for q in (q_function_1, q_function_2)]
        for t in (self.target_q_function_1, self.target_q_function_2):
            for p in t.network.parameters():
                p.requires_grad = False

    def _trainable(self):
        return [self.policy, self.q_function_1, self.q_function_2, self.value_function]

    def _nets(self):
        return self._trainable(), [self.target_q_function_1, self.target_q_function_2]

    def _engine_extra(self) -> dict:
        vsz, vact, vout, _ = describe_mlp(self.value_function.network)
        return dict(iql=(tuple(vsz), (vact, vout)))

    def iql_hparams(self) -> dict:
        """``OffPolicyEngine.set_iql``'s arguments."""
        lr, b1, b2, eps = adam_hparams(self.value_function.optimizer, describe_mlp(self.value_function.network)[3],
                                       "IQL value-function optimizer")
        return dict(expectile=self.expectile, beta=self.beta, max_weight=self.max_weight,
                    log_std_min=self.policy.log_std_min, log_std_max=self.policy.log_std_max, v_lr=lr,
                    v_betas=(b1, b2), v_eps=eps)

    def _train_schedule(self):
        return False, 1  # no noise, no policy delay

    def _hparams(self, noisy: bool, delay: int):
        hp = super()._hparams(False, 1)
        hp.action_limit = self.policy.action_limit  # the policy mean's bound
        return hp

    def _upload_state(self, e, trainable, targets, lins) -> None:
        super()._upload_state(e, trainable, targets, lins)
        e.set_iql(**self.iql_hparams())

    def learn(self, num_epochs: int = 2000, batch_size: int = 50, minibatch_size: int = 100,
              num_start_steps: int = 10000, num_steps_before_update: int = 1000, num_train_steps: int = 50,
              num_evaluation_episodes: int = 5, evaluation_interval: int = 4000, model_saving_interval: int = 4000,
              output_dir: str = ".") -> None:
        _learn(self, num_epochs, batch_size, minibatch_size, num_start_steps, num_steps_before_update, num_train_steps,
               num_evaluation_episodes, evaluation_interval, model_saving_interval, output_dir)

    def _record_train(self, out) -> None:
        mm, steps = getattr(self, "metrics_manager", None), getattr(self, "current_total_steps", 0)
        if mm is None or out is None:
            return
        mm.record_scalar("policy/average_loss", float(np.mean(out["policy_losses"])), steps, tensorboard=True)
        mm.record_scalar("q-function_1/average_loss", float(np.mean(out["q1_losses"])), steps, tensorboard=True)
        mm.record_scalar("q-function_2/average_loss", float(np.mean(out["q2_losses"])), steps, tensorboard=True)
        for i, key in ((1, "q1_values"), (2, "q2_values")):
            q = out[key].astype(np.float64)
            mm.record_scalar(f"q-function_{i}/avarage_q-value", float(np.mean(q)), steps, tensorboard=True)
            mm.record_scalar(f"q-function_{i}/max_q-value", float(np.max(q)))
            mm.record_scalar(f"q-function_{i}/min_q-value", float(np.min(q)))
        mm.record_scalar("value-function/average_loss", float(np.mean(out["value_losses"])), steps, tensorboard=True)
        mm.record_scalar("value-function/average_value", float(np.mean(out["value_means"])), steps, tensorboard=True)
        mm.record_scalar("iql/average_weight", float(np.mean(out["weight_means"])), steps, tensorboard=True)

    def save_model(self, current_epoch: int, model_path: str) -> None:
        """SAC's checkpoint keys without the temperature, plus the value function and its optimizer."""
        torch.save({
            "epoch": current_epoch, "total_steps": getattr(self, "current_total_steps", 0),
            "policy_state_dict": self.policy.network.state_dict(),
            "policy_optimizer_state_dict": self.policy.optimizer.state_dict(),
            "q_function_1_state_dict": self.q_function_1.network.state_dict(),
            "q_function_1_optimizer_state_dict": self.q_function_1.optimizer.state_dict(),
            "target_q_function_1_state_dict": self.target_q_function_1.network.state_dict(),
            "q_function_2_state_dict": self.q_function_2.network.state_dict(),
            "q_function_2_optimizer_state_dict": self.q_function_2.optimizer.state_dict(),
            "target_q_function_2_state_dict": self.target_q_function_2.network.state_dict(),
            "value_function_state_dict": self.value_function.network.state_dict(),
            "value_function_optimizer_state_dict": self.value_function.optimizer.state_dict(),
        }, model_path)

    def load_model(self, model_path: str, trust_checkpoint: bool = False) -> int:
        """Resume from a checkpoint written by ``save_model``; returns the saved epoch."""
        ckpt = torch.load(model_path, map_location="cpu", weights_only=not trust_checkpoint)
        self.policy.network.load_state_dict(ckpt["policy_state_dict"])
        self.policy.optimizer.load_state_dict(ckpt["policy_optimizer_state_dict"])
        for i, (q, t) in enumerate(((self.q_function_1, self.target_q_function_1),
                                    (self.q_function_2, self.target_q_function_2)), 1):
            q.network.load_state_dict(ckpt[f"q_function_{i}_state_dict"])
            q.optimizer.load_state_dict(ckpt[f"q_function_{i}_optimizer_state_dict"])
            t.network.load_state_dict(ckpt[f"target_q_function_{i}_state_dict"])
        self.value_function.network.load_state_dict(ckpt["value_function_state_dict"])
        self.value_function.optimizer.load_state_dict(ckpt["value_function_optimizer_state_dict"])
        self.current_total_steps = int(ckpt.get("total_steps", 0))
        return int(ckpt.get("epoch", 0))
