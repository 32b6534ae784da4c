"""Soft Actor-Critic (Spinning Up sac/sac.py, with an optional learned temperature) over the GPU off-policy engine.
``learn`` is the shared off-policy host loop; ``train`` is the hot path (enqueue_sac_steps in csrc/offpolicy.cu)."""
from __future__ import annotations

import copy
import math

import numpy as np
import torch
from torch import nn

from .._lib import SacHparams
from ..engine import OffPolicyEngine
from ..policies import SquashedGaussianPolicy
from ._onpolicy import adam_hparams, describe_mlp, refuse_noisy
from .td3 import _learn, _make_eval_env, _OffPolicyBase


class SAC(_OffPolicyBase):
    """Per train step: one Adam step on each critic towards the soft target
    r + gamma (1 - d) (min(Q1targ, Q2targ)(s', a') - alpha log pi(a' | s')), one Adam step on the policy loss
    mean(alpha log pi - min(Q1, Q2)(s, a_pi)), optionally one Adam step on log_alpha for
    -mean(log_alpha (log pi + target_entropy)), and polyak averaging of both target critics.  alpha = exp(log_alpha);
    with learn_alpha=False it stays at ``alpha``.  target_entropy defaults to -A."""
    n_q = 2
    algo = OffPolicyEngine.SAC
    target_slots = (4, 5)  # no target policy

    def __init__(self, policy, exploration_policy, q_function_1, q_function_2, env, sampler, replay_buffer, evaluator,
                 gamma: float = 0.99, polyak_rho: float = 0.995, alpha: float = 0.2, learn_alpha: bool = False,
                 target_entropy=None, alpha_lr: float = 3e-4) -> None:
        if not isinstance(policy, SquashedGaussianPolicy):
            raise TypeError(f"SAC needs a SquashedGaussianPolicy, got {type(policy).__name__}")
        refuse_noisy("SAC", policy, q_function_1, q_function_2)
        A = int(np.prod(env.action_space.shape))
        psz, _, _, plin = describe_mlp(policy.network)
        O = psz[0]
        if psz[-1] != 2 * A:
            raise ValueError(f"the SAC policy network must output [mean | log_std] = {2 * A} values, got {psz[-1]}")
        limit = float(env.action_space.high[0])
        if policy.action_limit != limit:
            raise ValueError(f"policy.action_limit {policy.action_limit} != the action space's bound {limit}")
        adam_hparams(policy.optimizer, plin, "policy optimizer")
        for q in (q_function_1, q_function_2):
            qsz, _, _, qlin = describe_mlp(q.network)
            width = self._critic_width(q)
            if qsz[0] != O + A or qsz[-1] != width:
                raise ValueError(f"a Q network must map [obs {O} + act {A}] -> {width}, got {qsz[0]} -> {qsz[-1]}")
            adam_hparams(q.optimizer, qlin, "q-function optimizer")
        if alpha <= 0:
            raise ValueError("alpha must be > 0")
        self.policy, self.exploration_policy = policy, exploration_policy
        self.q_function_1, self.q_function_2 = q_function_1, q_function_2
        self.env, self.sampler, self.replay_buffer, self.evaluator = env, sampler, replay_buffer, evaluator
        self.gamma, self.polyak_rho = gamma, polyak_rho
        self.learn_alpha = bool(learn_alpha)
        self.alpha = float(alpha)  # the fixed coefficient (learn_alpha=False)
        self.target_entropy = float(-A if target_entropy is None else target_entropy)
        self.action_dim = A
        self.log_alpha = nn.Parameter(torch.tensor(math.log(alpha), dtype=torch.float32))
        self.alpha_optimizer = torch.optim.Adam([self.log_alpha], lr=alpha_lr)
        self.noised_policy = policy  # after warm-up the policy explores by sampling
        self.evaluation_policy = policy.deterministic()
        self.evaluation_env = _make_eval_env(env)
        self.target_q_function_1, self.target_q_function_2 = [copy.deepcopy(q) for q in (q_function_1, q_function_2)]
        for t in (self.target_q_function_1, self.target_q_function_2):
            for p in t.network.parameters():
                p.requires_grad = False

    def _critic_width(self, q_function) -> int:
        """The output width each critic network must have."""
        return 1

    def _nets(self):
        return self._trainable(), [self.target_q_function_1, self.target_q_function_2]

    def _noise(self, S: int, B: int) -> np.ndarray:
        """[S, 2, B, A]: per step torch.randn(B, A) for s' (compute_loss_q), then for s (compute_loss_pi) -- the order
        in which Spinning Up's update() draws its two rsample()s."""
        A = self.action_dim
        out = np.empty((S, 2, B, A), dtype=np.float32)
        for i in range(S):
            out[i, 0] = torch.randn(B, A).numpy()
            out[i, 1] = torch.randn(B, A).numpy()
        return out

    def _sac_hparams(self) -> SacHparams:
        sp = SacHparams()
        sp.alpha, sp.learn_alpha, sp.target_entropy = self.alpha, int(self.learn_alpha), self.target_entropy
        sp.alpha_lr, sp.alpha_beta1, sp.alpha_beta2, sp.alpha_eps = adam_hparams(
            self.alpha_optimizer, [], "alpha optimizer", extra=[self.log_alpha])
        sp.log_std_min, sp.log_std_max = self.policy.log_std_min, self.policy.log_std_max
        return sp

    # log_alpha and its Adam state travel with the networks' state on every train() call
    def _upload_state(self, e, trainable, targets, lins) -> None:
        super()._upload_state(e, trainable, targets, lins)
        e.set_sac(self._sac_hparams())
        e.set_alpha(*self._alpha_state())

    def _download_state(self, e, trainable, targets, lins) -> None:
        super()._download_state(e, trainable, targets, lins)
        self._store_alpha_state(*e.get_alpha())

    def _alpha_state(self):
        """(log_alpha, exp_avg, exp_avg_sq, step) of the temperature, as the engine takes it."""
        st = self.alpha_optimizer.state.get(self.log_alpha, {})
        step = int(float(st["step"])) if "exp_avg" in st else 0
        m = float(st["exp_avg"]) if step else 0.0
        v = float(st["exp_avg_sq"]) if step else 0.0
        return float(self.log_alpha.detach()), m, v, step

    def _store_alpha_state(self, log_alpha, m, v, step) -> None:
        with torch.no_grad():
            self.log_alpha.fill_(log_alpha)
        if step > 0:
            st = self.alpha_optimizer.state[self.log_alpha]
            st["step"] = torch.tensor(float(step))
            st["exp_avg"] = torch.tensor(m, dtype=torch.float32)
            st["exp_avg_sq"] = torch.tensor(v, dtype=torch.float32)

    def learn(self, num_epochs: int = 2000, batch_size: int = 50, minibatch_size: int = 100,
              num_start_steps: int = 10000, num_steps_before_update: int = 1000, num_train_steps: int = 50,
              num_evaluation_episodes: int = 5, evaluation_interval: int = 4000, model_saving_interval: int = 4000,
              output_dir: str = ".") -> None:
        _learn(self, num_epochs, batch_size, minibatch_size, num_start_steps, num_steps_before_update, num_train_steps,
               num_evaluation_episodes, evaluation_interval, model_saving_interval, output_dir)

    def _train_schedule(self):
        return True, 1

    def _record_train(self, out) -> None:
        mm, steps = getattr(self, "metrics_manager", None), getattr(self, "current_total_steps", 0)
        if mm is None or out is None:
            return
        mm.record_scalar("policy/average_loss", float(np.mean(out["policy_losses"])), steps, tensorboard=True)
        mm.record_scalar("policy/average_log_prob", float(np.mean(out["log_prob_means"])), steps, tensorboard=True)
        mm.record_scalar("alpha/value", float(out["alphas"][-1]), steps, tensorboard=True)
        mm.record_scalar("q-function_1/average_loss", float(np.mean(out["q1_losses"])), steps, tensorboard=True)
        mm.record_scalar("q-function_2/average_loss", float(np.mean(out["q2_losses"])), steps, tensorboard=True)
        for i, key in ((1, "q1_values"), (2, "q2_values")):
            q = out[key].astype(np.float64)
            mm.record_scalar(f"q-function_{i}/avarage_q-value", float(np.mean(q)), steps, tensorboard=True)
            mm.record_scalar(f"q-function_{i}/max_q-value", float(np.max(q)))
            mm.record_scalar(f"q-function_{i}/min_q-value", float(np.min(q)))

    def save_model(self, current_epoch: int, model_path: str) -> None:
        """TD3's checkpoint keys without the target policy, plus log_alpha and its optimizer."""
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
            "log_alpha": self.log_alpha.detach().clone(),
            "alpha_optimizer_state_dict": self.alpha_optimizer.state_dict(),
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
        with torch.no_grad():
            self.log_alpha.copy_(ckpt["log_alpha"])
        self.alpha_optimizer.load_state_dict(ckpt["alpha_optimizer_state_dict"])
        self.current_total_steps = int(ckpt.get("total_steps", 0))
        return int(ckpt.get("epoch", 0))
