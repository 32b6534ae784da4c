"""CQL (Kumar, Zhou, Tucker & Levine 2020, "Conservative Q-Learning for Offline Reinforcement Learning"), CQL(H) on
SAC, over the GPU off-policy engine: SAC's networks, acting, evaluation and checkpoints, with a log-sum-exp penalty over
sampled actions in each critic's loss.  Built for a fixed dataset (``ReplayBuffer.from_dataset`` and ``learn_offline``);
on the device SAC's step program with the critics fanned out over the sampled actions (enqueue_sac_steps in
csrc/offpolicy.cu)."""
from __future__ import annotations

import math

import numpy as np
import torch
from torch import nn

from ..critics import ContinuousQuantileQFunction
from ..engine import OffPolicyEngine
from ..networks import DuelingMLP, ImplicitQuantileMLP
from ..replay_buffer import PrioritizedReplayBuffer
from ._onpolicy import adam_hparams
from .sac import SAC

MAX_ACTIONS = 64  # N: the engine's penalty head takes at most 3 x 64 values per row


class CQL(SAC):
    """Per train step, on a minibatch (s, a, r, s', d) (b200rl.h, "CQL"): SAC's draws a', log pi' at s' and a_pi,
    log pi at s; N uniform actions u in [-L, L]^A (log density -A log 2L) and N policy samples each at s and at s' per
    row, all evaluated by each critic at s; the target r + gamma (1 - d) (min(Q1targ, Q2targ)(s', a') -
    [backup_entropy] alpha log pi'); each critic's loss is the MSE to it plus w_eff (mean_i T logsumexp_j(c_ij / T) -
    mean_i Q(s_i, a_i)) over the 3N values c_ij = Q(s_i, sample) - its log density; w_eff = ``cql_weight``, or
    alpha' ``cql_weight`` with the Lagrange step (``cql_target_action_gap`` not None), which runs one Adam step on
    log alpha' for -1/2 sum_k alpha' (w gap_k - tau).  Then SAC's policy step, optional temperature step and polyak.

    The constructor takes SAC's arguments and defaults (``sampler`` and ``exploration_policy`` may be None for offline
    training) plus ``cql_weight``, ``cql_n_actions`` (1..64), ``cql_temperature``, ``cql_target_action_gap``,
    ``cql_alpha_lr`` and ``backup_entropy``.  Metric tags are SAC's plus ``cql/penalty_1`` / ``cql/penalty_2`` (the
    mean gap of each critic over the call) and ``cql/alpha_prime`` with the Lagrange step; the checkpoint is SAC's plus
    ``log_alpha_prime`` and ``alpha_prime_optimizer_state_dict``.  Prioritized replay, n-step returns and quantile,
    noisy, dueling and IQN networks are not implemented for CQL."""
    algo = OffPolicyEngine.CQL

    def __init__(self, policy, exploration_policy, q_function_1, q_function_2, env, sampler, replay_buffer, evaluator,
                 gamma: float = 0.99, polyak_rho: float = 0.995, alpha: float = 0.2, learn_alpha: bool = False,
                 target_entropy=None, alpha_lr: float = 3e-4, cql_weight: float = 5.0, cql_n_actions: int = 10,
                 cql_temperature: float = 1.0, cql_target_action_gap=None, cql_alpha_lr: float = 3e-4,
                 backup_entropy: bool = False) -> None:
        for what, q in (("q_function_1", q_function_1), ("q_function_2", q_function_2)):
            if isinstance(q, ContinuousQuantileQFunction):
                raise TypeError(f"CQL: {what} is a quantile critic; CQL trains plain QFunction critics")
        for what, m in (("policy", policy), ("q_function_1", q_function_1), ("q_function_2", q_function_2)):
            if isinstance(m.network, (DuelingMLP, ImplicitQuantileMLP)):
                raise NotImplementedError(f"CQL: the {what} network is a {type(m.network).__name__}: dueling and IQN "
                                          "networks are not implemented for CQL (plain MLPs only)")
        if isinstance(replay_buffer, PrioritizedReplayBuffer):
            raise ValueError("CQL does not train on a PrioritizedReplayBuffer: prioritized replay is not implemented "
                             "for CQL")
        n = cql_n_actions
        if isinstance(n, bool) or not isinstance(n, int) or not 1 <= n <= MAX_ACTIONS:
            raise ValueError(f"CQL: cql_n_actions must be an integer from 1 to {MAX_ACTIONS}, got {n!r}")
        for name, v in (("cql_weight", cql_weight), ("cql_temperature", cql_temperature), ("cql_alpha_lr", cql_alpha_lr),
                        ("cql_target_action_gap", 0.0 if cql_target_action_gap is None else cql_target_action_gap)):
            if not math.isfinite(float(v)):
                raise ValueError(f"CQL: {name} must be finite, got {v!r}")
        if cql_weight < 0:
            raise ValueError(f"CQL: cql_weight must be >= 0, got {cql_weight}")
        if cql_temperature <= 0:
            raise ValueError(f"CQL: cql_temperature must be > 0, got {cql_temperature}")
        super().__init__(policy, exploration_policy, q_function_1, q_function_2, env, sampler, replay_buffer, evaluator,
                         gamma=gamma, polyak_rho=polyak_rho, alpha=alpha, learn_alpha=learn_alpha,
                         target_entropy=target_entropy, alpha_lr=alpha_lr)
        self.cql_weight, self.cql_n_actions = float(cql_weight), int(n)
        self.cql_temperature = float(cql_temperature)
        self.cql_target_action_gap = None if cql_target_action_gap is None else float(cql_target_action_gap)
        self.backup_entropy = bool(backup_entropy)
        self.log_alpha_prime = nn.Parameter(torch.tensor(0.0, dtype=torch.float32))
        self.alpha_prime_optimizer = torch.optim.Adam([self.log_alpha_prime], lr=cql_alpha_lr)

    @property
    def lagrange(self) -> bool:
        return self.cql_target_action_gap is not None

    @property
    def cql_config(self):
        """(N, lagrange), fixed when the engine is created."""
        return self.cql_n_actions, self.lagrange

    def _engine_extra(self) -> dict:
        return dict(cql=self.cql_config)

    def cql_hparams(self) -> dict:
        """``OffPolicyEngine.set_cql``'s arguments."""
        lr, b1, b2, eps = adam_hparams(self.alpha_prime_optimizer, [], "alpha' optimizer", extra=[self.log_alpha_prime])
        return dict(weight=self.cql_weight, temperature=self.cql_temperature,
                    target_action_gap=self.cql_target_action_gap or 0.0, alpha_lr=lr, alpha_betas=(b1, b2),
                    alpha_eps=eps, backup_entropy=self.backup_entropy)

    def _noise(self, S: int, B: int):
        """(SAC's [S, 2, B, A], CQL's [S, 3, B, N, A]): per step SAC's two torch.randn(B, A) (s', then s), then
        torch.rand(B, N, A) for the uniform actions, torch.randn(B, N, A) at s and torch.randn(B, N, A) at s'."""
        A, N = self.action_dim, self.cql_n_actions
        sac = np.empty((S, 2, B, A), dtype=np.float32)
        cql = np.empty((S, 3, B, N, A), dtype=np.float32)
        for i in range(S):
            sac[i, 0] = torch.randn(B, A).numpy()
            sac[i, 1] = torch.randn(B, A).numpy()
            cql[i, 0] = torch.rand(B, N, A).numpy()
            cql[i, 1] = torch.randn(B, N, A).numpy()
            cql[i, 2] = torch.randn(B, N, A).numpy()
        return sac, cql

    def _upload_state(self, e, trainable, targets, lins) -> None:
        super()._upload_state(e, trainable, targets, lins)
        e.set_cql(**self.cql_hparams())
        e.set_alpha_prime(*self._alpha_prime_state())

    def _download_state(self, e, trainable, targets, lins) -> None:
        super()._download_state(e, trainable, targets, lins)
        self._store_alpha_prime_state(*e.get_alpha_prime())

    def _alpha_prime_state(self):
        """(log_alpha', exp_avg, exp_avg_sq, step) of the Lagrange multiplier, as the engine takes it."""
        st = self.alpha_prime_optimizer.state.get(self.log_alpha_prime, {})
        step = int(float(st["step"])) if "exp_avg" in st else 0
        m = float(st["exp_avg"]) if step else 0.0
        v = float(st["exp_avg_sq"]) if step else 0.0
        return float(self.log_alpha_prime.detach()), m, v, step

    def _store_alpha_prime_state(self, log_alpha_prime, m, v, step) -> None:
        with torch.no_grad():
            self.log_alpha_prime.fill_(log_alpha_prime)
        if step > 0:
            st = self.alpha_prime_optimizer.state[self.log_alpha_prime]
            st["step"] = torch.tensor(float(step))
            st["exp_avg"] = torch.tensor(m, dtype=torch.float32)
            st["exp_avg_sq"] = torch.tensor(v, dtype=torch.float32)

    def _record_train(self, out) -> None:
        super()._record_train(out)
        mm, steps = getattr(self, "metrics_manager", None), getattr(self, "current_total_steps", 0)
        if mm is None or out is None:
            return
        mm.record_scalar("cql/penalty_1", float(np.mean(out["cql_gap_1"])), steps, tensorboard=True)
        mm.record_scalar("cql/penalty_2", float(np.mean(out["cql_gap_2"])), steps, tensorboard=True)
        if self.lagrange:
            mm.record_scalar("cql/alpha_prime", float(out["alpha_primes"][-1]), steps, tensorboard=True)

    def save_model(self, current_epoch: int, model_path: str) -> None:
        """SAC's checkpoint keys plus log_alpha_prime and its optimizer."""
        super().save_model(current_epoch, model_path)
        ckpt = torch.load(model_path, map_location="cpu", weights_only=True)
        ckpt["log_alpha_prime"] = self.log_alpha_prime.detach().clone()
        ckpt["alpha_prime_optimizer_state_dict"] = self.alpha_prime_optimizer.state_dict()
        torch.save(ckpt, model_path)

    def load_model(self, model_path: str, trust_checkpoint: bool = False) -> int:
        epoch = super().load_model(model_path, trust_checkpoint)
        ckpt = torch.load(model_path, map_location="cpu", weights_only=not trust_checkpoint)
        with torch.no_grad():
            self.log_alpha_prime.copy_(ckpt["log_alpha_prime"])
        self.alpha_prime_optimizer.load_state_dict(ckpt["alpha_prime_optimizer_state_dict"])
        return epoch
