"""Discrete SAC (Christodoulou 2019, "Soft Actor-Critic for Discrete Action Settings") over the GPU off-policy engine.
``learn`` is the shared off-policy host loop; ``train`` is the hot path (enqueue_dsac_steps in csrc/offpolicy.cu)."""
from __future__ import annotations

import copy
import math

import numpy as np
import torch
from torch import nn

from .._lib import SacHparams
from ..critics import DiscreteQFunction
from ..engine import OffPolicyEngine
from ..networks import DuelingMLP, ImplicitQuantileMLP
from ..policies import CategoricalPolicy, GreedyPolicy
from ..replay_buffer import PrioritizedReplayBuffer
from ._onpolicy import adam_hparams, describe_mlp, refuse_noisy
from .sac import SAC
from .td3 import _make_eval_env, _OffPolicyBase


class DiscreteSAC(SAC):
    """SAC for a discrete action space of n >= 2 actions.  The policy network maps obs -> [n] logits (a
    ``CategoricalPolicy``), both critics obs -> [n] Q-values (``critics.DiscreteQFunction``s).  Per train step, with
    log pi = log_softmax of the logits and alpha = exp(log_alpha) at the start of the step:
    one Adam step on each critic on mean((Qk(s)[a] - y)^2) with y = r + gamma (1 - d) V(s'),
    V(s') = sum_a' pi(a'|s') (min(Q1targ, Q2targ)(s', a') - alpha log pi(a'|s')); one Adam step on the policy loss
    mean_B sum_a pi(a|s) (alpha log pi(a|s) - min(Q1, Q2)(s, a)) with the critics just updated; optionally one Adam step
    on log_alpha for -mean_B(log_alpha (E + target_entropy)), E = sum_a pi(a|s) log pi(a|s); and polyak averaging of
    both target critics.  Every expectation is exact: nothing is sampled.  target_entropy defaults to 0.98 log(n).

    Acting: ``exploration_policy`` before ``num_start_steps``, then samples of the policy; evaluation is greedy on the
    logits.  Checkpoints and metrics are SAC's; ``policy/average_log_prob`` logs the mean of E.  Prioritized replay,
    n-step returns and noisy, dueling and IQN networks are not implemented for discrete SAC and are refused."""
    n_q = 2
    algo = OffPolicyEngine.DSAC
    target_slots = (4, 5)  # no target policy

    def __init__(self, policy, exploration_policy, q_function_1, q_function_2, env, sampler, replay_buffer, evaluator,
                 gamma: float = 0.99, polyak_rho: float = 0.995, alpha: float = 0.2, learn_alpha: bool = False,
                 target_entropy=None, alpha_lr: float = 3e-4) -> None:
        n = getattr(env.action_space, "n", None)
        if n is None:
            raise ValueError("DiscreteSAC needs a discrete action space (one with .n)")
        n = int(n)
        if n < 2:
            raise ValueError(f"DiscreteSAC needs at least 2 actions, the action space has {n}")
        if not isinstance(policy, CategoricalPolicy):
            raise TypeError(f"DiscreteSAC needs a CategoricalPolicy, got {type(policy).__name__}")
        refuse_noisy("DiscreteSAC", policy, q_function_1, q_function_2)
        for what, m in (("policy", policy), ("q_function_1", q_function_1), ("q_function_2", q_function_2)):
            if isinstance(m.network, (DuelingMLP, ImplicitQuantileMLP)):
                raise NotImplementedError(f"DiscreteSAC: the {what} network is a {type(m.network).__name__}: dueling "
                                          "and IQN networks are not implemented for discrete SAC (plain MLPs only)")
        for what, q in (("q_function_1", q_function_1), ("q_function_2", q_function_2)):
            if not isinstance(q, DiscreteQFunction):
                raise TypeError(f"DiscreteSAC: {what} must be a DiscreteQFunction, got {type(q).__name__}")
        if isinstance(replay_buffer, PrioritizedReplayBuffer):
            raise ValueError("DiscreteSAC does not train on a PrioritizedReplayBuffer: prioritized replay is not "
                             "implemented for discrete SAC")
        psz, _, _, plin = describe_mlp(policy.network)
        obs_shape = getattr(getattr(env, "observation_space", None), "shape", None)
        O = int(np.prod(obs_shape)) if obs_shape else psz[0]
        if psz[0] != O or psz[-1] != n:
            raise ValueError(f"the policy network must map obs {O} -> {n} logits, got {psz[0]} -> {psz[-1]}")
        adam_hparams(policy.optimizer, plin, "policy optimizer")
        for q in (q_function_1, q_function_2):
            qsz, _, _, qlin = describe_mlp(q.network)
            if qsz[0] != O or qsz[-1] != n:
                raise ValueError(f"a Q network must map obs {O} -> {n} values (one per action), got {qsz[0]} -> "
                                 f"{qsz[-1]}")
            adam_hparams(q.optimizer, qlin, "q-function optimizer")
        if alpha <= 0:
            raise ValueError("alpha must be > 0")
        self.policy, self.exploration_policy = policy, exploration_policy
        self.q_function_1, self.q_function_2 = q_function_1, q_function_2
        self.env, self.sampler, self.replay_buffer, self.evaluator = env, sampler, replay_buffer, evaluator
        self.gamma, self.polyak_rho = gamma, polyak_rho
        self.learn_alpha = bool(learn_alpha)
        self.alpha = float(alpha)  # the fixed coefficient (learn_alpha=False)
        self.target_entropy = float(0.98 * math.log(n) if target_entropy is None else target_entropy)
        self.n_actions = n
        self.log_alpha = nn.Parameter(torch.tensor(math.log(alpha), dtype=torch.float32))
        self.alpha_optimizer = torch.optim.Adam([self.log_alpha], lr=alpha_lr)
        self.noised_policy = policy  # after warm-up the policy explores by sampling
        self.evaluation_policy = GreedyPolicy(policy.network)  # argmax of the logits
        self.evaluation_env = _make_eval_env(env)
        self.target_q_function_1, self.target_q_function_2 = [copy.deepcopy(q) for q in (q_function_1, q_function_2)]
        for t in (self.target_q_function_1, self.target_q_function_2):
            for p in t.network.parameters():
                p.requires_grad = False

    def _train_schedule(self):
        return False, 1  # no noise draws: every expectation over actions is exact

    def _sac_hparams(self) -> SacHparams:
        sp = SacHparams()
        sp.alpha, sp.learn_alpha, sp.target_entropy = self.alpha, int(self.learn_alpha), self.target_entropy
        sp.alpha_lr, sp.alpha_beta1, sp.alpha_beta2, sp.alpha_eps = adam_hparams(
            self.alpha_optimizer, [], "alpha optimizer", extra=[self.log_alpha])
        sp.log_std_min, sp.log_std_max = 0.0, 0.0  # ignored by discrete SAC
        return sp

    def _stage_inputs(self, replay_buffer, S: int, B: int, noisy: bool):
        mode, inputs = _OffPolicyBase._stage_inputs(self, replay_buffer, S, B, noisy)
        if mode == "host":  # the action column as [S, B] indices
            obs, act, rew, nobs, done, _ = inputs
            inputs = (obs, act.reshape(S, B), rew, nobs, done, None)
        return mode, inputs
