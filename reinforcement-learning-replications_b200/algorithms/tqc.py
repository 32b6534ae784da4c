"""TQC (Kuznetsov, Shvechikov, Grishin & Vetrov 2020, "Controlling Overestimation Bias with Truncated Mixture of
Continuous Distributional Quantile Critics") over the GPU off-policy engine: SAC with two quantile critics whose pooled,
truncated target atoms replace SAC's min(Q1, Q2).  SAC's host loop, acting, evaluation and checkpoints; on the device
SAC's step program with quantile heads (enqueue_sac_steps in csrc/offpolicy.cu)."""
from __future__ import annotations

from ..critics import ContinuousQuantileQFunction
from ..engine import OffPolicyEngine
from ..networks import DuelingMLP, ImplicitQuantileMLP
from ..replay_buffer import PrioritizedReplayBuffer
from .sac import SAC


class TQC(SAC):
    """Per train step, on a minibatch (s, a, r, s', d), with N = 2 critics of M quantiles each, d =
    ``top_quantiles_to_drop_per_net`` and kN = N (M - d) (b200rl.h, "TQC"): a', log pi' from the policy at s' as for
    SAC; the 2M atoms of both target critics at (s', a') sorted ascending and the smallest kN kept, z_(1..kN); the target
    atoms y_i = r + gamma (1 - d) (z_(i) - alpha log pi'); one Adam step on each critic's quantile Huber loss
    (1 / (kN M)) sum_m sum_i |tau_m - 1{u < 0}| h(u), u = y_i - theta^m(s, a) (mean over the minibatch); one Adam step
    on the policy loss mean(alpha log pi - mean over both critics' 2M quantiles at (s, a_pi)) with the critics just
    updated; SAC's optional temperature step; and polyak averaging of both target critics.  Dropping atoms from the
    pooled target replaces SAC's min(Q1, Q2) as the guard against overestimation.

    The constructor takes SAC's arguments and defaults, with two ``ContinuousQuantileQFunction`` critics of equal
    ``n_quantiles`` whose networks map [obs | act] to their quantiles, plus ``top_quantiles_to_drop_per_net`` (0..M - 1;
    the paper's default is 2).  Acting, evaluation, metric tags and checkpoint keys are SAC's; the Q-value tags log the
    critics' quantile means and ``q-function_{1,2}/average_loss`` their quantile Huber losses.  Prioritized replay,
    n-step returns, more than two critics and noisy, dueling and IQN networks are not implemented for TQC."""
    algo = OffPolicyEngine.TQC

    def __init__(self, policy, exploration_policy, q_function_1, q_function_2, env, sampler, replay_buffer, evaluator,
                 gamma: float = 0.99, polyak_rho: float = 0.995, alpha: float = 0.2, learn_alpha: bool = False,
                 target_entropy=None, alpha_lr: float = 3e-4, top_quantiles_to_drop_per_net: int = 2) -> None:
        for what, q in (("q_function_1", q_function_1), ("q_function_2", q_function_2)):
            if not isinstance(q, ContinuousQuantileQFunction):
                raise TypeError(f"TQC: {what} must be a ContinuousQuantileQFunction, got {type(q).__name__}")
        for what, m in (("policy", policy), ("q_function_1", q_function_1), ("q_function_2", q_function_2)):
            if isinstance(m.network, (DuelingMLP, ImplicitQuantileMLP)):
                raise NotImplementedError(f"TQC: the {what} network is a {type(m.network).__name__}: dueling and IQN "
                                          "networks are not implemented for TQC (plain MLPs only)")
        if q_function_1.n_quantiles != q_function_2.n_quantiles:
            raise ValueError(f"TQC: both critics need the same n_quantiles, got {q_function_1.n_quantiles} and "
                             f"{q_function_2.n_quantiles}")
        M, d = q_function_1.n_quantiles, top_quantiles_to_drop_per_net
        if isinstance(d, bool) or not isinstance(d, int) or not 0 <= d <= M - 1:
            raise ValueError(f"TQC: top_quantiles_to_drop_per_net must be an integer from 0 to n_quantiles - 1 = {M - 1}, "
                             f"got {d!r}")
        if isinstance(replay_buffer, PrioritizedReplayBuffer):
            raise ValueError("TQC does not train on a PrioritizedReplayBuffer: prioritized replay is not implemented "
                             "for TQC")
        super().__init__(policy, exploration_policy, q_function_1, q_function_2, env, sampler, replay_buffer, evaluator,
                         gamma=gamma, polyak_rho=polyak_rho, alpha=alpha, learn_alpha=learn_alpha,
                         target_entropy=target_entropy, alpha_lr=alpha_lr)
        self.top_quantiles_to_drop_per_net = int(d)

    def _critic_width(self, q_function) -> int:
        return q_function.n_quantiles

    @property
    def tqc_config(self):
        """(n_quantiles, top_quantiles_to_drop_per_net), fixed when the engine is created."""
        return self.q_function_1.n_quantiles, self.top_quantiles_to_drop_per_net

    def _engine_extra(self) -> dict:
        return dict(tqc=self.tqc_config)
