"""IQN (Dabney, Ostrovski, Silver & Munos 2018): implicit quantile networks over the GPU off-policy engine.  DQN's
host loop, acting, prioritized replay, n-step returns and checkpoints; on the device its own step program branch:
quantile fractions drawn and embedded per step, and a sampled-fraction quantile Huber head (iqn_loss_kernel in
csrc/offpolicy.cu)."""
from __future__ import annotations

from ..critics import ImplicitQuantileQFunction
from ..engine import OffPolicyEngine
from ..networks import DuelingMLP, ImplicitQuantileMLP, has_noisy_layers
from .dqn import DQN


class IQN(DQN):
    """Per train step, on a minibatch (s, a, r, s', d) with a the action index, the engine draws per row N + N' + K
    fractions tau ~ U(0, 1) (N = ``n_quantiles``, N' = ``n_target_quantiles``, K = ``n_policy_quantiles`` of the
    ``ImplicitQuantileQFunction``) and takes
    a* = argmax_a' (1/K) sum_k Z(s', tau~_k, a') (Q_targ's, or the online network's with ``double_q``), the target
    samples T_j = r + gamma (1 - d) Z_targ(s', tau'_j, a*), and one Adam step on the quantile Huber loss
    (1/N') sum_i sum_j |tau_i - 1{u_ij < 0}| h(u_ij) with u_ij = T_j - Z(s, tau_i, a) and h the Huber loss with
    kappa = 1 (mean over the minibatch); Q_targ <- Q as DQN copies it.

    The constructor takes DQN's arguments and defaults, ``n_step`` included, with an ``ImplicitQuantileQFunction``
    over an ``ImplicitQuantileMLP``.  With a ``PrioritizedReplayBuffer`` the loss is weighted by the importance weights
    and a row's priority is computed from its quantile loss (b200rl.h).  The fractions are drawn on the device, keyed by
    ``device_rng_seed`` and the learner's own count of train calls, whatever ``use_device_rng`` says.  Acting and
    evaluation use the critic's mean over K fixed midpoint fractions.  Dueling and noisy IQN networks are not
    implemented."""
    algo = OffPolicyEngine.IQN

    def __init__(self, q_function, exploration_policy, env, sampler, replay_buffer, evaluator, **kwargs) -> None:
        if not isinstance(q_function, ImplicitQuantileQFunction):
            raise ValueError(f"IQN needs an ImplicitQuantileQFunction, got {type(q_function).__name__}")
        net = q_function.network
        if isinstance(net, DuelingMLP):
            raise NotImplementedError("IQN does not take a DuelingMLP: dueling IQN networks are not implemented")
        if has_noisy_layers(net):
            raise NotImplementedError("IQN does not take networks with noisy layers (NoisyLinear): noisy IQN networks "
                                      "are not implemented")
        if not isinstance(net, ImplicitQuantileMLP):
            raise ValueError(f"IQN needs an ImplicitQuantileMLP Q network, got {type(net).__name__}")
        super().__init__(q_function, exploration_policy, env, sampler, replay_buffer, evaluator, **kwargs)

    @property
    def iqn_config(self):
        """(n_cos, N, N', K): the engine's cosine features and fractions per row."""
        q = self.q_function
        return q.network.n_cos, q.n_quantiles, q.n_target_quantiles, q.n_policy_quantiles

    def _engine_config(self):
        qsz, qacts, kw = super()._engine_config()
        return qsz, qacts, dict(kw, iqn=self.iqn_config)

    def _needs_draw_keys(self) -> bool:
        return True
