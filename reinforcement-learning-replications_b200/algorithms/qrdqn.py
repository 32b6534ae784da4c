"""QR-DQN (Dabney, Rowland, Bellemare & Munos 2018): quantile regression DQN over the GPU off-policy engine.  DQN's
step program, host loop, acting, prioritized replay, n-step returns and checkpoints, with a quantile Huber head
(qr_loss_kernel in csrc/offpolicy.cu)."""
from __future__ import annotations

from ..critics import QuantileQFunction
from .dqn import DQN


class QRDQN(DQN):
    """Per train step, on a minibatch (s, a, r, s', d) with a the action index and the critic's N quantile midpoints
    tau_i = (2i + 1) / (2N): a* = argmax_a' Q(s', a') over quantile means (Q_targ's, or the online network's with
    ``double_q``), target quantiles T_j = r + gamma (1 - d) theta_j(s', a*) from Q_targ, one Adam step on the quantile
    Huber loss (1/N) sum_i sum_j |tau_i - 1{u_ij < 0}| h(u_ij) with u_ij = T_j - theta_i(s, a) and h the Huber loss
    with kappa = 1 (mean over the minibatch), and Q_targ <- Q as DQN copies it.

    The constructor takes DQN's arguments and defaults, ``n_step`` included, with a ``QuantileQFunction`` whose network
    outputs n_actions x n_quantiles values.  With a ``PrioritizedReplayBuffer`` the loss is weighted by the importance
    weights and a row's priority is computed from its quantile loss (b200rl.h)."""

    def __init__(self, q_function, exploration_policy, env, sampler, replay_buffer, evaluator, **kwargs) -> None:
        if not isinstance(q_function, QuantileQFunction):
            raise ValueError(f"QRDQN needs a QuantileQFunction, got {type(q_function).__name__}")
        super().__init__(q_function, exploration_policy, env, sampler, replay_buffer, evaluator, **kwargs)

    @staticmethod
    def _output_width(q_function, n: int):
        N = q_function.n_quantiles
        return n * N, f"{n} actions x {N} quantiles"

    @staticmethod
    def _outputs_per_action(q_function):
        return q_function.n_quantiles, "n_quantiles locations per action"

    def _upload_state(self, e, trainable, targets, lins) -> None:
        super()._upload_state(e, trainable, targets, lins)
        e.set_qr(self.q_function.n_quantiles)
