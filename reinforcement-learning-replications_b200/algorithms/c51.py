"""C51 (Bellemare, Dabney & Munos 2017): categorical distributional DQN over the GPU off-policy engine.  DQN's step
program, host loop, acting and checkpoints, with a projected cross-entropy head (c51_loss_kernel in
csrc/offpolicy.cu)."""
from __future__ import annotations

from ..critics import CategoricalQFunction
from ..engine import OffPolicyEngine
from ..replay_buffer import PrioritizedReplayBuffer
from .dqn import DQN


class C51(DQN):
    """Per train step, on a minibatch (s, a, r, s', d) with a the action index and the critic's support z:
    a* = argmax_a' Q(s', a') over expected values (Q_targ's, or the online network's with ``double_q``), the target
    distribution m = Q_targ's p(s', a*) projected onto z after Tz = clamp(r + gamma (1 - d) z, v_min, v_max), one Adam
    step on the cross-entropy -sum_i m_i log p_i(s, a) (mean over the minibatch), and Q_targ <- Q as DQN copies it.

    The constructor takes DQN's arguments and defaults with a ``CategoricalQFunction`` whose network outputs
    n_actions x n_atoms logits.  Prioritized replay is not implemented for C51."""
    algo = OffPolicyEngine.C51

    def __init__(self, q_function, exploration_policy, env, sampler, replay_buffer, evaluator, **kwargs) -> None:
        if not isinstance(q_function, CategoricalQFunction):
            raise ValueError(f"C51 needs a CategoricalQFunction, got {type(q_function).__name__}")
        _refuse_prioritized(replay_buffer)
        super().__init__(q_function, exploration_policy, env, sampler, replay_buffer, evaluator, **kwargs)

    @staticmethod
    def _output_width(q_function, n: int):
        N = q_function.n_atoms
        return n * N, f"{n} actions x {N} atoms logits"

    @staticmethod
    def _outputs_per_action(q_function):
        return q_function.n_atoms, "n_atoms logits per action"

    def _upload_state(self, e, trainable, targets, lins) -> None:
        super()._upload_state(e, trainable, targets, lins)
        q = self.q_function
        e.set_c51(q.n_atoms, q.v_min, q.v_max)

    def _stage_inputs(self, replay_buffer, S: int, B: int, noisy: bool):
        _refuse_prioritized(replay_buffer)  # the buffer may have been replaced since construction
        return super()._stage_inputs(replay_buffer, S, B, noisy)


def _refuse_prioritized(replay_buffer) -> None:
    if isinstance(replay_buffer, PrioritizedReplayBuffer):
        raise ValueError("C51 does not train on a PrioritizedReplayBuffer: prioritized replay is implemented for DQN "
                         "only")
