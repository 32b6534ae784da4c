"""DQN (Mnih et al. 2015) with optional Double DQN targets (van Hasselt et al. 2016) over the GPU off-policy engine.
``learn`` is the shared off-policy host loop; ``train`` is the hot path (enqueue_dqn_steps in csrc/offpolicy.cu)."""
from __future__ import annotations

import copy

import numpy as np
import torch

from .._lib import OffPolicyHparams
from ..engine import OffPolicyEngine
from ..networks import DuelingMLP, ImplicitQuantileMLP, NoisyLinear
from ..policies import EpsilonGreedyPolicy, GreedyPolicy, NoisyGreedyPolicy
from ._onpolicy import _ACT_NAMES, adam_hparams, describe_mlp
from .td3 import _learn, _make_eval_env, _OffPolicyBase


def describe_q_network(module):
    """(sizes, hidden activation, output activation, Linear layers in parameters() order, dueling K) of a DQN-family Q
    network: an ``MLP`` as ``describe_mlp`` reads it (K = 0), or a ``DuelingMLP`` with sizes [obs, h_trunk, h_stream,
    n_actions * K] and its five Linear layers (trunk, value hidden, value out, advantage hidden, advantage out), or an
    ``ImplicitQuantileMLP`` with sizes [obs, d, h, n_actions] and its four (psi, phi, head hidden, head out; K = 0)."""
    if isinstance(module, ImplicitQuantileMLP):
        acts = {type(m) for m in (module.embedding[1], module.tau_embedding[1], module.head[1])}
        if len(acts) != 1 or next(iter(acts)) not in _ACT_NAMES:
            raise NotImplementedError(f"ImplicitQuantileMLP activations must be one of Tanh, ReLU, Identity throughout, "
                                      f"got {sorted(a.__name__ for a in acts)}")
        linears = [module.embedding[0], module.tau_embedding[0], module.head[0], module.head[2]]
        return module.sizes + [module.n_actions], _ACT_NAMES[acts.pop()], "identity", linears, 0
    if not isinstance(module, DuelingMLP):
        return describe_mlp(module, allow_noisy=True) + (0,)
    acts = {type(m) for m in (module.trunk[1], module.value[1], module.advantage[1])}
    if len(acts) != 1 or next(iter(acts)) not in _ACT_NAMES:
        raise NotImplementedError(f"DuelingMLP activations must be one of Tanh, ReLU, Identity throughout, got "
                                  f"{sorted(a.__name__ for a in acts)}")
    linears = [module.trunk[0], module.value[0], module.value[2], module.advantage[0], module.advantage[2]]
    sizes = module.sizes + [module.n_actions * module.outputs_per_action]
    return sizes, _ACT_NAMES[acts.pop()], "identity", linears, module.outputs_per_action


def noisy_mask(linears) -> int:
    """The engine's noisy_layers: bit l set for each NoisyLinear among the Q network's layers in flat order."""
    return sum(1 << l for l, lin in enumerate(linears) if isinstance(lin, NoisyLinear))


class DQN(_OffPolicyBase):
    """Per train step, on a minibatch (s, a, r, s', d) with a the action index:
    y = r + gamma (1 - d) Q_targ(s', argmax_a' Q(s', a')) (``double_q``) or r + gamma (1 - d) max_a' Q_targ(s', a'),
    one Adam step on F.smooth_l1_loss(Q(s, a), y), and Q_targ <- Q whenever the Q optimizer's step count reaches a
    multiple of ``target_update_interval`` (the count carries across train() calls and checkpoints).

    With a ``PrioritizedReplayBuffer`` every train() call takes the prioritized device path (draws keyed by
    ``device_rng_seed``, whatever ``use_device_rng`` says): minibatches drawn in proportion to the priorities, the loss
    weighted by the importance weights, and the rows' priorities updated from their TD errors (b200rl.h).

    ``n_step`` (1..32) > 1 trains on n-step returns (b200rl.h, "n-step returns"): from a drawn row the window takes up to
    n consecutive transitions of its episode, R = r_0 + gamma r_1 + ... + gamma^(k-1) r_(k-1) with the k rows it took,
    and the target bootstraps from the last row's next observation with discount gamma^k: y = R + gamma^k (1 - d) v,
    d and v (Double DQN's argmax too) taken at that row.  A window stops at a done row and at the last row of an episode
    in the append that wrote it -- a segment ``BatchSampler`` cut off at the end of a ``sample()`` call included, also
    with ``is_continuous=True``: such a row bootstraps from its own next observation with a shorter horizon.  Windows
    are assembled on the device from the replay ring (with prioritized replay too, where the priority is the n-step
    TD error's), so n_step > 1 needs ``use_device_replay = True`` and a replay buffer with ``device_episode_ends``.
    ``n_step = 1`` is exactly the one-step update.  n_step is a constructor argument, not part of checkpoints.

    The Q network is an ``MLP`` or a ``networks.DuelingMLP`` with ``n_actions`` = the action count and
    ``outputs_per_action`` = 1 (C51: ``n_atoms``, QR-DQN: ``n_quantiles``); the engine runs either (b200rl.h).

    Acting: ``exploration_policy`` before ``num_start_steps``, then epsilon-greedy with epsilon falling linearly from
    ``epsilon_start`` to ``epsilon_end`` over the first ``epsilon_decay_steps`` environment steps; evaluation is greedy.

    Noisy networks (Fortunato et al. 2018): a Q network with ``networks.NoisyLinear`` layers (a ``NoisyMLP``, or a
    ``DuelingMLP(..., noisy=True)``) explores through its weight noise instead: past ``num_start_steps`` acting is a
    ``NoisyGreedyPolicy`` (fresh noise per action, then greedy; epsilon is not used), evaluation is greedy on the mean
    weights.  Each train step draws the online and the target network's noise on the device (b200rl.h, "Noisy
    networks"), keyed by ``device_rng_seed`` and the learner's own count of train calls, whatever ``use_device_rng``
    says."""
    n_q = 1
    algo = OffPolicyEngine.DQN
    trainable_slots = (1,)  # the Q network is engine network 1, its optimizer row 1
    target_slots = (4,)

    def __init__(self, q_function, exploration_policy, env, sampler, replay_buffer, evaluator, gamma: float = 0.99,
                 target_update_interval: int = 1000, double_q: bool = False, epsilon_start: float = 1.0,
                 epsilon_end: float = 0.05, epsilon_decay_steps: int = 10000, n_step: int = 1) -> None:
        n = getattr(env.action_space, "n", None)
        if n is None:
            raise ValueError("DQN needs a discrete action space (one with .n)")
        net = q_function.network
        if isinstance(net, DuelingMLP):
            k, what_k = self._outputs_per_action(q_function)
            if net.n_actions != int(n):
                raise ValueError(f"the DuelingMLP has n_actions = {net.n_actions}, the action space has {int(n)} actions")
            if net.outputs_per_action != k:
                raise ValueError(f"{type(self).__name__} needs a DuelingMLP with outputs_per_action = {k} ({what_k}), "
                                 f"got {net.outputs_per_action}")
        sizes, _, _, lins, _ = describe_q_network(net)
        obs_shape = getattr(getattr(env, "observation_space", None), "shape", None)
        width, what = self._output_width(q_function, int(n))
        if sizes[-1] != width or (obs_shape and sizes[0] != int(np.prod(obs_shape))):
            want = f"{int(np.prod(obs_shape))} -> {width}" if obs_shape else f"obs -> {width}"
            raise ValueError(f"the Q network must map {want} ({what}), got {sizes[0]} -> {sizes[-1]}")
        adam_hparams(q_function.optimizer, lins, "q-function optimizer")
        if int(target_update_interval) < 1:
            raise ValueError(f"target_update_interval must be >= 1, got {target_update_interval}")
        if isinstance(n_step, bool) or not isinstance(n_step, (int, np.integer)) or not 1 <= n_step <= 32:
            raise ValueError(f"n_step must be an integer from 1 to 32, got {n_step!r}")
        self.q_function, self.exploration_policy = q_function, exploration_policy
        self.env, self.sampler, self.replay_buffer, self.evaluator = env, sampler, replay_buffer, evaluator
        self.gamma = gamma
        self.target_update_interval, self.double_q = int(target_update_interval), bool(double_q)
        self.epsilon_start, self.epsilon_end = float(epsilon_start), float(epsilon_end)
        self.epsilon_decay_steps = int(epsilon_decay_steps)
        self.n_actions = int(n)
        self.n_step = int(n_step)
        self.epsilon_greedy_policy = EpsilonGreedyPolicy(q_function, env.action_space, epsilon_start)
        self.policy = self.evaluation_policy = GreedyPolicy(q_function)  # acting greedily (evaluation)
        self.noisy = noisy_mask(lins) != 0
        if self.noisy:  # explores with its weight noise; evaluation on the mean weights
            self.noisy_policy = NoisyGreedyPolicy(q_function)
            self.policy = self.evaluation_policy = self.noisy_policy.deterministic()
        self.evaluation_env = _make_eval_env(env)
        self.target_q_function = copy.deepcopy(q_function)
        for p in self.target_q_function.network.parameters():
            p.requires_grad = False

    @staticmethod
    def _output_width(q_function, n: int):
        """(width of the Q network's output for n actions, what it holds)."""
        return n, "one value per action"

    @staticmethod
    def _outputs_per_action(q_function):
        """(outputs per action a DuelingMLP Q network must have, what they are)."""
        return 1, "one value per action"

    def epsilon(self) -> float:
        """epsilon at the current total step count: linear from epsilon_start to epsilon_end, then constant."""
        t = getattr(self, "current_total_steps", 0)
        frac = min(t / self.epsilon_decay_steps, 1.0) if self.epsilon_decay_steps > 0 else 1.0
        return self.epsilon_start + frac * (self.epsilon_end - self.epsilon_start)

    @property
    def noised_policy(self):
        """The acting policy after warm-up (the shared learn loop's name for it), at the current epsilon; a noisy Q
        network's NoisyGreedyPolicy."""
        if self.noisy:
            return self.noisy_policy
        self.epsilon_greedy_policy.epsilon = self.epsilon()
        return self.epsilon_greedy_policy

    def _trainable(self):
        return [self.q_function]

    def _nets(self):
        return [self.q_function], [self.target_q_function]

    def _engine_config(self):
        """(Q network sizes, its (hidden, output) activations, the other OffPolicyEngine arguments) of this learner's
        engine."""
        qsz, qact, qout, lins, dk = describe_q_network(self.q_function.network)
        return qsz, (qact, qout), dict(dueling_k=dk, noisy_layers=noisy_mask(lins))

    def _needs_draw_keys(self) -> bool:
        """Whether every train call hands the engine (seed, call) keys for its device draws (set_noise_keys)."""
        return self.noisy

    def _ensure_engine(self, S: int, B: int) -> OffPolicyEngine:
        qsz, qacts, kw = self._engine_config()
        e = getattr(self, "_engine", None)
        if (e is None or e.q_sizes != qsz or e.max_minibatch < B or e.max_steps < S or e.q_acts != qacts
                or any(getattr(e, k) != v for k, v in kw.items())):
            if e is not None:
                e.close()
            e = OffPolicyEngine(None, qsz, 1, B, S, q_acts=qacts, algo=self.algo, **kw)
            self._engine = e
        return e

    def _hparams(self, noisy: bool, delay: int) -> OffPolicyHparams:
        hp = OffPolicyHparams()
        hp.gamma, hp.policy_delay = self.gamma, 1
        lr, b1, b2, eps = adam_hparams(self.q_function.optimizer, describe_q_network(self.q_function.network)[3],
                                       "q-function optimizer")
        hp.q1_lr, hp.q2_lr, hp.q_beta1, hp.q_beta2, hp.q_eps = lr, lr, b1, b2, eps
        return hp

    def _upload_state(self, e, trainable, targets, lins) -> None:
        super()._upload_state(e, trainable, targets, lins)
        e.set_dqn(self.target_update_interval, self.double_q)

    def _stage_inputs(self, replay_buffer, S: int, B: int, noisy: bool):
        if self._needs_draw_keys() and S > 0:  # the device draws' keys: this learner's own count of train calls
            self._noise_calls = getattr(self, "_noise_calls", 0) + 1
            self.noise_key = (getattr(self, "device_rng_seed", 0), self._noise_calls)
        staged = self._stage_nstep_and_prioritized(replay_buffer, S, self.q_function.optimizer,
                                                   describe_q_network(self.q_function.network)[3])
        if staged is not None:
            return staged
        mode, inputs = super()._stage_inputs(replay_buffer, S, B, noisy)
        if mode == "host":  # the action column as [S, B] indices
            obs, act, rew, nobs, done, _ = inputs
            inputs = (obs, act.reshape(S, B), rew, nobs, done, None)
        return mode, inputs

    def _call_engine(self, e, hp, replay_buffer, S: int, B: int, mode, inputs):
        if mode is not None and self._needs_draw_keys():
            e.set_noise_keys(*([k] for k in self.noise_key))
        return self._call_nstep_and_prioritized(e, hp, replay_buffer, S, B, mode, inputs)

    def _train_schedule(self):
        return False, 1

    def _learner_nets(self):
        trainable, targets = self._nets()
        return trainable, targets, [describe_q_network(m.network)[3] for m in trainable + targets]

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
        q = out["q1_values"].astype(np.float64)  # DDPG's critic tags
        mm.record_scalar("q-function/average_loss", float(np.mean(out["q1_losses"])), steps, tensorboard=True)
        mm.record_scalar("q-function/avarage_q-value", float(np.mean(q)), steps, tensorboard=True)
        mm.record_scalar("q-function/max_q-value", float(np.max(q)))
        mm.record_scalar("q-function/min_q-value", float(np.min(q)))
        if not self.noisy:
            mm.record_scalar("exploration/epsilon", self.epsilon(), steps, tensorboard=True)
        if getattr(self, "_last_beta", None) is not None:
            mm.record_scalar("replay/beta", self._last_beta, steps, tensorboard=True)

    def save_model(self, current_epoch: int, model_path: str) -> None:
        torch.save({
            "epoch": current_epoch, "total_steps": getattr(self, "current_total_steps", 0),
            "q_function_state_dict": self.q_function.network.state_dict(),
            "q_function_optimizer_state_dict": self.q_function.optimizer.state_dict(),
            "target_q_function_state_dict": self.target_q_function.network.state_dict(),
        }, model_path)

    def load_model(self, model_path: str, trust_checkpoint: bool = False) -> int:
        """Resume from a checkpoint written by ``save_model``: the Q network, its Adam state (and so the step count
        the target-copy schedule follows), the target network and the step total; returns the saved epoch."""
        ckpt = torch.load(model_path, map_location="cpu", weights_only=not trust_checkpoint)
        self.q_function.network.load_state_dict(ckpt["q_function_state_dict"])
        self.q_function.optimizer.load_state_dict(ckpt["q_function_optimizer_state_dict"])
        self.target_q_function.network.load_state_dict(ckpt["target_q_function_state_dict"])
        self.current_total_steps = int(ckpt.get("total_steps", 0))
        return int(ckpt.get("epoch", 0))
