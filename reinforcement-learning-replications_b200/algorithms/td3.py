"""TD3 and DDPG -- the reference's class surfaces (ref: algorithms/td3.py:25-382, algorithms/ddpg.py:24-314) over the
GPU off-policy engine.  ``learn`` keeps the reference's host-side loop; ``train`` is the hot path."""
from __future__ import annotations

import copy
import logging
import os
import time
from typing import List

import numpy as np
import torch

from .._lib import OffPolicyHparams
from ..engine import OffPolicyEngine
from ..metrics_manager import MetricsManager
from ..replay_buffer import PrioritizedReplayBuffer
from ..utils import add_noise_to_get_action
from ._onpolicy import adam_hparams, describe_mlp, layer_params, refuse_noisy

logger = logging.getLogger(__name__)


class _OffPolicyBase:
    n_q = 1
    algo = OffPolicyEngine.TD3  # the engine's step program (DDPG / TD3 by n_q, or SAC)
    trainable_slots = (0, 1, 2)  # engine network (and optimizer) index of each trainable network, _trainable() order
    target_slots = (3, 4, 5)    # engine network index of each target network
    use_device_replay = True  # replay columns mirrored in HBM, minibatches gathered on the device (SURVEY 8f-4)
    use_device_rng = False    # opt-in: indices and target-smoothing noise drawn on the device (Philox) instead of with
    device_rng_seed = 0       # the reference's numpy / torch CPU streams -- same distributions, different numbers

    def _trainable(self):
        return [self.policy] + ([self.q_function_1, self.q_function_2] if self.n_q == 2 else [self.q_function])

    def _nets(self):
        tq = [self.target_q_function_1, self.target_q_function_2] if self.n_q == 2 else [self.target_q_function]
        return self._trainable(), [self.target_policy] + tq

    def load_model(self, model_path: str, trust_checkpoint: bool = False) -> int:
        """Resume from a checkpoint written by ``save_model`` or by the reference (same layout, ref td3.py:367-382 /
        ddpg.py:295-314): trainable networks, their Adam states, the target networks; returns the saved epoch."""
        ckpt = torch.load(model_path, map_location="cpu", weights_only=not trust_checkpoint)
        names = ["policy"] + (["q_function_1", "q_function_2"] if self.n_q == 2 else ["q_function"])
        trainable, targets = self._nets()
        for name, module, target in zip(names, trainable, targets):
            module.network.load_state_dict(ckpt[name + "_state_dict"])
            module.optimizer.load_state_dict(ckpt[name + "_optimizer_state_dict"])
            target.network.load_state_dict(ckpt["target_" + name + "_state_dict"])
        self.current_total_steps = int(ckpt.get("total_steps", 0))
        return int(ckpt.get("epoch", 0))

    def _make_targets(self):
        targets = [copy.deepcopy(m) for m in self._trainable()]
        for t in targets:
            for p in t.network.parameters():
                p.requires_grad = False
        return targets

    def _engine_extra(self) -> dict:
        """OffPolicyEngine arguments beyond the shapes and the algo (D4PG: its critic's support)."""
        return {}

    def _ensure_engine(self, S: int, B: int) -> OffPolicyEngine:
        psz, pact, pout, _ = describe_mlp(self.policy.network)
        trainable, _ = self._nets()
        qsz, qact, qout, _ = describe_mlp(trainable[1].network)
        kw = self._engine_extra()
        e = getattr(self, "_engine", None)
        if (e is None or e.policy_sizes != psz or e.q_sizes != qsz or e.max_minibatch < B or e.max_steps < S
                or e.policy_acts != (pact, pout) or e.q_acts != (qact, qout)
                or any(getattr(e, k) != v for k, v in kw.items())):
            if e is not None:
                e.close()
            e = OffPolicyEngine(psz, qsz, self.n_q, B, S, (pact, pout), (qact, qout), algo=self.algo, **kw)
            self._engine = e
        return e

    # The host modules stay the reference point between train() calls (the sampler acts with self.policy on the CPU, a
    # user may edit or load weights), so every call moves the whole learner state down and up again -- as ONE blob per
    # direction with one synchronisation each (24 separate synchronous copies per call before: the transfers cost more
    # than the 50 train steps between them).
    def _state_plan(self, e, trainable, targets, lins, lane: int = 0):
        """[(kind, host parameter, owning module, numpy view into the engine's host blob)] in blob order, built once per
        (engine, learner, networks): the blob is persistent (page-locked), so the views stay valid between calls.
        ``lane``: this learner's place in a group engine's blob."""
        key = (id(e), lane) + tuple(id(l) for ls in lins for l in ls)
        plan = getattr(self, "_plan", None)
        if plan is not None and plan[0] == key:
            return plan[1]
        layout, total = e.state_layout()
        blob = e.state_buffer()
        assert blob.numel() == total * getattr(e, "K", 1)
        blob_np = blob.numpy()[lane * total:(lane + 1) * total]  # shares the page-locked memory
        mods = {i: (m, l) for i, m, l in zip(self.trainable_slots, trainable, lins)}
        mods.update({k: (m, l) for k, m, l in zip(self.target_slots, targets, lins[len(trainable):])})
        slots = []
        for kind, i, off, count in layout:
            m, l = mods[i]
            o = off
            for lin in l:
                for p_ in layer_params(lin):
                    slots.append((kind, p_, m, blob_np[o:o + p_.numel()].reshape(tuple(p_.shape))))
                    o += p_.numel()
            assert o == off + count
        self._plan = (key, slots)
        return slots

    @staticmethod
    def _adam_step_count(optimizer, linears) -> int:
        ps = [t for l in linears for t in layer_params(l)]
        if not all(p_ in optimizer.state and "exp_avg" in optimizer.state[p_] for p_ in ps):
            return 0
        steps = {int(float(optimizer.state[p_]["step"])) for p_ in ps}
        if len(steps) != 1:
            raise NotImplementedError("parameters of one optimizer have different step counts")
        return steps.pop()

    # The copies between the host modules and the page-locked blob are plain numpy copies on purpose: torch's CPU copy
    # kernels go parallel above 32768 elements (the 256 x 256 weights), and on a many-core host the OpenMP workers that
    # linger after such a region cost the calling thread tens of milliseconds every few train() calls.
    def _upload_state(self, e, trainable, targets, lins) -> None:
        e.set_state(None, self._fill_state(self._state_plan(e, trainable, targets, lins), trainable, lins))

    def _fill_state(self, slots, trainable, lins):
        """Host modules and Adam states -> this learner's part of the blob; returns its Adam step counts, one per engine
        optimizer row (3, or 4 with IQL's value network in slot 3)."""
        steps = [0] * max(3, 1 + max(self.trainable_slots))
        for i, m, l in zip(self.trainable_slots, trainable, lins):
            adam_hparams(m.optimizer, l, "optimizer")  # refuses anything but a plain Adam over exactly this network
            steps[i] = self._adam_step_count(m.optimizer, l)
        index = {id(m): i for i, m in zip(self.trainable_slots, trainable)}
        for kind, p_, m, view in slots:
            if kind == "params":
                src = p_.detach()
            else:
                st = m.optimizer.state.get(p_) if steps[index[id(m)]] > 0 else None
                src = st["exp_avg" if kind == "m" else "exp_avg_sq"] if st else None
            if src is None:
                view.fill(0.0)
            else:
                np.copyto(view, src.numpy(), casting="same_kind")
        return steps

    def _download_state(self, e, trainable, targets, lins) -> None:
        slots = self._state_plan(e, trainable, targets, lins)
        _, steps = e.get_state()
        self._read_state(slots, trainable, steps)

    def _read_state(self, slots, trainable, steps) -> None:
        """This learner's part of the blob -> host modules and Adam states."""
        index = {id(m): i for i, m in zip(self.trainable_slots, trainable)}
        for kind, p_, m, view in slots:
            if kind == "params":
                np.copyto(p_.detach().numpy(), view, casting="same_kind")
                continue
            step = steps[index[id(m)]]
            if step == 0:
                continue
            st = m.optimizer.state[p_]
            key = "exp_avg" if kind == "m" else "exp_avg_sq"
            if key in st and st[key].shape == p_.shape and not st[key].is_cuda:
                np.copyto(st[key].numpy(), view, casting="same_kind")
            else:
                st[key] = torch.from_numpy(view.copy())
            if kind == "m":
                cur = st.get("step")
                if torch.is_tensor(cur) and cur.dim() == 0 and not cur.is_cuda:
                    cur.fill_(float(step))
                else:
                    st["step"] = torch.tensor(float(step))  # torch keeps the step as a float32 scalar tensor

    def _hparams(self, noisy: bool, delay: int) -> OffPolicyHparams:
        trainable, _ = self._nets()
        lin = lambda m: describe_mlp(m.network)[3]
        hp = OffPolicyHparams()
        hp.gamma, hp.polyak_rho = self.gamma, self.polyak_rho
        hp.target_noise_scale = getattr(self, "target_noise_scale", 0.0)
        hp.target_noise_clip = getattr(self, "target_noise_clip", 0.0)
        hp.action_limit = float(self.env.action_space.high[0]) if noisy else 0.0
        hp.policy_delay, hp.use_target_noise = int(delay), int(noisy)
        hp.policy_lr, hp.policy_beta1, hp.policy_beta2, hp.policy_eps = adam_hparams(
            self.policy.optimizer, lin(self.policy), "policy optimizer")
        q_last = trainable[2] if self.n_q == 2 else trainable[1]  # IQL's value function follows the critics
        q1 = adam_hparams(trainable[1].optimizer, lin(trainable[1]), "q-function optimizer")
        q2 = adam_hparams(q_last.optimizer, lin(q_last), "q-function optimizer")
        if q1[1:] != q2[1:]:
            raise NotImplementedError("both Q optimizers must share betas / eps")
        hp.q1_lr, hp.q2_lr = q1[0], q2[0]
        hp.q_beta1, hp.q_beta2, hp.q_eps = q1[1], q1[2], q1[3]
        return hp

    def _noise(self, S: int, B: int) -> np.ndarray:
        """S draws of torch.randn(B, A), the reference's stream (td3.py:328), gathered without torch.stack."""
        A = self.policy.network.sizes[-1] if hasattr(self.policy.network, "sizes") else describe_mlp(self.policy.network)[0][-1]
        out = np.empty((S, B, A), dtype=np.float32)
        for i in range(S):
            out[i] = torch.randn(B, A).numpy()
        return out

    # A train() call in three phases -- draw and stage the inputs (_stage_inputs), the engine call (_call_engine), the
    # write-back (_download_state) -- so that a LearnerGroup can run the host phases per learner and make ONE engine
    # call for all of them.
    def _stage_inputs(self, replay_buffer, S: int, B: int, noisy: bool):
        """Everything of one train() call that uses the host's random streams: the minibatch indices (or, without a
        device replay, the gathered minibatches) and the noise.  Returns (mode, inputs)."""
        # host side, same random streams as the reference: numpy RNG for the indices (replay_buffer.py:58), torch CPU
        # RNG for the target-smoothing noise (td3.py:328); the two streams are independent, so drawing all minibatches
        # first and all noise second consumes each exactly as the interleaved reference loop does.
        if isinstance(replay_buffer, PrioritizedReplayBuffer):
            raise ValueError(f"{type(self).__name__} does not train on a PrioritizedReplayBuffer: prioritized replay is "
                             "implemented for DQN only")
        device_replay = (S > 0 and getattr(self, "use_device_replay", True) and hasattr(replay_buffer, "device_columns")
                         and hasattr(replay_buffer, "sample_indices"))
        # opt-in (SURVEY 8f-4): indices and smoothing noise drawn on the device -- not the reference's random streams
        device_rng = device_replay and getattr(self, "use_device_rng", False) and hasattr(replay_buffer, "ring")
        def noise_of():
            return self._noise(S, B) if noisy and S > 0 else None
        if S == 0:
            return None, None
        if device_rng:
            self._device_rng_calls = getattr(self, "_device_rng_calls", 0) + 1
            return "rng", (getattr(self, "device_rng_seed", 0), self._device_rng_calls)
        if device_replay:
            # device-resident replay columns: S index draws on the host (the same numpy stream as S sample_minibatch
            # calls); the gather happens on the GPU, only indices and noise cross PCIe
            idx = replay_buffer.physical_rows(np.stack([replay_buffer.sample_indices(B) for _ in range(S)]))
            return "gather", (idx, noise_of())
        else:
            if S > 0 and hasattr(replay_buffer, "sample_indices") and hasattr(replay_buffer, "gather"):
                idx_l = np.stack([replay_buffer.sample_indices(B) for _ in range(S)])
                cols = replay_buffer.gather(idx_l)
                stack = lambda k, dt: np.ascontiguousarray(cols[k], dtype=dt).reshape((S, B) + cols[k].shape[2:])
            else:  # any object with the reference's sample_minibatch
                mbs = [replay_buffer.sample_minibatch(B) for _ in range(S)]
                stack = lambda k, dt: np.stack([np.asarray(m[k]) for m in mbs]).astype(dt) if S > 0 else np.zeros((0, B), dt)
            noise = noise_of()
            obs, act = stack("observations", np.float32), stack("actions", np.float32)
            rew = stack("rewards", np.float32)                      # rewards f64 -> .float() (td3.py:226)
            nobs = stack("next_observations", np.float32)
            done = stack("dones", np.float32)                       # bool -> .int() (td3.py:228), used as (1 - d)
            return "host", (obs, act, rew, nobs, done, noise)

    # n-step returns and prioritized replay (DQN's family and D4PG): what _stage_inputs / _call_engine add to the
    # uniform paths above
    def _stage_nstep_and_prioritized(self, replay_buffer, S: int, critic_optimizer, critic_linears):
        """The n-step checks, then for a PrioritizedReplayBuffer the staging of the prioritized device call: its keys
        (``device_rng_seed``, this learner's count of device-drawn calls) and the last step's beta, logged as
        replay/beta (beta follows ``critic_optimizer``'s step count).  Returns ("per", keys) or (None, None) for S = 0
        with a prioritized buffer, and None for any other buffer (the uniform paths stage the call)."""
        n_step = getattr(self, "n_step", 1)
        if n_step > 1:  # the windows are assembled on the device from the replay ring
            if not getattr(self, "use_device_replay", True):
                raise ValueError(f"n_step = {n_step} needs use_device_replay = True: n-step windows are assembled on "
                                 "the device from the replay columns")
            if not hasattr(replay_buffer, "device_episode_ends"):
                raise ValueError(f"n_step = {n_step} needs a replay buffer with device_episode_ends (a ReplayBuffer "
                                 f"or PrioritizedReplayBuffer), got {type(replay_buffer).__name__}")
        if not isinstance(replay_buffer, PrioritizedReplayBuffer):
            self._last_beta = None
            return None
        # always the prioritized device path, keyed like the uniform device draws (device_rng_seed, call count)
        if not getattr(self, "use_device_replay", True):
            raise ValueError("a PrioritizedReplayBuffer needs use_device_replay = True: its draws and priority "
                             "updates run on the device")
        if S == 0:
            return None, None
        self._device_rng_calls = getattr(self, "_device_rng_calls", 0) + 1
        t0 = self._adam_step_count(critic_optimizer, critic_linears)
        self._last_beta = replay_buffer.beta(t0 + S - 1)  # the last step's beta, logged as replay/beta
        return "per", (getattr(self, "device_rng_seed", 0), self._device_rng_calls)

    def _call_nstep_and_prioritized(self, e, hp, replay_buffer, S: int, B: int, mode, inputs):
        """The engine call of a learner with n-step returns and prioritized replay: the window length (and episode
        ends) first, then the prioritized call for mode "per" or the uniform paths' call."""
        if mode is not None:
            n_step = getattr(self, "n_step", 1)
            e.set_nstep(n_step, [replay_buffer.device_episode_ends()] if n_step > 1 else None)
        if mode != "per":
            return _OffPolicyBase._call_engine(e, hp, replay_buffer, S, B, mode, inputs)
        e.set_per(*replay_buffer.per_settings())
        tree = replay_buffer.device_tree()
        columns, rows = replay_buffer.device_columns()
        return e.train_prioritized(hp, columns, rows, tree, S, B, *inputs)

    @staticmethod
    def _call_engine(e, hp, replay_buffer, S: int, B: int, mode, inputs):
        """The engine call of one learner (``e`` solo) on what ``_stage_inputs`` returned."""
        if mode is None:
            return None
        if mode == "rng":
            columns, rows = replay_buffer.device_columns()
            start, size, _ = replay_buffer.ring()
            return e.train_gather_rng(hp, columns, rows, start, size, S, B, *inputs)
        if mode == "gather":
            columns, rows = replay_buffer.device_columns()
            return e.train_gather(hp, columns, rows, *inputs)
        return e.train(hp, *inputs)

    def _learner_nets(self):
        """(trainable, targets, Linear layers of each) in the blob's order."""
        trainable, targets = self._nets()
        return trainable, targets, [describe_mlp(m.network)[3] for m in trainable + targets]

    def _run(self, replay_buffer, num_train_steps: int, minibatch_size: int, noisy: bool, delay: int):
        S, B = int(num_train_steps), int(minibatch_size)
        mode, inputs = self._stage_inputs(replay_buffer, S, B, noisy)
        e = self._ensure_engine(max(S, 1), B)
        trainable, targets, lins = self._learner_nets()
        self._upload_state(e, trainable, targets, lins)
        out = self._call_engine(e, self._hparams(noisy, delay), replay_buffer, S, B, mode, inputs)
        self._download_state(e, trainable, targets, lins)
        self.last_train_output = out
        return out

    def _train_schedule(self):
        """(noisy, policy delay) of this algorithm's train steps."""
        return True, int(self.policy_delay)

    def train(self, replay_buffer, num_train_steps: int, minibatch_size: int) -> None:
        noisy, delay = self._train_schedule()
        self._record_train(self._run(replay_buffer, num_train_steps, minibatch_size, noisy=noisy, delay=delay))

    def learn_offline(self, num_epochs: int, num_train_steps: int = 1000, minibatch_size: int = 256,
                      num_evaluation_episodes: int = 10, evaluation_interval: int = 1, model_saving_interval: int = 1,
                      output_dir: str = ".") -> None:
        """Train on the fixed contents of ``self.replay_buffer`` (e.g. ``ReplayBuffer.from_dataset``) with no sampler:
        each epoch runs ``num_train_steps`` train steps, logs ``epoch`` and ``total_train_steps``, then evaluates every
        ``evaluation_interval`` and saves ``model.pt`` every ``model_saving_interval`` epochs as ``learn`` does."""
        started = _learn_begin(self, output_dir)
        mm = self.metrics_manager
        for epoch in range(1, num_epochs + 1):
            self.current_total_steps += int(num_train_steps)  # the train steps so far: the x-axis of the logs
            self.train(self.replay_buffer, num_train_steps, minibatch_size)
            mm.record_scalar("epoch", epoch)
            mm.record_scalar("total_train_steps", self.current_total_steps)
            _learn_evaluate_save(self, epoch, started, num_evaluation_episodes, evaluation_interval,
                                 model_saving_interval, output_dir, progress=epoch)
        mm.close()


class TD3(_OffPolicyBase):
    """Same constructor arguments / defaults as ref algorithms/td3.py:46-62."""
    n_q = 2

    def __init__(self, policy, exploration_policy, q_function_1, q_function_2, env, sampler, replay_buffer, evaluator,
                 gamma: float = 0.99, polyak_rho: float = 0.995, action_noise_scale: float = 0.1,
                 target_noise_scale: float = 0.2, target_noise_clip: float = 0.5, policy_delay: int = 2) -> None:
        refuse_noisy("TD3", policy, q_function_1, q_function_2)
        self.policy, self.exploration_policy = policy, exploration_policy
        self.q_function_1, self.q_function_2 = q_function_1, q_function_2
        self.env, self.sampler, self.replay_buffer, self.evaluator = env, sampler, replay_buffer, evaluator
        self.gamma, self.polyak_rho, self.action_noise_scale = gamma, polyak_rho, action_noise_scale
        self.target_noise_scale, self.target_noise_clip, self.policy_delay = target_noise_scale, target_noise_clip, policy_delay
        self.noised_policy = add_noise_to_get_action(self.policy, self.env.action_space, self.action_noise_scale)
        self.evaluation_env = _make_eval_env(env)
        self.target_policy, self.target_q_function_1, self.target_q_function_2 = self._make_targets()

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
        # ref td3.py:265-299 (tag typos are part of the API)
        mm.record_scalar("policy/average_loss", float(np.mean(out["policy_losses"])), steps, tensorboard=True)
        mm.record_scalar("q-function_1/average_loss", float(np.mean(out["q1_losses"])), steps, tensorboard=True)
        mm.record_scalar("q-function_2/average_loss", float(np.mean(out["q2_losses"])), steps, tensorboard=True)
        for i, key in ((1, "q1_values"), (2, "q2_values")):
            q = out[key].astype(np.float64)
            mm.record_scalar(f"q-function_{i}/avarage_q-value", float(np.mean(q)), steps, tensorboard=True)
            mm.record_scalar(f"q-function_{i}/max_q-value", float(np.max(q)))
            mm.record_scalar(f"q-function_{i}/min_q-value", float(np.min(q)))

    def save_model(self, current_epoch: int, model_path: str) -> None:
        """ref td3.py:360-382"""
        torch.save({
            "epoch": current_epoch, "total_steps": self.current_total_steps,
            "policy_state_dict": self.policy.network.state_dict(),
            "policy_optimizer_state_dict": self.policy.optimizer.state_dict(),
            "target_policy_state_dict": self.target_policy.network.state_dict(),
            "q_function_1_state_dict": self.q_function_1.network.state_dict(),
            "q_function_1_optimizer_state_dict": self.q_function_1.optimizer.state_dict(),
            "target_q_function_1_state_dict": self.target_q_function_1.network.state_dict(),
            "q_function_2_state_dict": self.q_function_2.network.state_dict(),
            "q_function_2_optimizer_state_dict": self.q_function_2.optimizer.state_dict(),
            "target_q_function_2_state_dict": self.target_q_function_2.network.state_dict(),
        }, model_path)


class DDPG(_OffPolicyBase):
    """Same constructor arguments / defaults as ref algorithms/ddpg.py:41-53."""
    n_q = 1

    def __init__(self, policy, exploration_policy, q_function, env, sampler, replay_buffer, evaluator,
                 gamma: float = 0.99, polyak_rho: float = 0.995, action_noise_scale: float = 0.1) -> None:
        refuse_noisy("DDPG", policy, q_function)
        self.policy, self.exploration_policy, self.q_function = policy, exploration_policy, q_function
        self.env, self.sampler, self.replay_buffer, self.evaluator = env, sampler, replay_buffer, evaluator
        self.gamma, self.polyak_rho, self.action_noise_scale = gamma, polyak_rho, action_noise_scale
        self.noised_policy = add_noise_to_get_action(self.policy, self.env.action_space, self.action_noise_scale)
        self.evaluation_env = _make_eval_env(env)
        self.target_policy, self.target_q_function = self._make_targets()

    def learn(self, num_epochs: int = 2000, batch_size: int = 50, minibatch_size: int = 100,
              num_start_steps: int = 10000, num_steps_before_update: int = 1000, num_train_steps: int = 50,
              num_evaluation_episodes: int = 5, evaluation_interval: int = 4000, model_saving_interval: int = 4000,
              output_dir: str = ".") -> None:
        _learn(self, num_epochs, batch_size, minibatch_size, num_start_steps, num_steps_before_update, num_train_steps,
               num_evaluation_episodes, evaluation_interval, model_saving_interval, output_dir)

    def _train_schedule(self):
        return False, 1

    def _record_train(self, out) -> None:
        mm, steps = getattr(self, "metrics_manager", None), getattr(self, "current_total_steps", 0)
        if mm is None or out is None:
            return
        q = out["q1_values"].astype(np.float64)  # ref ddpg.py:232-253
        mm.record_scalar("policy/average_loss", float(np.mean(out["policy_losses"])), steps, tensorboard=True)
        mm.record_scalar("q-function/average_loss", float(np.mean(out["q1_losses"])), steps, tensorboard=True)
        mm.record_scalar("q-function/avarage_q-value", float(np.mean(q)), steps, tensorboard=True)
        mm.record_scalar("q-function/max_q-value", float(np.max(q)))
        mm.record_scalar("q-function/min_q-value", float(np.min(q)))

    def save_model(self, current_epoch: int, model_path: str) -> None:
        """ref ddpg.py:295-314"""
        torch.save({
            "epoch": current_epoch, "total_steps": self.current_total_steps,
            "policy_state_dict": self.policy.network.state_dict(),
            "policy_optimizer_state_dict": self.policy.optimizer.state_dict(),
            "target_policy_state_dict": self.target_policy.network.state_dict(),
            "q_function_state_dict": self.q_function.network.state_dict(),
            "q_function_optimizer_state_dict": self.q_function.optimizer.state_dict(),
            "target_q_function_state_dict": self.target_q_function.network.state_dict(),
        }, model_path)


def _make_eval_env(env):
    """gym.make(env.spec.id) when gymnasium knows the environment (ref td3.py:76); otherwise an independent copy of
    ``env`` -- evaluation must not step the environment the sampler is in the middle of an episode with."""
    try:
        import gymnasium as gym
        return gym.make(env.spec.id)
    except Exception:
        try:
            return copy.deepcopy(env)
        except Exception:
            return env


def _learn(self, num_epochs, batch_size, minibatch_size, num_start_steps, num_steps_before_update, num_train_steps,
           num_evaluation_episodes, evaluation_interval, model_saving_interval, output_dir) -> None:
    """Shared host loop of TD3.learn / DDPG.learn / SAC.learn / DQN.learn (ref: td3.py:94-212, ddpg.py:85-193).  One epoch is three
    phases (sample, train, evaluate and save), which LearnerGroup.learn runs in lockstep for its learners."""
    if self.sampler is None or self.exploration_policy is None:
        raise ValueError(f"{type(self).__name__}.learn needs a sampler and an exploration policy; without them "
                         "(offline data) use learn_offline")
    started = _learn_begin(self, output_dir)
    for epoch in range(1, num_epochs + 1):
        if _learn_sample(self, epoch, batch_size, num_start_steps, num_steps_before_update):
            self.train(self.replay_buffer, num_train_steps, minibatch_size)
        _learn_evaluate_save(self, epoch, started, num_evaluation_episodes, evaluation_interval, model_saving_interval,
                             output_dir)
    self.metrics_manager.close()


def _learn_begin(self, output_dir) -> float:
    started = time.time()
    self.current_total_steps = 0
    self.current_total_episodes = 0
    os.makedirs(output_dir, exist_ok=True)
    self.metrics_manager = MetricsManager(output_dir)
    return started


def _learn_sample(self, epoch, batch_size, num_start_steps, num_steps_before_update) -> bool:
    """Sample, add to the replay buffer and log; returns whether this epoch trains."""
    mm = self.metrics_manager
    actor = self.exploration_policy if self.current_total_steps < num_start_steps else self.noised_policy
    experience = self.sampler.sample(batch_size, actor)
    self.replay_buffer.add_experience(experience)
    returns, lengths = experience.episode_returns, experience.episode_lengths
    self.current_total_steps += sum(lengths)
    self.current_total_episodes += sum(experience.flattened_dones)
    mm.record_scalar("epoch", epoch)
    mm.record_scalar("total_steps", self.current_total_steps)
    mm.record_scalar("total_episodes", self.current_total_episodes)
    if len(lengths) > 0:
        mm.record_scalar("sampling/average_episode_return", float(np.mean(returns)), self.current_total_steps,
                         tensorboard=True)
        mm.record_scalar("sampling/episode_return_std", float(np.std(returns)))
        mm.record_scalar("sampling/max_episode_return", float(np.max(returns)))
        mm.record_scalar("sampling/min_episode_return", float(np.min(returns)))
        mm.record_scalar("sampling/average_episode_length", float(np.mean(lengths)), self.current_total_steps,
                         tensorboard=True)
    return self.current_total_steps >= num_steps_before_update


def _learn_evaluate_save(self, epoch, started, num_evaluation_episodes, evaluation_interval, model_saving_interval,
                         output_dir, progress=None) -> None:
    """Evaluate and save when ``progress`` (the environment steps so far unless given) is a multiple of the interval."""
    mm = self.metrics_manager
    progress = self.current_total_steps if progress is None else progress
    if num_evaluation_episodes > 0 and progress % evaluation_interval == 0:
        ev_policy = getattr(self, "evaluation_policy", self.policy)  # SAC: the deterministic view of its policy
        ev_returns, ev_lengths = self.evaluator.evaluate(ev_policy, self.evaluation_env, num_evaluation_episodes)
        mm.record_scalar("evaluation/average_episode_return", float(np.mean(ev_returns)), self.current_total_steps,
                         tensorboard=True)
        mm.record_scalar("evaluation/episode_return_std", float(np.std(ev_returns)))
        mm.record_scalar("evaluation/max_episode_return", float(np.max(ev_returns)))
        mm.record_scalar("evaluation/min_episode_return", float(np.min(ev_returns)))
        mm.record_scalar("evaluation/average_episode_length", float(np.mean(ev_lengths)), self.current_total_steps,
                         tensorboard=True)
    if progress % model_saving_interval == 0:
        self.save_model(epoch, os.path.join(output_dir, "model.pt"))
    mm.record_scalar("time", time.time() - started)
    mm.dump()
