"""LearnerGroup: several independent TD3 / DDPG / D4PG / SAC / TQC / CQL / IQL / REDQ / EDAC / discrete SAC / DQN / C51 / QR-DQN / IQN learners (typically one per seed) trained side by side by ONE
off-policy engine, every operation of a train step one launch for all of them (b200rl_offpolicy_create_group).

The contract: each member ends up bit for bit where it would be had it run alone.  Members keep everything of their
own -- environment, sampler, replay buffer, evaluator, networks, Adam states and step counts, temperature -- and their
own random streams: ``add`` records the current state of the generators ``set_seed_for_libraries`` seeds (Python
``random``, NumPy's global ``np.random``, torch's default CPU generator) as that member's stream, and every piece of
host work the group does for a member (minibatch index draws, target-smoothing / SAC noise, sampling, exploration,
evaluation) runs with that stream installed.  After a group call the global generators are as they were before it.

    group = LearnerGroup()
    for seed in (0, 1, 2):
        set_seed_for_libraries(seed)
        group.add(build_td3(seed))
    group.learn(num_epochs=..., output_dirs=["seed-0", "seed-1", "seed-2"])
"""
from __future__ import annotations

import contextlib
import random
from typing import List, Sequence

import numpy as np
import torch

from .._lib import MAX_LEARNERS
from ..engine import OffPolicyEngine
from ..networks import ImplicitQuantileMLP
from ..replay_buffer import PrioritizedReplayBuffer
from ._onpolicy import adam_hparams, describe_mlp
from .dqn import describe_q_network, noisy_mask
from .qrdqn import QRDQN
from .td3 import _learn_begin, _learn_evaluate_save, _learn_sample, _OffPolicyBase


def _signature(agent) -> list:
    """[(attribute, value)] that every member of a group shares (one engine trains them all), in the order in which a
    refusal reports the first difference."""
    trainable, _ = agent._nets()
    dqn = agent.algo in OffPolicyEngine.DISCRETE
    names = ["q_function"] if dqn else ["policy"] + (["q_function_1", "q_function_2"] if agent.n_q == 2 else ["q_function"])
    if agent.algo == OffPolicyEngine.IQL:
        names.append("value_function")
    if agent.algo in (OffPolicyEngine.REDQ, OffPolicyEngine.EDAC):
        names = ["policy"] + [f"q_function_{i}" for i in range(1, agent.n_critics + 1)]
    sig = [("class", type(agent).__name__)]
    for name, m in zip(names, trainable):
        if dqn:
            sizes, hidden_act, out_act, lins, k = describe_q_network(m.network)
            kind = type(m.network).__name__ if isinstance(m.network, ImplicitQuantileMLP) else "DuelingMLP" if k else "MLP"
            sig.append((f"{name} network kind", kind))
            sig.append((f"{name} dueling (h_trunk, h_stream, outputs_per_action)", (sizes[1], sizes[2], k) if k else None))
            sig.append((f"{name} noisy layers", noisy_mask(lins)))
        else:
            sizes, hidden_act, out_act, lins = describe_mlp(m.network)
        sig.append((f"{name} network", (tuple(sizes), hidden_act, out_act)))
        sig.append((f"{name} optimizer (lr, beta1, beta2, eps)", adam_hparams(m.optimizer, lins, f"{name} optimizer")))
    if dqn:
        sig.append(("action count", agent.n_actions))
        for attr in ("gamma", "target_update_interval", "double_q", "epsilon_start", "epsilon_end", "epsilon_decay_steps",
                     "use_device_replay", "use_device_rng", "n_step"):
            sig.append((attr, getattr(agent, attr, None)))
        if agent.algo == OffPolicyEngine.C51:
            for attr in ("n_atoms", "v_min", "v_max"):
                sig.append((attr, getattr(agent.q_function, attr)))
        sig.append(("n_quantiles", getattr(agent.q_function, "n_quantiles", None)))
        sig.append(("IQN (n_cos, n_quantiles, n_target_quantiles, n_policy_quantiles)", getattr(agent, "iqn_config", None)))
        return sig + _prioritized_signature(agent)
    if agent.algo == OffPolicyEngine.DSAC:
        sig.append(("action count", agent.n_actions))
    else:
        sig.append(("action limit", float(agent.env.action_space.high[0])))
    for attr in ("gamma", "polyak_rho", "target_noise_scale", "target_noise_clip", "policy_delay", "use_device_replay",
                 "use_device_rng"):
        sig.append((attr, getattr(agent, attr, None)))
    if agent.algo in OffPolicyEngine.SOFT:
        sig += [("alpha", agent.alpha), ("learn_alpha", agent.learn_alpha), ("target_entropy", agent.target_entropy),
                ("alpha optimizer (lr, beta1, beta2, eps)",
                 adam_hparams(agent.alpha_optimizer, [], "alpha optimizer", extra=[agent.log_alpha]))]
    if agent.algo in OffPolicyEngine.SQUASHED:
        sig.append(("log_std bounds", (agent.policy.log_std_min, agent.policy.log_std_max)))
    if agent.algo == OffPolicyEngine.TQC:
        sig.append(("(n_quantiles, top_quantiles_to_drop_per_net)", agent.tqc_config))
    if agent.algo == OffPolicyEngine.REDQ:
        sig.append(("(n_critics, n_min)", agent.redq_config))
    if agent.algo == OffPolicyEngine.EDAC:
        sig.append(("(n_critics, eta)", agent.edac_config))
    if agent.algo == OffPolicyEngine.CQL:
        sig.append(("(cql_n_actions, lagrange)", agent.cql_config))
        sig.append(("CQL hyper-parameters", agent.cql_hparams()))
    if agent.algo == OffPolicyEngine.IQL:
        sig.append(("log_std bounds", (agent.policy.log_std_min, agent.policy.log_std_max)))
        sig.append(("IQL hyper-parameters (expectile, beta, max_weight)", (agent.expectile, agent.beta, agent.max_weight)))
    if agent.algo == OffPolicyEngine.D4PG:
        sig.append(("(n_atoms, v_min, v_max)", agent.d4pg_config))
        sig.append(("n_step", agent.n_step))
        sig += _prioritized_signature(agent)
    return sig


def _prioritized_signature(agent) -> list:
    """Whether the member trains on a PrioritizedReplayBuffer, and its settings (the engine takes one set)."""
    rb = getattr(agent, "replay_buffer", None)
    per = isinstance(rb, PrioritizedReplayBuffer)
    return [("prioritized replay", per)] + [(f"prioritized replay {attr}", getattr(rb, attr, None) if per else None)
                                            for attr in ("alpha", "eps", "beta_start", "beta_anneal_steps")]


def _check_prioritized_buffers(members) -> None:
    """Each member's PrioritizedReplayBuffer must be its own: the priority updates of all members run at once, and two
    of them writing one sum tree would race."""
    seen = {}
    for k, m in enumerate(members):
        rb = getattr(m, "replay_buffer", None)
        if isinstance(rb, PrioritizedReplayBuffer):
            if id(rb) in seen:
                raise ValueError(f"LearnerGroup: members {seen[id(rb)]} and {k} share one PrioritizedReplayBuffer; "
                                 "every prioritized member needs a buffer of its own")
            seen[id(rb)] = k


def _stack_noise(parts):
    """The members' inputs stacked on a leading [K] axis; a tuple (CQL's noise) part by part; None stays None."""
    if parts[0] is None:
        return None
    if isinstance(parts[0], tuple):
        return tuple(np.stack(x) for x in zip(*parts))
    return np.stack(parts)


def _rng_state():
    return random.getstate(), np.random.get_state(), torch.get_rng_state()


def _set_rng_state(state) -> None:
    random.setstate(state[0])
    np.random.set_state(state[1])
    torch.set_rng_state(state[2])


class LearnerGroup:
    """Up to ``MAX_LEARNERS`` (16) off-policy learners of one class with the same network shapes and hyper-parameters
    (Adam step counts may differ), trained in lockstep by one engine."""

    def __init__(self) -> None:
        self.members: List[_OffPolicyBase] = []
        self._streams: list = []
        self._engine = None

    def __len__(self) -> int:
        return len(self.members)

    def add(self, agent) -> None:
        """Add ``agent``; the current state of the global random generators becomes its private stream."""
        if not isinstance(agent, _OffPolicyBase):
            raise ValueError(f"LearnerGroup: members must be TD3, DDPG or SAC (or D4PG / TQC / CQL / IQL / REDQ / EDAC / DiscreteSAC / DQN / C51 / QR-DQN / IQN) learners, got {type(agent).__name__}")
        if any(m is agent for m in self.members):
            raise ValueError("LearnerGroup: this agent is already a member")
        if len(self.members) >= MAX_LEARNERS:
            raise ValueError(f"LearnerGroup: at most {MAX_LEARNERS} members")
        if self.members:
            for (name, want), (_, got) in zip(_signature(self.members[0]), _signature(agent)):
                if got != want:
                    raise ValueError(f"LearnerGroup: {name} differs from the first member's ({got!r} != {want!r})")
        _check_prioritized_buffers(self.members + [agent])
        self.members.append(agent)
        self._streams.append(_rng_state())
        self._close_engine()

    @contextlib.contextmanager
    def stream(self, k: int):
        """Run the body with member ``k``'s random stream installed; its advance is kept for the member, and the global
        generators are restored afterwards."""
        saved = _rng_state()
        _set_rng_state(self._streams[k])
        try:
            yield
        finally:
            self._streams[k] = _rng_state()
            _set_rng_state(saved)

    def _check(self) -> List[_OffPolicyBase]:
        if not self.members:
            raise ValueError("LearnerGroup: the group has no members")
        return self.members

    def _close_engine(self) -> None:
        if self._engine is not None:
            self._engine.close()
            self._engine = None

    def _ensure_engine(self, S: int, B: int) -> OffPolicyEngine:
        m = self.members[0]
        discrete = m.algo in OffPolicyEngine.DISCRETE
        if discrete:  # no policy network
            psz, pact, pout = None, "relu", "tanh"
            qsz, (qact, qout), kw = m._engine_config()
        else:
            psz, pact, pout, _ = describe_mlp(m.policy.network)
            qsz, qact, qout, _ = describe_mlp(m._nets()[0][1].network)
            kw = dict(dueling_k=0, noisy_layers=0, **m._engine_extra())
        e = self._engine
        if (e is None or e.K != len(self.members) or e.max_minibatch < B or e.max_steps < S or e.policy_sizes != psz
                or e.q_sizes != qsz or e.policy_acts != (pact, pout) or e.q_acts != (qact, qout)
                or any(getattr(e, k) != v for k, v in kw.items())):
            self._close_engine()
            e = OffPolicyEngine(psz, qsz, m.n_q, B, S, (pact, pout), (qact, qout), algo=m.algo,
                                n_learners=len(self.members), **kw)
            self._engine = e
        return e

    def train(self, num_train_steps: int, minibatch_size: int) -> None:
        """``agent.train(agent.replay_buffer, num_train_steps, minibatch_size)`` for every member, each on its own replay
        buffer and random stream, as one engine call."""
        members = self._check()
        _check_prioritized_buffers(members)  # a member's buffer may have been replaced since add()
        S, B = int(num_train_steps), int(minibatch_size)
        if len(members) == 1 or S == 0:  # nothing to batch: the members' own calls
            for k, m in enumerate(members):
                with self.stream(k):
                    m.train(m.replay_buffer, S, B)
            return
        noisy, delay = members[0]._train_schedule()
        staged = []
        for k, m in enumerate(members):
            with self.stream(k):
                staged.append(m._stage_inputs(m.replay_buffer, S, B, noisy))
        mode = staged[0][0]
        if any(st[0] != mode for st in staged):
            raise ValueError("LearnerGroup: the members' replay buffers do not all support the same minibatch path")
        e = self._ensure_engine(S, B)
        plans, steps = [], []
        for k, m in enumerate(members):
            trainable, targets, lins = m._learner_nets()
            slots = m._state_plan(e, trainable, targets, lins, lane=k)
            steps.append(m._fill_state(slots, trainable, lins))
            plans.append((slots, trainable))
        e.set_state(None, steps)
        sac = members[0].algo in OffPolicyEngine.SOFT
        if sac:
            e.set_sac(members[0]._sac_hparams())
            e.set_alpha_group([m._alpha_state() for m in members])
        cql = members[0].algo == OffPolicyEngine.CQL
        if members[0].algo == OffPolicyEngine.IQL:
            e.set_iql(**members[0].iql_hparams())
        if cql:
            e.set_cql(**members[0].cql_hparams())
            e.set_alpha_prime_group([m._alpha_prime_state() for m in members])
        if members[0].algo in OffPolicyEngine.DISCRETE:
            e.set_dqn(members[0].target_update_interval, members[0].double_q)
        if members[0].algo == OffPolicyEngine.C51:
            q = members[0].q_function
            e.set_c51(q.n_atoms, q.v_min, q.v_max)
        if isinstance(members[0], QRDQN):
            e.set_qr(members[0].q_function.n_quantiles)
        hp = members[0]._hparams(noisy, delay)
        if members[0].algo in OffPolicyEngine.DISCRETE and members[0]._needs_draw_keys():
            e.set_noise_keys(*zip(*[m.noise_key for m in members]))
        if members[0].algo in OffPolicyEngine.DISCRETE + (OffPolicyEngine.D4PG,):
            n = members[0].n_step
            e.set_nstep(n, [m.replay_buffer.device_episode_ends() for m in members] if n > 1 else None)
        if mode == "per":
            e.set_per(*members[0].replay_buffer.per_settings())
            trees = [m.replay_buffer.device_tree() for m in members]
            replays = [m.replay_buffer.device_columns() for m in members]
            out = e.train_prioritized_group(hp, replays, trees, S, B, [st[1][0] for st in staged],
                                            [st[1][1] for st in staged])
        elif mode == "rng":
            replays = [m.replay_buffer.device_columns() for m in members]
            rings = [m.replay_buffer.ring() for m in members]
            out = e.train_gather_rng_group(hp, replays, [r[0] for r in rings], [r[1] for r in rings], S, B,
                                           [st[1][0] for st in staged], [st[1][1] for st in staged])
        elif mode == "gather":
            replays = [m.replay_buffer.device_columns() for m in members]
            noise = _stack_noise([st[1][1] for st in staged])
            out = e.train_gather_group(hp, replays, np.stack([st[1][0] for st in staged]), noise)
        else:
            cols = [_stack_noise([st[1][i] for st in staged]) for i in range(6)]
            out = e.train(hp, *cols)
        _, steps = e.get_state()
        for (slots, trainable), m, st in zip(plans, members, steps):
            m._read_state(slots, trainable, st)
        if sac:
            for m, a in zip(members, e.get_alpha_group()):
                m._store_alpha_state(*a)
        if cql:
            for m, a in zip(members, e.get_alpha_prime_group()):
                m._store_alpha_prime_state(*a)
        for k, m in enumerate(members):
            m.last_train_output = {key: v[k] for key, v in out.items()}
            m._record_train(m.last_train_output)

    def learn(self, output_dirs: Sequence[str], num_epochs: int = 2000, batch_size: int = 50, minibatch_size: int = 100,
              num_start_steps: int = 10000, num_steps_before_update: int = 1000, num_train_steps: int = 50,
              num_evaluation_episodes: int = 5, evaluation_interval: int = 4000, model_saving_interval: int = 4000) -> None:
        """Every member's ``learn`` (TD3.learn's arguments, one output directory per member) in lockstep: per epoch each
        member samples under its own stream, the members train in one group call, then each evaluates and saves.  An
        epoch in which only some members train (their step counts differ) trains those alone."""
        members = self._check()
        if len(output_dirs) != len(members):
            raise ValueError(f"LearnerGroup.learn: {len(members)} members need {len(members)} output_dirs, "
                             f"got {len(output_dirs)}")
        started = []
        for k, m in enumerate(members):
            with self.stream(k):
                started.append(_learn_begin(m, output_dirs[k]))
        for epoch in range(1, num_epochs + 1):
            trains = []
            for k, m in enumerate(members):
                with self.stream(k):
                    trains.append(_learn_sample(m, epoch, batch_size, num_start_steps, num_steps_before_update))
            if all(trains):
                self.train(num_train_steps, minibatch_size)
            else:
                for k, m in enumerate(members):
                    if trains[k]:
                        with self.stream(k):
                            m.train(m.replay_buffer, num_train_steps, minibatch_size)
            for k, m in enumerate(members):
                with self.stream(k):
                    _learn_evaluate_save(m, epoch, started[k], num_evaluation_episodes, evaluation_interval,
                                         model_saving_interval, output_dirs[k])
        for m in members:
            m.metrics_manager.close()
