from typing import List, Optional

import numpy as np


class Experience:
    """Trajectory container with the reference's nested-list layout (ref: experience.py:6-84):
    ``observations[e][t]``, ``actions[e][t]``, ``rewards[e][t]``, ``dones[e][t]`` and one ``last_observations[e]``."""

    _FIELDS = ("observations", "actions", "rewards", "last_observations", "dones", "episode_returns", "episode_lengths")

    def __init__(self, observations: Optional[List[List[np.ndarray]]] = None,
                 actions: Optional[List[List[np.ndarray]]] = None, rewards: Optional[List[List[float]]] = None,
                 last_observations: Optional[List[np.ndarray]] = None, dones: Optional[List[List[bool]]] = None,
                 episode_returns: Optional[List[float]] = None, episode_lengths: Optional[List[int]] = None):
        given = (observations, actions, rewards, last_observations, dones, episode_returns, episode_lengths)
        for name, value in zip(self._FIELDS, given):
            setattr(self, name, value if value else [])

    @property
    def observations_with_last_observation(self):
        return [list(obs) + [last] for obs, last in zip(self.observations, self.last_observations)]

    @property
    def next_observations(self):
        return [list(obs[1:]) + [last] for obs, last in zip(self.observations, self.last_observations)]

    @property
    def episode_dones(self) -> List[bool]:
        return [episode[-1] for episode in self.dones]

    @staticmethod
    def _flat(nested):
        return [item for episode in nested for item in episode]

    @property
    def flattened_observations(self):
        return self._flat(self.observations)

    @property
    def flattened_actions(self):
        return self._flat(self.actions)

    @property
    def flattened_rewards(self):
        return self._flat(self.rewards)

    @property
    def flattened_next_observations(self):
        return self._flat(self.next_observations)

    @property
    def flattened_dones(self):
        return self._flat(self.dones)


class PackedExperience(Experience):
    """Contiguous backing store for one epoch of rollouts (SURVEY 8f-1): structure-of-arrays ``obs [N,O]`` f32,
    ``act [N,A]`` f32, ``rew [N]`` f64, ``done [N]`` bool, ``last_obs [E,O]`` f32 and CSR ``ep_offsets [E+1]`` --
    exactly the layout the update engine uploads, so ``PPO.train(experience)`` skips the nested-list flattening the
    reference pays inside ``train`` (``np.concatenate`` / ``np.stack`` per episode: ppo.py:153-154, utils.py:66-70;
    18 % of its epoch at 64 k transitions, seconds at 1 M).  A sampler appends steps with ``append_step`` and closes
    episodes with ``end_episode``; the reference's nested-list attributes and ``flattened_*`` properties remain
    available as views built on demand, so code written against ``Experience`` keeps working.
    ``pinned=True`` allocates the arrays in page-locked memory (one DMA per column to the GPU)."""

    def __init__(self, capacity: int, observation_size: int, action_size: int, pinned: bool = False,
                 scalar_actions: bool = False):
        """``scalar_actions=True`` (or ``action_size=0``): actions are 0-d values (Discrete spaces: the index a
        CategoricalPolicy samples); ``packed()["act"]`` is then ``[N]`` as the engine's categorical path expects,
        and the ``actions`` view holds 0-d entries like the reference's lists."""
        self.episode_returns, self.episode_lengths = [], []  # the five trajectory fields are views (properties below)
        self.capacity, self._n, self._start = int(capacity), 0, 0
        self._o = int(observation_size)
        self._a = 0 if scalar_actions else int(action_size)

        def alloc(shape, dtype):
            if pinned:
                import torch
                return torch.empty(shape, dtype=getattr(torch, np.dtype(dtype).name), pin_memory=True).numpy()
            return np.empty(shape, dtype=dtype)

        self._obs = alloc((self.capacity, self._o), np.float32)
        self._act = alloc((self.capacity, max(self._a, 1)), np.float32)
        self._rew = alloc((self.capacity,), np.float64)
        self._done = np.zeros(self.capacity, dtype=bool)
        self._last: List[np.ndarray] = []
        self._offsets: List[int] = [0]

    # ---- producer side ----
    def append_step(self, observation, action, reward: float, done: bool) -> None:
        i = self._n
        if i >= self.capacity:
            raise IndexError("PackedExperience is full")
        self._obs[i] = np.asarray(observation, dtype=np.float32).reshape(-1)
        self._act[i] = np.asarray(action, dtype=np.float32).reshape(-1)
        self._rew[i] = reward
        self._done[i] = done
        self._n = i + 1

    def end_episode(self, last_observation, episode_return: Optional[float] = None) -> None:
        if self._n == self._offsets[-1]:
            raise ValueError("end_episode: the episode is empty")
        begin = self._offsets[-1]
        self._offsets.append(self._n)
        self._last.append(np.asarray(last_observation, dtype=np.float32).reshape(-1).copy())
        self.episode_returns.append(float(self._rew[begin:self._n].sum()) if episode_return is None else episode_return)
        self.episode_lengths.append(self._n - begin)

    def append_episode(self, observations, actions, rewards, dones, last_observation) -> None:
        """A whole episode at once: ``[L,O]`` / ``[L,A]`` (or ``[L]``) / ``[L]`` / ``[L]`` arrays, one slice copy per
        column (what a vectorised sampler flushes; ``append_step`` per transition is a Python call per row)."""
        n = len(rewards)
        i = self._n
        if n == 0:
            raise ValueError("append_episode: the episode is empty")
        if i + n > self.capacity:
            raise IndexError("PackedExperience is full")
        self._obs[i:i + n] = np.asarray(observations, dtype=np.float32).reshape(n, -1)
        self._act[i:i + n] = np.asarray(actions, dtype=np.float32).reshape(n, -1)
        self._rew[i:i + n] = rewards
        self._done[i:i + n] = dones
        self._n = i + n
        self.end_episode(last_observation)

    # ---- consumer side: what the engine uploads (views, no copy) ----
    def packed(self):
        n, e = self._offsets[-1], len(self._offsets) - 1
        if e == 0:
            raise ValueError("experience must hold at least one episode and no empty episode")
        act = self._act[:n] if self._a >= 1 else self._act[:n, 0]
        done = np.asarray([bool(self._done[self._offsets[k + 1] - 1]) for k in range(e)], dtype=bool)
        return dict(obs=self._obs[:n], act=act, rew=self._rew[:n], last_obs=np.stack(self._last).astype(np.float32),
                    ep_offsets=np.asarray(self._offsets, dtype=np.int64), ep_done=done)

    def transition_columns(self):
        """(observations [n,O], actions [n,A] or [n], rewards [n], next_observations [n,O], dones [n]) as arrays: what a
        replay buffer appends (``flattened_*`` of the reference, experience.py:60-84) without building Python lists."""
        n = self._offsets[-1]
        obs = self._obs[:n]
        nxt = np.empty_like(obs)
        nxt[:-1] = obs[1:]
        for k, end in enumerate(self._offsets[1:]):
            nxt[end - 1] = self._last[k]  # the step that closes an episode is followed by its last observation
        act = self._act[:n] if self._a >= 1 else self._act[:n, 0]
        return obs, act, self._rew[:n], nxt, self._done[:n]

    @property
    def ep_offsets(self) -> np.ndarray:
        """[E+1] int64: episode k holds rows ep_offsets[k] .. ep_offsets[k+1] - 1."""
        return np.asarray(self._offsets, dtype=np.int64)

    # ---- the reference's nested-list API, as views ----
    def _episodes(self, column):
        return [list(column[b:e]) for b, e in zip(self._offsets[:-1], self._offsets[1:])]

    observations = property(lambda self: self._episodes(self._obs))
    actions = property(lambda self: self._episodes(self._act if self._a >= 1 else self._act[:, 0]))
    rewards = property(lambda self: [[float(x) for x in ep] for ep in self._episodes(self._rew)])
    dones = property(lambda self: [[bool(x) for x in ep] for ep in self._episodes(self._done)])
    last_observations = property(lambda self: list(self._last))
