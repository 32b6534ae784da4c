import ctypes as C
from typing import Dict, List, Optional

import numpy as np

from .experience import Experience


class ReplayBuffer:
    """FIFO transition store with the reference's interface (ref: replay_buffer.py:9-74): ``add_experience`` appends
    the flattened transitions and drops the oldest beyond ``buffer_size``; ``sample_minibatch`` draws indices with
    ``np.random.randint`` (global numpy RNG, with replacement) -- the same random stream and the same logical order
    (index 0 = oldest kept transition) as the reference.

    Storage (SURVEY.md section 8f-4) is a structure-of-arrays ring: one contiguous float32 array per column, allocated
    on the first ``add_experience`` and grown geometrically up to ``buffer_size`` rows, so appending is a slice copy
    and a minibatch is ONE fancy-index gather per column instead of the reference's per-transition Python-list walk
    (1.2 ms per 256-sample minibatch there, SURVEY a20).  ``sample_indices`` + ``gather`` expose the two halves so the
    off-policy trainer can draw all S minibatches of a ``train`` call at once.  The reference's list attributes
    (``observations`` ...) remain available as read-only views in logical order.

    Beside the five columns the buffer keeps one flag per row for n-step returns: ``episode_ends[i]`` is true when row i
    was the last row of an episode in the experience that appended it -- the episode boundaries of a ``PackedExperience``
    (``ep_offsets``) or of a nested-list ``Experience`` (its episode lengths; a segment a sampler cut off at the end of a
    ``sample()`` call is an episode there), and only the last row for any other object with ``transition_columns()``.
    Every append ends on a marked row, so the newest live row is always marked: a window of consecutive rows that stops
    at the first marked or done row never reads past the ring's head, nor a row a ring overwrite replaced."""

    COLUMNS = ("observations", "actions", "rewards", "next_observations", "dones")

    def __init__(self, buffer_size: int = int(1e6)) -> None:
        self.buffer_size = int(buffer_size)
        self.current_size: int = 0
        self._head: int = 0           # physical row of logical index 0
        self._capacity: int = 0       # allocated rows (<= buffer_size)
        self._cols: Dict[str, Optional[np.ndarray]] = {k: None for k in self.COLUMNS}
        self._ends: Optional[np.ndarray] = None  # [capacity] bool: the row ended an episode of its append
        self._dev = None              # device mirror (torch CUDA tensors, float32), built lazily by device_columns()
        self._dev_ends = None         # device mirror of _ends (float32 0/1), built by the first device_episode_ends()
        self._dev_dirty: List = []    # physical row ranges written since the mirror was last refreshed

    @classmethod
    def from_dataset(cls, dataset, buffer_size: Optional[int] = None) -> "ReplayBuffer":
        """A buffer holding a fixed dataset with D4RL's keys: ``observations`` [n, O], ``actions`` [n, A], ``rewards``
        [n], ``next_observations`` [n, O], ``terminals`` [n] and optionally ``timeouts`` [n].  dones = terminals; a row
        ends an episode (for n-step windows) when it is terminal, timed out or the last row.  ``buffer_size`` defaults to
        the dataset's length and may not be smaller: an offline learner cannot afford to drop rows silently."""
        keys = ("observations", "actions", "rewards", "next_observations", "terminals")
        missing = [k for k in keys if k not in dataset]
        if missing:
            raise ValueError(f"from_dataset: the dataset lacks {missing}")
        cols = {k: np.asarray(dataset[k]) for k in keys}
        if "timeouts" in dataset and dataset["timeouts"] is not None:
            cols["timeouts"] = np.asarray(dataset["timeouts"])
        n = len(cols["observations"])
        if n == 0:
            raise ValueError("from_dataset: the dataset has no rows")
        lengths = {k: len(v) for k, v in cols.items()}
        if any(m != n for m in lengths.values()):
            raise ValueError(f"from_dataset: the columns differ in length: {lengths}")
        for k in ("observations", "actions", "rewards", "next_observations"):
            if not np.all(np.isfinite(cols[k].astype(np.float64))):
                raise ValueError(f"from_dataset: {k} holds non-finite values")
        size = n if buffer_size is None else int(buffer_size)
        if size < n:
            raise ValueError(f"from_dataset: buffer_size {size} is smaller than the dataset's {n} rows")
        rb = cls(size)
        terminals = cols["terminals"].astype(np.bool_).reshape(n)
        new = (cols["observations"], cols["actions"], cols["rewards"].reshape(n), cols["next_observations"], terminals)
        rb._allocate(n, new)
        if rb._capacity < n:  # _allocate starts at 1024 rows at least, buffer_size rows at most
            rb._grow(n)
        for k, v in zip(cls.COLUMNS, new):
            col = rb._cols[k]
            col[:n] = np.asarray(v, dtype=col.dtype).reshape((n,) + col.shape[1:])
        ends = terminals.copy()
        if "timeouts" in cols:
            ends |= cols["timeouts"].astype(np.bool_).reshape(n)
        ends[-1] = True
        rb._ends[:n] = ends
        rb.current_size = n
        return rb

    # ---- storage ----
    def _allocate(self, rows: int, samples) -> None:
        rows = min(max(rows, 1024), self.buffer_size)
        for k, v in zip(self.COLUMNS, samples):
            first = np.asarray(v[0])
            # rewards stay float64 and dones bool, like the values the reference's lists hold
            dt = np.float64 if k == "rewards" else (np.bool_ if k == "dones" else np.float32)
            self._cols[k] = np.empty((rows,) + first.shape, dtype=dt)
        self._ends = np.zeros(rows, dtype=np.bool_)
        self._capacity = rows

    def _grow(self, need: int) -> None:
        new_cap = self._capacity
        while new_cap < need:
            new_cap *= 2
        new_cap = min(new_cap, self.buffer_size)
        order = self._physical(np.arange(self.current_size))
        for k in self.COLUMNS:
            old = self._cols[k]
            new = np.empty((new_cap,) + old.shape[1:], dtype=old.dtype)
            new[:self.current_size] = old[order]
            self._cols[k] = new
        ends = np.zeros(new_cap, dtype=np.bool_)
        ends[:self.current_size] = self._ends[order]
        self._ends = ends
        self._head, self._capacity = 0, new_cap
        self._dev = self._dev_ends = None  # reallocated: the mirrors are rebuilt on their next request

    def _physical(self, logical: np.ndarray) -> np.ndarray:
        return (self._head + logical) % self._capacity if self._capacity else logical

    def add_experience(self, experience: Experience) -> None:
        if hasattr(experience, "transition_columns"):  # PackedExperience: contiguous columns, no per-row Python objects
            new = experience.transition_columns()
        else:
            new = (experience.flattened_observations, experience.flattened_actions, experience.flattened_rewards,
                   experience.flattened_next_observations, experience.flattened_dones)
        n = len(new[0])
        if n == 0:
            return
        ends = self._episode_ends_of(experience, n)
        if self._capacity == 0:
            self._allocate(n, new)
        if n >= self.buffer_size:  # only the newest buffer_size transitions survive (front deletion in the reference)
            new = tuple(v[n - self.buffer_size:] for v in new)
            ends = ends[n - self.buffer_size:]
            n = self.buffer_size
        total = self.current_size + n
        if min(total, self.buffer_size) > self._capacity:
            self._grow(min(total, self.buffer_size))
        overflow = max(0, total - self.buffer_size)  # oldest rows dropped
        self._head = (self._head + overflow) % self._capacity
        self.current_size -= overflow
        start = (self._head + self.current_size) % self._capacity
        first = min(n, self._capacity - start)
        for k, v in zip(self.COLUMNS, new):
            col = self._cols[k]
            arr = np.asarray(v, dtype=col.dtype).reshape((n,) + col.shape[1:])
            col[start:start + first] = arr[:first]
            if first < n:
                col[:n - first] = arr[first:]
        self._ends[start:start + first] = ends[:first]
        if first < n:
            self._ends[:n - first] = ends[first:]
        self.current_size += n
        if self._dev is not None:  # no mirror yet: its first build uploads everything anyway
            self._dev_dirty.append((start, first))
            if first < n:
                self._dev_dirty.append((0, n - first))
            if len(self._dev_dirty) > 256:  # many small appends between two train() calls: one full refresh is cheaper
                self._dev_dirty = self._live_ranges()

    @staticmethod
    def _episode_ends_of(experience, n: int) -> np.ndarray:
        """[n] bool: the rows of this append that end an episode (see the class docstring); the last is always set."""
        ends = np.zeros(n, dtype=np.bool_)
        offsets = getattr(experience, "ep_offsets", None)
        if offsets is not None:  # PackedExperience
            ends[np.asarray(offsets, np.int64)[1:] - 1] = True
        elif not hasattr(experience, "transition_columns"):  # nested lists: one list per episode
            ends[np.cumsum([len(ep) for ep in experience.rewards]) - 1] = True
        ends[-1] = True
        return ends

    @property
    def episode_ends(self) -> List:
        """The episode-end flags in logical order (a read-only view, like ``dones``)."""
        if self._ends is None:
            return []
        return [bool(x) for x in self._ends[self._physical(np.arange(self.current_size))]]

    def _live_ranges(self) -> List:
        first = min(self.current_size, self._capacity - self._head)  # the rows that hold data, wrap-around aware
        return [(self._head, first)] + ([(0, self.current_size - first)] if first < self.current_size else [])

    # ---- device mirror (SURVEY 8f-4): the columns as float32 CUDA tensors, refreshed incrementally ----
    def physical_rows(self, logical: np.ndarray) -> np.ndarray:
        return self._physical(np.asarray(logical)).astype(np.int64)

    def ring(self):
        """(physical row of logical index 0, live rows, allocated rows): what a device-side index draw needs."""
        return self._head, self.current_size, self._capacity

    def device_columns(self):
        """(obs, act, rew, next_obs, done) float32 CUDA tensors with ``capacity`` rows each, in PHYSICAL row order
        (use ``physical_rows`` on the logical indices).  rewards float64 -> float32 and dones bool -> 0/1 are the casts
        the reference applies to every minibatch (td3.py:226-228).  Only rows written since the last call are uploaded."""
        import torch
        if self._capacity == 0:
            raise ValueError("device_columns: the buffer is empty")
        if self._dev is None:
            self._dev = tuple(torch.zeros(self._cols[k].shape, dtype=torch.float32, device="cuda") for k in self.COLUMNS)
            self._dev_dirty = self._live_ranges()
        for start, count in self._dev_dirty:
            for k, d in zip(self.COLUMNS, self._dev):
                host = np.ascontiguousarray(self._cols[k][start:start + count], dtype=np.float32)
                d[start:start + count].copy_(torch.from_numpy(host))
            if self._dev_ends is not None:
                self._dev_ends[start:start + count].copy_(torch.from_numpy(self._ends[start:start + count].astype(np.float32)))
        self._dev_dirty = []
        return self._dev, self._capacity

    def device_episode_ends(self):
        """The episode-end flags as a float32 0/1 CUDA tensor with ``capacity`` rows in physical row order, beside
        ``device_columns()`` (what n-step returns walk).  Built on the first request, then refreshed from the same
        written row ranges as the columns."""
        import torch
        if self._capacity == 0:
            raise ValueError("device_episode_ends: the buffer is empty")
        if self._dev_ends is None:
            self._dev_ends = torch.from_numpy(self._ends.astype(np.float32)).to("cuda")
        self.device_columns()
        return self._dev_ends

    # ---- sampling ----
    def sample_indices(self, minibatch_size: int) -> np.ndarray:
        """The reference's draw (replay_buffer.py:58): logical indices, with replacement, global numpy RNG."""
        return np.random.randint(0, self.current_size, minibatch_size)

    def gather(self, indices: np.ndarray) -> Dict[str, np.ndarray]:
        """Rows at logical ``indices`` (any shape); the result has the shapes / dtypes ``sample_minibatch`` returns."""
        phys = self._physical(np.asarray(indices))
        return {k: self._cols[k][phys] for k in self.COLUMNS}

    def sample_minibatch(self, minibatch_size: int = 32) -> Dict[str, np.ndarray]:
        return self.gather(self.sample_indices(minibatch_size))

    # ---- reference-compatible read-only views (logical order) ----
    def _view(self, k: str) -> List:
        if self._cols[k] is None:
            return []
        return list(self._cols[k][self._physical(np.arange(self.current_size))])

    observations = property(lambda self: self._view("observations"))
    actions = property(lambda self: self._view("actions"))
    rewards = property(lambda self: [float(x) for x in self._view("rewards")])
    next_observations = property(lambda self: self._view("next_observations"))
    dones = property(lambda self: [bool(x) for x in self._view("dones")])


class PrioritizedReplayBuffer(ReplayBuffer):
    """A ``ReplayBuffer`` with one priority per physical row for prioritized experience replay (Schaul et al. 2016,
    proportional variant), used by ``DQN.train``: each train step draws its minibatch in proportion to the priorities,
    weighs the rows by (min_k p_k / p_j)^beta and writes (|TD error| + ``eps``)^``alpha`` back for the rows it drew, all on
    the device (b200rl.h, "Prioritized experience replay").  beta rises linearly from ``beta_start`` to 1 over
    ``beta_anneal_steps`` Q optimizer steps.

    The priorities live in a sum tree on the device (a torch CUDA tensor owned here).  Rows that are not live have
    priority 0; rows written by ``add_experience`` (ring overwrites included) get the running max of all priorities so
    far (1 at the start) when the device mirror is next refreshed.  The columns are allocated at ``buffer_size`` rows on
    the first append, so rows never move.  There is no host-side draw: ``sample_indices`` and ``sample_minibatch``
    refuse rather than sample uniformly.  Priorities are not part of checkpoints."""

    def __init__(self, buffer_size: int = int(1e6), alpha: float = 0.6, beta_start: float = 0.4,
                 beta_anneal_steps: int = 100_000, eps: float = 1e-6) -> None:
        super().__init__(buffer_size)
        if not alpha >= 0.0:
            raise ValueError(f"alpha must be >= 0, got {alpha}")
        if not 0.0 <= beta_start <= 1.0:
            raise ValueError(f"beta_start must be in [0, 1], got {beta_start}")
        if int(beta_anneal_steps) < 1:
            raise ValueError(f"beta_anneal_steps must be >= 1, got {beta_anneal_steps}")
        if not eps > 0.0:
            raise ValueError(f"eps must be > 0, got {eps}")
        if self.buffer_size >= 2 ** 31:
            raise ValueError(f"buffer_size must be below 2^31, got {self.buffer_size}")
        self.alpha, self.beta_start, self.beta_anneal_steps, self.eps = float(alpha), float(beta_start), \
            int(beta_anneal_steps), float(eps)
        self._tree = None             # the sum tree (built with the device mirror)
        self._prio_dirty: List = []   # physical row ranges appended since the tree was last refreshed

    def per_settings(self):
        """(alpha, eps, beta_start, beta_anneal_steps): what the engine's b200rl_per_hparams take."""
        return self.alpha, self.eps, self.beta_start, self.beta_anneal_steps

    def beta(self, t: int) -> float:
        """beta of a train step taken at Q optimizer step count ``t`` (the count before the step)."""
        return min(1.0, self.beta_start + (1.0 - self.beta_start) * t / self.beta_anneal_steps)

    def _allocate(self, rows: int, samples) -> None:
        super()._allocate(self.buffer_size, samples)  # full size at once: rows keep their place, and so their priority

    def add_experience(self, experience: Experience) -> None:
        if hasattr(experience, "transition_columns"):
            n = len(experience.transition_columns()[0])
        else:
            n = len(experience.flattened_rewards)
        super().add_experience(experience)
        n = min(n, self.buffer_size)
        if n == 0 or self._tree is None:  # no tree yet: its first build gives every live row the initial max
            return
        start = (self._head + self.current_size - n) % self._capacity
        if self._prio_dirty:  # consecutive appends continue the previous range
            s0, c0 = self._prio_dirty[-1]
            if (s0 + c0) % self._capacity == start:
                self._prio_dirty[-1] = (s0, min(c0 + n, self._capacity))
                return
        self._prio_dirty.append((start, n))

    def device_columns(self):
        from . import _lib
        from .engine import current_stream_handle
        import torch
        cols, rows = super().device_columns()
        lib = _lib.load()
        if self._tree is None:
            n = int(lib.b200rl_per_tree_floats(rows))
            self._tree = torch.zeros(n, dtype=torch.float32, device="cuda")
            self._tree[n - 31] = 1.0  # the running max m (b200rl.h: the last level is [root, m, 0 ...])
            self._prio_dirty = self._live_ranges()
        stream = current_stream_handle()
        for start, count in self._prio_dirty:
            _lib.check(lib.b200rl_per_tree_set_range(C.c_void_p(self._tree.data_ptr()), rows, start, count, stream),
                       "per_tree_set_range")
        self._prio_dirty = []
        return cols, rows

    def device_tree(self):
        """The sum tree (CUDA float32 tensor, b200rl.h layout) with every append so far given its priority."""
        self.device_columns()
        return self._tree

    def priorities(self) -> np.ndarray:
        """The leaves: one priority per physical row (``capacity`` rows), as float32 on the host."""
        return self.device_tree()[:self._capacity].cpu().numpy()

    def max_priority(self) -> float:
        """The running max m that new rows receive."""
        t = self.device_tree()
        return float(t[t.numel() - 31])

    def sample_indices(self, minibatch_size: int) -> np.ndarray:
        raise NotImplementedError("PrioritizedReplayBuffer draws its minibatches on the device, in proportion to the "
                                  "priorities, inside DQN.train; it has no uniform host-side draw")
