"""Python handle of the native on-policy update engine (C ABI: include/b200rl.h).

PyTorch is used for plumbing only: picking the CUDA device / current stream, exposing engine-owned device memory
as tensors (``view``) and torch.distributed collectives for data-parallel runs.  All arithmetic of the update path
runs in libb200rl.so's CUDA kernels; there is no fallback.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional, Sequence

import numpy as np

from . import _lib
from ._lib import DIST, MlpDesc, OnPolicyConfig, PpoHparams, TrpoHparams, TrpoStats, UpdateStats, check

POLICY, OLD_POLICY, VALUE = 0, 1, 2
_OPENED_IPC: Dict[bytes, int] = {}  # CUDA IPC handle -> device pointer of the mapping in this process


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else C.c_void_p(a.ctypes.data)


def _c(a, dtype) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=dtype)


class _CudaArray:
    """Minimal __cuda_array_interface__ carrier so torch can wrap engine-owned device memory without copying."""

    def __init__(self, ptr: int, count: int, typestr: str):
        self.__cuda_array_interface__ = {"shape": (count,), "typestr": typestr, "data": (ptr, False), "version": 3}


def current_stream_handle() -> int:
    import torch
    if not torch.cuda.is_available():
        raise _lib.B200RLError("no CUDA device: the update engine has no CPU fallback")
    return int(torch.cuda.current_stream().cuda_stream)


class OnPolicyEngine:
    """Device-resident state of one PPO / VPG / TRPO learner."""

    def __init__(self, policy_sizes: Sequence[int], value_sizes: Sequence[int], dist: str, max_rows: int,
                 max_episodes: int, hidden_act: str = "tanh", rewards_f64: bool = True, train_log_std: bool = False):
        self.lib = _lib.load()
        current_stream_handle()  # fail early and loudly without a GPU
        cfg = OnPolicyConfig()
        cfg.policy = MlpDesc.make(policy_sizes, hidden_act, "identity")
        cfg.value = MlpDesc.make(value_sizes, hidden_act, "identity")
        cfg.dist = DIST[dist]
        cfg.rewards_f64 = int(rewards_f64)
        cfg.max_rows, cfg.max_episodes = int(max_rows), int(max_episodes)
        self.cfg = cfg
        self.dist = dist
        self.policy_sizes, self.value_sizes = list(policy_sizes), list(value_sizes)
        self.rewards_f64 = rewards_f64
        self.n_policy = int(self.lib.b200rl_mlp_param_count(cfg.policy))
        self.n_value = int(self.lib.b200rl_mlp_param_count(cfg.value))
        self.max_rows, self.max_episodes = int(max_rows), int(max_episodes)
        h = C.c_void_p()
        check(self.lib.b200rl_onpolicy_create(C.byref(cfg), C.byref(h)), "onpolicy_create")
        self.h = h
        self.train_log_std = bool(train_log_std)
        if self.train_log_std:  # the policy vector becomes [network parameters | log_std]
            check(self.lib.b200rl_onpolicy_set_train_log_std(h, 1), "set_train_log_std")
            self.n_policy += int(policy_sizes[-1])
        self.n_rows = 0
        self.n_episodes = 0
        self._allreduce_cb = None
        self._keep = []
        self.peer_exchange = False

    def close(self):
        if getattr(self, "h", None):
            self.lib.b200rl_onpolicy_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- parameters / optimiser state -------------------------------------------------------------------------
    def _n(self, which):
        return self.n_value if which == VALUE else self.n_policy

    def set_params(self, which: int, flat: np.ndarray):
        a = _c(flat, np.float32)
        self._keep.append(a)
        check(self.lib.b200rl_onpolicy_set_params(self.h, which, _ptr(a), a.size, current_stream_handle()), "set_params")

    def get_params(self, which: int) -> np.ndarray:
        out = np.empty(self._n(which), dtype=np.float32)
        check(self.lib.b200rl_onpolicy_get_params(self.h, which, _ptr(out), out.size, current_stream_handle()), "get_params")
        return out

    def set_adam(self, which: int, exp_avg: Optional[np.ndarray], exp_avg_sq: Optional[np.ndarray], step: int):
        m = None if exp_avg is None else _c(exp_avg, np.float32)
        v = None if exp_avg_sq is None else _c(exp_avg_sq, np.float32)
        self._keep += [m, v]
        check(self.lib.b200rl_onpolicy_set_adam(self.h, which, _ptr(m), _ptr(v), self._n(which), int(step),
                                                current_stream_handle()), "set_adam")

    def get_adam(self, which: int):
        m = np.empty(self._n(which), dtype=np.float32)
        v = np.empty(self._n(which), dtype=np.float32)
        step = C.c_int64()
        check(self.lib.b200rl_onpolicy_get_adam(self.h, which, _ptr(m), _ptr(v), m.size, C.byref(step),
                                                current_stream_handle()), "get_adam")
        return m, v, int(step.value)

    def set_log_std(self, log_std: np.ndarray):
        a = _c(log_std, np.float32)
        self._keep.append(a)
        check(self.lib.b200rl_onpolicy_set_log_std(self.h, _ptr(a), a.size, current_stream_handle()), "set_log_std")

    # ---- batch ----------------------------------------------------------------------------------------------
    def load_batch(self, batch: Dict[str, np.ndarray]):
        """Copy a packed HOST batch (see synthetic.py for the layout) to the device."""
        obs = _c(batch["obs"], np.float32)
        act = _c(batch["act"], np.float32)
        rew = _c(batch["rew"], np.float64 if self.rewards_f64 else np.float32)
        last = _c(batch["last_obs"], np.float32)
        off = _c(batch["ep_offsets"], np.int64)
        done = _c(batch["ep_done"], np.uint8)
        n, e = obs.shape[0], done.shape[0]
        if obs.ndim != 2 or obs.shape[1] != self.policy_sizes[0]:
            raise ValueError(f"observations must be [N,{self.policy_sizes[0]}], got {obs.shape}")
        want_act = (n, self.policy_sizes[-1]) if self.dist == "gaussian" else (n,)
        if act.shape != want_act:
            raise ValueError(f"actions must have shape {want_act}, got {act.shape}")
        if rew.shape != (n,) or last.shape != (e, obs.shape[1]) or off.shape != (e + 1,):
            raise ValueError("inconsistent packed batch shapes")
        self._keep += [obs, act, rew, last, off, done]  # keep host buffers alive until the stream has consumed them
        check(self.lib.b200rl_onpolicy_load_batch(self.h, _ptr(obs), _ptr(act), _ptr(rew), _ptr(last), _ptr(off),
                                                  _ptr(done), n, e, 0, current_stream_handle()), "load_batch")
        self.n_rows, self.n_episodes = n, e

    def load_batch_device(self, obs, act, rew, last_obs, ep_offsets, ep_done):
        """Same from torch CUDA tensors already resident in HBM (device-to-device copies)."""
        n, e = obs.shape[0], ep_done.shape[0]
        ts = [obs, act, rew, last_obs, ep_offsets, ep_done]
        assert all(t.is_cuda and t.is_contiguous() for t in ts)
        check(self.lib.b200rl_onpolicy_load_batch(self.h, *[C.c_void_p(t.data_ptr()) for t in ts], n, e, 1,
                                                  current_stream_handle()), "load_batch(device)")
        self.n_rows, self.n_episodes = n, e

    # ---- update ---------------------------------------------------------------------------------------------
    @staticmethod
    def hparams(gamma=0.99, gae_lambda=0.97, clip_range=0.2, max_kl_divergence=0.01, num_policy_gradients=80,
                num_value_gradients=80, policy_adam=(3e-4, 0.9, 0.999, 1e-8), value_adam=(1e-3, 0.9, 0.999, 1e-8),
                n_global_rows=0) -> PpoHparams:
        hp = PpoHparams()
        hp.gamma, hp.gae_lambda, hp.clip_range, hp.max_kl_divergence = gamma, gae_lambda, clip_range, max_kl_divergence
        hp.num_policy_gradients, hp.num_value_gradients = int(num_policy_gradients), int(num_value_gradients)
        hp.policy_lr, hp.policy_beta1, hp.policy_beta2, hp.policy_eps = policy_adam
        hp.value_lr, hp.value_beta1, hp.value_beta2, hp.value_eps = value_adam
        hp.n_global_rows = int(n_global_rows)
        return hp

    def _make_allreduce(self, process_group):
        import torch
        import torch.distributed as dist

        def cb(user, buf, count, dtype, stream):
            try:
                t = torch.as_tensor(_CudaArray(buf, count, "<f8" if dtype == 1 else "<f4"), device="cuda")
                dist.all_reduce(t, op=dist.ReduceOp.SUM, group=process_group)
                return 0
            except Exception as exc:  # surfaced by the engine as a failed update
                import traceback
                traceback.print_exc()
                return 1

        return _lib.ALLREDUCE_FN(cb)

    def _make_allreduce_from(self, fn):
        import torch

        def cb(user, buf, count, dtype, stream):
            try:
                fn(torch.as_tensor(_CudaArray(buf, count, "<f8" if dtype == 1 else "<f4"), device="cuda"))
                return 0
            except Exception:
                import traceback
                traceback.print_exc()
                return 1

        return _lib.ALLREDUCE_FN(cb)

    # ---- one-shot gradient exchange over peer-mapped memory (one node, NVLink) ---------------------------------
    def comm_export(self):
        """(64-byte CUDA IPC handle, local device pointer) of this engine's exchange buffer."""
        handle = (C.c_uint8 * 64)()
        ptr = C.c_void_p()
        check(self.lib.b200rl_onpolicy_comm_export(self.h, handle, C.byref(ptr)), "comm_export")
        return bytes(handle), int(ptr.value)

    def comm_attach(self, rank: int, peer_ptrs: Sequence[int]):
        arr = (C.c_void_p * len(peer_ptrs))(*peer_ptrs)
        check(self.lib.b200rl_onpolicy_comm_attach(self.h, int(rank), len(peer_ptrs), arr), "comm_attach")
        self.peer_exchange = True

    def enable_peer_exchange(self, process_group=None) -> bool:
        """Exchange IPC handles over torch.distributed and map every rank's buffer (all ranks on ONE node).  Returns
        False (and leaves the NCCL all-reduce in place) when the ranks cannot map each other's memory."""
        import torch
        import torch.distributed as dist
        rank, world = dist.get_rank(process_group), dist.get_world_size(process_group)
        if world < 2 or world > 16:
            return False
        ok = 1
        try:
            handle, mine = self.comm_export()
        except _lib.B200RLError:
            handle, mine, ok = b"", 0, 0
        gathered = [None] * world
        dist.all_gather_object(gathered, (handle, ok), group=process_group)
        ptrs = []
        if all(g[1] for g in gathered):
            # mappings of buffers that no longer exist on their rank (its engine was replaced) go first: a new
            # allocation may land where the old one was, and that cannot be mapped twice
            live = {hd for r, (hd, _) in enumerate(gathered) if r != rank}
            for hd in [h_ for h_ in _OPENED_IPC if h_ not in live]:
                self.lib.b200rl_ipc_close(C.c_void_p(_OPENED_IPC.pop(hd)))
            for r, (hd, _) in enumerate(gathered):
                if r == rank:
                    ptrs.append(mine)
                    continue
                if hd not in _OPENED_IPC:  # a handle can be mapped once per process: keep the mapping
                    p = C.c_void_p()
                    buf = (C.c_uint8 * 64).from_buffer_copy(hd)
                    if self.lib.b200rl_ipc_open(buf, C.byref(p)) != 0:
                        ok = 0
                        break
                    _OPENED_IPC[hd] = int(p.value)
                ptrs.append(_OPENED_IPC[hd])
        else:
            ok = 0
        t = torch.tensor([ok], dtype=torch.int32, device="cuda")
        dist.all_reduce(t, op=dist.ReduceOp.MIN, group=process_group)  # all or nobody
        if int(t.item()) != 1:
            return False
        self.comm_attach(rank, ptrs)
        return True

    def update(self, hp: PpoHparams, algo: str = "ppo", process_group=None, distributed: bool = False,
               allreduce=None) -> UpdateStats:
        """``distributed``: all-reduce through torch.distributed on ``process_group`` (NCCL).  ``allreduce``: a callable
        ``fn(tensor)`` that sums the given CUDA tensor over the data-parallel group in place, for transports other than
        torch.distributed (and for tests)."""
        stats = UpdateStats()
        cb = None
        if allreduce is not None:
            self._allreduce_cb = self._make_allreduce_from(allreduce)
            cb = C.cast(self._allreduce_cb, C.c_void_p)
        elif distributed:
            self._allreduce_cb = self._make_allreduce(process_group)
            cb = C.cast(self._allreduce_cb, C.c_void_p)
        fn = {"ppo": self.lib.b200rl_ppo_update, "vpg": self.lib.b200rl_vpg_update}[algo]
        check(fn(self.h, C.byref(hp), cb, None, C.byref(stats), current_stream_handle()), f"{algo}_update")
        self._keep.clear()  # the update synchronised the stream: staged host buffers are no longer in flight
        return stats

    def trpo_update(self, hp: PpoHparams, max_constraint=0.01, n_conjugate_gradients=10, max_backtracks=15,
                    backtrack_ratio=0.8, hvp_damping_coefficient=1e-5, process_group=None, distributed: bool = False,
                    allreduce=None):
        """The reference's TRPO.train on the loaded batch; returns (UpdateStats, TrpoStats).  ``distributed`` /
        ``allreduce`` as in ``update``: every rank holds a block of episodes, ``hp.n_global_rows`` the global row count,
        and every batch-derived sum of the step is all-reduced (b200rl_trpo_update_dp)."""
        cg = TrpoHparams()
        cg.max_constraint, cg.n_conjugate_gradients = float(max_constraint), int(n_conjugate_gradients)
        cg.max_backtracks, cg.backtrack_ratio = int(max_backtracks), float(backtrack_ratio)
        cg.hvp_damping_coefficient = float(hvp_damping_coefficient)
        stats, ts = UpdateStats(), TrpoStats()
        cb = None
        if allreduce is not None:
            self._allreduce_cb = self._make_allreduce_from(allreduce)
            cb = C.cast(self._allreduce_cb, C.c_void_p)
        elif distributed:
            self._allreduce_cb = self._make_allreduce(process_group)
            cb = C.cast(self._allreduce_cb, C.c_void_p)
        check(self.lib.b200rl_trpo_update_dp(self.h, C.byref(hp), C.byref(cg), cb, None, C.byref(stats), C.byref(ts),
                                             current_stream_handle()), "trpo_update")
        self._keep.clear()
        return stats, ts

    def fvp(self, v: np.ndarray, damping: float = 1e-5) -> np.ndarray:
        """(F + damping I) v at the current policy parameters on the loaded batch (one fused FVP launch)."""
        v = _c(v, np.float32)
        out = np.empty_like(v)
        check(self.lib.b200rl_onpolicy_fvp(self.h, _ptr(v), _ptr(out), v.size, float(damping), current_stream_handle()),
              "fvp")
        return out

    def scalar_history(self) -> np.ndarray:
        """[slots, 8] float64 scalar sums of the last update (see b200rl_onpolicy_scalar_history)."""
        n = C.c_int32()
        probe = np.zeros((1, _lib.N_SCALARS))
        check(self.lib.b200rl_onpolicy_scalar_history(self.h, _ptr(probe), 0, C.byref(n)), "scalar_history")
        out = np.zeros((max(int(n.value), 1), _lib.N_SCALARS))
        check(self.lib.b200rl_onpolicy_scalar_history(self.h, _ptr(out), int(n.value), C.byref(n)), "scalar_history")
        return out[:int(n.value)]

    def run_stage(self, stage: str, hp: PpoHparams):
        check(self.lib.b200rl_onpolicy_run_stage(self.h, stage.encode(), C.byref(hp), current_stream_handle()),
              f"run_stage({stage})")

    def view(self, name: str):
        """Engine-owned device buffer as a torch tensor (zero copy)."""
        import torch
        p, n, d = C.c_void_p(), C.c_int64(), C.c_int32()
        check(self.lib.b200rl_onpolicy_device_view(self.h, name.encode(), C.byref(p), C.byref(n), C.byref(d)), "device_view")
        return torch.as_tensor(_CudaArray(p.value, int(n.value), "<f8" if d.value == 1 else "<f4"), device="cuda")


class OffPolicyEngine:
    """Device-resident state of one DDPG / TD3 (``algo`` 0), SAC (``algo`` 1), DQN (``algo`` 2) or C51 (``algo`` 3)
    learner (C ABI: b200rl_offpolicy_*).  SAC: ``n_q`` = 2, the policy maps obs -> [mean | log_std] (2A outputs), there
    is no target policy (network 3), and ``set_sac`` must be called before the first train call.  DQN: ``policy_sizes``
    = None, ``n_q`` = 1, the Q network maps obs -> [n actions], only networks 1 (Q) and 4 (target Q) exist, actions are
    indices (act [S,B]), and ``set_dqn`` must be called before the first train call.  C51 is a DQN engine whose Q
    network maps obs -> [n actions x n atoms] logits; it needs ``set_c51`` as well as ``set_dqn``.  QR-DQN is a DQN
    engine after ``set_qr``: its Q network maps obs -> [n actions x n quantiles] quantile locations.  ``dueling_k`` = K
    >= 1 (DQN / QR-DQN / C51): the Q network is a dueling one, ``q_sizes`` = [obs, h_trunk, h_stream, n actions x K]
    (b200rl.h, "Dueling Q networks").  ``noisy_layers`` (DQN / QR-DQN / C51): bit mask of the Q network's noisy Linear
    layers in flat order; every train call then needs ``set_noise_keys`` first (b200rl.h, "Noisy networks").  IQN
    (``algo`` 4) is a DQN engine over an implicit quantile network: ``q_sizes`` = [obs, d, h, n actions] and ``iqn`` =
    (n_cos, N, N', K); every train call needs ``set_noise_keys`` first, the keys of its fraction draws (b200rl.h, "IQN").
    Discrete SAC (``algo`` 5) has SAC's networks, temperature and outputs over a discrete action space: the policy maps
    obs -> [n] logits, both critics obs -> [n] values, actions are indices (act [S,B]) as for DQN, no noise is used,
    and ``set_sac`` must be called before the first train call (b200rl.h, "Discrete SAC").  D4PG (``algo`` 6) has
    DDPG's networks with a categorical critic: ``q_sizes`` = [obs + act, ..., N] and ``d4pg`` = (N, v_min, v_max), the
    critic's support; it takes ``set_per`` / ``train_prioritized`` and ``set_nstep`` as DQN does (b200rl.h, "D4PG").
    TQC (``algo`` 7) is a SAC engine whose critics map [s | a] to M quantiles: ``q_sizes`` = [obs + act, ..., M] and
    ``tqc`` = (M, d), d the atoms per critic dropped from the pooled target (b200rl.h, "TQC").  CQL (``algo`` 8) is a SAC
    engine whose critic step also runs on 3N sampled actions per row: ``cql`` = (N, lagrange); ``set_cql`` is required,
    and a call with host draws takes ``noise`` = (SAC's [S, 2, B, A], CQL's [S, 3, B, N, A]) (b200rl.h, "CQL").  IQL
    (``algo`` 9) has SAC's policy and critics and a trained value network in slot 3: ``iql`` = (sizes, (hidden, out
    activation)) of V; ``set_iql`` is required, no noise is used, and the state has four optimizers (b200rl.h, "IQL").
    REDQ (``algo`` 10) has SAC's policy, temperature and noise over N critics: ``redq`` = (N, M), M the target critics
    drawn per step; networks 1..N are the critics and N+1..2N their targets, the state has 1 + N optimizers, and a call
    with host draws takes ``noise`` = (SAC's [S, 2, B, A], subsets [S, M]) (b200rl.h, "REDQ").  EDAC (``algo`` 11)
    has REDQ's layout with every target critic in the target, a policy step every step on the min over the critics, and
    a diversity penalty of weight eta on the critics' action gradients: ``edac`` = (N, eta), eta = 0 being SAC-N; a call
    takes SAC's noise alone, and ``edac_outputs`` returns the penalty D per step (b200rl.h, "EDAC").

    ``n_learners`` = K > 1: a group of K independent learners with the same shapes and hyper-parameters, every step one
    launch for all K (b200rl_offpolicy_create_group).  Inputs and outputs then carry a leading [K] axis, the state blob
    is [K][per-learner blob] with [K][n_opt] step counts (n_opt = 3, 4 for IQL), and the per-network accessors are
    refused."""

    NETS = {"policy": 0, "q1": 1, "q2": 2, "target_policy": 3, "target_q1": 4, "target_q2": 5}
    TD3, SAC, DQN, C51, IQN, DSAC, D4PG, TQC, CQL, IQL, REDQ, EDAC = 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11
    DISCRETE = (DQN, C51, IQN)  # the algos with DQN's networks, inputs and outputs
    INDEX_ACTIONS = DISCRETE + (DSAC,)  # the algos whose action column holds an action index
    SOFT = (SAC, DSAC, TQC, CQL, REDQ, EDAC)  # the algos with SAC's temperature and outputs
    SQUASHED = (SAC, TQC, CQL, REDQ, EDAC)  # the algos with SAC's squashed-Gaussian policy and its [S, 2, B, A] noise

    def __init__(self, policy_sizes, q_sizes, n_q: int, max_minibatch: int, max_steps: int, policy_acts=("relu", "tanh"),
                 q_acts=("relu", "identity"), algo: int = 0, n_learners: int = 1, dueling_k: int = 0,
                 noisy_layers: int = 0, iqn=None, d4pg=None, tqc=None, cql=None, iql=None, redq=None, edac=None):
        from ._lib import OffPolicyConfig
        self.lib = _lib.load()
        current_stream_handle()
        cfg = OffPolicyConfig()
        if policy_sizes is not None:  # DQN: no policy, the description stays zeroed
            cfg.policy = MlpDesc.make(policy_sizes, *policy_acts)
        cfg.q = MlpDesc.make(q_sizes, *q_acts)
        cfg.n_q, cfg.max_minibatch, cfg.max_steps = int(n_q), int(max_minibatch), int(max_steps)
        cfg.algo, cfg.dueling_k, cfg.noisy_layers = int(algo), int(dueling_k), int(noisy_layers)
        self.algo, self.dueling_k, self.noisy_layers = int(algo), int(dueling_k), int(noisy_layers)
        self.iqn = None if iqn is None else tuple(int(x) for x in iqn)
        self.d4pg = None if d4pg is None else (int(d4pg[0]), float(d4pg[1]), float(d4pg[2]))
        self.tqc = None if tqc is None else (int(tqc[0]), int(tqc[1]))
        self.cql = None if cql is None else (int(cql[0]), int(bool(cql[1])))
        self.iql = None if iql is None else (tuple(int(x) for x in iql[0]), tuple(iql[1]))
        self.edac = None if edac is None else (int(edac[0]), float(edac[1]))
        # an EDAC engine has REDQ's layout and outputs with M = N
        self.redq = (self.edac[0], self.edac[0]) if self.edac is not None else None if redq is None else \
            (int(redq[0]), int(redq[1]))
        # optimizers in the state blob and the step counts
        self.n_opt = 4 if self.iql is not None else 1 + self.redq[0] if self.redq is not None else 3
        self.n_value = 0
        self.discrete = self.algo in self.DISCRETE  # DQN's networks and outputs
        self.index_actions = self.algo in self.INDEX_ACTIONS  # act [S,B] indices, no noise
        self.n_q, self.max_minibatch, self.max_steps = int(n_q), int(max_minibatch), int(max_steps)
        self.policy_sizes, self.q_sizes = None if policy_sizes is None else list(policy_sizes), list(q_sizes)
        self.policy_acts, self.q_acts = tuple(policy_acts), tuple(q_acts)
        self.n_policy = 0 if policy_sizes is None else int(self.lib.b200rl_mlp_param_count(cfg.policy))
        self.n_qp = int(self.lib.b200rl_mlp_param_count(cfg.q))
        if self.dueling_k and len(self.q_sizes) == 4:  # trunk, both streams' hidden layers, V and A (b200rl.h)
            O, h1, h2, w = self.q_sizes
            self.n_qp = h1 * (O + 1) + 2 * h2 * (h1 + 1) + (self.dueling_k + w) * (h2 + 1)
        if self.iqn is not None and len(self.q_sizes) == 4:  # psi, phi, head hidden, head out (b200rl.h, "IQN")
            O, d, hh, n = self.q_sizes
            self.n_qp = d * (O + 1) + d * (self.iqn[0] + 1) + hh * (d + 1) + n * (hh + 1)
        noisy = [(i, o) for l, (i, o) in enumerate(self.q_layers()) if self.noisy_layers >> l & 1]
        self.n_qp += sum(o * (i + 1) for i, o in noisy)  # W_sigma and b_sigma of each noisy layer
        self.noise_width = sum(i + o for i, o in noisy)  # E: draws per network and step
        self.K = int(n_learners)
        h = C.c_void_p()
        if self.iqn is not None:  # IQN's counts size its per-row buffers (b200rl.h, "IQN")
            check(self.lib.b200rl_offpolicy_create_iqn(C.byref(cfg), C.byref(_lib.IqnConfig(*self.iqn)), self.K,
                                                       C.byref(h)), "offpolicy_create_iqn")
        elif self.d4pg is not None:  # the critic's support is fixed at creation (b200rl.h, "D4PG")
            n_atoms, v_min, v_max = self.d4pg
            check(self.lib.b200rl_offpolicy_create_d4pg(C.byref(cfg), C.byref(_lib.D4pgConfig(n_atoms, 0, v_min, v_max)),
                                                        self.K, C.byref(h)), "offpolicy_create_d4pg")
        elif self.tqc is not None:  # the quantile counts size the critics' heads (b200rl.h, "TQC")
            check(self.lib.b200rl_offpolicy_create_tqc(C.byref(cfg), C.byref(_lib.TqcConfig(*self.tqc)), self.K,
                                                       C.byref(h)), "offpolicy_create_tqc")
        elif self.iql is not None:  # the value network's description (b200rl.h, "IQL")
            vdesc = MlpDesc.make(list(self.iql[0]), *self.iql[1])
            self.n_value = int(self.lib.b200rl_mlp_param_count(vdesc))
            check(self.lib.b200rl_offpolicy_create_iql(C.byref(cfg), C.byref(_lib.IqlConfig(vdesc)), self.K,
                                                       C.byref(h)), "offpolicy_create_iql")
        elif self.edac is not None:  # the ensemble's size and the diversity weight (b200rl.h, "EDAC")
            check(self.lib.b200rl_offpolicy_create_edac(C.byref(cfg), C.byref(_lib.EdacConfig(self.edac[0], 0,
                                                                                                self.edac[1])),
                                                        self.K, C.byref(h)), "offpolicy_create_edac")
        elif self.redq is not None:  # the ensemble's size (b200rl.h, "REDQ")
            check(self.lib.b200rl_offpolicy_create_redq(C.byref(cfg), C.byref(_lib.RedqConfig(*self.redq)), self.K,
                                                        C.byref(h)), "offpolicy_create_redq")
        elif self.cql is not None:  # N and the Lagrange switch size the buffers (b200rl.h, "CQL")
            check(self.lib.b200rl_offpolicy_create_cql(C.byref(cfg), C.byref(_lib.CqlConfig(*self.cql)), self.K,
                                                       C.byref(h)), "offpolicy_create_cql")
        else:
            check(self.lib.b200rl_offpolicy_create_group(C.byref(cfg), self.K, C.byref(h)), "offpolicy_create")
        self.h = h

    def q_layers(self):
        """(in, out) of the Q network's Linear layers in flat order (a dueling network: trunk, value hidden, value out,
        advantage hidden, advantage out)."""
        if self.dueling_k and len(self.q_sizes) == 4:
            O, h1, h2, w = self.q_sizes
            return [(O, h1), (h1, h2), (h2, self.dueling_k), (h1, h2), (h2, w)]
        return list(zip(self.q_sizes[:-1], self.q_sizes[1:]))

    def close(self):
        if getattr(self, "h", None):
            self.lib.b200rl_offpolicy_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _n(self, which):
        if self.redq is not None:  # 0 the policy, 1..2N the critics and their targets
            return self.n_policy if which == 0 else self.n_qp
        if which == 3 and self.iql is not None:
            return self.n_value
        return self.n_policy if which in (0, 3) else self.n_qp

    def set_params(self, which: int, flat: np.ndarray):
        a = _c(flat, np.float32)
        check(self.lib.b200rl_offpolicy_set_params(self.h, which, _ptr(a), a.size, current_stream_handle()), "set_params")
        import torch
        torch.cuda.current_stream().synchronize()  # `a` may be a temporary

    def get_params(self, which: int) -> np.ndarray:
        out = np.empty(self._n(which), dtype=np.float32)
        check(self.lib.b200rl_offpolicy_get_params(self.h, which, _ptr(out), out.size, current_stream_handle()), "get_params")
        return out

    def set_adam(self, which: int, m, v, step: int):
        m = None if m is None else _c(m, np.float32)
        v = None if v is None else _c(v, np.float32)
        check(self.lib.b200rl_offpolicy_set_adam(self.h, which, _ptr(m), _ptr(v), self._n(which), int(step),
                                                 current_stream_handle()), "set_adam")
        import torch
        torch.cuda.current_stream().synchronize()

    def get_adam(self, which: int):
        m, v = np.empty(self._n(which), np.float32), np.empty(self._n(which), np.float32)
        step = C.c_int64()
        check(self.lib.b200rl_offpolicy_get_adam(self.h, which, _ptr(m), _ptr(v), m.size, C.byref(step),
                                                 current_stream_handle()), "get_adam")
        return m, v, int(step.value)

    # ---- whole state in one transfer ----
    def state_layout(self):
        """[(kind, net index, offset, count)] of one learner's state blob: ("params", 0..5) then ("m" / "v", 0..2; IQL
        0..3); every segment starts on a multiple of 64 floats (b200rl.h).  A group's blob is K of these back to back."""
        pad = lambda n: (n + 63) & ~63
        if self.discrete:
            present, optimized = [1, 4], [1]
        elif self.redq is not None:
            present, optimized = list(range(1 + 2 * self.redq[0])), list(range(1 + self.redq[0]))
        else:
            present = [0, 1] + ([2] if self.n_q == 2 else []) + ([] if self.algo in self.SOFT else [3]) + [4] + \
                ([5] if self.n_q == 2 else [])
            optimized = [0, 1] + ([2] if self.n_q == 2 else []) + ([3] if self.iql is not None else [])
        out, off = [], 0
        for i in present:
            out.append(("params", i, off, self._n(i)))
            off += pad(self._n(i))
        for i in optimized:
            for kind in ("m", "v"):
                out.append((kind, i, off, self._n(i)))
                off += pad(self._n(i))
        assert off * self.K == int(self.lib.b200rl_offpolicy_state_floats(self.h))
        return out, off

    def state_buffer(self):
        """The engine's persistent host-side state blob (a float32 torch tensor, page-locked when CUDA allows it): filled
        by ``get_state()``, sent by ``set_state()``.  Views into it stay valid for the engine's lifetime."""
        import torch
        buf = getattr(self, "_state_buf", None)
        if buf is None:
            n = int(self.lib.b200rl_offpolicy_state_floats(self.h))
            buf = torch.zeros(n, dtype=torch.float32)
            try:
                buf = buf.pin_memory()
            except RuntimeError:  # pragma: no cover  (no page-locked memory available)
                pass
            self._state_buf = buf
        return buf

    def get_state(self):
        """Device -> the persistent blob; returns (blob as numpy view, [n_opt Adam step counts]; a group: [K][n_opt])."""
        buf = self.state_buffer()
        n = self.n_opt
        steps = (C.c_int64 * (n * self.K))()
        check(self.lib.b200rl_offpolicy_get_state(self.h, C.c_void_p(buf.data_ptr()), buf.numel(), steps,
                                                  current_stream_handle()), "get_state")
        st = [int(x) for x in steps]
        return buf.numpy(), st if self.K == 1 else [st[n * z:n * z + n] for z in range(self.K)]

    def set_state(self, blob, steps):
        """``blob`` = None sends the persistent blob (fill ``state_buffer()`` first), else any float32 array of that size.
        ``steps``: [n_opt] Adam step counts (a group: [K][n_opt])."""
        buf = self.state_buffer()
        if blob is not None and not (isinstance(blob, np.ndarray) and blob.ctypes.data == buf.data_ptr()):
            buf.numpy()[:] = np.asarray(blob, dtype=np.float32).reshape(-1)
        flat = np.asarray(steps, dtype=np.int64).reshape(-1)
        n = self.n_opt * self.K
        if flat.size != n:
            raise ValueError(f"set_state: expected {n} step counts, got {flat.size}")
        st = (C.c_int64 * n)(*[int(x) for x in flat])
        check(self.lib.b200rl_offpolicy_set_state(self.h, C.c_void_p(buf.data_ptr()), buf.numel(), st,
                                                  current_stream_handle()), "set_state")

    # ---- SAC ----
    def set_sac(self, sp) -> None:
        """``sp``: a ``_lib.SacHparams`` (fixed or learned temperature, its Adam settings, the log_std clamp)."""
        check(self.lib.b200rl_offpolicy_set_sac(self.h, C.byref(sp)), "set_sac")

    def set_alpha(self, log_alpha: float, exp_avg: float = 0.0, exp_avg_sq: float = 0.0, step: int = 0) -> None:
        check(self.lib.b200rl_offpolicy_set_alpha(self.h, float(log_alpha), float(exp_avg), float(exp_avg_sq), int(step)),
              "set_alpha")

    def get_alpha(self):
        """(log_alpha, exp_avg, exp_avg_sq, step) of the temperature, float32 values as Python floats."""
        la, m, v, step = C.c_float(), C.c_float(), C.c_float(), C.c_int64()
        check(self.lib.b200rl_offpolicy_get_alpha(self.h, C.byref(la), C.byref(m), C.byref(v), C.byref(step)),
              "get_alpha")
        return la.value, m.value, v.value, int(step.value)

    def set_alpha_group(self, states) -> None:
        """``states``: K tuples (log_alpha, exp_avg, exp_avg_sq, step), one per learner."""
        la, m, v = (np.array([float(x[i]) for x in states], np.float32) for i in range(3))
        st = np.array([int(x[3]) for x in states], np.int64)
        if st.size != self.K:
            raise ValueError(f"set_alpha_group: expected {self.K} learners, got {st.size}")
        check(self.lib.b200rl_offpolicy_set_alpha_group(self.h, _ptr(la), _ptr(m), _ptr(v), _ptr(st)), "set_alpha")

    def get_alpha_group(self):
        """[(log_alpha, exp_avg, exp_avg_sq, step)] of every learner."""
        la, m, v = (np.zeros(self.K, np.float32) for _ in range(3))
        st = np.zeros(self.K, np.int64)
        check(self.lib.b200rl_offpolicy_get_alpha_group(self.h, _ptr(la), _ptr(m), _ptr(v), _ptr(st)), "get_alpha")
        return [(float(la[z]), float(m[z]), float(v[z]), int(st[z])) for z in range(self.K)]

    # ---- IQL ----
    def set_iql(self, expectile: float, beta: float, max_weight: float, log_std_min: float, log_std_max: float,
                v_lr: float, v_betas=(0.9, 0.999), v_eps: float = 1e-8) -> None:
        """The expectile, the AWR inverse temperature and weight cap, the policy's log-std clamp and the value
        network's Adam settings (b200rl.h, "IQL")."""
        ip = _lib.IqlHparams(float(expectile), float(beta), float(max_weight), float(log_std_min), float(log_std_max),
                             float(v_lr), float(v_betas[0]), float(v_betas[1]), float(v_eps))
        check(self.lib.b200rl_offpolicy_set_iql(self.h, C.byref(ip)), "set_iql")

    def iql_outputs(self, S: int):
        """(value losses [S], mean V(s) before each value step [S], mean AWR weight [S]) of the last train call; a
        group: each [K, S]."""
        out = tuple(np.zeros((self.K, S), np.float32) for _ in range(3))
        check(self.lib.b200rl_offpolicy_iql_outputs(self.h, int(S), *[_ptr(x) for x in out]), "iql_outputs")
        return tuple(x[0] for x in out) if self.K == 1 else out

    # ---- REDQ ----
    def set_redq_subsets(self, subsets) -> None:
        """The target subsets int32 [S, M] (a group: [K, S, M]) of the next train / train_gather call."""
        sub = self._lead(subsets, np.int32, 3)
        if sub.shape[2] != self.redq[1]:
            raise ValueError(f"REDQ subsets: expected {self.redq[1]} critics per step, got shape {sub.shape}")
        check(self.lib.b200rl_offpolicy_set_redq_subsets(self.h, int(sub.shape[1]), _ptr(sub)), "set_redq_subsets")

    def get_redq_subsets(self, S: int):
        """The subsets [S, M] of the last train call (a group: [K, S, M])."""
        sub = np.empty((self.K, S, self.redq[1]), np.int32)
        check(self.lib.b200rl_offpolicy_get_redq_subsets(self.h, int(S), _ptr(sub)), "get_redq_subsets")
        return sub[0] if self.K == 1 else sub

    def redq_outputs(self, S: int, B: int):
        """(every critic's values [N, S, B] before each step's update, its losses [N, S]) of the last train call; a
        group: each with a leading [K] axis."""
        N = self.redq[0]
        qv, ql = np.zeros((self.K, N, S, B), np.float32), np.zeros((self.K, N, S), np.float32)
        check(self.lib.b200rl_offpolicy_redq_outputs(self.h, int(S), _ptr(qv), _ptr(ql)), "redq_outputs")
        return (qv[0], ql[0]) if self.K == 1 else (qv, ql)

    # ---- EDAC ----
    def edac_outputs(self, S: int):
        """The diversity penalty D [S] of every step of the last train call (0 with eta = 0; a group: [K, S])."""
        d = np.zeros((self.K, S), np.float32)
        check(self.lib.b200rl_offpolicy_edac_outputs(self.h, int(S), _ptr(d)), "edac_outputs")
        return d[0] if self.K == 1 else d

    # ---- CQL ----
    def set_cql(self, weight: float, temperature: float, target_action_gap: float = 0.0, alpha_lr: float = 3e-4,
                alpha_betas=(0.9, 0.999), alpha_eps: float = 1e-8, backup_entropy: bool = False) -> None:
        """The penalty's weight and temperature, the Lagrange step's gap and Adam settings, and whether the backup keeps
        SAC's entropy term (b200rl.h, "CQL")."""
        cp = _lib.CqlHparams(float(weight), float(temperature), float(target_action_gap), float(alpha_lr),
                             float(alpha_betas[0]), float(alpha_betas[1]), float(alpha_eps), int(bool(backup_entropy)), 0)
        check(self.lib.b200rl_offpolicy_set_cql(self.h, C.byref(cp)), "set_cql")

    def set_alpha_prime(self, log_alpha_prime: float, exp_avg: float = 0.0, exp_avg_sq: float = 0.0,
                        step: int = 0) -> None:
        self.set_alpha_prime_group([(log_alpha_prime, exp_avg, exp_avg_sq, step)])

    def get_alpha_prime(self):
        """(log_alpha', exp_avg, exp_avg_sq, step) of the Lagrange multiplier, float32 values as Python floats."""
        return self.get_alpha_prime_group()[0]

    def set_alpha_prime_group(self, states) -> None:
        """``states``: K tuples (log_alpha', exp_avg, exp_avg_sq, step), one per learner."""
        la, m, v = (np.array([float(x[i]) for x in states], np.float32) for i in range(3))
        st = np.array([int(x[3]) for x in states], np.int64)
        if st.size != self.K:
            raise ValueError(f"set_alpha_prime_group: expected {self.K} learners, got {st.size}")
        check(self.lib.b200rl_offpolicy_set_alpha_prime_group(self.h, _ptr(la), _ptr(m), _ptr(v), _ptr(st)),
              "set_alpha_prime")

    def get_alpha_prime_group(self):
        la, m, v = (np.zeros(self.K, np.float32) for _ in range(3))
        st = np.zeros(self.K, np.int64)
        check(self.lib.b200rl_offpolicy_get_alpha_prime_group(self.h, _ptr(la), _ptr(m), _ptr(v), _ptr(st)),
              "get_alpha_prime")
        return [(float(la[z]), float(m[z]), float(v[z]), int(st[z])) for z in range(self.K)]

    def cql_outputs(self, S: int):
        """(gap_1 [S], gap_2 [S], alpha' [S]) of the last train call's steps (alpha' 1 without the Lagrange step); a
        group: each with a leading [K] axis."""
        gaps, ap = np.zeros((self.K, 2, S), np.float32), np.zeros((self.K, S), np.float32)
        check(self.lib.b200rl_offpolicy_cql_outputs(self.h, int(S), _ptr(gaps), _ptr(ap)), "cql_outputs")
        out = gaps[:, 0], gaps[:, 1], ap
        return tuple(x[0] for x in out) if self.K == 1 else out

    def _cql_draws_shape(self, S, B):
        return (self.K, S, 3, B, self.cql[0], self.policy_sizes[-1] // 2)

    def get_cql_draws(self, S: int, B: int):
        """CQL's draws [S, 3, B, N, A] of the last train call (x in [0, 1), eps at s, eps at s'); a group: [K, ...]."""
        d = np.empty(self._cql_draws_shape(S, B), np.float32)
        check(self.lib.b200rl_offpolicy_get_cql_draws(self.h, int(S), int(B), _ptr(d)), "get_cql_draws")
        return d[0] if self.K == 1 else d

    def _split_noise(self, noise, S, B):
        """A CQL engine's (SAC noise, CQL draws) or a REDQ engine's (SAC noise, subsets): stages the draws for the
        call, returns SAC's part."""
        if self.algo not in (self.CQL, self.REDQ) or not isinstance(noise, tuple):  # the engine asks for the draws
            return noise
        sac, draws = noise
        if self.algo == self.REDQ:
            self.set_redq_subsets(draws)
            return sac
        draws = self._lead(draws, np.float32, 6)
        if draws.shape != self._cql_draws_shape(S, B):
            raise ValueError(f"CQL draws: expected shape {self._cql_draws_shape(S, B)}, got {draws.shape}")
        check(self.lib.b200rl_offpolicy_set_cql_draws(self.h, int(S), int(B), _ptr(draws)), "set_cql_draws")
        return sac

    # ---- DQN ----
    def set_dqn(self, target_update_interval: int, double_q: bool) -> None:
        from ._lib import DqnHparams
        dp = DqnHparams()
        dp.target_update_interval, dp.double_q = int(target_update_interval), int(bool(double_q))
        check(self.lib.b200rl_offpolicy_set_dqn(self.h, C.byref(dp)), "set_dqn")

    # ---- noisy networks (DQN / C51) ----
    def set_noise_keys(self, seeds, calls) -> None:
        """The (seed, call) keys of the next train call's weight noise, one of each per learner (b200rl.h, "Noisy
        networks"); an engine with noisy layers refuses a train call without fresh keys."""
        keys = [np.asarray([int(x) & (2 ** 64 - 1) for x in v], np.uint64) for v in (seeds, calls)]
        if any(k.size != self.K for k in keys):
            raise ValueError(f"set_noise_keys: expected the keys of {self.K} learners")
        check(self.lib.b200rl_offpolicy_set_noise_keys(self.h, *[_ptr(k) for k in keys]), "set_noise_keys")

    def get_noisy_draws(self, S: int):
        """Raw N(0, 1) draws [S, 2, E] (per step the online network's, then the target's; E = sum(in + out) over the
        noisy layers, eps_in then eps_out of each in layer order) of the last train call; a group: [K, S, 2, E]."""
        eps = np.empty((self.K, S, 2, self.noise_width), np.float32)
        check(self.lib.b200rl_offpolicy_get_noisy_draws(self.h, int(S), _ptr(eps)), "get_noisy_draws")
        return eps[0] if self.K == 1 else eps

    # ---- IQN ----
    def get_iqn_draws(self, S: int):
        """The fractions [S, B, N + N' + K] (per row the online, target and argmax ones) of the first S steps of the
        last train call that ran steps, B its minibatch; a group: [K, S, B, N + N' + K]."""
        _, N, Nt, K = self.iqn
        buf = np.empty(self.K * S * self.max_minibatch * (N + Nt + K), np.float32)  # room for any call's minibatch
        check(self.lib.b200rl_offpolicy_get_iqn_draws(self.h, int(S), _ptr(buf)), "get_iqn_draws")
        B = getattr(self, "_last_B", 0)
        taus = buf[:self.K * S * B * (N + Nt + K)].reshape(self.K, S, B, N + Nt + K)
        return taus[0] if self.K == 1 else taus

    # ---- C51 ----
    def set_c51(self, n_atoms: int, v_min: float, v_max: float) -> None:
        """The categorical head's support: ``n_atoms`` atoms from ``v_min`` to ``v_max`` (b200rl.h)."""
        from ._lib import C51Hparams
        cp = C51Hparams()
        cp.n_atoms, cp.v_min, cp.v_max = int(n_atoms), float(v_min), float(v_max)
        check(self.lib.b200rl_offpolicy_set_c51(self.h, C.byref(cp)), "set_c51")

    # ---- QR-DQN ----
    def set_qr(self, n_quantiles: int) -> None:
        """Makes the loss head QR-DQN's quantile Huber loss over ``n_quantiles`` quantiles for every later train call
        (a DQN engine only; b200rl.h)."""
        from ._lib import QrHparams
        qp = QrHparams()
        qp.n_quantiles = int(n_quantiles)
        check(self.lib.b200rl_offpolicy_set_qr(self.h, C.byref(qp)), "set_qr")

    # ---- prioritized replay (DQN, D4PG) ----
    def set_per(self, alpha: float, eps: float, beta_start: float, beta_anneal_steps: int) -> None:
        from ._lib import PerHparams
        pp = PerHparams()
        pp.alpha, pp.eps, pp.beta_start, pp.beta_anneal_steps = float(alpha), float(eps), float(beta_start), \
            int(beta_anneal_steps)
        check(self.lib.b200rl_offpolicy_set_per(self.h, C.byref(pp)), "set_per")

    def train_prioritized(self, hp, columns, rows: int, tree, S: int, B: int, seed: int, call: int):
        """S prioritized DQN steps on a device replay (``columns``, ``rows``) and its sum tree ``tree`` (a CUDA float32
        tensor, b200rl_per_tree_floats(rows) long; the steps update it in place), draws keyed by (``seed``, ``call``)."""
        return self.train_prioritized_group(hp, [(columns, rows)], [tree], S, B, [seed], [call])

    def train_prioritized_group(self, hp, replays, trees, S: int, B: int, seeds, calls):
        """``train_prioritized`` for every learner: K (columns, rows) pairs, K trees, K seeds and calls."""
        rb = self._replays(replays)
        if len(trees) != self.K:
            raise ValueError(f"expected the trees of {self.K} learners, got {len(trees)}")
        import torch
        for z, (t, (_, rows)) in enumerate(zip(trees, replays)):
            need = int(self.lib.b200rl_per_tree_floats(int(rows)))
            if not (torch.is_tensor(t) and t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()
                    and t.numel() == need):
                raise ValueError(f"learner {z}: the tree must be a contiguous float32 CUDA tensor of "
                                 f"b200rl_per_tree_floats({int(rows)}) = {need} floats, got "
                                 f"{getattr(t, 'dtype', type(t))} {tuple(getattr(t, 'shape', ()))} "
                                 f"on {getattr(t, 'device', '?')}")
        tp = (C.c_void_p * self.K)(*[t.data_ptr() for t in trees])
        keys = [np.asarray([int(x) & (2 ** 64 - 1) for x in v], np.uint64) for v in (seeds, calls)]
        q1v, _, l1, _, lp, npol = self._out_buffers(S, B)
        check(self.lib.b200rl_offpolicy_train_prioritized_group(self.h, C.byref(hp), S, B, rb, tp, *[_ptr(x) for x in keys],
                                                                _ptr(q1v), _ptr(l1), current_stream_handle()),
              "offpolicy_train_prioritized")
        out = dict(q1_values=q1v, q1_losses=l1)
        if not self.discrete:  # D4PG: the policy losses the call logged
            check(self.lib.b200rl_offpolicy_get_policy_losses(self.h, int(S), _ptr(lp), C.byref(npol)),
                  "get_policy_losses")
            out["policy_losses"] = lp[:, :npol.value]
        return {k: v[0] for k, v in out.items()} if self.K == 1 else out

    def get_per_draws(self, S: int, B: int):
        """(rows [S,B] int64, importance weights [S,B], new priorities [S,B] (NaN where a row wrote none)) of the last
        prioritized call; a group: each with a leading [K] axis."""
        idx = np.empty((self.K, S, B), np.int64)
        w, p = np.empty((self.K, S, B), np.float32), np.empty((self.K, S, B), np.float32)
        check(self.lib.b200rl_offpolicy_get_per_draws(self.h, S, B, _ptr(idx), _ptr(w), _ptr(p), current_stream_handle()),
              "get_per_draws")
        return (idx[0], w[0], p[0]) if self.K == 1 else (idx, w, p)

    # ---- n-step returns (DQN / C51 / D4PG) ----
    def set_nstep(self, n_step: int, episode_ends=None) -> None:
        """Window length ``n_step`` (1..32; 1 clears it) of the next train calls, with ``episode_ends`` = K float32 CUDA
        tensors (each learner's ``device_episode_ends()``, over the rows of the replay it trains on) when n_step > 1."""
        import torch
        ptrs = None
        if int(n_step) > 1:
            if episode_ends is None or len(episode_ends) != self.K:
                raise ValueError(f"set_nstep: n_step = {n_step} needs the episode-end columns of {self.K} learners")
            for z, t in enumerate(episode_ends):
                if not (torch.is_tensor(t) and t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()):
                    raise ValueError(f"set_nstep: learner {z}: the episode-end column must be a contiguous float32 CUDA "
                                     f"tensor, got {getattr(t, 'dtype', type(t))} on {getattr(t, 'device', '?')}")
            ptrs = (C.c_void_p * self.K)(*[t.data_ptr() for t in episode_ends])
        check(self.lib.b200rl_offpolicy_set_nstep(self.h, int(n_step), ptrs), "set_nstep")

    def get_nstep_draws(self, S: int, B: int):
        """(last window row [S,B] int64, return R [S,B], discount [S,B] float32) of each row of the last n-step call;
        a group: each with a leading [K] axis."""
        last = np.empty((self.K, S, B), np.int64)
        R, g = np.empty((self.K, S, B), np.float32), np.empty((self.K, S, B), np.float32)
        check(self.lib.b200rl_offpolicy_get_nstep_draws(self.h, S, B, _ptr(last), _ptr(R), _ptr(g),
                                                        current_stream_handle()), "get_nstep_draws")
        return (last[0], R[0], g[0]) if self.K == 1 else (last, R, g)

    def sac_outputs(self, S: int):
        """(mean log pi per step [S], alpha used by each step [S]) of the last train call (a group: [K, S] each)."""
        lp, al = np.zeros((self.K, S), np.float32), np.zeros((self.K, S), np.float32)
        check(self.lib.b200rl_offpolicy_sac_outputs(self.h, int(S), _ptr(lp), _ptr(al)), "sac_outputs")
        return (lp[0], al[0]) if self.K == 1 else (lp, al)

    def _out_buffers(self, S, B):
        K = self.K
        if S > 0:
            self._last_B = B  # the minibatch of the call's steps, get_iqn_draws's
        return (np.zeros((K, S, B), np.float32), np.zeros((K, S, B), np.float32), np.zeros((K, S), np.float32),
                np.zeros((K, S), np.float32), np.zeros((K, max(S, 1)), np.float32), C.c_int32())

    def _outputs(self, S, q1v, q2v, l1, l2, lp, npol):
        """The logged quantities; a solo engine drops the leading [K] axis."""
        if self.discrete:
            out = dict(q1_values=q1v, q1_losses=l1)
        else:
            out = dict(q1_values=q1v, q2_values=q2v, q1_losses=l1, q2_losses=l2, policy_losses=lp[:, :npol.value])
        if self.K == 1:
            out = {k: v[0] for k, v in out.items()}
        if self.algo in self.SOFT:
            out["log_prob_means"], out["alphas"] = self.sac_outputs(S)
        if self.algo == self.CQL:
            out["cql_gap_1"], out["cql_gap_2"], out["alpha_primes"] = self.cql_outputs(S)
        if self.algo == self.IQL:
            out["value_losses"], out["value_means"], out["weight_means"] = self.iql_outputs(S)
        if self.algo in (self.REDQ, self.EDAC) and S > 0:  # one mean log pi per policy step; every critic's values
            out["log_prob_means"] = out["log_prob_means"][..., :npol.value]  # and losses
            out["redq_q_values"], out["redq_q_losses"] = self.redq_outputs(S, self._last_B)
        if self.algo == self.EDAC and S > 0:
            out["edac_diversity"] = self.edac_outputs(S)
        return out

    def _lead(self, a, dtype, ndim):
        """A solo engine's input without the [K] axis, a group's with it, as one contiguous [K, ...] array."""
        a = _c(a, dtype)
        if self.K == 1 and a.ndim == ndim - 1:
            a = a[None]
        if a.shape[0] != self.K:
            raise ValueError(f"expected a leading axis of {self.K} learners, got shape {a.shape}")
        return a

    def train(self, hp, obs, act, rew, next_obs, done, noise=None):
        """obs/next_obs [S,B,O], act [S,B,A], rew/done [S,B], noise [S,B,A] or None (SAC: [S,2,B,A], required) -> dict
        of logged quantities (SAC adds log_prob_means and alphas).  A group: every array with a leading [K] axis.
        DQN: act [S,B] action indices, noise None; the dict holds q1_values and q1_losses.  Discrete SAC: act [S,B]
        action indices, noise None; the dict is SAC's."""
        if self.index_actions:
            act = np.asarray(act, np.float32)[..., None]
        obs, act, next_obs = (self._lead(x, np.float32, 4) for x in (obs, act, next_obs))
        rew, done = self._lead(rew, np.float32, 3), self._lead(done, np.float32, 3)
        S, B = obs.shape[1], obs.shape[2]
        noise = self._split_noise(noise, S, B)
        noise = None if noise is None else self._lead(noise, np.float32, 5 if self.algo in self.SQUASHED else 4)
        q1v, q2v, l1, l2, lp, npol = self._out_buffers(S, B)
        check(self.lib.b200rl_offpolicy_train(self.h, C.byref(hp), S, B, _ptr(obs), _ptr(act), _ptr(rew), _ptr(next_obs),
                                              _ptr(done), _ptr(noise), _ptr(q1v), _ptr(q2v), _ptr(l1), _ptr(l2), _ptr(lp),
                                              C.byref(npol), current_stream_handle()), "offpolicy_train")
        return self._outputs(S, q1v, q2v, l1, l2, lp, npol)

    def train_gather_rng(self, hp, columns, rows: int, ring_start: int, ring_size: int, S: int, B: int, seed: int, call: int):
        """``train_gather`` with the indices and the smoothing noise drawn on the device (Philox keyed by ``seed``, block
        ``call``); ``ring_size`` live rows, logical row u at physical ``(ring_start + u) % rows``.  Opt-in: the streams
        are not the reference's numpy / torch ones."""
        return self.train_gather_rng_group(hp, [(columns, rows)], [ring_start], [ring_size], S, B, [seed], [call])

    def train_gather_rng_group(self, hp, replays, ring_starts, ring_sizes, S: int, B: int, seeds, calls):
        """``train_gather_rng`` for every learner: ``replays`` = K (columns, rows) pairs, the other sequences K long;
        learner z's draws are those of a solo engine keyed by (seeds[z], calls[z])."""
        rb = self._replays(replays)
        ring = [np.asarray(x, np.int64).reshape(-1) for x in (ring_starts, ring_sizes)]
        keys = [np.asarray([int(x) & (2 ** 64 - 1) for x in v], np.uint64) for v in (seeds, calls)]
        q1v, q2v, l1, l2, lp, npol = self._out_buffers(S, B)
        check(self.lib.b200rl_offpolicy_train_gather_rng_group(self.h, C.byref(hp), S, B, rb, *[_ptr(x) for x in ring],
                                                               *[_ptr(x) for x in keys], _ptr(q1v), _ptr(q2v), _ptr(l1),
                                                               _ptr(l2), _ptr(lp), C.byref(npol), current_stream_handle()),
              "offpolicy_train_gather_rng")
        return self._outputs(S, q1v, q2v, l1, l2, lp, npol)

    def get_draws(self, S: int, B: int, with_noise: bool = True):
        """(physical rows [S,B] int64, noise [S,B,A] (SAC: [S,2,B,A]) float32 or None) of the last train_gather /
        train_gather_rng call; a group: both with a leading [K] axis."""
        idx = np.empty((self.K, S, B), np.int64)
        with_noise = with_noise and not self.index_actions and self.algo != self.IQL  # these draw indices only
        noise = None
        if with_noise and self.algo in self.SQUASHED:
            noise = np.empty((self.K, S, 2, B, self.policy_sizes[-1] // 2), np.float32)
        elif with_noise:
            noise = np.empty((self.K, S, B, self.policy_sizes[-1]), np.float32)
        check(self.lib.b200rl_offpolicy_get_draws(self.h, S, B, _ptr(idx), _ptr(noise), current_stream_handle()), "get_draws")
        if self.K == 1:
            return idx[0], None if noise is None else noise[0]
        return idx, noise

    def _replays(self, replays):
        if len(replays) != self.K:
            raise ValueError(f"expected the replay columns of {self.K} learners, got {len(replays)}")
        rb = (_lib.OffPolicyReplay * self.K)()
        for z, (columns, rows) in enumerate(replays):
            rb[z] = _lib.OffPolicyReplay(*[t.data_ptr() for t in columns], int(rows))
        return rb

    def train_gather(self, hp, columns, rows: int, idx, noise=None):
        """Minibatches gathered on the device: ``columns`` = CUDA float32 tensors (obs [rows,O], act [rows,A], rew [rows],
        next_obs [rows,O], done [rows]) of a device-resident replay buffer, ``idx`` [S,B] int64 physical rows (host)."""
        return self.train_gather_group(hp, [(columns, rows)], idx, noise)

    def train_gather_group(self, hp, replays, idx, noise=None):
        """``train_gather`` for every learner: ``replays`` = K (columns, rows) pairs, one replay buffer per learner;
        ``idx`` [K,S,B], ``noise`` [K,S,B,A] (SAC [K,S,2,B,A]); a solo engine also takes them without the [K] axis."""
        rb = self._replays(replays)
        idx = self._lead(idx, np.int64, 3)
        S, B = idx.shape[1], idx.shape[2]
        noise = self._split_noise(noise, S, B)
        noise = None if noise is None else self._lead(noise, np.float32, 5 if self.algo in self.SQUASHED else 4)
        q1v, q2v, l1, l2, lp, npol = self._out_buffers(S, B)
        check(self.lib.b200rl_offpolicy_train_gather_group(self.h, C.byref(hp), S, B, rb, _ptr(idx), _ptr(noise),
                                                           _ptr(q1v), _ptr(q2v), _ptr(l1), _ptr(l2), _ptr(lp),
                                                           C.byref(npol), current_stream_handle()),
              "offpolicy_train_gather")
        return self._outputs(S, q1v, q2v, l1, l2, lp, npol)
