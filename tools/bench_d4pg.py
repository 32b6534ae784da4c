"""D4PG.train throughput at the HalfCheetah shape, against DDPG at the same shape in the same process.

    python tools/bench_d4pg.py [--calls 20] [--warmup 3] [--rounds 3]

Workload: obs 17, act 6, 256-256 ReLU networks, minibatch 256, 50 train steps per train() call, a replay of 1 M
transitions (episodes of 1000) resident on the device; D4PG's critic has 51 atoms on [-10, 10].  Arms, alternated
round by round within the run: DDPG and D4PG on uniform device draws, D4PG with n = 5, D4PG with prioritized replay, and
LearnerGroup.train of D4PG learners at K = 1, 4 and 16 (uniform device draws, one replay each).  For every arm: median ms
per train() call end to end (host state sync included) and engine-only, train steps/s of both (a group: learner steps/s,
K x steps over the call), launches per step, and, from a torch.profiler pass after the timed rounds, the loss heads'
share of the device time per step (c51_loss_kernel and d4pg_policy_loss_kernel over every kernel of the call).  Prints
one JSON line with the card's name and power limit read in this run.  Needs a GPU; there is no CPU fallback."""
import argparse
import json
import os
import subprocess
import sys
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

O_DIM, A_DIM, H, B, S, N_REPLAY, N_ATOMS, EP = 17, 6, 256, 256, 50, 1_000_000, 51, 1000
HEADS = ("c51_loss_kernel", "d4pg_policy_loss_kernel")


class _Columns:
    """A replay-buffer input in column form (no per-transition Python objects), episodes of EP transitions."""

    def __init__(self, rng, n):
        obs = rng.standard_normal((n + 1, O_DIM)).astype(np.float32)
        done = np.zeros(n, bool)
        done[EP - 1::EP] = True
        self.cols = (obs[:n], rng.uniform(-1, 1, (n, A_DIM)).astype(np.float32), rng.standard_normal(n), obs[1:], done)
        self.ep_offsets = np.arange(0, n + 1, EP)

    def transition_columns(self):
        return self.cols


def card():
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = r.stdout.strip() or "unknown"
    except Exception:
        power = "unknown"
    return name, power


def replay(kind, seed):
    from rl_replicas_b200.replay_buffer import PrioritizedReplayBuffer, ReplayBuffer
    rb = PrioritizedReplayBuffer(N_REPLAY) if kind == "per" else ReplayBuffer(buffer_size=N_REPLAY)
    rb.add_experience(_Columns(np.random.default_rng(seed), N_REPLAY))
    return rb


def make(kind, rb, seed=0):
    from rl_replicas_b200.algorithms import D4PG, DDPG
    from rl_replicas_b200.critics import DistributionalQFunction, QFunction
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import DeterministicPolicy, RandomPolicy
    torch.manual_seed(seed)
    hi = np.ones(A_DIM, np.float32)
    env = types.SimpleNamespace(action_space=types.SimpleNamespace(high=hi, low=-hi, shape=(A_DIM,)),
                                observation_space=types.SimpleNamespace(shape=(O_DIM,)), spec=types.SimpleNamespace(id="stub"))
    pnet = MLP([O_DIM, H, H, A_DIM], torch.nn.ReLU, torch.nn.Tanh)
    policy = DeterministicPolicy(pnet, torch.optim.Adam(pnet.parameters(), lr=1e-3))
    if kind == "ddpg":
        q = MLP([O_DIM + A_DIM, H, H, 1], torch.nn.ReLU)
        algo = DDPG(policy, RandomPolicy(None), QFunction(q, torch.optim.Adam(q.parameters(), lr=1e-3)), env, None, rb,
                    None)
    else:
        q = MLP([O_DIM + A_DIM, H, H, N_ATOMS], torch.nn.ReLU)
        qf = DistributionalQFunction(q, torch.optim.Adam(q.parameters(), lr=1e-3), n_atoms=N_ATOMS)
        algo = D4PG(policy, RandomPolicy(None), qf, env, None, rb, None, n_step=5 if kind == "nstep" else 1)
    algo.metrics_manager = None
    algo.use_device_rng, algo.device_rng_seed = True, seed
    return algo


class Arm:
    """One timed configuration: ``call()`` runs one train() call; ``engine`` the engine whose calls are timed."""

    def __init__(self, name, learners, group=None):
        self.name, self.learners, self.group = name, learners, group
        self.call_ms, self.engine_ms, self.launches = [], [], []

    def call(self):
        if self.group is not None:
            self.group.train(S, B)
        else:
            a = self.learners[0]
            a.train(a.replay_buffer, S, B)

    def engine(self):  # a group of one trains through its member's own engine
        return self.group._engine if self.group is not None and self.group._engine else self.learners[0]._engine

    def timed(self, calls, lib):
        e = self.engine()
        names = ("train_gather_rng_group", "train_prioritized_group")
        orig = {n: getattr(e, n) for n in names}

        def wrap(f):
            def timed_call(*a, **k):
                t0 = time.perf_counter()
                r = f(*a, **k)  # reads the logs back: ends in a stream synchronisation
                self.engine_ms.append((time.perf_counter() - t0) * 1e3)
                return r
            return timed_call
        for n in names:
            setattr(e, n, wrap(orig[n]))
        try:
            for _ in range(calls):
                torch.cuda.synchronize()
                n0 = lib.b200rl_launch_count()
                t0 = time.perf_counter()
                self.call()
                torch.cuda.synchronize()
                self.call_ms.append((time.perf_counter() - t0) * 1e3)
                self.launches.append(lib.b200rl_launch_count() - n0)
        finally:
            for n in names:
                setattr(e, n, orig[n])

    def head_share(self):
        """The heads' share of the device time of one call, from a profiler pass (None for DDPG)."""
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            self.call()
            torch.cuda.synchronize()
        total = head = 0.0
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                total += ev.device_time
                if any(h in ev.name for h in HEADS):
                    head += ev.device_time
        return None if total == 0 or head == 0 else round(head / total, 4)

    def result(self):
        K = len(self.learners)
        med, eng = float(np.median(self.call_ms)), float(np.median(self.engine_ms))
        return {"train_call_ms": round(med, 3), "engine_ms": round(eng, 3),
                "train_steps_per_s": round(K * S / med * 1e3, 1), "engine_steps_per_s": round(K * S / eng * 1e3, 1),
                "launches_per_step": round(float(np.median(self.launches)) / S, 2), "head_device_share": self.share}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_d4pg.py needs a CUDA device: there is no CPU fallback")
    from rl_replicas_b200 import _lib
    from rl_replicas_b200.algorithms import LearnerGroup
    lib = _lib.load()
    np.random.seed(0)
    uniform = replay("uniform", 0)
    arms = [Arm("ddpg_uniform", [make("ddpg", uniform)]), Arm("d4pg_uniform", [make("d4pg", uniform)]),
            Arm("d4pg_nstep5", [make("nstep", uniform)]), Arm("d4pg_prioritized", [make("d4pg", replay("per", 1))])]
    for K in (1, 4, 16):
        members = [make("d4pg", replay("uniform", 10 + k) if k else uniform, seed=k) for k in range(K)]
        g = LearnerGroup()
        for m in members:
            g.add(m)
        arms.append(Arm(f"group_k{K}", members, g))
    for arm in arms:  # builds every engine (and graph)
        for _ in range(args.warmup):
            arm.call()
    for _ in range(args.rounds):  # alternated: every arm sees the same conditions
        for arm in arms:
            arm.timed(max(args.calls // args.rounds, 1), lib)
    for arm in arms:
        arm.share = arm.head_share()
    name, power = card()
    print(json.dumps({
        "workload": f"D4PG.train ({N_ATOMS} atoms) vs DDPG.train, obs {O_DIM} act {A_DIM}, {H}-{H} ReLU, B {B}, {S} "
                    f"steps per call, {N_REPLAY} transitions on the device",
        **{arm.name: arm.result() for arm in arms}, "gpu": name, "power_limit": power}))


if __name__ == "__main__":
    main()
