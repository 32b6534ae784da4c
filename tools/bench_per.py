"""Prioritized experience replay against uniform device draws for DQN.train at a LunarLander shape, alone and as learner
groups.

    python tools/bench_per.py [--calls 20] [--warmup 3] [--rounds 3]

Workload: obs 8, 4 actions, 256-256 ReLU Q network, minibatch 256, 50 train steps per train() call, Double DQN, replay
of 1 M transitions resident on the device.  The uniform path is DQN.train with device-side index draws
(use_device_rng); the prioritized path is DQN.train on a PrioritizedReplayBuffer (draw, weights and gather inside the
step graph, priority update beside the backward pass).  The two alternate in `rounds` rounds of `calls` timed calls
each, so both see the same machine state; the medians over all timed calls are reported.  Prints one JSON line: ms per
DQN.train call end to end (host state sync included) and engine-only, train steps/s, launches per step, LearnerGroup
.train with prioritized members at K = 1, 4 and 16 (learner steps/s summed over the members), and the card's name and
power limit read in this run.  Needs a GPU; there is no CPU fallback."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_dqn import B, N_REPLAY, S, _Columns, make  # noqa: E402
from bench_sac import card  # noqa: E402


def build(prioritized: bool, cols, seed=0):
    from rl_replicas_b200.replay_buffer import PrioritizedReplayBuffer, ReplayBuffer
    rb = PrioritizedReplayBuffer(N_REPLAY) if prioritized else ReplayBuffer(buffer_size=N_REPLAY)
    rb.add_experience(cols)
    algo = make(rb, seed=seed)
    algo.use_device_rng = True  # the uniform path's device draws; the prioritized path draws on the device anyway
    algo.device_rng_seed = seed
    return algo


class Timer:
    """DQN.train calls of one learner, with the engine call inside timed on its own (it ends in a synchronisation)."""

    def __init__(self, algo, prioritized: bool):
        from rl_replicas_b200 import _lib
        self.algo, self.lib = algo, _lib.load()
        algo.train(algo.replay_buffer, S, B)  # builds the engine and the graph
        self.name = "train_prioritized" if prioritized else "train_gather_rng"
        self.f = getattr(algo._engine, self.name)
        self.engine_ms, self.call_ms, self.launches = [], [], []

        def timed(*a, **k):
            t0 = time.perf_counter()
            r = self.f(*a, **k)
            self.engine_ms.append((time.perf_counter() - t0) * 1e3)
            return r
        setattr(algo._engine, self.name, timed)

    def run(self, calls, warmup):
        for _ in range(warmup):
            self.algo.train(self.algo.replay_buffer, S, B)
        del self.engine_ms[len(self.engine_ms) - warmup:]
        for _ in range(calls):
            torch.cuda.synchronize()
            n0 = self.lib.b200rl_launch_count()
            t0 = time.perf_counter()
            self.algo.train(self.algo.replay_buffer, S, B)
            torch.cuda.synchronize()
            self.call_ms.append((time.perf_counter() - t0) * 1e3)
            self.launches.append(self.lib.b200rl_launch_count() - n0)

    def result(self):
        med, eng = float(np.median(self.call_ms)), float(np.median(self.engine_ms))
        return {"train_call_ms": round(med, 3), "engine_ms": round(eng, 3), "train_steps_per_s": round(S / med * 1e3, 1),
                "engine_steps_per_s": round(S / eng * 1e3, 1), "launches_per_step": float(np.median(self.launches)) / S,
                "timed_calls": len(self.call_ms)}


def time_group(cols, K, calls, warmup):
    from rl_replicas_b200.algorithms import LearnerGroup
    g = LearnerGroup()
    for k in range(K):
        np.random.seed(k)
        g.add(build(True, cols, seed=k))
    for _ in range(warmup + 1):
        g.train(S, B)
    per_call = []
    for _ in range(calls):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        g.train(S, B)
        torch.cuda.synchronize()
        per_call.append((time.perf_counter() - t0) * 1e3)
    med = float(np.median(per_call))
    return {"train_call_ms": round(med, 3), "learner_steps_per_s": round(K * S / med * 1e3, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_per.py needs a CUDA device: there is no CPU fallback")
    cols = _Columns(np.random.default_rng(0), N_REPLAY)
    timers = {"uniform": Timer(build(False, cols), False), "prioritized": Timer(build(True, cols), True)}
    for _ in range(args.rounds):
        for t in timers.values():
            t.run(args.calls, args.warmup)
    res = {k: t.result() for k, t in timers.items()}
    res["prioritized_over_uniform_engine_time"] = round(res["prioritized"]["engine_ms"] / res["uniform"]["engine_ms"], 3)
    groups = {f"K={K}": time_group(cols, K, args.calls, args.warmup) for K in (1, 4, 16)}
    name, power = card()
    print(json.dumps({
        "workload": f"DQN.train, obs 8, 4 actions, 256-256 ReLU, B {B}, {S} steps per call, {N_REPLAY} transitions on "
                    "the device, Double DQN; uniform device draws vs prioritized replay (alpha 0.6, beta 0.4 -> 1)",
        **res, "prioritized_groups": groups, "gpu": name, "power_limit": power}))


if __name__ == "__main__":
    main()
