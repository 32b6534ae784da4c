"""Learner groups against back-to-back solo learners at the SAC / TD3 benchmark shape, in one process.

    python tools/bench_group.py [--calls 10] [--warmup 2] [--ks 1,2,3,4,8,16]

Workload (tools/bench_sac.py's): obs 17, act 6, 256-256 ReLU networks, minibatch 256, 50 train steps per call, SAC
with a learned temperature; every member has its own device replay of 1 M transitions (168 MB).  For TD3 and SAC and
each K, the same K learners are trained alternately as one LearnerGroup.train call and as K back-to-back solo
agent.train calls.  Prints one JSON line: per K the median engine-only ms per call of the group and of the K solo calls
together, the aggregate train steps/s of both, the group's end-to-end LearnerGroup.train ms (host state sync included),
and the card's name and power limit read in this run.  Needs a GPU; there is no CPU fallback."""
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

from bench_sac import B, N_REPLAY, S, _Columns, card, make  # noqa: E402


class _EngineClock:
    """Wall time of the engine's train calls (each ends in a stream synchronisation when it reads the logs back)."""

    def __init__(self):
        self.ms = 0.0

    def wrap(self, e, name):
        f = getattr(e, name)

        def timed(*a, **k):
            t0 = time.perf_counter()
            r = f(*a, **k)
            self.ms += (time.perf_counter() - t0) * 1e3
            return r
        setattr(e, name, timed)


def bench(kind, K, cols, calls, warmup):
    from rl_replicas_b200.algorithms import LearnerGroup
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    agents = []
    group = LearnerGroup()
    for k in range(K):
        rb = ReplayBuffer(buffer_size=N_REPLAY)
        rb.add_experience(cols)
        np.random.seed(k)
        a = make(kind, rb)
        agents.append(a)
        group.add(a)
    clock = _EngineClock()
    group.train(S, B)  # builds the group engine (K = 1: the member's own)
    for a in agents:
        a.train(a.replay_buffer, S, B)  # builds each solo engine
    for a in agents:
        clock.wrap(a._engine, "train_gather")
    if group._engine is not None:
        clock.wrap(group._engine, "train_gather_group")
    g_eng, g_e2e, s_eng = [], [], []
    for i in range(warmup + calls):
        clock.ms = 0.0
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        group.train(S, B)
        torch.cuda.synchronize()
        e2e, eng = (time.perf_counter() - t0) * 1e3, clock.ms
        clock.ms = 0.0
        for a in agents:
            a.train(a.replay_buffer, S, B)
        if i >= warmup:
            g_eng.append(eng)
            g_e2e.append(e2e)
            s_eng.append(clock.ms)
    for a in agents:
        a._engine.close()
    group._close_engine()
    ge, se, gt = (float(np.median(x)) for x in (g_eng, s_eng, g_e2e))
    return {"K": K, "group_engine_ms": round(ge, 3), "group_engine_steps_per_s": round(K * S / ge * 1e3, 1),
            "solo_engine_ms_sum": round(se, 3), "solo_engine_steps_per_s": round(K * S / se * 1e3, 1),
            "engine_speedup": round(se / ge, 3), "group_train_call_ms": round(gt, 3),
            "group_train_steps_per_s": round(K * S / gt * 1e3, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--ks", default="1,2,3,4,8,16")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_group.py needs a CUDA device: there is no CPU fallback")
    cols = _Columns(np.random.default_rng(0), N_REPLAY)
    res = {}
    for kind in ("td3", "sac"):
        res[kind] = [bench(kind, int(k), cols, args.calls, args.warmup) for k in args.ks.split(",")]
    name, power = card()
    print(json.dumps({
        "workload": f"K learners, obs 17 act 6, 256-256 ReLU, B {B}, {S} steps per call, {N_REPLAY} transitions on "
                    "the device per learner, SAC with learned alpha; group vs K back-to-back solo calls",
        **res, "gpu": name, "power_limit": power}))


if __name__ == "__main__":
    main()
