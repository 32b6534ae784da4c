"""DiscreteSAC.train throughput at DQN's LunarLander shape, alternated in one process with Double DQN at the same shape
and continuous SAC at the HalfCheetah shape of tools/bench_sac.py, and as learner groups.

    python tools/bench_discrete_sac.py [--calls 10] [--warmup 3] [--rounds 3]

Workload: obs 8, 4 actions, 256-256 ReLU policy and critics, minibatch 256, 50 train steps per train() call, learned
temperature, replay of 1 M transitions resident on the device, indices drawn on the device (use_device_rng).  DQN
(Double DQN, same shape) and SAC (obs 17, act 6, learned temperature) take the same path.  The three learners are timed
in turn, ``--rounds`` times over, and every figure is the median over all rounds.  Prints one JSON line: ms per train()
call end to end (host state sync included) and engine-only, train steps/s for each, LearnerGroup.train at K = 1, 4 and
16 (learner steps/s summed over the members), the launches per call and per step of discrete SAC, and the card's name
and power limit read in this run.  Needs a GPU; there is no CPU fallback."""
import argparse
import json
import os
import sys
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench_dqn  # noqa: E402
import bench_sac  # noqa: E402
from bench_sac import card  # noqa: E402

O_DIM, N_ACT, H, B, S, N_REPLAY = 8, 4, 256, 256, 50, 1_000_000


def make_dsac(rb, seed=0):
    from rl_replicas_b200.algorithms import DiscreteSAC
    from rl_replicas_b200.critics import DiscreteQFunction
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import CategoricalPolicy
    torch.manual_seed(seed)
    env = types.SimpleNamespace(action_space=types.SimpleNamespace(n=N_ACT, shape=()), spec=types.SimpleNamespace(id="stub"),
                                observation_space=types.SimpleNamespace(shape=(O_DIM,)))
    pnet, q1, q2 = (MLP([O_DIM, H, H, N_ACT], torch.nn.ReLU) for _ in range(3))
    algo = DiscreteSAC(CategoricalPolicy(pnet, torch.optim.Adam(pnet.parameters(), lr=3e-4)), None,
                       DiscreteQFunction(q1, torch.optim.Adam(q1.parameters(), lr=3e-4)),
                       DiscreteQFunction(q2, torch.optim.Adam(q2.parameters(), lr=3e-4)), env, None, rb, None,
                       learn_alpha=True)
    algo.metrics_manager = None
    algo.use_device_rng = True
    return algo


class Timer:
    """Times one learner's train() calls end to end and its engine call alone (train_gather_rng reads the logs back, so
    it ends in a stream synchronisation)."""

    def __init__(self, algo, rb):
        self.algo, self.rb = algo, rb
        self.call_ms, self.engine_ms = [], []
        algo.train(rb, S, B)  # builds the engine and captures the graph
        f = algo._engine.train_gather_rng

        def timed(*a, **k):
            t0 = time.perf_counter()
            r = f(*a, **k)
            self.engine_ms.append((time.perf_counter() - t0) * 1e3)
            return r
        algo._engine.train_gather_rng = timed

    def run(self, calls, keep=True):
        n_eng = len(self.engine_ms)
        for _ in range(calls):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            self.algo.train(self.rb, S, B)
            torch.cuda.synchronize()
            if keep:
                self.call_ms.append((time.perf_counter() - t0) * 1e3)
        if not keep:
            del self.engine_ms[n_eng:]

    def result(self):
        med, eng = float(np.median(self.call_ms)), float(np.median(self.engine_ms))
        return {"train_call_ms": round(med, 3), "engine_ms": round(eng, 3),
                "train_steps_per_s": round(S / med * 1e3, 1), "engine_steps_per_s": round(S / eng * 1e3, 1)}


def time_group(rb, K, calls, warmup):
    from rl_replicas_b200.algorithms import LearnerGroup
    g = LearnerGroup()
    for k in range(K):
        np.random.seed(k)
        g.add(make_dsac(rb, seed=k))
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
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_discrete_sac.py needs a CUDA device: there is no CPU fallback")
    from rl_replicas_b200 import _lib
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    rng = np.random.default_rng(0)
    rb_d = ReplayBuffer(buffer_size=N_REPLAY)
    rb_d.add_experience(bench_dqn._Columns(rng, N_REPLAY))  # obs 8, action indices 0..3
    rb_c = ReplayBuffer(buffer_size=N_REPLAY)
    rb_c.add_experience(bench_sac._Columns(rng, N_REPLAY))  # obs 17, act 6
    np.random.seed(0)
    dqn, sac = bench_dqn.make(rb_d), bench_sac.make("sac", rb_c)
    dqn.use_device_rng = sac.use_device_rng = True
    timers = {"discrete_sac": Timer(make_dsac(rb_d), rb_d), "dqn_same_shape": Timer(dqn, rb_d),
              "sac_halfcheetah": Timer(sac, rb_c)}
    for t in timers.values():
        t.run(args.warmup, keep=False)
    for _ in range(args.rounds):
        for t in timers.values():
            t.run(args.calls)
    lib = _lib.load()
    d = timers["discrete_sac"]
    n0 = lib.b200rl_launch_count()
    d.algo.train(rb_d, S, B)
    per_call = int(lib.b200rl_launch_count() - n0)
    groups = {f"K={K}": time_group(rb_d, K, args.calls, args.warmup) for K in (1, 4, 16)}
    name, power = card()
    print(json.dumps({
        "workload": f"DiscreteSAC.train, obs {O_DIM}, {N_ACT} actions, {H}-{H} ReLU, B {B}, {S} steps per call, "
                    f"{N_REPLAY} transitions on the device, device index draws, learned alpha",
        **{k: t.result() for k, t in timers.items()}, "discrete_sac_groups": groups,
        # per call: the index draw, five column gathers and the temperature table
        "discrete_sac_launches": {"per_call": per_call, "per_step": (per_call - 7) / S},
        "rounds": args.rounds, "gpu": name, "power_limit": power}))


if __name__ == "__main__":
    main()
