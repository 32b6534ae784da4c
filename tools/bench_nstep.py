"""n-step returns against one-step targets for DQN.train (and C51.train) at a LunarLander shape.

    python tools/bench_nstep.py [--calls 20] [--warmup 3] [--rounds 3]

Workload: obs 8, 4 actions, 256-256 ReLU Q network, minibatch 256, 50 train steps per train() call, Double DQN, replay
of 1 M transitions resident on the device in episodes of 200 rows (so windows stop at episode ends as they would on
LunarLander).  Arms: DQN at n = 1, 3 and 10 on uniform device draws (use_device_rng) and on prioritized replay, and C51
(51 atoms) at n = 1 and 3 on uniform device draws.  The arms alternate in `rounds` rounds of `calls` timed calls each,
so all see the same machine state; the medians over all timed calls are reported.  Prints one JSON line: per arm ms per
train() call end to end (host state sync included) and engine-only, train steps/s and launches per step, and the
card's name and power limit read in this run.  Needs a GPU; there is no CPU fallback."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_dqn import B, N_ACT, N_REPLAY, S, _Columns, make  # noqa: E402
from bench_per import Timer  # noqa: E402
from bench_sac import card  # noqa: E402

EPISODE = 200


class _Episodes(_Columns):
    """The column stub with episode boundaries every EPISODE rows (what a PackedExperience reports)."""

    def __init__(self, rng, n):
        super().__init__(rng, n)
        self.ep_offsets = np.append(np.arange(0, n, EPISODE), n)


def build(kind: str, n_step: int, cols, seed=0):
    from bench_c51 import make as make_c51
    from rl_replicas_b200.replay_buffer import PrioritizedReplayBuffer, ReplayBuffer
    rb = PrioritizedReplayBuffer(N_REPLAY) if kind == "per" else ReplayBuffer(buffer_size=N_REPLAY)
    rb.add_experience(cols)
    algo = make_c51("c51", N_ACT, rb, seed=seed) if kind == "c51" else make(rb, seed=seed)
    algo.n_step = n_step
    algo.use_device_rng = True  # uniform device draws; the prioritized path draws on the device anyway
    algo.device_rng_seed = seed
    return algo


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_nstep.py needs a CUDA device: there is no CPU fallback")
    cols = _Episodes(np.random.default_rng(0), N_REPLAY)
    arms = [("dqn", n) for n in (1, 3, 10)] + [("per", n) for n in (1, 3, 10)] + [("c51", n) for n in (1, 3)]
    timers = {f"{kind} n={n}": Timer(build(kind, n, cols), kind == "per") for kind, n in arms}
    for _ in range(args.rounds):
        for t in timers.values():
            t.run(args.calls, args.warmup)
    res = {k: t.result() for k, t in timers.items()}
    ratios = {f"{k} over n=1 engine time": round(res[k]["engine_ms"] / res[k.split()[0] + " n=1"]["engine_ms"], 3)
              for k in res if not k.endswith("n=1")}
    name, power = card()
    print(json.dumps({
        "workload": f"train(), obs 8, {N_ACT} actions, 256-256 ReLU, B {B}, {S} steps per call, {N_REPLAY} transitions "
                    f"on the device in episodes of {EPISODE}, Double DQN; DQN uniform device draws (dqn), prioritized "
                    "replay (per), C51 51 atoms uniform device draws (c51)",
        **res, **ratios, "gpu": name, "power_limit": power}))


if __name__ == "__main__":
    main()
