"""DQN.train throughput at a LunarLander shape, alone and as learner groups, with the torch-CPU oracle as the baseline.

    python tools/bench_dqn.py [--calls 20] [--warmup 3] [--oracle-calls 2]

Workload: obs 8, 4 actions, 256-256 ReLU Q network, minibatch 256, 50 train steps per train() call, Double DQN, replay
of 1 M transitions resident on the device.  Prints one JSON line: median ms per DQN.train call end to end (host state
sync included) and engine-only, train steps/s, LearnerGroup.train at K = 1, 2, 4, 8 and 16 (learner steps/s summed over
the members), the torch-CPU oracle's ms per call (the CPU baseline), and the card's name and power limit read in this
run.  Needs a GPU; there is no CPU fallback."""
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

from bench_sac import card, time_calls  # noqa: E402
from oracle import dqn as OD  # noqa: E402

O_DIM, N_ACT, H, B, S, N_REPLAY = 8, 4, 256, 256, 50, 1_000_000


class _Columns:
    """A replay-buffer input that is already in column form (no per-transition Python objects)."""

    def __init__(self, rng, n):
        obs = rng.standard_normal((n + 1, O_DIM)).astype(np.float32)
        self.cols = (obs[:n], rng.integers(0, N_ACT, n).astype(np.float32), rng.standard_normal(n), obs[1:],
                     rng.random(n) < 0.001)

    def transition_columns(self):
        return self.cols


def make(rb, seed=0):
    from rl_replicas_b200.algorithms import DQN
    from rl_replicas_b200.critics import DiscreteQFunction
    from rl_replicas_b200.networks import MLP
    torch.manual_seed(seed)
    env = types.SimpleNamespace(action_space=types.SimpleNamespace(n=N_ACT, shape=()), spec=types.SimpleNamespace(id="stub"),
                                observation_space=types.SimpleNamespace(shape=(O_DIM,)))
    net = MLP([O_DIM, H, H, N_ACT], torch.nn.ReLU)
    algo = DQN(DiscreteQFunction(net, torch.optim.Adam(net.parameters(), lr=1e-3)), None, env, None, rb, None,
               target_update_interval=1000, double_q=True)
    algo.metrics_manager = None
    return algo


def time_group(rb, K, calls, warmup):
    from rl_replicas_b200.algorithms import LearnerGroup
    g = LearnerGroup()
    for k in range(K):
        np.random.seed(k)
        g.add(make(rb, seed=k))
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
    ap.add_argument("--oracle-calls", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dqn.py needs a CUDA device: there is no CPU fallback")
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    rng = np.random.default_rng(0)
    rb = ReplayBuffer(buffer_size=N_REPLAY)
    rb.add_experience(_Columns(rng, N_REPLAY))
    np.random.seed(0)
    algo = make(rb)
    res = time_calls(algo, rb, args.calls, args.warmup)
    groups = {f"K={K}": time_group(rb, K, args.calls, args.warmup) for K in (1, 2, 4, 8, 16)}
    oracle = OD.DqnOracle(algo.q_function.network, algo.target_q_function.network, algo.q_function.optimizer,
                          target_update_interval=1000, double_q=True)
    oracle_ms = []
    for _ in range(args.oracle_calls):
        mbs = [rb.sample_minibatch(B) for _ in range(S)]
        t0 = time.perf_counter()
        oracle.train(mbs)
        oracle_ms.append((time.perf_counter() - t0) * 1e3)
    name, power = card()
    print(json.dumps({
        "workload": f"DQN.train, obs {O_DIM}, {N_ACT} actions, {H}-{H} ReLU, B {B}, {S} steps per call, "
                    f"{N_REPLAY} transitions on the device, Double DQN",
        "dqn": res, "groups": groups,
        "oracle_cpu_ms_per_call": round(float(np.median(oracle_ms)), 1), "cpu_threads": torch.get_num_threads(),
        "gpu": name, "power_limit": power}))


if __name__ == "__main__":
    main()
