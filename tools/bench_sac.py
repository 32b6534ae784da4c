"""SAC.train throughput at the Spinning Up / reference recipe's shape, with TD3 at the same shape in the same process.

    python tools/bench_sac.py [--calls 20] [--warmup 3] [--oracle-calls 2]

Workload: HalfCheetah-shaped (obs 17, act 6), 256-256 ReLU networks, minibatch 256, 50 train steps per train() call
(the recipe's 50 updates every 50 env steps), replay of 1 M transitions resident on the device.  Prints one JSON line:
median ms per SAC.train call end to end (host state sync included) and engine-only, train steps/s, the same for TD3,
the torch-CPU oracle's ms per call (the CPU baseline), and the card's name and power limit read in this run.  Needs a
GPU; there is no CPU fallback."""
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

from oracle import sac as OS  # noqa: E402

O_DIM, A_DIM, H, B, S, N_REPLAY = 17, 6, 256, 256, 50, 1_000_000


class _Columns:
    """A replay-buffer input that is already in column form (no per-transition Python objects)."""

    def __init__(self, rng, n):
        obs = rng.standard_normal((n + 1, O_DIM)).astype(np.float32)
        self.cols = (obs[:n], rng.uniform(-1, 1, (n, A_DIM)).astype(np.float32), rng.standard_normal(n),
                     obs[1:], rng.random(n) < 0.001)

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


def make(kind, rb):
    from rl_replicas_b200.algorithms import SAC, TD3
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import DeterministicPolicy, RandomPolicy, SquashedGaussianPolicy
    from rl_replicas_b200.q_function import QFunction
    torch.manual_seed(0)
    hi = np.ones(A_DIM, np.float32)
    env = types.SimpleNamespace(action_space=types.SimpleNamespace(high=hi, low=-hi, shape=(A_DIM,)),
                                spec=types.SimpleNamespace(id="stub"))
    qs = [MLP([O_DIM + A_DIM, H, H, 1], torch.nn.ReLU) for _ in range(2)]
    qfs = [QFunction(q, torch.optim.Adam(q.parameters(), lr=1e-3)) for q in qs]
    if kind == "sac":
        pnet = MLP([O_DIM, H, H, 2 * A_DIM], torch.nn.ReLU)
        algo = SAC(SquashedGaussianPolicy(pnet, torch.optim.Adam(pnet.parameters(), lr=1e-3)), RandomPolicy(None),
                   qfs[0], qfs[1], env, None, rb, None, learn_alpha=True)
    else:
        pnet = MLP([O_DIM, H, H, A_DIM], torch.nn.ReLU, torch.nn.Tanh)
        algo = TD3(DeterministicPolicy(pnet, torch.optim.Adam(pnet.parameters(), lr=1e-3)), RandomPolicy(None),
                   qfs[0], qfs[1], env, None, rb, None)
    algo.metrics_manager = None
    return algo


def time_calls(algo, rb, calls, warmup):
    algo.train(rb, S, B)  # builds the engine
    engine_ms = []
    f = algo._engine.train_gather

    def timed(*a, **k):
        t0 = time.perf_counter()
        r = f(*a, **k)  # reads the logs back: ends in a stream synchronisation
        engine_ms.append((time.perf_counter() - t0) * 1e3)
        return r
    algo._engine.train_gather = timed
    for _ in range(warmup):
        algo.train(rb, S, B)
    engine_ms.clear()
    per_call = []
    for _ in range(calls):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        algo.train(rb, S, B)
        torch.cuda.synchronize()
        per_call.append((time.perf_counter() - t0) * 1e3)
    algo._engine.train_gather = f
    med, eng = float(np.median(per_call)), float(np.median(engine_ms))
    return {"train_call_ms": round(med, 3), "engine_ms": round(eng, 3), "train_steps_per_s": round(S / med * 1e3, 1),
            "engine_steps_per_s": round(S / eng * 1e3, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--oracle-calls", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sac.py needs a CUDA device: there is no CPU fallback")
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    rng = np.random.default_rng(0)
    rb = ReplayBuffer(buffer_size=N_REPLAY)
    rb.add_experience(_Columns(rng, N_REPLAY))
    np.random.seed(0)
    sac = make("sac", rb)
    res_sac = time_calls(sac, rb, args.calls, args.warmup)
    td3 = make("td3", rb)
    res_td3 = time_calls(td3, rb, args.calls, args.warmup)
    # the CPU baseline: the torch-autograd oracle on the same shape and the same kind of minibatches
    oracle = OS.SacOracle(sac.policy.network, sac.q_function_1.network, sac.q_function_2.network, learn_alpha=True)
    oracle_ms = []
    for _ in range(args.oracle_calls):
        mbs = [rb.sample_minibatch(B) for _ in range(S)]
        noise = np.random.standard_normal((S, 2, B, A_DIM)).astype(np.float32)
        t0 = time.perf_counter()
        oracle.train(mbs, noise)
        oracle_ms.append((time.perf_counter() - t0) * 1e3)
    name, power = card()
    print(json.dumps({
        "workload": f"SAC.train, obs {O_DIM} act {A_DIM}, {H}-{H} ReLU, B {B}, {S} steps per call, "
                    f"{N_REPLAY} transitions on the device, learned alpha",
        "sac": res_sac, "td3_same_shape": res_td3,
        "oracle_cpu_ms_per_call": round(float(np.median(oracle_ms)), 1), "cpu_threads": torch.get_num_threads(),
        "gpu": name, "power_limit": power}))


if __name__ == "__main__":
    main()
