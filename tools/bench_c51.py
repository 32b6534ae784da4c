"""C51.train throughput at a LunarLander shape and at a wide one, beside DQN.train at the same shapes, alone and as
learner groups, with the torch-CPU oracle as the baseline.

    python tools/bench_c51.py [--calls 20] [--warmup 3] [--oracle-calls 2]

Workloads: obs 8, 4 actions x 51 atoms (LunarLander) and 18 actions x 51 atoms (a full Atari action set), 256-256 ReLU
Q network, minibatch 256, 50 train steps per train() call, Double DQN, 1 M transitions resident on the device.  Prints
one JSON line: median ms per train() call end to end (host state sync included) and engine-only, train steps/s, for C51
and for DQN at the same shape, their ratio, LearnerGroup.train of C51 at K = 1, 4 and 16, kernel launches per step, the
torch-CPU oracle's ms per call (the CPU baseline), a torch.profiler breakdown of one C51 call at the LunarLander shape
(device time per step by kernel, taken in a separate profiled call), and the card's name and power limit read in this
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
from oracle import c51 as OC  # noqa: E402

O_DIM, H, B, S, N_REPLAY, N_ATOMS = 8, 256, 256, 50, 1_000_000, 51


class _Columns:
    """A replay-buffer input that is already in column form (no per-transition Python objects)."""

    def __init__(self, rng, n, n_actions):
        obs = rng.standard_normal((n + 1, O_DIM)).astype(np.float32)
        self.cols = (obs[:n], rng.integers(0, n_actions, n).astype(np.float32), rng.standard_normal(n), obs[1:],
                     rng.random(n) < 0.001)

    def transition_columns(self):
        return self.cols


def make(kind, n_actions, rb, seed=0):
    from rl_replicas_b200.algorithms import C51, DQN
    from rl_replicas_b200.critics import CategoricalQFunction, DiscreteQFunction
    from rl_replicas_b200.networks import MLP
    torch.manual_seed(seed)
    env = types.SimpleNamespace(action_space=types.SimpleNamespace(n=n_actions, shape=()),
                                spec=types.SimpleNamespace(id="stub"), observation_space=types.SimpleNamespace(shape=(O_DIM,)))
    width = n_actions * (N_ATOMS if kind == "c51" else 1)
    net = MLP([O_DIM, H, H, width], torch.nn.ReLU)
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    if kind == "c51":
        algo = C51(CategoricalQFunction(net, opt, n_atoms=N_ATOMS), None, env, None, rb, None,
                   target_update_interval=1000, double_q=True)
    else:
        algo = DQN(DiscreteQFunction(net, opt), None, env, None, rb, None, target_update_interval=1000, double_q=True)
    algo.metrics_manager = None
    return algo


def time_group(rb, n_actions, K, calls, warmup):
    from rl_replicas_b200.algorithms import LearnerGroup
    g = LearnerGroup()
    for k in range(K):
        np.random.seed(k)
        g.add(make("c51", n_actions, rb, seed=k))
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


def launches_per_step(algo, rb):
    from rl_replicas_b200 import _lib
    lib = _lib.load()
    n0 = lib.b200rl_launch_count()
    algo.train(rb, S, B)
    return (lib.b200rl_launch_count() - n0) / S


def profile_step(algo, rb):
    """Device time per train step by kernel name, from one profiled train() call (after the timed ones)."""
    from torch.profiler import ProfilerActivity, profile
    algo.train(rb, S, B)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        algo.train(rb, S, B)
        torch.cuda.synchronize()
    per = {}
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            key = ev.name.split("<")[0].split("(")[0].replace("void ", "").replace("b200rl::", "")
            per[key] = per.get(key, 0.0) + ev.device_time_total
    total = sum(per.values())
    top = sorted(per.items(), key=lambda kv: -kv[1])
    return {"device_us_per_step": round(total / S, 2),
            "by_kernel_us_per_step": {k: round(v / S, 2) for k, v in top[:8]}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--oracle-calls", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_c51.py needs a CUDA device: there is no CPU fallback")
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    out = {}
    for n_actions, label in ((4, "lunar"), (18, "wide")):
        rng = np.random.default_rng(0)
        rb = ReplayBuffer(buffer_size=N_REPLAY)
        rb.add_experience(_Columns(rng, N_REPLAY, n_actions))
        res = {}
        for kind in ("dqn", "c51"):  # in the same run, at the same shape
            np.random.seed(0)
            algo = make(kind, n_actions, rb)
            res[kind] = time_calls(algo, rb, args.calls, args.warmup)
            res[kind]["launches_per_step"] = launches_per_step(algo, rb)
        res["c51_over_dqn_call_time"] = round(res["c51"]["train_call_ms"] / res["dqn"]["train_call_ms"], 3)
        res["c51_over_dqn_engine_time"] = round(res["c51"]["engine_ms"] / res["dqn"]["engine_ms"], 3)
        if label == "lunar":
            res["groups"] = {f"K={K}": time_group(rb, n_actions, K, args.calls, args.warmup) for K in (1, 4, 16)}
            oracle = OC.C51Oracle(algo.q_function.network, algo.target_q_function.network, algo.q_function.optimizer,
                                  n_atoms=N_ATOMS, target_update_interval=1000, double_q=True)
            oracle_ms = []
            for _ in range(args.oracle_calls):
                mbs = [rb.sample_minibatch(B) for _ in range(S)]
                t0 = time.perf_counter()
                oracle.train(mbs)
                oracle_ms.append((time.perf_counter() - t0) * 1e3)
            res["oracle_cpu_ms_per_call"] = round(float(np.median(oracle_ms)), 1)
            res["profile"] = profile_step(algo, rb)
        out[label] = res
        del rb
    name, power = card()
    print(json.dumps({
        "workload": f"C51.train vs DQN.train, obs {O_DIM}, 4 and 18 actions x {N_ATOMS} atoms, {H}-{H} ReLU, B {B}, "
                    f"{S} steps per call, {N_REPLAY} transitions on the device, Double DQN",
        **out, "cpu_threads": torch.get_num_threads(), "gpu": name, "power_limit": power}))


if __name__ == "__main__":
    main()
