"""IQL.train throughput at the HalfCheetah shape, against SAC.train and CQL.train (N = 10) in the same process.

    python tools/bench_iql.py [--steps 200] [--calls 4] [--warmup 1] [--rounds 2] [--group-calls 2]

Workload: HalfCheetah-shaped (obs 17, act 6), 256-256 ReLU networks (V too), minibatch 256, ``--steps`` train steps
per call, a dataset of 1 M rows resident on the device (uniform host draws, device gather).  IQL, SAC and CQL calls are
timed in alternating rounds, so all see the same machine state; then LearnerGroup.train at K = 1 / 4 / 16 IQL learners
on the one dataset, and the device time per IQL step split by kernel family from torch.profiler (in a run of its own).
Prints one JSON line with median ms per call end to end and engine-only, train steps/s, and the card's name and power
limit read in this run.  Needs a GPU; there is no CPU fallback."""
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

from bench_cql import B, H, N_REPLAY, A_DIM, O_DIM, Timer  # noqa: E402
from bench_cql import make as make_sac_family  # noqa: E402
from bench_sac import _Columns, card  # noqa: E402


def make_iql(rb, seed=0):
    from rl_replicas_b200.algorithms import IQL
    from rl_replicas_b200.critics import ValueFunction
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import TanhMeanGaussianPolicy
    from rl_replicas_b200.q_function import QFunction
    torch.manual_seed(seed)
    hi = np.ones(A_DIM, np.float32)
    env = types.SimpleNamespace(action_space=types.SimpleNamespace(high=hi, low=-hi, shape=(A_DIM,)),
                                spec=types.SimpleNamespace(id="stub"))
    pnet = MLP([O_DIM, H, H, 2 * A_DIM], torch.nn.ReLU)
    qs = [MLP([O_DIM + A_DIM, H, H, 1], torch.nn.ReLU) for _ in range(2)]
    vnet = MLP([O_DIM, H, H, 1], torch.nn.ReLU)
    algo = IQL(TanhMeanGaussianPolicy(pnet, torch.optim.Adam(pnet.parameters(), lr=3e-4)), None,
               *[QFunction(q, torch.optim.Adam(q.parameters(), lr=3e-4)) for q in qs],
               ValueFunction(vnet, torch.optim.Adam(vnet.parameters(), lr=3e-4)), env, None, rb, None)
    algo.metrics_manager = None
    return algo


def time_group(rb, K, S, calls):
    from rl_replicas_b200.algorithms import LearnerGroup
    g = LearnerGroup()
    for k in range(K):
        g.add(make_iql(rb, seed=k))
    g.train(S, B)
    ms = []
    for _ in range(calls):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        g.train(S, B)
        torch.cuda.synchronize()
        ms.append((time.perf_counter() - t0) * 1e3)
    med = float(np.median(ms))
    return {"train_call_ms": round(med, 2), "learner_steps_per_s": round(K * S / med * 1e3, 1)}


def device_split(timer):
    """Device time per IQL step by kernel family, from one profiled call."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        timer.run(1, record=False)
    fam = {"gemm": 0.0, "iql_heads": 0.0, "critic_heads": 0.0, "adam": 0.0, "rest": 0.0}
    for ev in prof.key_averages():
        us = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        name = ev.key
        if "gemm_kernel" in name:
            fam["gemm"] += us
        elif "iql_value_loss" in name or "iql_policy_loss" in name:
            fam["iql_heads"] += us
        elif "sac_q_loss" in name:
            fam["critic_heads"] += us
        elif "adam" in name:
            fam["adam"] += us
        else:
            fam["rest"] += us
    total = sum(fam.values())
    return {"device_us_per_step": round(total / timer.S, 1),
            "share": {k: round(v / total, 4) for k, v in fam.items()} if total else {}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--calls", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--group-calls", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_iql.py needs a CUDA device: there is no CPU fallback")
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    S = args.steps
    rng = np.random.default_rng(0)
    rb = ReplayBuffer(buffer_size=N_REPLAY)
    rb.add_experience(_Columns(rng, N_REPLAY))
    np.random.seed(0)
    timers = {"iql": Timer(make_iql(rb), rb, S), "sac": Timer(make_sac_family("sac", rb), rb, S),
              "cql_N10": Timer(make_sac_family("cql", rb), rb, S)}
    for t in timers.values():
        t.run(args.warmup, record=False)
    per_round = max(1, args.calls // args.rounds)
    for _ in range(args.rounds):  # alternate the arms so that all see the same machine state
        for t in timers.values():
            t.run(per_round)
    results = {k: t.result() for k, t in timers.items()}
    split = device_split(timers["iql"])
    groups = {f"K={K}": time_group(rb, K, S, args.group_calls) for K in (1, 4, 16)}
    name, power = card()
    print(json.dumps({
        "workload": f"IQL.train, obs {O_DIM} act {A_DIM}, {H}-{H} ReLU, B {B}, {S} steps per call, "
                    f"{N_REPLAY} rows on the device, tau 0.7, beta 3",
        **results, "iql_device_split": split, "iql_learner_group": groups, "gpu": name, "power_limit": power}))


if __name__ == "__main__":
    main()
