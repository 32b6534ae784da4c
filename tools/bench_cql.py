"""CQL.train throughput at the HalfCheetah shape, against SAC.train at the same shape in the same process.

    python tools/bench_cql.py [--steps 1000] [--calls 4] [--warmup 1] [--rounds 2] [--group-calls 2]

Workload: HalfCheetah-shaped (obs 17, act 6), 256-256 ReLU networks, minibatch 256, ``--steps`` train steps per call
(offline training runs long calls), a dataset of 1 M rows resident on the device (uniform host draws, device gather),
fixed alpha.  CQL (N = 10, weight 5) and SAC calls are timed in alternating rounds, so both see the same machine
state; then CQL at N = 1 and 25 and with the Lagrange step, LearnerGroup.train at K = 1 / 4 / 16 CQL learners on the
one dataset, the device time per step split by kernel family from torch.profiler (in a run of its own), and the
torch-CPU oracle per call.  Prints one JSON line with median ms per call end to end and engine-only, train steps/s,
and the card's name and power limit read in this run.  Needs a GPU; there is no CPU fallback."""
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

from bench_sac import _Columns, card  # noqa: E402
from oracle import cql as OC  # noqa: E402

O_DIM, A_DIM, H, B, N_REPLAY = 17, 6, 256, 256, 1_000_000


def make(kind, rb, seed=0, **kw):
    from rl_replicas_b200.algorithms import CQL, SAC
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import SquashedGaussianPolicy
    from rl_replicas_b200.q_function import QFunction
    torch.manual_seed(seed)
    hi = np.ones(A_DIM, np.float32)
    env = types.SimpleNamespace(action_space=types.SimpleNamespace(high=hi, low=-hi, shape=(A_DIM,)),
                                spec=types.SimpleNamespace(id="stub"))
    pnet = MLP([O_DIM, H, H, 2 * A_DIM], torch.nn.ReLU)
    policy = SquashedGaussianPolicy(pnet, torch.optim.Adam(pnet.parameters(), lr=1e-3))
    qs = [MLP([O_DIM + A_DIM, H, H, 1], torch.nn.ReLU) for _ in range(2)]
    qfs = [QFunction(q, torch.optim.Adam(q.parameters(), lr=1e-3)) for q in qs]
    cls = CQL if kind == "cql" else SAC
    algo = cls(policy, None, qfs[0], qfs[1], env, None, rb, None, **kw)
    algo.metrics_manager = None
    return algo


class Timer:
    """Times algo.train end to end and its engine call (which ends in the read-back's stream synchronisation)."""

    def __init__(self, algo, rb, S):
        self.algo, self.rb, self.S, self.call_ms, self.engine_ms = algo, rb, S, [], []
        algo.train(rb, S, B)  # builds the engine and captures the graph
        f = algo._engine.train_gather

        def timed(*a, **k):
            t0 = time.perf_counter()
            r = f(*a, **k)
            self.engine_ms.append((time.perf_counter() - t0) * 1e3)
            return r
        algo._engine.train_gather = timed

    def run(self, calls, record=True):
        n_eng = len(self.engine_ms)
        for _ in range(calls):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            self.algo.train(self.rb, self.S, B)
            torch.cuda.synchronize()
            if record:
                self.call_ms.append((time.perf_counter() - t0) * 1e3)
        if not record:
            del self.engine_ms[n_eng:]

    def result(self):
        med, eng = float(np.median(self.call_ms)), float(np.median(self.engine_ms))
        return {"train_call_ms": round(med, 2), "engine_ms": round(eng, 2),
                "train_steps_per_s": round(self.S / med * 1e3, 1), "engine_steps_per_s": round(self.S / eng * 1e3, 1)}


def time_group(rb, K, S, calls):
    from rl_replicas_b200.algorithms import LearnerGroup
    g = LearnerGroup()
    for k in range(K):
        g.add(make("cql", rb, seed=k))
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
    """Device time per step by kernel family, from one profiled call."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        timer.run(1, record=False)
    fam = {"gemm": 0.0, "sampling": 0.0, "heads": 0.0, "rest": 0.0}
    for ev in prof.key_averages():
        us = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        name = ev.key
        if "gemm_kernel" in name:
            fam["gemm"] += us
        elif "cql_stage" in name or "cql_draw" in name or "sac_squash_kernel" in name:
            fam["sampling"] += us
        elif "loss_kernel" in name or "cql_penalty" in name or "cql_alpha_prime" in name:
            fam["heads"] += us
        else:
            fam["rest"] += us
    total = sum(fam.values())
    return {"device_us_per_step": round(total / timer.S, 1),
            "share": {k: round(v / total, 4) for k, v in fam.items()} if total else {}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--calls", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--group-calls", type=int, default=2)
    ap.add_argument("--oracle-steps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_cql.py needs a CUDA device: there is no CPU fallback")
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    S = args.steps
    rng = np.random.default_rng(0)
    rb = ReplayBuffer(buffer_size=N_REPLAY)
    rb.add_experience(_Columns(rng, N_REPLAY))
    np.random.seed(0)
    timers = {"cql_N10": Timer(make("cql", rb), rb, S), "sac": Timer(make("sac", rb), rb, S)}
    for t in timers.values():
        t.run(args.warmup, record=False)
    per_round = max(1, args.calls // args.rounds)
    for _ in range(args.rounds):  # alternate the two so that both see the same machine state
        for t in timers.values():
            t.run(per_round)
    variants = {"cql_N1": dict(cql_n_actions=1), "cql_N25": dict(cql_n_actions=25),
                "cql_N10_lagrange": dict(cql_target_action_gap=10.0)}
    results = {k: t.result() for k, t in timers.items()}
    for k, kw in variants.items():
        t = Timer(make("cql", rb, **kw), rb, S)
        t.run(per_round)
        results[k] = t.result()
    split = device_split(timers["cql_N10"])
    groups = {f"K={K}": time_group(rb, K, S, args.group_calls) for K in (1, 4, 16)}
    cql = timers["cql_N10"].algo
    oracle = OC.CqlOracle(cql.policy.network, cql.q_function_1.network, cql.q_function_2.network)
    So = args.oracle_steps
    mbs = [rb.sample_minibatch(B) for _ in range(So)]
    t0 = time.perf_counter()
    oracle.train(mbs, cql._noise(So, B))
    oracle_ms_per_step = (time.perf_counter() - t0) * 1e3 / So
    name, power = card()
    print(json.dumps({
        "workload": f"CQL.train, obs {O_DIM} act {A_DIM}, {H}-{H} ReLU, B {B}, {S} steps per call, "
                    f"{N_REPLAY} rows on the device, fixed alpha, weight 5",
        **results, "cql_N10_device_split": split, "cql_learner_group": groups,
        "oracle_cpu_ms_per_call": round(oracle_ms_per_step * S, 1), "cpu_threads": torch.get_num_threads(),
        "gpu": name, "power_limit": power}))


if __name__ == "__main__":
    main()
