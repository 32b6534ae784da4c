"""TQC.train throughput at the HalfCheetah shape, against SAC.train at the same shape in the same process.

    python tools/bench_tqc.py [--calls 20] [--warmup 3] [--rounds 3] [--oracle-calls 2]

Workload: HalfCheetah-shaped (obs 17, act 6), 256-256 ReLU networks, TQC with M = 25 quantiles per critic and d = 2
dropped per critic, minibatch 256, 50 train steps per train() call, learned alpha, replay of 1 M transitions resident
on the device (uniform host draws, device gather).  TQC and SAC calls are timed in alternating rounds, so both see the
same machine state.  Also times LearnerGroup.train at K = 1 / 4 / 16 TQC learners (one shared replay) and the
torch-CPU oracle per call.  Prints one JSON line with median ms per call end to end (host state sync included) and
engine-only, train steps/s, and the card's name and power limit read in this run.  Needs a GPU; there is no CPU
fallback."""
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
from oracle import tqc as OT  # noqa: E402

O_DIM, A_DIM, H, B, S, N_REPLAY, M, D_DROP = 17, 6, 256, 256, 50, 1_000_000, 25, 2


def make(kind, rb, seed=0):
    from rl_replicas_b200.algorithms import SAC, TQC
    from rl_replicas_b200.critics import ContinuousQuantileQFunction
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import RandomPolicy, SquashedGaussianPolicy
    from rl_replicas_b200.q_function import QFunction
    torch.manual_seed(seed)
    hi = np.ones(A_DIM, np.float32)
    env = types.SimpleNamespace(action_space=types.SimpleNamespace(high=hi, low=-hi, shape=(A_DIM,)),
                                spec=types.SimpleNamespace(id="stub"))
    pnet = MLP([O_DIM, H, H, 2 * A_DIM], torch.nn.ReLU)
    policy = SquashedGaussianPolicy(pnet, torch.optim.Adam(pnet.parameters(), lr=1e-3))
    if kind == "tqc":
        qs = [MLP([O_DIM + A_DIM, H, H, M], torch.nn.ReLU) for _ in range(2)]
        qfs = [ContinuousQuantileQFunction(q, torch.optim.Adam(q.parameters(), lr=1e-3), n_quantiles=M) for q in qs]
        algo = TQC(policy, RandomPolicy(None), qfs[0], qfs[1], env, None, rb, None, learn_alpha=True,
                   top_quantiles_to_drop_per_net=D_DROP)
    else:
        qs = [MLP([O_DIM + A_DIM, H, H, 1], torch.nn.ReLU) for _ in range(2)]
        qfs = [QFunction(q, torch.optim.Adam(q.parameters(), lr=1e-3)) for q in qs]
        algo = SAC(policy, RandomPolicy(None), qfs[0], qfs[1], env, None, rb, None, learn_alpha=True)
    algo.metrics_manager = None
    return algo


class Timer:
    """Times algo.train end to end and its engine call (which ends in the read-back's stream synchronisation)."""

    def __init__(self, algo, rb):
        self.algo, self.rb, self.call_ms, self.engine_ms = algo, rb, [], []
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
            self.algo.train(self.rb, S, B)
            torch.cuda.synchronize()
            if record:
                self.call_ms.append((time.perf_counter() - t0) * 1e3)
        if not record:
            del self.engine_ms[n_eng:]

    def result(self):
        med, eng = float(np.median(self.call_ms)), float(np.median(self.engine_ms))
        return {"train_call_ms": round(med, 3), "engine_ms": round(eng, 3),
                "train_steps_per_s": round(S / med * 1e3, 1), "engine_steps_per_s": round(S / eng * 1e3, 1)}


def time_group(rb, K, calls, warmup):
    from rl_replicas_b200.algorithms import LearnerGroup
    g = LearnerGroup()
    for k in range(K):
        g.add(make("tqc", rb, seed=k))
    for _ in range(warmup + 1):
        g.train(S, B)
    ms = []
    for _ in range(calls):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        g.train(S, B)
        torch.cuda.synchronize()
        ms.append((time.perf_counter() - t0) * 1e3)
    med = float(np.median(ms))
    return {"train_call_ms": round(med, 3), "learner_steps_per_s": round(K * S / med * 1e3, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--group-calls", type=int, default=10)
    ap.add_argument("--oracle-calls", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tqc.py needs a CUDA device: there is no CPU fallback")
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    rng = np.random.default_rng(0)
    rb = ReplayBuffer(buffer_size=N_REPLAY)
    rb.add_experience(_Columns(rng, N_REPLAY))
    np.random.seed(0)
    timers = {"tqc": Timer(make("tqc", rb), rb), "sac": Timer(make("sac", rb), rb)}
    for t in timers.values():
        t.run(args.warmup, record=False)
    per_round = max(1, args.calls // args.rounds)
    for _ in range(args.rounds):  # alternate the two so that both see the same machine state
        for t in timers.values():
            t.run(per_round)
    groups = {f"K={K}": time_group(rb, K, args.group_calls, args.warmup) for K in (1, 4, 16)}
    tqc = timers["tqc"].algo
    oracle = OT.TqcOracle(tqc.policy.network, tqc.q_function_1.network, tqc.q_function_2.network, n_quantiles=M,
                          n_drop=D_DROP, learn_alpha=True)
    oracle_ms = []
    for _ in range(args.oracle_calls):
        mbs = [rb.sample_minibatch(B) for _ in range(S)]
        noise = np.random.standard_normal((S, 2, B, A_DIM)).astype(np.float32)
        t0 = time.perf_counter()
        oracle.train(mbs, noise)
        oracle_ms.append((time.perf_counter() - t0) * 1e3)
    name, power = card()
    print(json.dumps({
        "workload": f"TQC.train, obs {O_DIM} act {A_DIM}, {H}-{H} ReLU, M {M} d {D_DROP}, B {B}, {S} steps per call, "
                    f"{N_REPLAY} transitions on the device, learned alpha",
        "tqc": timers["tqc"].result(), "sac_same_shape": timers["sac"].result(), "tqc_learner_group": groups,
        "oracle_cpu_ms_per_call": round(float(np.median(oracle_ms)), 1), "cpu_threads": torch.get_num_threads(),
        "gpu": name, "power_limit": power}))


if __name__ == "__main__":
    main()
