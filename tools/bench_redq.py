"""REDQ.train throughput at the HalfCheetah shape, against SAC.train at the same shape in the same process.

    python tools/bench_redq.py [--calls 6] [--rounds 3] [--steps 1000] [--profile]

Workload: HalfCheetah-shaped (obs 17, act 6), 256-256 ReLU networks, minibatch 256, REDQ with N = 10 critics, M = 2
drawn per step and a policy step every G = 20 critic steps (the paper's setting), 1000 train steps per train() call
(an update-to-data ratio of 20 at 50 environment steps per call), fixed alpha, a replay of 200k transitions resident on
the device (uniform host draws, device gather).  REDQ and SAC calls are timed in alternating rounds, so both see the
same machine state.  Also reports engine critic steps/s at N = 2 / 5 / 10 / 20, LearnerGroup.train at K = 1 / 4 / 16
REDQ learners (one shared replay), and the graph capture + instantiation time of the first S = 1000 call.  --profile
instead runs one call under torch.profiler and prints the device-time share of each kernel family.  Prints one JSON
line, with the card's name and power limit read in this run.  Needs a GPU; there is no CPU fallback."""
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

O_DIM, A_DIM, H, B, N_REPLAY = 17, 6, 256, 256, 200_000


def make(kind, rb, n=10, seed=0):
    from rl_replicas_b200.algorithms import REDQ, SAC
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import RandomPolicy, SquashedGaussianPolicy
    from rl_replicas_b200.q_function import QFunction
    torch.manual_seed(seed)
    hi = np.ones(A_DIM, np.float32)
    env = types.SimpleNamespace(action_space=types.SimpleNamespace(high=hi, low=-hi, shape=(A_DIM,)),
                                spec=types.SimpleNamespace(id="stub"))
    pnet = MLP([O_DIM, H, H, 2 * A_DIM], torch.nn.ReLU)
    policy = SquashedGaussianPolicy(pnet, torch.optim.Adam(pnet.parameters(), lr=3e-4))
    qs = [MLP([O_DIM + A_DIM, H, H, 1], torch.nn.ReLU) for _ in range(n if kind == "redq" else 2)]
    qfs = [QFunction(q, torch.optim.Adam(q.parameters(), lr=3e-4)) for q in qs]
    if kind == "redq":
        algo = REDQ(policy, RandomPolicy(None), qfs, env, None, rb, None, n_min=2, policy_delay=20)
    else:
        algo = SAC(policy, RandomPolicy(None), qfs[0], qfs[1], env, None, rb, None)
    algo.metrics_manager = None
    return algo


class Timer:
    """Times algo.train end to end and its engine call (which ends in the read-back's stream synchronisation)."""

    def __init__(self, algo, rb, S):
        self.algo, self.rb, self.S, self.call_ms, self.engine_ms = algo, rb, S, [], []
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        algo.train(rb, S, B)  # builds the engine and captures the graph
        torch.cuda.synchronize()
        self.first_ms = (time.perf_counter() - t0) * 1e3
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
                "train_steps_per_s": round(self.S / med * 1e3, 1), "engine_steps_per_s": round(self.S / eng * 1e3, 1),
                "first_call_ms": round(self.first_ms, 1),
                "graph_capture_and_instantiate_ms": round(self.first_ms - med, 1)}


def time_group(rb, K, S, calls):
    from rl_replicas_b200.algorithms import LearnerGroup
    g = LearnerGroup()
    for k in range(K):
        g.add(make("redq", rb, seed=k))
    for _ in range(2):
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


def profile(rb, S):
    """Device-time share of each kernel family over one REDQ.train call (N = 10) under torch.profiler."""
    from torch.profiler import ProfilerActivity, profile as prof
    algo = make("redq", rb)
    algo.train(rb, S, B)
    torch.cuda.synchronize()
    with prof(activities=[ProfilerActivity.CUDA]) as p:
        algo.train(rb, S, B)
        torch.cuda.synchronize()
    fam = {}
    for ev in p.key_averages():
        t = getattr(ev, "device_time_total", None)
        t = ev.cuda_time_total if t is None else t
        if t <= 0:
            continue
        n = ev.key
        k = next((f for f in ("gemm_ens_kernel", "gemm_kernel", "redq_q_loss", "redq_target", "redq_policy_loss",
                              "redq_squash_backward", "redq_draw", "adam_step", "polyak", "sac_", "gather_rows")
                  if f in n), "other")
        fam[k] = fam.get(k, 0.0) + t
    tot = sum(fam.values())
    return {k: round(v / tot, 4) for k, v in sorted(fam.items(), key=lambda x: -x[1])}, round(tot / 1e3 / S, 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=6)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_redq.py needs a CUDA device: there is no CPU fallback")
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    rng = np.random.default_rng(0)
    rb = ReplayBuffer(buffer_size=N_REPLAY)
    rb.add_experience(_Columns(rng, N_REPLAY))
    np.random.seed(0)
    S = args.steps
    name, power = card()
    if args.profile:
        shares, ms_per_step = profile(rb, 200)
        print(json.dumps({"workload": f"one REDQ.train call, N 10 M 2 G 20, B {B}, 200 steps, torch.profiler",
                          "device_time_share": shares, "device_ms_per_step": ms_per_step, "gpu": name,
                          "power_limit": power}))
        return
    timers = {"redq": Timer(make("redq", rb), rb, S), "sac": Timer(make("sac", rb), rb, S)}
    for t in timers.values():
        t.run(1, record=False)
    per_round = max(1, args.calls // args.rounds)
    for _ in range(args.rounds):  # alternate the two so that both see the same machine state
        for t in timers.values():
            t.run(per_round)
    scaling = {}
    for n in (2, 5, 10, 20):
        t = Timer(make("redq", rb, n=n), rb, S)
        t.run(1, record=False)
        t.run(max(2, args.calls // 2))
        scaling[f"N={n}"] = t.result()["engine_steps_per_s"]
    groups = {f"K={K}": time_group(rb, K, 200, 3) for K in (1, 4, 16)}
    print(json.dumps({
        "workload": f"REDQ.train, obs {O_DIM} act {A_DIM}, {H}-{H} ReLU, N 10 M 2 G 20, B {B}, {S} steps per call, "
                    f"{N_REPLAY} transitions on the device, fixed alpha",
        "redq": timers["redq"].result(), "sac_same_shape": timers["sac"].result(),
        "redq_engine_steps_per_s_by_n": scaling, "redq_learner_group_200_steps": groups,
        "gpu": name, "power_limit": power}))


if __name__ == "__main__":
    main()
