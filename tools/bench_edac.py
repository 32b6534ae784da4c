"""EDAC.train throughput at the HalfCheetah shape, against SAC-N, REDQ and SAC at the same shape in the same process.

    python tools/bench_edac.py [--calls 6] [--rounds 3] [--steps 200] [--profile]

Workload: HalfCheetah-shaped (obs 17, act 6), 256-256 ReLU networks, minibatch 256, learned alpha, a replay of 200k
transitions resident on the device (uniform host draws, device gather), S train steps per train() call.  Arms, timed in
alternating rounds so that all see the same machine state: EDAC with N = 10 critics at eta = 1, SAC-N (the same at
eta = 0), REDQ with N = 10, M = 2, G = 20, and SAC.  Also reports LearnerGroup.train at K = 1 / 4 / 16 EDAC learners
(one shared replay).  --profile instead runs one EDAC call at eta = 1 and one at eta = 0 under torch.profiler and prints
the device time per step of each kernel family; the diversity pass's cost is the difference of the two totals.  Prints
one JSON line, with the card's name and power limit read in this run.  Needs a GPU; there is no CPU fallback."""
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
    from rl_replicas_b200.algorithms import EDAC, REDQ, SAC
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import RandomPolicy, SquashedGaussianPolicy
    from rl_replicas_b200.q_function import QFunction
    torch.manual_seed(seed)
    hi = np.ones(A_DIM, np.float32)
    env = types.SimpleNamespace(action_space=types.SimpleNamespace(high=hi, low=-hi, shape=(A_DIM,)),
                                spec=types.SimpleNamespace(id="stub"))
    pnet = MLP([O_DIM, H, H, 2 * A_DIM], torch.nn.ReLU)
    policy = SquashedGaussianPolicy(pnet, torch.optim.Adam(pnet.parameters(), lr=3e-4))
    qs = [MLP([O_DIM + A_DIM, H, H, 1], torch.nn.ReLU) for _ in range(2 if kind == "sac" else n)]
    qfs = [QFunction(q, torch.optim.Adam(q.parameters(), lr=3e-4)) for q in qs]
    if kind == "edac":
        algo = EDAC(policy, RandomPolicy(None), qfs, env, None, rb, None, learn_alpha=True, eta=1.0)
    elif kind == "sac_n":
        algo = EDAC(policy, RandomPolicy(None), qfs, env, None, rb, None, learn_alpha=True, eta=0.0)
    elif kind == "redq":
        algo = REDQ(policy, RandomPolicy(None), qfs, env, None, rb, None, learn_alpha=True, n_min=2, policy_delay=20)
    else:
        algo = SAC(policy, RandomPolicy(None), qfs[0], qfs[1], env, None, rb, None, learn_alpha=True)
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
        g.add(make("edac", rb, seed=k))
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
    """Device time per step of each kernel family over one EDAC.train call at eta = 1 and one at eta = 0 (N = 10)."""
    from torch.profiler import ProfilerActivity, profile as prof
    out = {}
    for kind in ("edac", "sac_n"):
        algo = make(kind, rb)
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
            # gemm_ens_kernel<4, ...> is the diversity pass's tangent forward; its other products share the
            # instantiations of the TD pass, so the pass as a whole is the difference between the two runs' totals
            k = next((f for f in ("gemm_ens_kernel<4", "gemm_ens_kernel", "gemm_kernel", "edac_diversity",
                                  "edac_policy_loss", "redq_q_loss", "redq_target", "redq_squash_backward",
                                  "redq_adam", "adam_step", "polyak", "sac_", "gather_rows") if f in n), "other")
            fam[k] = fam.get(k, 0.0) + t
        out[kind] = {k: round(v / 1e3 / S, 4) for k, v in sorted(fam.items(), key=lambda x: -x[1])}
        out[kind]["total"] = round(sum(fam.values()) / 1e3 / S, 4)
    out["diversity_pass_ms_per_step"] = round(out["edac"]["total"] - out["sac_n"]["total"], 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=6)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_edac.py needs a CUDA device: there is no CPU fallback")
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    rng = np.random.default_rng(0)
    rb = ReplayBuffer(buffer_size=N_REPLAY)
    rb.add_experience(_Columns(rng, N_REPLAY))
    np.random.seed(0)
    S = args.steps
    name, power = card()
    if args.profile:
        print(json.dumps({"workload": f"one EDAC.train call each at eta 1 and eta 0, N 10, B {B}, 200 steps, learned "
                                      "alpha, torch.profiler", "device_ms_per_step": profile(rb, 200), "gpu": name,
                          "power_limit": power}))
        return
    arms = ("edac", "sac_n", "redq", "sac")
    timers = {k: Timer(make(k, rb), rb, S) for k in arms}
    for t in timers.values():
        t.run(1, record=False)
    per_round = max(1, args.calls // args.rounds)
    for _ in range(args.rounds):  # alternate the arms so that all see the same machine state
        for t in timers.values():
            t.run(per_round)
    groups = {f"K={K}": time_group(rb, K, S, 3) for K in (1, 4, 16)}
    print(json.dumps({
        "workload": f"obs {O_DIM} act {A_DIM}, {H}-{H} ReLU, N 10, B {B}, {S} steps per call, {N_REPLAY} transitions "
                    "on the device, learned alpha; edac eta 1, sac_n eta 0, redq M 2 G 20",
        **{k: timers[k].result() for k in arms}, "edac_learner_group": groups, "gpu": name, "power_limit": power}))


if __name__ == "__main__":
    main()
