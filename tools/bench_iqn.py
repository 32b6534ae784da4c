"""IQN.train throughput at a LunarLander shape beside QR-DQN's, at minibatches of 32 (the paper's) and 256, and as
learner groups.

    python tools/bench_iqn.py [--calls 20] [--warmup 3] [--rounds 3]

Workload: obs 8, 4 actions, a 256-256 ReLU network (IQN: d = 256, h = 256, n_cos = 64, N = N' = 64, K = 32; QR-DQN:
200 quantiles), 50 train steps per train() call, Double DQN, 1 M transitions resident on the device, uniform device
draws.  Arms, alternated in `rounds` rounds of `calls` timed calls each so all see the same machine state: IQN and
QR-DQN at B = 32 and B = 256.  Then LearnerGroup.train of IQN at K = 1, 4 and 16 (B = 32), and, in a separate
torch.profiler run, the device time per step by kernel of one IQN call at each minibatch, with the share of the GEMMs
(gemm_kernel).  Prints one JSON line: per arm the median ms per train() call end to end (host state sync included) and
engine-only, train steps/s and launches per step, the group rates, the profiles, and the card's name and power limit
read in this run.  Needs a GPU; there is no CPU fallback."""
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

from bench_dqn import H, N_REPLAY, O_DIM, S  # noqa: E402
from bench_sac import card  # noqa: E402

N_COS, N, N_TARGET, K_POLICY, N_QUANT = 64, 64, 64, 32, 200


def make(kind, rb, seed=0):
    from rl_replicas_b200.algorithms import IQN, QRDQN
    from rl_replicas_b200.critics import ImplicitQuantileQFunction, QuantileQFunction
    from rl_replicas_b200.networks import MLP, ImplicitQuantileMLP
    torch.manual_seed(seed)
    env = types.SimpleNamespace(action_space=types.SimpleNamespace(n=4, shape=()), spec=types.SimpleNamespace(id="stub"),
                                observation_space=types.SimpleNamespace(shape=(O_DIM,)))
    kw = dict(target_update_interval=1000, double_q=True)
    if kind == "iqn":
        net = ImplicitQuantileMLP([O_DIM, H, H], 4, n_cos=N_COS)
        qf = ImplicitQuantileQFunction(net, torch.optim.Adam(net.parameters(), lr=1e-3), N, N_TARGET, K_POLICY)
        algo = IQN(qf, None, env, None, rb, None, **kw)
    else:
        net = MLP([O_DIM, H, H, 4 * N_QUANT], torch.nn.ReLU)
        qf = QuantileQFunction(net, torch.optim.Adam(net.parameters(), lr=1e-3), n_quantiles=N_QUANT)
        algo = QRDQN(qf, None, env, None, rb, None, **kw)
    algo.metrics_manager = None
    algo.use_device_rng = True
    algo.device_rng_seed = seed
    return algo


class Timer:
    """train() calls of one learner at minibatch B, with the engine call inside timed on its own (it ends in a
    synchronisation)."""

    def __init__(self, algo, B):
        from rl_replicas_b200 import _lib
        self.algo, self.B, self.lib = algo, B, _lib.load()
        algo.train(algo.replay_buffer, S, B)  # builds the engine and the graph
        self.f = algo._engine.train_gather_rng
        self.engine_ms, self.call_ms, self.launches = [], [], []

        def timed(*a, **k):
            t0 = time.perf_counter()
            r = self.f(*a, **k)
            self.engine_ms.append((time.perf_counter() - t0) * 1e3)
            return r
        algo._engine.train_gather_rng = timed

    def run(self, calls, warmup):
        for _ in range(warmup):
            self.algo.train(self.algo.replay_buffer, S, self.B)
        del self.engine_ms[len(self.engine_ms) - warmup:]
        for _ in range(calls):
            torch.cuda.synchronize()
            n0 = self.lib.b200rl_launch_count()
            t0 = time.perf_counter()
            self.algo.train(self.algo.replay_buffer, S, self.B)
            torch.cuda.synchronize()
            self.call_ms.append((time.perf_counter() - t0) * 1e3)
            self.launches.append(self.lib.b200rl_launch_count() - n0)

    def result(self):
        call, eng = float(np.median(self.call_ms)), float(np.median(self.engine_ms))
        return {"train_call_ms": round(call, 3), "engine_ms": round(eng, 3),
                "train_steps_per_s": round(S / call * 1e3, 1), "engine_steps_per_s": round(S / eng * 1e3, 1),
                "launches_per_step": round(float(np.median(self.launches)) / S, 2)}


def time_group(rb, K, B, calls, warmup):
    from rl_replicas_b200.algorithms import LearnerGroup
    g = LearnerGroup()
    for k in range(K):
        np.random.seed(k)
        g.add(make("iqn", rb, seed=k))
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


def profile_step(algo, B):
    """Device time per train step by kernel name from one profiled train() call, and the GEMMs' share of it."""
    from torch.profiler import ProfilerActivity, profile
    rb = algo.replay_buffer
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
            "gemm_share": round(per.get("gemm_kernel", 0.0) / total, 3) if total else None,
            "by_kernel_us_per_step": {k: round(v / S, 2) for k, v in top[:8]}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_iqn.py needs a CUDA device: there is no CPU fallback")
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    rng = np.random.default_rng(0)
    obs = rng.standard_normal((N_REPLAY + 1, O_DIM)).astype(np.float32)
    rb = ReplayBuffer(buffer_size=N_REPLAY)
    rb.add_experience(types.SimpleNamespace(transition_columns=lambda: (
        obs[:N_REPLAY], rng.integers(0, 4, N_REPLAY).astype(np.float32), rng.standard_normal(N_REPLAY), obs[1:],
        rng.random(N_REPLAY) < 0.001), ep_offsets=np.append(np.arange(0, N_REPLAY, 200), N_REPLAY)))
    arms = {f"{kind} B={B}": Timer(make(kind, rb), B) for B in (32, 256) for kind in ("iqn", "qr")}
    for _ in range(args.rounds):
        for t in arms.values():
            t.run(args.calls, args.warmup)
    res = {k: t.result() for k, t in arms.items()}
    del arms
    groups = {f"K={K}": time_group(rb, K, 32, args.calls, args.warmup) for K in (1, 4, 16)}
    prof = {f"B={B}": profile_step(make("iqn", rb), B) for B in (32, 256)}
    name, power = card()
    print(json.dumps({
        "workload": f"train(), obs {O_DIM}, 4 actions, {H}-{H} ReLU, {S} steps per call, {N_REPLAY} transitions on the "
                    f"device, Double DQN, uniform device draws; IQN d {H}, n_cos {N_COS}, N {N}, N' {N_TARGET}, K "
                    f"{K_POLICY}; QR-DQN {N_QUANT} quantiles",
        **res, "iqn_groups_B32": groups, "iqn_profile": prof, "gpu": name, "power_limit": power}))


if __name__ == "__main__":
    main()
