"""QRDQN.train throughput at a LunarLander shape beside DQN.train and C51.train, with prioritized replay and n-step
returns, at 18 actions, and as learner groups.

    python tools/bench_qr.py [--calls 20] [--warmup 3] [--rounds 3]

Workload: obs 8, 4 actions x 200 quantiles (LunarLander), 256-256 ReLU Q network, minibatch 256, 50 train steps per
train() call, Double DQN, 1 M transitions resident on the device in episodes of 200 rows.  Arms, alternated in `rounds`
rounds of `calls` timed calls each so all see the same machine state: DQN, C51 (51 atoms), QR-DQN, QR-DQN with
prioritized replay and QR-DQN at n = 3, on uniform device draws (the prioritized arm draws from its tree), and DQN and
QR-DQN at 18 actions.  Then LearnerGroup.train of QR-DQN at K = 1, 4 and 16, and, in a separate torch.profiler run, the
device time per step by kernel of one QR-DQN call (the head is qr_loss_kernel).  Prints one JSON line: per arm the
median ms per train() call end to end (host state sync included) and engine-only, train steps/s and launches per step,
the engine-time ratios against DQN, the group rates, the profile, and the card's name and power limit read in this run.
Needs a GPU; there is no CPU fallback."""
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

from bench_c51 import profile_step  # noqa: E402
from bench_dqn import B, H, N_REPLAY, O_DIM, S  # noqa: E402
from bench_per import Timer  # noqa: E402
from bench_sac import card  # noqa: E402

N_QUANT, N_ATOMS, EPISODE = 200, 51, 200


class _Episodes:
    """Replay columns already in column form, with episode boundaries every EPISODE rows."""

    def __init__(self, rng, n, n_actions):
        obs = rng.standard_normal((n + 1, O_DIM)).astype(np.float32)
        self.cols = (obs[:n], rng.integers(0, n_actions, n).astype(np.float32), rng.standard_normal(n), obs[1:],
                     rng.random(n) < 0.001)
        self.ep_offsets = np.append(np.arange(0, n, EPISODE), n)

    def transition_columns(self):
        return self.cols


def make(kind, n_actions, rb, seed=0, n_step=1):
    from rl_replicas_b200.algorithms import C51, DQN, QRDQN
    from rl_replicas_b200.critics import CategoricalQFunction, DiscreteQFunction, QuantileQFunction
    from rl_replicas_b200.networks import MLP
    torch.manual_seed(seed)
    env = types.SimpleNamespace(action_space=types.SimpleNamespace(n=n_actions, shape=()),
                                spec=types.SimpleNamespace(id="stub"), observation_space=types.SimpleNamespace(shape=(O_DIM,)))
    width = n_actions * {"dqn": 1, "c51": N_ATOMS, "qr": N_QUANT}[kind]
    net = MLP([O_DIM, H, H, width], torch.nn.ReLU)
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    kw = dict(target_update_interval=1000, double_q=True, n_step=n_step)
    if kind == "c51":
        algo = C51(CategoricalQFunction(net, opt, n_atoms=N_ATOMS), None, env, None, rb, None, **kw)
    elif kind == "qr":
        algo = QRDQN(QuantileQFunction(net, opt, n_quantiles=N_QUANT), None, env, None, rb, None, **kw)
    else:
        algo = DQN(DiscreteQFunction(net, opt), None, env, None, rb, None, **kw)
    algo.metrics_manager = None
    algo.use_device_rng = True  # uniform device draws; the prioritized path draws on the device anyway
    algo.device_rng_seed = seed
    return algo


def buffer(cols, prioritized=False):
    from rl_replicas_b200.replay_buffer import PrioritizedReplayBuffer, ReplayBuffer
    rb = PrioritizedReplayBuffer(N_REPLAY) if prioritized else ReplayBuffer(buffer_size=N_REPLAY)
    rb.add_experience(cols)
    return rb


def time_group(rb, K, calls, warmup):
    from rl_replicas_b200.algorithms import LearnerGroup
    g = LearnerGroup()
    for k in range(K):
        np.random.seed(k)
        g.add(make("qr", 4, rb, seed=k))
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
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_qr.py needs a CUDA device: there is no CPU fallback")
    cols4 = _Episodes(np.random.default_rng(0), N_REPLAY, 4)
    cols18 = _Episodes(np.random.default_rng(1), N_REPLAY, 18)
    rb4, rb18 = buffer(cols4), buffer(cols18)
    arms = {
        "dqn": (make("dqn", 4, rb4), False), "c51": (make("c51", 4, rb4), False), "qr": (make("qr", 4, rb4), False),
        "qr per": (make("qr", 4, buffer(cols4, True)), True), "qr n=3": (make("qr", 4, rb4, n_step=3), False),
        "dqn 18 actions": (make("dqn", 18, rb18), False), "qr 18 actions": (make("qr", 18, rb18), False),
    }
    timers = {k: Timer(algo, per) for k, (algo, per) in arms.items()}
    for _ in range(args.rounds):
        for t in timers.values():
            t.run(args.calls, args.warmup)
    res = {k: t.result() for k, t in timers.items()}
    ratios = {f"{k} over dqn engine time": round(res[k]["engine_ms"] / res["dqn"]["engine_ms"], 3)
              for k in ("c51", "qr", "qr per", "qr n=3")}
    ratios["qr over dqn engine time, 18 actions"] = round(res["qr 18 actions"]["engine_ms"] /
                                                          res["dqn 18 actions"]["engine_ms"], 3)
    del timers, arms
    groups = {f"K={K}": time_group(rb4, K, args.calls, args.warmup) for K in (1, 4, 16)}
    prof = profile_step(make("qr", 4, rb4), rb4)
    head = prof["by_kernel_us_per_step"].get("qr_loss_kernel")
    name, power = card()
    print(json.dumps({
        "workload": f"train(), obs {O_DIM}, 4 and 18 actions, {H}-{H} ReLU, B {B}, {S} steps per call, {N_REPLAY} "
                    f"transitions on the device in episodes of {EPISODE}, Double DQN, uniform device draws; QR-DQN "
                    f"{N_QUANT} quantiles, C51 {N_ATOMS} atoms",
        **res, **ratios, "qr_groups": groups, "qr_profile": prof, "qr_head_us_per_step": head,
        "gpu": name, "power_limit": power}))


if __name__ == "__main__":
    main()
