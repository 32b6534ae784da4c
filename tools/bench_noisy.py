"""DQN, C51 and QR-DQN train() throughput with noisy Q networks beside the same networks without noise at a
LunarLander shape.

    python tools/bench_noisy.py [--calls 20] [--warmup 3] [--rounds 3]

Workload: obs 8, 4 actions, ReLU, minibatch 256, 50 train steps per train() call, Double DQN, 1 M transitions resident
on the device, uniform device draws; K = 1 for DQN, 51 atoms for C51, 200 quantiles for QR-DQN.  Per algorithm four
arms: MLP([8, 256, 256, 4 K]) against NoisyMLP([8, 256, 256, 4 K]), and DuelingMLP([8, 256, 256], 4, K) against
DuelingMLP(..., noisy=True).  The twelve arms alternate in `rounds` rounds of `calls` timed calls each, so all see the
same machine state.  Prints one JSON line: per arm the median ms per train() call end to end (host state sync
included) and engine-only, engine train steps/s and .train steps/s, launches per step, the noisy-over-plain
engine-time ratios, and the card's name and power limit read in this run.  Needs a GPU; there is no CPU fallback."""
import argparse
import json
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_dqn import B, H, N_REPLAY, O_DIM, S  # noqa: E402
from bench_per import Timer  # noqa: E402
from bench_qr import N_ATOMS, N_QUANT, _Episodes, buffer  # noqa: E402
from bench_sac import card  # noqa: E402

N_ACT = 4


def make(kind, dueling, noisy, rb, seed=0):
    from rl_replicas_b200.algorithms import C51, DQN, QRDQN
    from rl_replicas_b200.critics import CategoricalQFunction, DiscreteQFunction, QuantileQFunction
    from rl_replicas_b200.networks import MLP, DuelingMLP, NoisyMLP
    torch.manual_seed(seed)
    env = types.SimpleNamespace(action_space=types.SimpleNamespace(n=N_ACT, shape=()),
                                spec=types.SimpleNamespace(id="stub"), observation_space=types.SimpleNamespace(shape=(O_DIM,)))
    K = {"dqn": 1, "c51": N_ATOMS, "qr": N_QUANT}[kind]
    if dueling:
        net = DuelingMLP([O_DIM, H, H], N_ACT, K, torch.nn.ReLU, noisy=noisy)
    else:
        net = (NoisyMLP if noisy else MLP)([O_DIM, H, H, N_ACT * K], torch.nn.ReLU)
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    kw = dict(target_update_interval=1000, double_q=True)
    if kind == "c51":
        algo = C51(CategoricalQFunction(net, opt, n_atoms=N_ATOMS), None, env, None, rb, None, **kw)
    elif kind == "qr":
        algo = QRDQN(QuantileQFunction(net, opt, n_quantiles=N_QUANT), None, env, None, rb, None, **kw)
    else:
        algo = DQN(DiscreteQFunction(net, opt), None, env, None, rb, None, **kw)
    algo.metrics_manager = None
    algo.use_device_rng = True
    algo.device_rng_seed = seed
    return algo


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_noisy.py needs a CUDA device: there is no CPU fallback")
    rb = buffer(_Episodes(np.random.default_rng(0), N_REPLAY, N_ACT))
    arm = lambda kind, d, nz: f"{kind}{' dueling' if d else ''}{' noisy' if nz else ''}"
    timers = {arm(kind, d, nz): Timer(make(kind, d, nz, rb), False)
              for kind in ("dqn", "c51", "qr") for d in (False, True) for nz in (False, True)}
    for _ in range(args.rounds):
        for t in timers.values():
            t.run(args.calls, args.warmup)
    res = {k: t.result() for k, t in timers.items()}
    ratios = {f"{arm(k, d, True)} over {arm(k, d, False)} engine time":
              round(res[arm(k, d, True)]["engine_ms"] / res[arm(k, d, False)]["engine_ms"], 3)
              for k in ("dqn", "c51", "qr") for d in (False, True)}
    name, power = card()
    print(json.dumps({
        "workload": f"train(), obs {O_DIM}, {N_ACT} actions, NoisyMLP([{O_DIM}, {H}, {H}, {N_ACT} K]) against MLP, "
                    f"DuelingMLP([{O_DIM}, {H}, {H}], {N_ACT}, K, noisy=True) against noisy=False, ReLU, B {B}, {S} "
                    f"steps per call, {N_REPLAY} transitions on the device, Double DQN, uniform device draws; K = 1 "
                    f"(DQN), {N_ATOMS} (C51), {N_QUANT} (QR-DQN)",
        **res, **ratios, "gpu": name, "power_limit": power}))


if __name__ == "__main__":
    main()
