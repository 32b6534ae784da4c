"""The fused PPO step with both networks against each network alone.  Times, on BASELINE config 2, the stages
fused_step_kernel, fused_step_kernel_policy and fused_step_kernel_value alternately in one process and prints one JSON
line.

    python tools/bench_fused_split.py [--envs N] [--rounds R] [--reps N] [--lib-ms MS]

Every CTA of the step kernel runs one network on the tiles of its slot, so the two-network launch should take about
the sum of the two one-network launches (`one_network_sum_ratio` near 1): what each network costs, and how much the
two waves of CTAs overlap.

Under the timing build (tools/tc3_timing.sh, B200RL_TC3_TIMING=1 B200RL_LIB=...) it also reads the per-tile cycle
counters of CTA 0 (the policy network's, or the value network's in a value-only launch) and prints each chain
warpgroup's own work and waits per tile and each gradient warpgroup's waits and issue time.  `chain_bound_share` =
(policy chain work + value chain work per tile of the one-network launches) / (cycles per tile of the two-network
launch's CTA 0); with --lib-ms (the library's fused_step_kernel time) it is also given in ms.  The timing build runs
slower than the library, so its cycles are only used as shares of a tile.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import bench  # noqa: E402
from rl_replicas_b200 import synthetic  # noqa: E402

STAGES = ("fused_step_kernel", "fused_step_kernel_policy", "fused_step_kernel_value")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=1024)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--lib-ms", type=float, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fused_split.py needs a GPU")
    pl, vl, log_std = bench.make_nets()
    b = bench.make_batch(args.envs, 1000, pl, seed=0)
    ppo = synthetic.onpolicy_learner("ppo", pl, vl, log_std, num_policy_gradients=2, num_value_gradients=2,
                                     max_kl_divergence=float("inf"))
    ppo.train_packed(b)
    e = ppo._engine
    hp = ppo._hparams(e, 0)
    for s in ("preamble", "old_logp", "pack_obs"):
        e.run_stage(s, hp)

    def ms(stage, n):
        e.run_stage(stage, hp)
        torch.cuda.synchronize()
        a, z = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(n):
            e.run_stage(stage, hp)
        z.record()
        torch.cuda.synchronize()
        return a.elapsed_time(z) / n

    times = {s: [] for s in STAGES}
    for _ in range(args.rounds):
        for s in STAGES:
            times[s].append(ms(s, args.reps))
    med = {s: statistics.median(v) for s, v in times.items()}
    props = torch.cuda.get_device_properties(0)
    out = {"gpu": props.name, "sms": props.multi_processor_count, "ms": {s: round(v, 4) for s, v in med.items()},
           "ms_spread": {s: round(max(v) - min(v), 4) for s, v in times.items()},
           "one_network_sum_ms": round(med[STAGES[1]] + med[STAGES[2]], 4),
           "one_network_sum_ratio": round((med[STAGES[1]] + med[STAGES[2]]) / med[STAGES[0]], 4)}

    if os.environ.get("B200RL_TC3_TIMING"):
        import ctypes as C
        from rl_replicas_b200 import _lib
        lib = _lib.load()
        cyc = {}
        for s in STAGES:
            buf = (C.c_ulonglong * 64)()
            lib.b200rl_debug_tc3_timing(buf, 1)
            e.run_stage(s, hp)
            torch.cuda.synchronize()
            lib.b200rl_debug_tc3_timing(buf, 0)
            tiles = max(int(buf[52]), 1)
            chains = {}
            # CTA 0 runs the policy network unless only the value network runs
            net = "v" if s.endswith("value") else "p"
            for wg in range(2):
                wait = [int(buf[10 * wg + i]) // tiles for i in range(5)]
                work = [(int(buf[10 * wg + 5 + i]) - int(buf[10 * wg + i])) // tiles for i in range(5)]
                chains[f"{net}{wg}"] = {"work": sum(work), "wait": sum(wait), "work_by_stage": work, "wait_by_stage": wait}
            grad = {f"{'hl'[g]}": {"wait": [int(buf[40 + 3 * g + i]) // tiles for i in range(3)],
                                   "issue": [int(buf[46 + 3 * g + i]) // tiles for i in range(3)]} for g in range(2)}
            cyc[s] = {"tiles": tiles, "tile_cycles": int(buf[54]) // tiles, "chains": chains, "gradient": grad}
        out["timing_build"] = cyc

        def own(stage, net):
            return max(v["work"] for k, v in cyc[stage]["chains"].items() if k[0] == net)

        w_split = own(STAGES[1], "p") + own(STAGES[2], "v")
        out["chain_bound_share"] = round(w_split / cyc[STAGES[0]]["tile_cycles"], 4)
        if args.lib_ms:
            out["chain_bound_ms"] = round(args.lib_ms * out["chain_bound_share"], 4)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
