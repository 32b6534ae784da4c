"""BASELINE config 2 on the fused policy + value step: times the single stages with CUDA events and leaves the process
in a state ncu can capture (`ncu -k regex:mlp_tc3 ...`).  Usage: python tools/profile_fused.py [envs] [reps]"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
from rl_replicas_b200 import synthetic  # noqa: E402

if __name__ == "__main__":
    envs = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 10
    pl, vl, log_std = bench.make_nets()
    b = bench.make_batch(envs, 1000, pl, seed=0)
    ppo = synthetic.onpolicy_learner("ppo", pl, vl, log_std, num_policy_gradients=2, num_value_gradients=2,
                                     max_kl_divergence=float("inf"))
    ppo.train_packed(b)  # builds the engine, loads the batch, leaves values / advantages / old log-probs on the device
    e = ppo._engine
    hp = ppo._hparams(e, 0)
    e.run_stage("preamble", hp)
    e.run_stage("old_logp", hp)
    e.run_stage("pack_obs", hp)

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

    out = {s: ms(s, reps) for s in ("pack_obs", "fused_step_kernel", "fused_step", "policy_grad_kernel", "value_grad_kernel")}
    print({k: round(v, 4) for k, v in out.items()}, "fused update:", ppo.last_update_stats.fused)
    if os.environ.get("B200RL_TC3_TIMING"):
        import ctypes as C
        from rl_replicas_b200 import _lib
        lib = _lib.load()
        out = (C.c_ulonglong * 64)()
        lib.b200rl_debug_tc3_timing(out, 1)
        e.run_stage("fused_step_kernel", hp)
        torch.cuda.synchronize()
        lib.b200rl_debug_tc3_timing(out, 0)
        tiles = max(int(out[52]), 1)
        print("tiles of CTA 0:", tiles, "set-up", int(out[53]), "tile loop", int(out[54]), "read-out", int(out[55]), "cycles")
        # CTA 0: the policy network's CTA of slot 0 (the value network's when only the value network runs)
        for wg in range(2):  # chain warpgroups: rows 0..63, 64..127
            wait = [int(out[10 * wg + s]) // tiles for s in range(5)]
            work = [(int(out[10 * wg + 5 + s]) - int(out[10 * wg + s])) // tiles for s in range(5)]
            print(f"chain {wg} wait / tile:", dict(zip(("E1", "E2", "E3", "E4", "E5"), wait)), "sum", sum(wait))
            print(f"chain {wg} work / tile:", dict(zip(("E1", "E2", "E3", "E4", "E5"), work)), "sum", sum(work))
        keys = ("dW3", "dW2", "dW1")
        for g in range(2):  # gradient warpgroups: the h and the l half of the stacked A operands
            wait = [int(out[40 + 3 * g + i]) // tiles for i in range(3)]
            issue = [int(out[46 + 3 * g + i]) // tiles for i in range(3)]
            print(f"gradient {'hl'[g]} wait  / tile:", dict(zip(keys, wait)), "sum", sum(wait))
            print(f"gradient {'hl'[g]} issue / tile:", dict(zip(keys, issue)), "sum", sum(issue))
