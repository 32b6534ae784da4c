"""Short PPO update on BASELINE config 2 for ncu captures: `--steps p,v` policy/value gradient steps (default 2,2)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402

import bench  # noqa: E402
from oracle import onpolicy as O  # noqa: E402
from test_gpu_ppo import build as build_algo  # noqa: E402

if __name__ == "__main__":
    p, v = (int(x) for x in (sys.argv[1] if len(sys.argv) > 1 else "2,2").split(","))
    envs = int(sys.argv[2]) if len(sys.argv) > 2 else 1024
    pl, vl, log_std = bench.make_nets()
    b = bench.make_batch(envs, 1000, pl, seed=0)
    ppo = build_algo(bench.POLICY_SIZES, bench.VALUE_SIZES, "gaussian", O.flatten_layers(pl), O.flatten_layers(vl),
                     log_std, num_policy_gradients=p, num_value_gradients=v, max_kl_divergence=float("inf"))
    ppo.train_packed(b)
    st = ppo.last_update_stats
    print("launches", st.kernel_launches, "kl", st.kl_divergence, "vloss", st.value_loss_mean)
    if os.environ.get("B200RL_TC_TIMING"):
        import ctypes as C
        from rl_replicas_b200 import _lib
        import torch
        torch.cuda.synchronize()
        out = (C.c_ulonglong * 24)()
        _lib.load().b200rl_debug_tc2_timing(out)
        names = ["E0wait", "E0work", "E1wait", "E1work", "E2wait", "E2work", "E3wait", "E3work", "E4wait", "E4work",
                 "E5wait", "E5work", "-"]
        tiles = (envs * 1000 // 128 + 147) // 148
        print("cycles per tile (CTA 0, last backward launch):", {n: int(out[i]) // tiles for i, n in enumerate(names)},
              "total", sum(int(out[i]) for i in range(13)) // tiles)
        print("issuer cycles per tile:", {n: int(out[16 + i]) // tiles for i, n in
                                          enumerate(["F1", "F2", "F3", "S3", "S4", "S5", "idle"])})
    from rl_replicas_b200 import _lib as _L
    print("tc fallbacks:", _L.load().b200rl_tc_fallback_count())
