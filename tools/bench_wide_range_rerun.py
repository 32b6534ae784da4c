"""Cost and accuracy of the wide-range re-run: single-network steps whose fp16 pass leaves fp16's range.

    python tools/bench_wide_range_rerun.py [--rows N] [--reps R] [--save DIR]

Bench shapes (Gaussian policy [17, 64, 64, 6], value [17, 64, 64, 1]), 1024 x 1000 rows by default.  One step is one
b200rl_mlp_loss_grad launch (PPO clipped surrogate, or value MSE) and the fixed-order reduction of its partial rows, with
the range hints precomputed once, as the engine does.  Two batches: "in_range", the synthetic batch, and "obs_row_1e6",
the same with observation row 11 multiplied by 1e6, which trips the fp16 x 2 kernel's precision guard on every launch,
so the fp32 kernel queued behind it recomputes the launch.  Prints one JSON line: per batch and step the time per step,
the re-runs and launches per step, and the largest gradient error against oracle/onpolicy_f64, each gradient tensor
measured against its conditioning scale (as in tests/test_gpu_onpolicy_shapes.py).  B200RL_LIB selects another build of
the library; --save DIR writes the reduced gradients and scalar sums there for a bitwise comparison of two builds.
"""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import test_gpu_onpolicy_shapes as S  # noqa: E402
from gpu_helpers import dev, p, stream  # noqa: E402
from oracle import onpolicy_f64 as R  # noqa: E402
from rl_replicas_b200 import _lib  # noqa: E402
from rl_replicas_b200._lib import DIST, LOSS, N_SCALARS, LossGradArgs, MlpDesc, check  # noqa: E402

PS, VS = [17, 64, 64, 6], [17, 64, 64, 1]


def step_fn(lib, pb, obs, loss):
    """A closure running one step, and the device tensors of its reduced gradient and scalar sums."""
    sizes = PS if loss == "ppo_clip" else VS
    n = obs.shape[0]
    a = LossGradArgs()
    a.mlp = MlpDesc.make(sizes)
    a.n_rows, a.n_global, a.clip_range = n, n, S.CLIP
    keep = {"params": dev(pb["flat"] if loss == "ppo_clip" else pb["vflat"]), "obs": dev(obs),
            "obs_absmax": torch.zeros(32, device="cuda")}
    check(lib.b200rl_absmax_cols(p(keep["obs"]), n, sizes[0], p(keep["obs_absmax"]), stream()), "absmax_cols")
    if loss == "ppo_clip":
        a.loss, a.dist = LOSS["ppo_clip"], DIST["gaussian"]
        keep.update(actions=dev(pb["act"]), log_std=dev(pb["log_std"]), adv_raw=dev(pb["adv_raw"]),
                    adv_stats=dev(pb["stats"], np.float64), old_logp=dev(pb["old_logp"]))
    else:
        a.loss, a.dist = LOSS["mse"], DIST["none"]
        keep.update(target=dev(pb["ret"]), target_absmax=torch.zeros(1, device="cuda"))
        check(lib.b200rl_absmax(p(keep["target"]), n, p(keep["target_absmax"]), stream()), "absmax")
    for k, t in keep.items():
        setattr(a, k, t.data_ptr())
    P = int(lib.b200rl_mlp_param_count(a.mlp))
    grid = int(lib.b200rl_mlp_grid(a.mlp, n, 1))
    partials = torch.zeros(grid * P, dtype=torch.float32, device="cuda")
    sp = torch.zeros(grid * N_SCALARS, dtype=torch.float64, device="cuda")
    a.partials, a.scalar_partials = partials.data_ptr(), sp.data_ptr()
    grad = torch.zeros(P + N_SCALARS, dtype=torch.float32, device="cuda")
    scal = torch.zeros(N_SCALARS, dtype=torch.float64, device="cuda")

    def step():
        check(lib.b200rl_mlp_loss_grad(C.byref(a), stream()), "mlp_loss_grad")
        check(lib.b200rl_reduce_partials(p(partials), p(sp), grid, P, p(grad), p(scal), 0, None, stream()), "reduce")

    step.keep = keep  # the device inputs live as long as the closure
    return step, grad[:P], scal


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1024 * 1000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--save", metavar="DIR")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    lib = _lib.load()
    pb = S.policy_problem(PS, "gaussian", args.rows, seed=11, vs=VS)
    out = {"gpu": torch.cuda.get_device_name(0), "lib": _lib.LIB_PATH, "rows": args.rows}
    for case in ("in_range", "obs_row_1e6"):
        obs = pb["obs"].copy()
        if case == "obs_row_1e6":
            obs[11] *= np.float32(1e6)
        for loss in ("ppo_clip", "mse"):
            step, grad, scal = step_fn(lib, pb, obs, loss)
            for _ in range(3):
                step()
            torch.cuda.synchronize()
            f0, l0 = lib.b200rl_tc_fallback_count(), lib.b200rl_launch_count()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.reps):
                step()
            e1.record()
            torch.cuda.synchronize()
            g, s = grad.cpu().numpy(), scal.cpu().numpy()
            if loss == "ppo_clip":
                ref = R.policy_loss(pb["flat"], PS, obs, pb["act"], "gaussian", loss, pb["log_std"], pb["adv_raw"],
                                    pb["stats"], pb["old_logp"], S.CLIP)
                sizes, loss_scale = PS, ref["loss_abs_sum"]
            else:
                ref = R.value_loss(pb["vflat"], VS, obs, pb["ret"])
                sizes, loss_scale = VS, None
            out[f"{case}.{loss}"] = {
                "ms_per_step": e0.elapsed_time(e1) / args.reps,
                "reruns_per_step": (lib.b200rl_tc_fallback_count() - f0) / args.reps,
                "launches_per_step": (lib.b200rl_launch_count() - l0) / args.reps,
                "max_grad_err": max(S.grad_errs(g, ref, sizes).values()),
                "loss_err": S.scal_err(s[0], ref["loss_sum"], loss_scale)}
            if args.save:
                os.makedirs(args.save, exist_ok=True)
                np.save(os.path.join(args.save, f"{case}.{loss}.grad.npy"), g)
                np.save(os.path.join(args.save, f"{case}.{loss}.scalars.npy"), s)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
