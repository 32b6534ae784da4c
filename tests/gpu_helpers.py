"""Thin test-side wrappers that call the C ABI (through ctypes) on torch-allocated device memory."""
import ctypes as C

import numpy as np
import torch

from rl_replicas_b200 import _lib
from rl_replicas_b200._lib import DIST, LOSS, N_SCALARS, LossGradArgs, MlpDesc, check


def dev(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a if dtype is None else np.asarray(a, dtype=dtype)))
    return t.cuda()


def p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def stream():
    return int(torch.cuda.current_stream().cuda_stream)


def gae_scan(rew, values, last_values, ep_offsets, ep_done, gamma=0.99, lam=0.97):
    lib = _lib.load()
    n, e = len(values), len(ep_done)
    f64 = rew.dtype == np.float64
    d_rew, d_v, d_lv = dev(rew), dev(values, np.float32), dev(last_values, np.float32)
    d_off, d_done = dev(ep_offsets, np.int64), dev(np.asarray(ep_done, dtype=np.uint8))
    adv = torch.empty(max(n, 1), dtype=torch.float32, device="cuda")
    ret = torch.empty(max(n, 1), dtype=torch.float32, device="cuda")
    stats = torch.zeros(3, dtype=torch.float64, device="cuda")
    wsb = lib.b200rl_gae_scan_workspace_bytes(n)
    ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")  # zeroed once at allocation (ABI contract)
    check(lib.b200rl_gae_scan(p(d_rew), int(f64), p(d_v), p(d_lv), p(d_off), p(d_done), n, e, gamma, lam, p(adv), p(ret),
                              p(stats), p(ws), wsb, stream()), "gae_scan")
    torch.cuda.synchronize()
    return adv[:n].cpu().numpy(), ret[:n].cpu().numpy(), stats.cpu().numpy()


def loss_grad(sizes, flat, obs, loss, dist="none", act=None, log_std=None, adv_raw=None, adv_stats=None, old_logp=None,
              target=None, clip=0.2, hidden_act="tanh", n_global=0, want_rows=True, obs_absmax=None):
    """Returns dict(grad, scalars[8], rows).  obs_absmax: the per-feature range hint of the fp16 kernels (default: the
    library's pre-pass computes it)."""
    lib = _lib.load()
    a = LossGradArgs()
    a.mlp = MlpDesc.make(sizes, hidden_act, "identity")
    a.loss, a.dist = LOSS[loss], DIST[dist]
    n = obs.shape[0]
    a.n_rows, a.n_global, a.clip_range = n, n_global, clip
    P = int(lib.b200rl_mlp_param_count(a.mlp))
    backward = loss != "eval"
    grid = lib.b200rl_mlp_grid(a.mlp, n, int(backward))
    assert grid > 0
    keep = dict(params=dev(flat, np.float32), obs=dev(obs, np.float32))
    for k, v, dt in (("actions", act, np.float32), ("log_std", log_std, np.float32), ("adv_raw", adv_raw, np.float32),
                     ("adv_stats", adv_stats, np.float64), ("old_logp", old_logp, np.float32), ("target", target, np.float32),
                     ("obs_absmax", obs_absmax, np.float32)):
        if v is not None:
            keep[k] = dev(v, dt)
    rows = torch.zeros(max(n, 1), dtype=torch.float32, device="cuda") if want_rows else None
    partials = torch.zeros(grid * P, dtype=torch.float32, device="cuda")
    sp = torch.zeros(grid * N_SCALARS, dtype=torch.float64, device="cuda")
    for k, t in keep.items():
        setattr(a, k, t.data_ptr())
    a.row_out = rows.data_ptr() if rows is not None else None
    a.partials, a.scalar_partials = partials.data_ptr(), sp.data_ptr()
    check(lib.b200rl_mlp_loss_grad(C.byref(a), stream()), "mlp_loss_grad")
    grad = torch.zeros(P + N_SCALARS, dtype=torch.float32, device="cuda")
    scal = torch.zeros(N_SCALARS, dtype=torch.float64, device="cuda")
    check(lib.b200rl_reduce_partials(p(partials) if backward else None, p(sp), grid, P, p(grad), p(scal), 0, None,
                                     stream()), "reduce_partials")
    torch.cuda.synchronize()
    return dict(grad=grad[:P].cpu().numpy(), scalars=scal.cpu().numpy(), rows=None if rows is None else rows[:n].cpu().numpy())


def adam_step(params, grad, m, v, step, lr, b1=0.9, b2=0.999, eps=1e-8):
    lib = _lib.load()
    dp, dg, dm, dv = dev(params, np.float32), dev(grad, np.float32), dev(m, np.float32), dev(v, np.float32)
    check(lib.b200rl_adam_step(p(dp), p(dg), p(dm), p(dv), dp.numel(), step, lr, b1, b2, eps, None, 0, 1.0, 0.0, None,
                               None, None, None, stream()), "adam_step")
    torch.cuda.synchronize()
    return dp.cpu().numpy(), dm.cpu().numpy(), dv.cpu().numpy()


def fvp(sizes, flat, obs, dist, direction, log_std=None, hidden_act="tanh"):
    """One Fisher-vector product launch (B200RL_LOSS_FVP) + the fixed-order reduction: returns F v (no damping)."""
    lib = _lib.load()
    a = LossGradArgs()
    a.mlp = MlpDesc.make(sizes, hidden_act, "identity")
    a.loss, a.dist = LOSS["fvp"], DIST[dist]
    n = obs.shape[0]
    a.n_rows, a.n_global = n, 0
    P = int(lib.b200rl_mlp_param_count(a.mlp))
    grid = lib.b200rl_mlp_grid(a.mlp, n, 2)
    assert grid > 0
    keep = dict(params=dev(flat, np.float32), obs=dev(obs, np.float32), direction=dev(direction, np.float32))
    if log_std is not None:
        keep["log_std"] = dev(log_std, np.float32)
    partials = torch.full((grid * P,), float("nan"), dtype=torch.float32, device="cuda")  # every row must be written
    for k, t in keep.items():
        setattr(a, k, t.data_ptr())
    a.partials = partials.data_ptr()
    check(lib.b200rl_mlp_loss_grad(C.byref(a), stream()), "mlp_loss_grad(fvp)")
    out = torch.zeros(P + N_SCALARS, dtype=torch.float32, device="cuda")
    check(lib.b200rl_reduce_partials(p(partials), None, grid, P, p(out), None, 0, None, stream()), "reduce_partials")
    torch.cuda.synchronize()
    return out[:P].cpu().numpy()


def forward_outputs(sizes, flat, obs, dist, act, log_std=None, old_out=None, adv_raw=None, old_logp=None, loss="eval",
                    no_tc=False, hidden_act="tanh"):
    """A forward-only launch that asks for the raw outputs (out_full) and, with old_out, the true KL(old || new):
    returns dict(out, rows (log-probs), scalars[8])."""
    lib = _lib.load()
    a = LossGradArgs()
    a.mlp = MlpDesc.make(sizes, hidden_act, "identity")
    a.loss, a.dist = LOSS[loss], DIST[dist]
    a.flags = 1 | (2 if no_tc else 0)  # B200RL_FLAG_FORWARD_ONLY | B200RL_FLAG_NO_TC
    n = obs.shape[0]
    a.n_rows, a.n_global = n, 0
    grid = lib.b200rl_mlp_grid(a.mlp, n, 3)
    assert grid > 0
    keep = dict(params=dev(flat, np.float32), obs=dev(obs, np.float32), actions=dev(act, np.float32))
    for k, v in (("log_std", log_std), ("old_out", old_out), ("adv_raw", adv_raw), ("old_logp", old_logp)):
        if v is not None:
            keep[k] = dev(v, np.float32)
    out = torch.full((max(n, 1) * sizes[-1],), float("nan"), dtype=torch.float32, device="cuda")
    rows = torch.full((max(n, 1),), float("nan"), dtype=torch.float32, device="cuda")
    sp = torch.full((grid * N_SCALARS,), float("nan"), dtype=torch.float64, device="cuda")  # every row must be written
    for k, t in keep.items():
        setattr(a, k, t.data_ptr())
    a.out_full, a.row_out, a.scalar_partials = out.data_ptr(), rows.data_ptr(), sp.data_ptr()
    check(lib.b200rl_mlp_loss_grad(C.byref(a), stream()), "mlp_loss_grad(forward)")
    scal = torch.zeros(N_SCALARS, dtype=torch.float64, device="cuda")
    check(lib.b200rl_reduce_partials(None, p(sp), grid, int(lib.b200rl_mlp_param_count(a.mlp)), None, p(scal), 0, None,
                                     stream()), "reduce_partials")
    torch.cuda.synchronize()
    return dict(out=out[: n * sizes[-1]].cpu().numpy().reshape(n, sizes[-1]), rows=rows[:n].cpu().numpy(),
                scalars=scal.cpu().numpy())
