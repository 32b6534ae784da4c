"""GPU: every on-policy kernel against the float64 reference oracle/onpolicy_f64.py from identical inputs, tensor by
tensor, at the edges of each kernel's shape gate and at the edges of the distributions.

Paths, chosen with the switches the library reads on every call:
* "tc2": fp16 x 2 tensor-core kernel (mlp_tc2.cu), the default for 3-layer Tanh networks with obs <= 32, hidden <= 64,
  out <= 15.  Asserted by the fallback counter staying put (a launch that leaves fp16's range is redone by the fp32
  kernel, mlp_fused.cu).
* "rerun": the default path with an obs_absmax hint 1e6 times the largest |observation|, which puts every row below
  the fp16 kernel's precision guard: each launch is redone by the fp32 kernel queued behind it, into the tensor-core
  path's partial rows.  Asserted by the fallback counter (+1 per launch) and by the grid.
* "fp32": the CUDA-core kernel (mlp_fused.cu), B200RL_DISABLE_TC=1 or any shape outside the gate.  Asserted by its grid
  at 640 rows: 10, 20 or 40 CTAs for tiles of 64, 32 or 16 rows.
* FVP: mlp_tc_fvp.cu inside the gate, the fp32 kernel's FVP mode outside it (or under B200RL_DISABLE_TC=1).
* the fused PPO step (mlp_tc3.cu) through the engine, asserted by last_update_stats.fused.

Bars.  One per arithmetic: BAR["fp16x2"] (mlp_tc2 and mlp_tc3), BAR["fp32"], BAR["fvp"] (both FVP kernels), each
about 4x the largest error measured on an H100 over all cases of its path.  Every quantity is measured
against the scale of its own float32 rounding: per-row vectors and F v against max |ref| of that tensor; each W / b
gradient against the largest, over its entries, sum over rows of |that row's contribution| (oracle/onpolicy_f64),
since a gradient whose rows cancel is only known to ~2^-24 of that however the kernel sums it; the loss sum against
sum |term| and the KL / log-prob sums against sum |log pi|; the other sums against their value.

Inputs near a discontinuity are moved off it, never excused by a looser bar: old log-probs whose ratio lands within
1e-3 of a clip bound are shifted by 5e-3, and with ReLU hidden layers only rows whose pre-activations clear 1e-6
(relative) are used (see oracle/offpolicy_f64.mlp)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from conftest import rel_err
from oracle import onpolicy_f64 as R

pytestmark = pytest.mark.gpu

# Largest errors measured on an H100 over all cases of each path (gradients against their conditioning scale):
# fp16x2 2.1e-6, fp32 1.8e-6, fvp 1.4e-6; each bar is about 4x that.  The first two are the one-row
# case, whose single row gets no averaging of its rounding errors; every multi-row case stays under 1.5e-6.  The fused
# step (mlp_tc3, fp16x2) measured on an H100 80GB HBM3 at 700 W: gradients at most 4.1e-7 (one tile of 65 rows), with
# no growth in tiles per CTA (largest policy / value tensor 6.6e-8 / 3.0e-8 at 1 tile per CTA, 3.8e-8 / 1.2e-7 at 4-5,
# 3.4e-8 / 1.6e-7 at 9); its scalar sums at most 1.2e-6 (the PPO loss sum with 8-sigma actions).
BAR = {"fp16x2": 8e-6, "fp32": 7e-6, "fvp": 6e-6}
ARITH = {"tc2": "fp16x2", "rerun": "fp32", "fp32": "fp32"}
CLIP, CLIP_MARGIN, KINK = 0.2, 1e-3, 1e-6
# the fp32 kernel's limits for a [17, h, h, 6] policy: the largest equal hidden width whose backward layout fits
# 227 KiB of shared memory, and the largest whose Fisher-vector-product layout does (README)
FP32_MAX_H, FVP_MAX_H = 111, 92


def lib():
    from rl_replicas_b200 import _lib
    return _lib.load()


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def fallbacks():
    return int(lib().b200rl_tc_fallback_count())


def grid(sizes, n, mode, hidden="tanh"):
    from rl_replicas_b200._lib import MlpDesc
    return int(lib().b200rl_mlp_grid(C.byref(MlpDesc.make(sizes, hidden, "identity")), n, mode))


def tc_grid(n):
    return min(max(-(-n // 128), 1), sms())


def full_round():  # one 128-row tile for every SM
    return sms() * 128


def mixed_tiles():
    """2.5 tiles per SM with a ragged last tile: half of the CTAs get 3 tiles (both of tc2's slots busy, then one), the
    rest 2 (one per slot)."""
    return (2 * sms() + sms() // 2) * 128 - 51


@pytest.fixture
def path(request, monkeypatch):
    for k in ("B200RL_DISABLE_TC", "B200RL_FUSED_STEP"):
        monkeypatch.delenv(k, raising=False)
    name = getattr(request, "param", "default")
    if name == "fp32":
        monkeypatch.setenv("B200RL_DISABLE_TC", "1")
    return name


# ---- problems ------------------------------------------------------------------------------------------------------
def net(rng, sizes):
    return np.concatenate([np.concatenate([(rng.standard_normal((o, i)) / np.sqrt(i)).reshape(-1),
                                           0.1 * rng.standard_normal(o)]) for i, o in zip(sizes[:-1], sizes[1:])]
                          ).astype(np.float32)


def narrow_tanh(flat, sizes, obs):
    """per row, the largest |h| over the units of hidden layers one unit wide (0 if there are none)"""
    import torch as T
    with T.no_grad():
        _, _, layers = R._forward(T.as_tensor(flat.astype(np.float64)), sizes, T.as_tensor(obs.astype(np.float64)), "tanh")
    hs = [np.abs(np.tanh(z.numpy()))[:, 0] for z, _ in layers[:-1] if z.shape[1] == 1]
    return np.max(hs, axis=0) if hs else np.zeros(obs.shape[0])


def draw_obs(rng, sizes_list, n, hidden):
    """n observation rows; with ReLU only rows whose pre-activations in every network clear KINK.  With Tanh, a hidden
    layer one unit wide passes the whole gradient of the layers below through one tanh'(z) = 1 - h^2, which a float32
    h gives only to ~2^-24 h^2 / (1 - h^2); rows are kept with |h| <= 0.8 there, so that conditioning is not what is
    measured."""
    if hidden != "relu" and all(min(sizes[1:-1]) > 1 for sizes, _ in sizes_list):
        return rng.standard_normal((n, sizes_list[0][0][0])).astype(np.float32)
    pool = rng.standard_normal((3 * n + 16, sizes_list[0][0][0])).astype(np.float32)
    margin = np.full(pool.shape[0], np.inf)
    for sizes, flat in sizes_list:
        if hidden == "relu":
            margin = np.minimum(margin, R.policy_loss(flat, sizes, pool, np.zeros((pool.shape[0], sizes[-1]), np.float32),
                                                      "gaussian", "eval", np.zeros(sizes[-1], np.float32),
                                                      hidden=hidden)["margin"])
        elif min(sizes[1:-1]) == 1:
            margin = np.where(narrow_tanh(flat, sizes, pool) <= 0.8, margin, 0.0)
    keep = np.flatnonzero(margin >= KINK)[:n]
    assert keep.size == n
    return pool[keep]


def policy_problem(sizes, dist, n, seed, hidden="tanh", log_std=None, sigmas=None, out_scale=None, obs_outlier=None,
                   vs=None, obs_scale=None, ret_scale=None):
    """Policy and value networks, observations, actions, advantages and old log-probs.  log_std: the value of every
    entry, or one value per entry (default a spread over [-0.8, -0.2]); sigmas: in every row one action coordinate (at
    random) exactly this many standard deviations from the mean, the others a normal draw; out_scale: the policy's last
    layer scaled so that max |output| (mean or logit) is this; obs_outlier: observation row 11 multiplied by this; vs:
    the value network's sizes (default the policy's with one output); obs_scale: observation column j multiplied by
    obs_scale[j] (a scalar: every column) and column j of both first layers divided by it, so that the networks see
    inputs of the usual size (a column scaled by 0 is all zeros and its weights stay); ret_scale: the returns
    multiplied by this."""
    rng = np.random.default_rng(seed)
    A = sizes[-1]
    vs = sizes[:-1] + [1] if vs is None else vs
    flat, vflat = net(rng, sizes), net(rng, vs)
    obs = draw_obs(rng, [(sizes, flat), (vs, vflat)], n, hidden)
    if obs_outlier is not None:
        obs[11] *= np.float32(obs_outlier)
    if obs_scale is not None:
        col = np.broadcast_to(np.asarray(obs_scale, np.float32), (sizes[0],))
        obs *= col[None, :]
        for f, s in ((flat, sizes), (vflat, vs)):
            w1 = f[:s[0] * s[1]].reshape(s[1], s[0])
            w1 /= np.where(col != 0, col, np.float32(1))[None, :]
    ls = None
    if dist == "gaussian":
        ls = np.full(A, log_std, np.float32) if log_std is not None else np.linspace(-0.8, -0.2, A).astype(np.float32)
    mean = R.forward_kl(flat, sizes, obs, dist, np.zeros((n, A), np.float32), ls, hidden)["out"]
    if out_scale is not None:
        k = len(sizes) - 2
        o = sum(sizes[l] * sizes[l + 1] + sizes[l + 1] for l in range(k))
        flat[o:] *= np.float32(out_scale / np.abs(mean).max())
        mean = R.forward_kl(flat, sizes, obs, dist, np.zeros((n, A), np.float32), ls, hidden)["out"]
    if dist == "gaussian":
        z = rng.standard_normal((n, A))
        if sigmas is not None:
            z[np.arange(n), rng.integers(0, A, n)] = rng.choice([-sigmas, sigmas], n)
        act = (mean + np.exp(ls.astype(np.float64)) * z).astype(np.float32)
    else:
        act = rng.integers(0, A, n).astype(np.float32)
    adv_raw = (2.0 * rng.standard_normal(n) + 0.5).astype(np.float32)
    a64 = adv_raw.astype(np.float64)
    stats = np.asarray([a64.sum(), (a64 ** 2).sum(), n]) if n > 1 else None  # one row has no unbiased std
    logp = R.policy_loss(flat, sizes, obs, act, dist, "eval", ls, hidden=hidden)["logp"]
    old_logp = (logp + 0.3 * rng.standard_normal(n)).astype(np.float32)
    near = R.clip_margin(np.exp(logp - old_logp), CLIP) < CLIP_MARGIN
    old_logp[near] += np.float32(5e-3)
    assert R.clip_margin(np.exp(logp - old_logp), CLIP).min() >= CLIP_MARGIN
    ret = (5.0 * (1.0 if ret_scale is None else ret_scale) * rng.standard_normal(n)).astype(np.float32)
    return dict(sizes=sizes, vs=vs, dist=dist, flat=flat, vflat=vflat, obs=obs, act=act, log_std=ls, adv_raw=adv_raw,
                stats=stats, old_logp=old_logp, ret=ret, hidden=hidden, n=n)


def tensor_errs(got_flat, ref_tensors, sizes, prefix=""):
    return {f"{prefix}{k}": rel_err(g, ref_tensors[k]) for k, g in R.split(got_flat, sizes).items()}


def scaled_err(got, ref, scale):
    """max |got - ref| / max(scale): a gradient against the sum over rows of |contribution| (oracle/onpolicy_f64)."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    return float(np.max(np.abs(got - ref)) / max(float(np.max(scale)), 1e-300))


def grad_errs(got_flat, ref, sizes, prefix=""):
    """Every W / b gradient tensor against its conditioning scale."""
    return {f"{prefix}{k}": scaled_err(g, ref["grads"][k], ref["scales"][k])
            for k, g in R.split(got_flat, sizes).items()}


def scal_err(got, ref, scale=None):
    return abs(float(got) - ref) / max(abs(ref) if scale is None else scale, 1e-300)


def report(label, arith, errs):
    print(f"\n[{arith}] {label}: " + ", ".join(f"{k} {v:.1e}" for k, v in errs.items()))
    for k, v in errs.items():
        assert v < BAR[arith], (label, k, v, BAR[arith])


def run_policy_and_value(pb, launch_check, obs_absmax=None):
    """Every policy loss, the evaluation launch, the value MSE and the value evaluation of one problem; returns the
    per-quantity errors.  launch_check(what) is a context manager around each launch (Fired); obs_absmax: the range
    hint every launch passes (default none: the library's pre-pass)."""
    from gpu_helpers import loss_grad
    s, dist, n, h = pb["sizes"], pb["dist"], pb["n"], pb["hidden"]
    errs = {}
    for loss in ("ppo_clip", "vpg", "trpo_surrogate"):
        with launch_check(loss):
            got = loss_grad(s, pb["flat"], pb["obs"], loss, dist, act=pb["act"], log_std=pb["log_std"],
                            adv_raw=pb["adv_raw"], adv_stats=pb["stats"], old_logp=pb["old_logp"], clip=CLIP,
                            hidden_act=h, obs_absmax=obs_absmax)
        ref = R.policy_loss(pb["flat"], s, pb["obs"], pb["act"], dist, loss, pb["log_std"], pb["adv_raw"], pb["stats"],
                            pb["old_logp"], CLIP, h)
        errs.update(grad_errs(got["grad"], ref, s, f"{loss}.d"))
        sc = got["scalars"]
        errs[f"{loss}.loss"] = scal_err(sc[0], ref["loss_sum"], ref["loss_abs_sum"])
        errs[f"{loss}.logp"] = rel_err(got["rows"], ref["logp"])
        if loss != "vpg":
            errs[f"{loss}.kl"] = scal_err(sc[1], ref["kl_sum"], ref["logp_abs_sum"])
        assert sc[5] == n
        if loss == "ppo_clip" and n >= 100:
            assert (ref["ratio"] > 1 + CLIP).any() and (ref["ratio"] < 1 - CLIP).any()  # the clip binds both ways
    with launch_check("eval"):
        got = loss_grad(s, pb["flat"], pb["obs"], "eval", dist, act=pb["act"], log_std=pb["log_std"], hidden_act=h,
                        obs_absmax=obs_absmax)
    ref = R.policy_loss(pb["flat"], s, pb["obs"], pb["act"], dist, "eval", pb["log_std"], hidden=h)
    sc = got["scalars"]
    errs["eval.logp"] = rel_err(got["rows"], ref["logp"])
    errs["eval.entropy_sum"] = scal_err(sc[2], ref["entropy_sum"])
    errs["eval.logp_sum"] = scal_err(sc[3], ref["logp_sum"], ref["logp_abs_sum"])
    errs["eval.logp2_sum"] = scal_err(sc[4], ref["logp2_sum"])
    assert sc[5] == n
    with launch_check("mse"):
        got = loss_grad(pb["vs"], pb["vflat"], pb["obs"], "mse", "none", target=pb["ret"], hidden_act=h,
                        obs_absmax=obs_absmax)
    ref = R.value_loss(pb["vflat"], pb["vs"], pb["obs"], pb["ret"], h)
    errs.update(grad_errs(got["grad"], ref, pb["vs"], "mse.d"))
    errs["mse.loss"] = scal_err(got["scalars"][0], ref["loss_sum"])
    with launch_check("values"):
        got = loss_grad(pb["vs"], pb["vflat"], pb["obs"], "eval", "none", hidden_act=h, obs_absmax=obs_absmax)
    errs["values"] = rel_err(got["rows"], ref["values"])
    return errs


class Fired(dict):
    """Counts, per launch, how often the fp16 range guard fired (launches that left fp16's range are redone by the
    fp32 kernel): ``with fired("ppo_clip"): ...``.  Checked after the errors are printed."""

    def __call__(self, what):
        return _Count(self, what)


class _Count:
    def __init__(self, d, what):
        self.d, self.what = d, what

    def __enter__(self):
        self.before = fallbacks()

    def __exit__(self, *exc):
        n = fallbacks() - self.before
        if n:
            self.d[self.what] = self.d.get(self.what, 0) + n


# ---- cases inside the tensor-core gate: every path ----------------------------------------------------------------
GATE_CASES = {
    # obs = 32 fills all 32 input columns of tc2's XD operand; 15 outputs put the last dOut column (46) next to the
    # ones column (47); one full round of tiles + 1 row
    "obs32_out15": dict(sizes=[32, 64, 64, 15], dist="gaussian", n="full+1"),
    # the same edges, categorical, h2 = 63 (one zero-padded column); 129 rows: one tile + 1 row
    "obs32_out15_cat": dict(sizes=[32, 64, 63, 15], dist="categorical", n=129),
    # obs = 31 (the widest the fused step takes), one action, h1 = 63; 127 rows: one tile less one row
    "obs31_out1": dict(sizes=[31, 63, 64, 1], dist="gaussian", n=127),
    # one observation column and a hidden width of 1; exactly one tile
    "obs1_h1": dict(sizes=[1, 1, 64, 2], dist="categorical", n=128),
    # h2 = 1; a single row (no advantage normalisation: one row has no unbiased std)
    "h2_1_one_row": dict(sizes=[17, 64, 1, 6], dist="gaussian", n=1),
    # exactly one full round of 128-row tiles over all SMs
    "full_round": dict(sizes=[8, 64, 64, 15], dist="categorical", n="full"),
    # 3 tiles on some CTAs, 2 on the others, ragged last tile
    "mixed_tiles": dict(sizes=[17, 64, 64, 6], dist="gaussian", n="mixed"),
    # distributions at their edges.  sigma = e^-5 with means of order 1 would lose 2^-24 |mu| / sigma ~ 1e-5 of
    # a - mu to the float32 rounding of mu alone (a float32 reference shares that loss), so those means are of order
    # sigma; and one coordinate per row at 8 sigma, not all six: |log pi| ~ 200 would move every PPO ratio by its own
    # float32 rounding, 2^-24 * 200 ~ 1e-5
    "log_std_-5": dict(sizes=[17, 64, 64, 6], dist="gaussian", n=3000, log_std=-5.0, out_scale=0.02),
    "log_std_+1": dict(sizes=[17, 64, 64, 6], dist="gaussian", n=3000, log_std=1.0),
    "actions_8_sigma": dict(sizes=[17, 64, 64, 6], dist="gaussian", n=3000, log_std=-0.5, sigmas=8.0),
    "logits_30": dict(sizes=[8, 64, 64, 15], dist="categorical", n=3000, out_scale=30.0),
    # one observation row 1e6 times the others: after scaling, the other rows would lose their low fp16 splits, so the
    # default path's guard has the fp32 kernel redo its launches (the predicated re-run)
    "obs_row_1e6": dict(sizes=[17, 64, 64, 6], dist="gaussian", n=2000, obs_outlier=1e6),
}
# launches of the default path that legitimately leave fp16's range (and are redone by the fp32 kernel):
# {case: {launch: count}}.  The power-of-two pre-scales absorb log_std -5 / +1, 8-sigma actions and logits of +-30;
# only the outlier row trips the guard, in every launch.
LAUNCHES = ("ppo_clip", "vpg", "trpo_surrogate", "eval", "mse", "values")
TC2_TRIPS = {"obs_row_1e6": {k: 1 for k in LAUNCHES}}


def rows_of(n):
    return {"full": full_round(), "full+1": full_round() + 1, "mixed": mixed_tiles()}.get(n, n)


def make(case, seed, hidden="tanh"):
    c = dict(case)
    sizes, dist, n = c.pop("sizes"), c.pop("dist"), rows_of(c.pop("n"))
    return policy_problem(sizes, dist, n, seed, hidden, **c)


@pytest.mark.parametrize("path", ["tc2", "rerun", "fp32"], indirect=True)
@pytest.mark.parametrize("name", list(GATE_CASES))
def test_gate_case(name, path):
    pb = make(GATE_CASES[name], seed=list(GATE_CASES).index(name))
    n = pb["n"]
    if path == "fp32":
        assert grid(pb["sizes"], 640, 1) == 10
    else:  # the fp32 re-run writes the tensor-core path's partial rows, zeroing those past its own grid
        assert grid(pb["sizes"], n, 1) == 2 * tc_grid(n)
    hint = np.full(pb["sizes"][0], 1e6 * np.abs(pb["obs"]).max(), np.float32) if path == "rerun" else None
    fired = Fired()
    errs = run_policy_and_value(pb, fired, hint)
    # launches the guard sent to the fp32 kernel carry that kernel's arithmetic
    report(f"{name} n={n}" + (f" fp16 range trips {dict(fired)}" if fired else ""),
           "fp32" if fired else ARITH[path], errs)
    expect = {"tc2": TC2_TRIPS.get(name, {}), "rerun": {k: 1 for k in LAUNCHES}, "fp32": {}}[path]
    assert fired == expect


# ---- cases outside the gate: the fp32 kernel, at every tile height ------------------------------------------------
FP32_CASES = {
    # one past each bound of the gate
    "obs33": (dict(sizes=[33, 64, 64, 6], dist="gaussian", n=641), 64),
    "out16_gaussian": (dict(sizes=[17, 64, 64, 16], dist="gaussian", n=641), 64),  # dls[16] of train_log_std full
    "out16_categorical": (dict(sizes=[17, 64, 64, 16], dist="categorical", n=641), 64),
    "h65": (dict(sizes=[17, 65, 65, 6], dist="gaussian", n=641), 64),
    # Tanh networks wider than 64 land on 32- and 16-row tiles
    "h80": (dict(sizes=[17, 80, 80, 6], dist="categorical", n=641), 32),
    # the widest 32-row layout (97) leaves room for the kernel's static shared arrays; at 98 only 16 rows do
    "h98": (dict(sizes=[17, 98, 98, 6], dist="gaussian", n=641), 16),
    "h100": (dict(sizes=[17, 100, 100, 6], dist="gaussian", n=641), 16),
    f"h{FP32_MAX_H}": (dict(sizes=[17, FP32_MAX_H, FP32_MAX_H, 6], dist="gaussian", n=641), 16),  # the widest
    "h65_63_ragged": (dict(sizes=[9, 65, 63, 3], dist="categorical", n=100), 64),
}


@pytest.mark.parametrize("name", list(FP32_CASES))
def test_fp32_case(name, path):
    case, tile = FP32_CASES[name]
    pb = make(case, seed=100 + list(FP32_CASES).index(name))
    assert grid(pb["sizes"], 640, 1) == 640 // tile
    fired = Fired()
    errs = run_policy_and_value(pb, fired)
    report(f"{name} n={pb['n']} tile={tile}", "fp32", errs)
    assert not fired


def test_fp32_relu(path):
    pb = make(dict(sizes=[17, 64, 64, 6], dist="gaussian", n=641), seed=7, hidden="relu")
    assert grid(pb["sizes"], 640, 1, "relu") == 10
    fired = Fired()
    report("relu n=641", "fp32", run_policy_and_value(pb, fired))
    assert not fired


# ---- trainable log_std: the fp32 kernel's dLoss/dlog_std columns --------------------------------------------------
def loss_grad_log_std(pb, loss):
    """One launch with train_log_std: partial rows of P + A columns (b200rl_mlp_grid mode 4)."""
    from gpu_helpers import dev, p, stream
    from rl_replicas_b200._lib import DIST, LOSS, N_SCALARS, LossGradArgs, MlpDesc, check
    a = LossGradArgs()
    a.mlp = MlpDesc.make(pb["sizes"], pb["hidden"], "identity")
    a.loss, a.dist = LOSS[loss], DIST["gaussian"]
    n, A = pb["n"], pb["sizes"][-1]
    a.n_rows, a.n_global, a.clip_range, a.train_log_std = n, n, CLIP, 1
    P = int(lib().b200rl_mlp_param_count(a.mlp))
    g = grid(pb["sizes"], n, 4)
    keep = dict(params=dev(pb["flat"]), obs=dev(pb["obs"]), actions=dev(pb["act"]), log_std=dev(pb["log_std"]),
                adv_raw=dev(pb["adv_raw"]), adv_stats=dev(pb["stats"], np.float64), old_logp=dev(pb["old_logp"]))
    for k, t in keep.items():
        setattr(a, k, t.data_ptr())
    partials = torch.full((g * (P + A),), float("nan"), dtype=torch.float32, device="cuda")
    sp = torch.zeros(g * N_SCALARS, dtype=torch.float64, device="cuda")
    a.partials, a.scalar_partials = partials.data_ptr(), sp.data_ptr()
    check(lib().b200rl_mlp_loss_grad(C.byref(a), stream()), "mlp_loss_grad(train_log_std)")
    out = torch.zeros(P + A + N_SCALARS, dtype=torch.float32, device="cuda")
    check(lib().b200rl_reduce_partials(p(partials), p(sp), g, P + A, p(out), None, 0, None, stream()), "reduce")
    torch.cuda.synchronize()
    out = out.cpu().numpy()
    return out[:P], out[P:P + A]


@pytest.mark.parametrize("A,log_std", [(1, -5.0), (16, 1.0), (16, None)])
def test_train_log_std_columns(A, log_std, path):
    """A = 1 and A = 16 (every entry of the kernel's dls[16] in use), log_std at -5 (means of order sigma, see
    GATE_CASES), +1 and spread."""
    pb = policy_problem([17, 64, 64, A], "gaussian", 641, 200 + A, log_std=log_std,
                        out_scale=0.02 if log_std == -5.0 else None)
    assert grid(pb["sizes"], 640, 4) == 10
    errs = {}
    for loss in ("ppo_clip", "vpg"):
        g, gls = loss_grad_log_std(pb, loss)
        ref = R.policy_loss(pb["flat"], pb["sizes"], pb["obs"], pb["act"], "gaussian", loss, pb["log_std"],
                            pb["adv_raw"], pb["stats"], pb["old_logp"], CLIP)
        errs.update(grad_errs(g, ref, pb["sizes"], f"{loss}.d"))
        errs[f"{loss}.dlog_std"] = scaled_err(gls, ref["grad_log_std"], ref["scale_log_std"])
    report(f"train_log_std A={A} log_std={log_std}", "fp32", errs)


# ---- forward-only launches: raw outputs and the true KL -----------------------------------------------------------
FWD_CASES = {
    "obs32_out15": (dict(sizes=[32, 64, 64, 15], dist="gaussian", n="full+1"), True),
    "logits_30": (dict(sizes=[8, 64, 64, 15], dist="categorical", n="mixed", out_scale=30.0), True),
    "log_std_-5": (dict(sizes=[17, 64, 63, 6], dist="gaussian", n=129, log_std=-5.0, out_scale=0.02), True),
    "out16_categorical": (dict(sizes=[33, 64, 64, 16], dist="categorical", n=641), False),  # fp32 kernel only
}


@pytest.mark.parametrize("no_tc", [False, True])
@pytest.mark.parametrize("name", list(FWD_CASES))
def test_forward_outputs_and_true_kl(name, no_tc, path):
    from gpu_helpers import forward_outputs
    case, in_gate = FWD_CASES[name]
    pb = make(case, seed=300 + list(FWD_CASES).index(name))
    s, dist, n = pb["sizes"], pb["dist"], pb["n"]
    rng = np.random.default_rng(7)
    old_out = R.forward_kl(pb["flat"], s, pb["obs"], dist, np.zeros((n, s[-1]), np.float32), pb["log_std"])["out"]
    old_out = (old_out + 0.3 * np.abs(old_out).max() * rng.standard_normal(old_out.shape)).astype(np.float32)
    fired = Fired()
    with fired("forward"):
        got = forward_outputs(s, pb["flat"], pb["obs"], dist, pb["act"], log_std=pb["log_std"], old_out=old_out,
                              no_tc=no_tc)
    ref = R.forward_kl(pb["flat"], s, pb["obs"], dist, old_out, pb["log_std"])
    lp = R.policy_loss(pb["flat"], s, pb["obs"], pb["act"], dist, "eval", pb["log_std"])
    errs = {"out_full": rel_err(got["out"], ref["out"]), "logp": rel_err(got["rows"], lp["logp"]),
            "kl_sum": scal_err(got["scalars"][6], float(ref["kl"].sum()))}
    assert got["scalars"][5] == n
    arith = "fp16x2" if in_gate and not no_tc else "fp32"
    report(f"forward {name} n={n} no_tc={no_tc}" + (f" fp16 range trips {dict(fired)}" if fired else ""), arith, errs)
    assert not fired


# ---- Fisher-vector products ----------------------------------------------------------------------------------------
FVP_CASES = {
    # the FVP kernel's largest shape, obs = 32 and 15 outputs
    "obs32_out15": (dict(sizes=[32, 64, 64, 15], dist="gaussian", n="full+1"), "tc"),
    "obs32_out15_cat": (dict(sizes=[32, 64, 64, 15], dist="categorical", n="mixed"), "tc"),
    "obs1_h1": (dict(sizes=[1, 1, 63, 2], dist="categorical", n=1), "tc"),
    "log_std_-5": (dict(sizes=[31, 63, 64, 1], dist="gaussian", n=127, log_std=-5.0, out_scale=0.02), "tc"),
    "logits_30": (dict(sizes=[8, 64, 64, 15], dist="categorical", n=3000, out_scale=30.0), "tc"),
    # the fp32 kernel's FVP mode: inside the gate under B200RL_DISABLE_TC (32-row tiles) ...
    "obs32_out15_fp32": (dict(sizes=[32, 64, 64, 15], dist="gaussian", n=641), 32),
    # ... and its largest shape, 16-row tiles
    f"h{FVP_MAX_H}": (dict(sizes=[17, FVP_MAX_H, FVP_MAX_H, 6], dist="gaussian", n=641), 16),
    f"h{FVP_MAX_H}_cat": (dict(sizes=[17, FVP_MAX_H, FVP_MAX_H, 6], dist="categorical", n=641), 16),
}


@pytest.mark.parametrize("name", list(FVP_CASES))
def test_fvp(name, path, monkeypatch):
    from gpu_helpers import fvp
    case, kernel = FVP_CASES[name]
    pb = make(case, seed=400 + list(FVP_CASES).index(name))
    s, n = pb["sizes"], pb["n"]
    if kernel == "tc":  # a full round: the FVP kernel's two partial rows per CTA (the fp32 kernel would have one)
        assert grid(s, full_round(), 2) == 2 * sms()
    else:
        if s[1] <= 64:
            monkeypatch.setenv("B200RL_DISABLE_TC", "1")
        assert grid(s, 640, 2) == 640 // kernel
    v = np.random.default_rng(1).standard_normal(pb["flat"].size).astype(np.float32)
    fired = Fired()
    with fired("fvp"):
        got = fvp(s, pb["flat"], pb["obs"], pb["dist"], v, log_std=pb["log_std"])
    ref = R.fvp(pb["flat"], s, pb["obs"], pb["dist"], v, pb["log_std"])
    report(f"fvp {name} n={n}" + (f" fp16 range trips {dict(fired)}" if fired else ""), "fvp",
           tensor_errs(got, ref["tensors"], s, "Fv."))
    assert not fired


# ---- the fused PPO step (mlp_tc3.cu) through the engine ----------------------------------------------------------
def engine_for(ps, vs, dist, n_envs, horizon, seed):
    from rl_replicas_b200 import synthetic
    from rl_replicas_b200.engine import OnPolicyEngine
    rng = np.random.default_rng(seed)
    pol, val = net(rng, ps), net(rng, vs)
    A = ps[-1]
    log_std = np.linspace(-0.7, -0.2, A).astype(np.float32)
    b = synthetic.fixed_batch(n_envs, horizon, ps[0], A, discrete=dist == "categorical", seed=seed, frac_not_done=0.3)
    e = OnPolicyEngine(ps, vs, dist, b["obs"].shape[0], n_envs)
    e.set_params(0, pol)
    e.set_params(1, pol)
    e.set_params(2, val)
    if dist == "gaussian":
        e.set_log_std(log_std)
    e.set_adam(0, None, None, 0)
    e.set_adam(2, None, None, 0)
    e.load_batch(b)
    return e, b, (log_std if dist == "gaussian" else None), pol, val


def engine_grad_errs(e, b, ps, vs, dist, log_std):
    """policy_grad / value_grad views against the reference at the engine's current parameters, from its own inputs
    (advantages with their statistics, returns, old log-probs)."""
    v = lambda k: e.view(k).cpu().numpy()
    pol, val = e.get_params(0), e.get_params(2)
    ref_p = R.policy_loss(pol, ps, b["obs"], b["act"], dist, "ppo_clip", log_std, v("adv_raw"), v("adv_stats"),
                          v("old_logp"), CLIP)
    ref_v = R.value_loss(val, vs, b["obs"], v("ret"))
    errs = grad_errs(v("policy_grad")[:pol.size], ref_p, ps, "policy.d")
    errs.update(grad_errs(v("value_grad")[:val.size], ref_v, vs, "value.d"))
    return errs


def test_engine_step_gradients(path):
    """One PPO update with one policy and one value step from zeroed Adam state: the policy_grad / value_grad views hold
    the gradients at the initial parameters, from the engine's own advantages, returns and old log-probs.  obs 32: the
    fused step refuses it, so PPO takes the two-loop path with the absmax hint slots 0..31 (batch) and 32..63 (last
    observations) exactly full.  (The fused step's gradients: test_fused_step_gradients.)"""
    from rl_replicas_b200.engine import OnPolicyEngine
    ps, vs, dist, n_envs, horizon = [32, 64, 64, 15], [32, 64, 64, 1], "gaussian", 7, 139
    e, b, log_std, pol0, val0 = engine_for(ps, vs, dist, n_envs, horizon, seed=ps[-1] + n_envs)
    st = e.update(OnPolicyEngine.hparams(num_policy_gradients=1, num_value_gradients=1, max_kl_divergence=math.inf))
    assert st.fused == 0 and st.policy_steps_applied == 1 and st.value_steps_applied == 1
    errs = {}
    v = lambda k: e.view(k).cpu().numpy()
    ref_p = R.policy_loss(pol0, ps, b["obs"], b["act"], dist, "ppo_clip", log_std, v("adv_raw"), v("adv_stats"),
                          v("old_logp"), CLIP)
    ref_v = R.value_loss(val0, vs, b["obs"], v("ret"))
    errs.update(grad_errs(v("policy_grad")[:pol0.size], ref_p, ps, "policy.d"))
    errs.update(grad_errs(v("value_grad")[:val0.size], ref_v, vs, "value.d"))
    errs["values"] = rel_err(v("values"), R.values(val0, vs, b["obs"]))
    e.close()
    report(f"two-loop step {ps} {vs} n={b['obs'].shape[0]}", "fp16x2", errs)


def test_run_stage_views_show_the_buffer_the_stage_wrote(path):
    """run_stage("policy_grad" / "value_grad") and run_stage("fused_step") each leave device_view("policy_grad" /
    "value_grad") on the buffer they wrote, whichever path the previous update took."""
    from rl_replicas_b200.engine import OnPolicyEngine
    ps, vs = [17, 64, 64, 6], [17, 64, 64, 1]
    e, b, log_std, _, _ = engine_for(ps, vs, "gaussian", 5, 100, seed=3)
    hp = OnPolicyEngine.hparams(num_policy_gradients=1, num_value_gradients=1, max_kl_divergence=math.inf)
    assert e.update(hp).fused == 1
    for st in ("preamble", "old_logp", "policy_grad", "value_grad"):
        e.run_stage(st, hp)
    report("run_stage two-loop after a fused update", "fp16x2", engine_grad_errs(e, b, ps, vs, "gaussian", log_std))
    assert e.update(hp, algo="vpg").fused == 0
    for st in ("preamble", "old_logp", "pack_obs", "fused_step"):
        e.run_stage(st, hp)
    report("run_stage fused after a two-loop update", "fp16x2", engine_grad_errs(e, b, ps, vs, "gaussian", log_std))
    e.close()


# One fused launch on chosen inputs.  Rows may depend on S, the SM count: the grid is min(tiles, S) and CTA b runs tiles
# b, b + S, b + 2 S, ..., so 128 S rows are one tile per CTA.  Each row keeps its b3 gradient in four running sums, one
# per tile class k mod 4, that add to an earlier tile's sum from tile k = 4 on: 5 tiles per CTA and more.
OBS_COLUMNS = np.r_[10.0 ** np.linspace(-3, 3, 16), 0.0]  # 16 feature scales 1e-3 .. 1e3 and an all-zero column
FUSED_CASES = {
    # one tile: the second 64-row half empty, holding one row, one row short of full
    "one_tile_64": dict(sizes=[17, 64, 64, 6], dist="gaussian", n=64),
    "one_tile_65": dict(sizes=[17, 64, 64, 6], dist="gaussian", n=65),
    "one_tile_127": dict(sizes=[17, 64, 64, 6], dist="gaussian", n=127),
    "one_tile_64_cat": dict(sizes=[8, 64, 64, 15], dist="categorical", n=64),
    "one_tile_65_cat": dict(sizes=[8, 64, 64, 15], dist="categorical", n=65),
    "one_tile_127_cat": dict(sizes=[8, 64, 64, 15], dist="categorical", n=127),
    # obs 31, 15 outputs; 973 rows: 7 tiles + 77 rows
    "obs31_out15_973": dict(sizes=[31, 64, 64, 15], dist="gaussian", n=973),
    # uneven widths, a value network whose first hidden layer is one unit wide; 129 rows: one tile + 1 row
    "uneven_129_cat": dict(sizes=[31, 63, 32, 15], vs=[31, 1, 64, 1], dist="categorical", n=129),
    # one full round, 1 tile per CTA: the widest observation, the most outputs
    "full_round": dict(sizes=[31, 64, 64, 15], dist="gaussian", n=lambda S: 128 * S),
    # 2 tiles per CTA (both observation buffers and their phases), the last tile half full
    "2_tiles": dict(sizes=[31, 64, 63, 15], dist="categorical", n=lambda S: 128 * 2 * S - 64),
    # 5 tiles on half of the CTAs, 4 on the others, the last tile one row
    "4_5_tiles": dict(sizes=[17, 64, 64, 6], dist="gaussian", n=lambda S: 128 * (4 * S + S // 2) + 1),
    "4_5_tiles_cat": dict(sizes=[8, 64, 64, 15], dist="categorical", n=lambda S: 128 * (4 * S + S // 2) + 1),
    # 9 tiles per CTA, ragged last tile
    "9_tiles": dict(sizes=[17, 64, 64, 6], dist="gaussian", n=lambda S: 128 * 9 * S - 51),
    # hidden layers one unit wide in both networks
    "narrow": dict(sizes=[1, 1, 64, 2], vs=[1, 64, 1, 1], dist="categorical", n=3000),
    # distributions at their edges (see GATE_CASES)
    "log_std_-5": dict(sizes=[17, 64, 64, 6], dist="gaussian", n=3000, log_std=-5.0, out_scale=0.02),
    "log_std_+1": dict(sizes=[17, 64, 64, 6], dist="gaussian", n=3000, log_std=1.0),
    "actions_8_sigma": dict(sizes=[17, 64, 64, 6], dist="gaussian", n=3000, log_std=-0.5, sigmas=8.0),
    "logits_30": dict(sizes=[8, 64, 64, 15], dist="categorical", n=3000, out_scale=30.0),
    # sigmas e^-5 .. e^1 under one gradient scale (set by the smallest)
    "log_std_spread": dict(sizes=[17, 64, 64, 6], dist="gaussian", n=3000, log_std=np.linspace(-5.0, 1.0, 6),
                           out_scale=0.02),
    # data-parallel: these rows are a quarter of the global batch
    "n_global_4n": dict(sizes=[17, 64, 64, 6], dist="gaussian", n=3000, dp=4),
    # operand ranges the power-of-two scales absorb: the step stays on the fused path
    "obs_x1e3": dict(sizes=[17, 64, 64, 6], dist="gaussian", n=3000, obs_scale=1e3),
    "obs_x1e-4": dict(sizes=[17, 64, 64, 6], dist="gaussian", n=3000, obs_scale=1e-4),
    "ret_x3e4": dict(sizes=[17, 64, 64, 6], dist="gaussian", n=3000, ret_scale=3e4),
    "ret_x1e-3": dict(sizes=[17, 64, 64, 6], dist="gaussian", n=3000, ret_scale=1e-3),
    "obs_columns": dict(sizes=[17, 64, 64, 6], dist="gaussian", n=3000, obs_scale=OBS_COLUMNS),
}


def fused_problem(name):
    c = dict(FUSED_CASES[name])
    n, dp = c.pop("n"), c.pop("dp", 1)
    n = n(sms()) if callable(n) else n
    pb = policy_problem(c.pop("sizes"), c.pop("dist"), n, seed=500 + list(FUSED_CASES).index(name), **c)
    pb["n_global"] = dp * n
    return pb


def perturbed(pb, seed):
    """The policy with its output bias moved in a random direction, by 0.5 in sigma units (Gaussian: log-ratios of
    rows about N(-1/8, 1/4)) or by 1 (logits): PPO ratios spread past both clip bounds, the KL from the unperturbed
    policy is clearly positive, and no ratio is so large that a gradient row leaves fp16's range."""
    A = pb["sizes"][-1]
    w = np.random.default_rng(seed).standard_normal(A)
    w /= np.linalg.norm(w)
    flat = pb["flat"].copy()
    flat[-A:] += (0.5 * np.exp(pb["log_std"].astype(np.float64)) * w if pb["dist"] == "gaussian" else w
                  ).astype(np.float32)
    return flat


def fused_engine(pb, policy, old_policy):
    """An engine whose batch holds the problem's observations and actions, with its returns as the rewards (episodes of
    100 rows, every other one done): with gamma = 0 the scan's returns are the rewards, so the returns' absmax, which
    sets the value gradient's scale, is the problem's."""
    from rl_replicas_b200.engine import OLD_POLICY, POLICY, VALUE, OnPolicyEngine
    n = pb["n"]
    off = np.r_[np.arange(0, n, 100), n].astype(np.int64)
    b = dict(obs=pb["obs"], act=pb["act"], rew=pb["ret"].astype(np.float64), last_obs=pb["obs"][off[1:] - 1],
             ep_offsets=off, ep_done=np.arange(off.size - 1) % 2 == 0)
    e = OnPolicyEngine(pb["sizes"], pb["vs"], pb["dist"], n, off.size - 1)
    e.set_params(POLICY, policy)
    e.set_params(OLD_POLICY, old_policy)
    e.set_params(VALUE, pb["vflat"])
    if pb["log_std"] is not None:
        e.set_log_std(pb["log_std"])
    e.set_adam(POLICY, None, None, 0)
    e.set_adam(VALUE, None, None, 0)
    e.load_batch(b)
    return e


def fused_hp(pb, K=1, Kv=1, max_kl=math.inf):
    from rl_replicas_b200.engine import OnPolicyEngine
    return OnPolicyEngine.hparams(gamma=0.0, gae_lambda=0.0, max_kl_divergence=max_kl, num_policy_gradients=K,
                                  num_value_gradients=Kv, n_global_rows=pb["n_global"])


def bits(x):
    return np.ascontiguousarray(x).view(np.uint32 if x.dtype == np.float32 else np.uint64)


def assert_clip_binds_both_ways(ref, n):
    if n >= 100:
        assert (ref["ratio"] > 1 + CLIP).any() and (ref["ratio"] < 1 - CLIP).any()


@pytest.mark.parametrize("name", list(FUSED_CASES))
def test_fused_step_gradients(name, path):
    """policy_grad / value_grad of one fused launch (run_stage "fused_step") on the problem's advantages, statistics
    and old log-probs, against the reference."""
    pb = fused_problem(name)
    s, vs, n, ng = pb["sizes"], pb["vs"], pb["n"], pb["n_global"]
    e = fused_engine(pb, pb["flat"], pb["flat"])
    hp = fused_hp(pb)
    e.run_stage("preamble", hp)
    np.testing.assert_array_equal(bits(e.view("ret").cpu().numpy()), bits(pb["ret"]))
    for k in ("adv_raw", "stats", "old_logp"):
        e.view("adv_stats" if k == "stats" else k).copy_(torch.from_numpy(pb[k]))
    e.run_stage("pack_obs", hp)
    e.run_stage("fused_step", hp)
    got_p, got_v = e.view("policy_grad").cpu().numpy(), e.view("value_grad").cpu().numpy()
    e.close()
    ref_p = R.policy_loss(pb["flat"], s, pb["obs"], pb["act"], pb["dist"], "ppo_clip", pb["log_std"], pb["adv_raw"],
                          pb["stats"], pb["old_logp"], CLIP, n_global=ng)
    ref_v = R.value_loss(pb["vflat"], vs, pb["obs"], pb["ret"], n_global=ng)
    assert_clip_binds_both_ways(ref_p, n)
    errs = grad_errs(got_p, ref_p, s, "policy.d")
    errs.update(grad_errs(got_v, ref_v, vs, "value.d"))
    report(f"fused step {name} {s} {vs} n={n} n_global={ng}", "fp16x2", errs)


@pytest.mark.parametrize("name", list(FUSED_CASES))
def test_fused_step_scalar_sums(name, path):
    """One PPO update with one step of each loop, the policy moved off the network the actions were drawn around: it
    stays on the fused path, and the scalar sums of its launch (slot 0: policy, slot K + 1 = 2: value) match the
    reference from the engine's own advantages, statistics and old log-probs."""
    pb = fused_problem(name)
    s, vs, n, ng = pb["sizes"], pb["vs"], pb["n"], pb["n_global"]
    pol = perturbed(pb, 1 + list(FUSED_CASES).index(name))
    e = fused_engine(pb, pol, pb["flat"])
    st = e.update(fused_hp(pb))
    v = lambda k: e.view(k).cpu().numpy()
    adv_raw, stats, old_logp = v("adv_raw"), v("adv_stats"), v("old_logp")
    slots = e.scalar_history()
    e.close()
    assert st.fused == 1 and st.policy_steps_applied == 1 and st.value_steps_applied == 1
    ref = R.policy_loss(pol, s, pb["obs"], pb["act"], pb["dist"], "ppo_clip", pb["log_std"], adv_raw, stats, old_logp,
                        CLIP, n_global=ng)
    assert_clip_binds_both_ways(ref, n)
    ref_v = R.value_loss(pb["vflat"], vs, pb["obs"], pb["ret"], n_global=ng)
    s0 = slots[0]
    errs = {"loss": scal_err(s0[0], ref["loss_sum"], ref["loss_abs_sum"]),
            "kl": scal_err(s0[1], ref["kl_sum"], ref["logp_abs_sum"]),
            "entropy_sum": scal_err(s0[2], ref["entropy_sum"]),
            "logp_sum": scal_err(s0[3], ref["logp_sum"], ref["logp_abs_sum"]),
            "logp2_sum": scal_err(s0[4], ref["logp2_sum"]),
            "mse.loss": scal_err(slots[2][0], ref_v["loss_sum"])}
    assert s0[5] == n
    report(f"fused step sums {name} {s} {vs} n={n} n_global={ng}", "fp16x2", errs)


@pytest.mark.parametrize("tiles", [1, 5])
def test_fused_value_only_launches_match_full_launches(tiles, path):
    """The device-side KL stop fires at step 0 of three: launches 1 and 2 run the value chain alone (no host poll in
    between).  Everything of the value loop is bit-identical to the same update without a KL limit."""
    from rl_replicas_b200.engine import POLICY, VALUE
    K = 3
    pb = policy_problem([17, 64, 64, 6], "gaussian", 128 * tiles * sms() - 37, seed=600 + tiles)
    pb["n_global"] = pb["n"]
    pol = perturbed(pb, 2)
    args = (pb["sizes"], pb["obs"], pb["act"], "gaussian", "eval", pb["log_std"])
    kl0 = float(np.mean(R.policy_loss(pb["flat"], *args)["logp"] - R.policy_loss(pol, *args)["logp"]))
    assert kl0 > 1e-3  # the KL carried by step 0 (POLICY against the OLD_POLICY the actions came from)
    runs = {}
    for label, max_kl in (("stop", kl0 / 3), ("no limit", math.inf)):
        e = fused_engine(pb, pol, pb["flat"])
        st = e.update(fused_hp(pb, K=K, Kv=K, max_kl=max_kl))
        m, vv, _ = e.get_adam(VALUE)
        runs[label] = dict(st=st, pol=e.get_params(POLICY), val=e.get_params(VALUE), m=m, v=vv,
                           grad=e.view("value_grad").cpu().numpy(), slots=e.scalar_history()[K + 1:2 * K + 1])
        e.close()
    a, b = runs["stop"], runs["no limit"]
    assert (a["st"].policy_steps_applied, a["st"].value_steps_applied, a["st"].fused) == (0, K, 1)
    assert (b["st"].policy_steps_applied, b["st"].value_steps_applied, b["st"].fused) == (K, K, 1)
    np.testing.assert_array_equal(bits(a["pol"]), bits(pol))
    for k in ("val", "m", "v", "grad", "slots"):
        np.testing.assert_array_equal(bits(a[k]), bits(b[k]), err_msg=k)


# ---- refusals: host-side checks before any launch ------------------------------------------------------------------
def test_out17_is_refused(path):
    from gpu_helpers import loss_grad
    from rl_replicas_b200._lib import B200RLError
    pb = policy_problem([17, 64, 64, 16], "categorical", 64, 9)
    act17 = np.zeros((64, 17), np.float32)
    flat17 = net(np.random.default_rng(0), [17, 64, 64, 17])
    for dist, act, ls in (("gaussian", act17, np.zeros(17, np.float32)), ("categorical", pb["act"], None)):
        with pytest.raises(B200RLError, match="at most 16 action dimensions"):
            loss_grad([17, 64, 64, 17], flat17, pb["obs"], "ppo_clip", dist, act=act, log_std=ls, adv_raw=pb["adv_raw"],
                      adv_stats=pb["stats"], old_logp=pb["old_logp"])
    torch.cuda.synchronize()


@pytest.mark.parametrize("h,what", [(FP32_MAX_H + 1, "ppo_clip"), (FVP_MAX_H + 1, "fvp")])
def test_one_past_the_fp32_layout_is_refused(h, what, path):
    from gpu_helpers import fvp, loss_grad
    from rl_replicas_b200._lib import B200RLError
    pb = policy_problem([17, h, h, 6], "gaussian", 100, 11)
    with pytest.raises(B200RLError, match="shared memory"):
        if what == "fvp":
            fvp(pb["sizes"], pb["flat"], pb["obs"], "gaussian", np.ones(pb["flat"].size, np.float32), pb["log_std"])
        else:
            loss_grad(pb["sizes"], pb["flat"], pb["obs"], "ppo_clip", "gaussian", act=pb["act"], log_std=pb["log_std"],
                      adv_raw=pb["adv_raw"], adv_stats=pb["stats"], old_logp=pb["old_logp"])
    torch.cuda.synchronize()


def test_engine_refuses_layouts_that_do_not_fit(path):
    """A [17, 128, 128, 6] PPO update, and TRPO on a shape PPO can train but whose FVP layout does not fit, fail with
    the shared-memory message, and the device stays usable."""
    from rl_replicas_b200._lib import B200RLError
    from rl_replicas_b200.engine import OnPolicyEngine
    hp = OnPolicyEngine.hparams(num_policy_gradients=1, num_value_gradients=1, max_kl_divergence=math.inf)
    e = engine_for([17, 128, 128, 6], [17, 64, 64, 1], "gaussian", 4, 50, seed=1)[0]
    with pytest.raises(B200RLError, match="shared memory"):
        e.update(hp)
    e.close()
    h = FVP_MAX_H + 1
    e = engine_for([17, h, h, 6], [17, 64, 64, 1], "gaussian", 4, 50, seed=2)[0]
    assert e.update(hp).policy_steps_applied == 1  # PPO fits
    with pytest.raises(B200RLError, match="shared memory"):
        e.trpo_update(hp)
    e.close()
    torch.cuda.synchronize()
