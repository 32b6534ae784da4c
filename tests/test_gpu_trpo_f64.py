"""GPU: the TRPO step (trpo.cu with its driver b200rl_trpo_update_dp) against the float64 reference, one stage at a
time, on every kernel path and every branch of the line search.

A float32 conjugate-gradient run and a float64 one drift apart chaotically, so whole runs are never compared.  Every
stage is replayed from the engine's own state instead: the engine is run-to-run deterministic (asserted once per case),
so running the update with n_conjugate_gradients = k and then k + 1 exposes iteration k + 1 as a function of the
engine's iterate k, which oracle/onpolicy_f64.cg_iteration replays with the exact Fisher matrix.  The same holds for
the later stages: the step size from the engine's x, the line search at the engine's descent step.

Stages and what each checks (views "cg_x", "cg_r", "cg_p", "cg_z", "cg_descent", "policy_grad", scalar_history()):
* gradient: policy_grad against the float64 surrogate gradient from the engine's advantages, statistics and old
  log-probs, against its conditioning scale (see test_gpu_onpolicy_shapes); loss_before against sum |term|.
* CG: x', r', p' against cg_iteration's elementwise term scales (the largest of them; p' carries the rounding of
  r'); convergence: where the replay
  puts r'.r' below the kernel's 1e-10 with a 10x margin the engine must have stopped there, and later iterations are
  bit-identical no-ops; r'.r' within 10x of 1e-10 is a case on a boundary, and fails.
* step size: xHx against x.(F x + damping x) with the engine's x (a positive form: relative), cg_z against F x, and
  cg_descent bit-identical to the float32 replay of trpo.cu's rule from the engine's xHx and x.
* line search: slot k + 1 of scalar_history() against line_search_eval at the engine's step k (the loss sum against
  sum |term|, the KL sum relative); accepted_index / rejected against the float64 decision, whose margins must be at
  least 10x the bars; every slot after the accepted one exactly zero.
* final parameters: within 1 ulp of prev - fl32(ratio^k) descent (the kernel may contract it to an FMA) when accepted,
  bit-identical to prev when rejected; fvp_launches == n_cg + 1.

Advantages: gamma = lambda = 0 and an all-zero value network make the advantages the rewards, so each case chooses
them; the engine's own adv_raw / adv_stats / old_logp views feed the reference either way.  num_value_gradients = 0
keeps the value network, and with it the preamble, identical across runs.

Bars: about 4x the largest error measured on an H100 over every case of a path (measured figures below)."""
import math
import threading

import numpy as np
import pytest
import torch

from conftest import rel_err
from oracle import onpolicy_f64 as R
from test_gpu_onpolicy_shapes import bits, draw_obs, fallbacks, net, scal_err, scaled_err, sms

pytestmark = pytest.mark.gpu

# Largest errors measured on an H100 80GB HBM3 (power limit 700 W) over all cases, each quantity against its scale:
# gradient 2.9e-7 fp16x2 (the three-row case) / 2.0e-7 fp32; loss_before 4.6e-8; CG iterates 5.3e-6 (the categorical
# [4, 64, 64, 2] case: F v's own error against the iterates' scales); cg_z against F x 5.8e-6; xHx 2.5e-6 (100k rows);
# line-search loss sums 2.5e-7 fp16x2 / 7.0e-8 fp32, KL sums 2.4e-6 fp16x2 / 6.0e-7 fp32.  Each bar about 4x that.
BAR = {"grad.fp16x2": 1.2e-6, "grad.fp32": 8e-7, "loss_before": 2e-7, "cg": 2.4e-5, "xhx": 1e-5, "Fx": 2.4e-5,
       "ls.loss.fp16x2": 1e-6, "ls.loss.fp32": 3e-7, "ls.kl.fp16x2": 1e-5, "ls.kl.fp32": 2.4e-6}
TOL_CG, TOL_MARGIN = 1e-10, 10.0  # the kernel's residual tolerance; decisions and convergence keep 10x off a boundary

# sizes, dist, n (rows, or "full": one 128-row tile per SM); optional: path ("tc": the tensor-core kernels inside
# their gate, "notc": B200RL_DISABLE_TC=1; any shape outside the gate runs the fp32 kernels either way), hidden,
# obs_outlier (row 11 of the observations times this: every launch is redone by the fp32 kernel), n_cg, delta,
# max_backtracks, ratio, damping, accept (the line-search branch the case is built to take: the accepted index, -1 for
# a rejected step), converge (the iteration at which CG stops early), ep (episode length), seed, dp (two ranks: all
# episodes but the last, and the last).
F64_CASES = {
    # ---- tensor-core path: mlp_tc2 forward / backward, mlp_tc_fvp
    "tc_27_64_64_8_n20011": dict(sizes=[27, 64, 64, 8], dist="gaussian", n=20011),  # tail tile, 2 tiles on some CTAs
    "tc_4_64_64_2_cat": dict(sizes=[4, 64, 64, 2], dist="categorical", n=4000),
    "tc_17_64_32_6": dict(sizes=[17, 64, 32, 6], dist="gaussian", n=3001),
    "tc_9_33_20_3_cat": dict(sizes=[9, 33, 20, 3], dist="categorical", n=2000),
    # one input and one output: F's spectrum falls off so fast that from the fifth iteration on p lies where F p is
    # a cancelling sum, known to the FVP kernel only to ~1e-6 of its terms, not of the result; four iterations
    "tc_1_64_64_1": dict(sizes=[1, 64, 64, 1], dist="gaussian", n=2000, n_cg=4),
    "tc_32_64_64_15": dict(sizes=[32, 64, 64, 15], dist="gaussian", n=3000),  # the edge of the gate
    "tc_full_round": dict(sizes=[17, 64, 64, 6], dist="gaussian", n="full"),
    "tc_n100k": dict(sizes=[17, 64, 64, 6], dist="gaussian", n=100003, n_cg=4),  # several tiles per CTA
    # ---- fp32 kernels (mlp_fused.cu, its FVP mode)
    "fp32_obs33": dict(sizes=[33, 64, 64, 6], dist="gaussian", n=641),
    "fp32_out16_cat": dict(sizes=[17, 64, 64, 16], dist="categorical", n=641),
    "fp32_h92": dict(sizes=[17, 92, 92, 6], dist="gaussian", n=641),  # the FVP layout's widest
    "fp32_7_48_5": dict(sizes=[7, 48, 5], dist="gaussian", n=641),
    "fp32_7_64_48_40_5_cat": dict(sizes=[7, 64, 48, 40, 5], dist="categorical", n=641),
    "fp32_relu": dict(sizes=[17, 64, 64, 6], dist="gaussian", n=641, hidden="relu"),
    "notc_27_64_64_8": dict(sizes=[27, 64, 64, 8], dist="gaussian", n=3000, path="notc"),
    # ---- the fp16 range re-run: every forward and FVP launch of the step redone by the fp32 kernel
    "rerun_27_64_64_8": dict(sizes=[27, 64, 64, 8], dist="gaussian", n=3000, obs_outlier=1e6),
    # ---- parameter counts at the 1024-thread stride of the one-CTA CG kernels
    "p1024": dict(sizes=[20, 20, 24, 4], dist="gaussian", n=1500),
    "p1025": dict(sizes=[6, 21, 24, 14], dist="categorical", n=1500),
    "p17": dict(sizes=[2, 3, 2], dist="gaussian", n=700),
    # ---- decision branches; the deltas come from a seeded scan of the float64 step and keep every decision at least
    # 10% of delta (KL) off its boundary.  Moderate damping: x^T F x / x^T H x < 1 keeps the full step's KL below delta
    "accept_0": dict(sizes=[17, 64, 64, 6], dist="gaussian", n=3000, damping=0.1, accept=0),
    # the full step's KL 8% above delta (higher-order terms), the next within it
    "accept_1_kl": dict(sizes=[17, 64, 64, 6], dist="gaussian", n=3000, delta=0.1, accept=1),
    # a huge trust region: the full step's KL is 10% of delta, but it raises the surrogate loss; the next lowers it.
    # Two CG iterations: few enough that the float32 and float64 iterates, and so the branch, agree
    "accept_1_loss": dict(sizes=[4, 64, 64, 2], dist="categorical", n=3000, delta=30.0, n_cg=2, accept=1),
    # both evaluations over the KL limit: rejected, parameters restored
    "reject": dict(sizes=[17, 64, 64, 6], dist="gaussian", n=3000, delta=1.0, max_backtracks=2, accept=-1),
    # damping ~300 ||F||: the damping terms dominate every product; CG meets its tolerance at iteration 2.  The step's
    # KL is ~delta / 300; delta 3 keeps it ~1e-2, where the KL sum is not dominated by the outputs' float32 rounding
    "damping_5e3": dict(sizes=[17, 64, 64, 6], dist="gaussian", n=3000, damping=5e3, delta=3.0, accept=0, converge=2),
    # three rows, two actions: F has rank 3 and g lies in its range, so CG stops at iteration 3
    "early_converge": dict(sizes=[4, 64, 64, 2], dist="categorical", n=3, ep=3, converge=3),
    # ---- data-parallel, two ranks through an in-process all-reduce hook: rank 1 holds the last episode alone, 7 rows
    "dp_uneven": dict(sizes=[17, 64, 64, 6], dist="gaussian", n=2907, dp=True),
}
DEFAULTS = dict(path="tc", hidden="tanh", obs_outlier=None, n_cg=10, delta=0.01, max_backtracks=15, ratio=0.8,
                damping=1e-5, accept=None, converge=None, ep=100, seed=None, dp=False)


def cfg_of(name):
    c = dict(DEFAULTS)
    c.update(F64_CASES[name])
    if c["seed"] is None:
        c["seed"] = 700 + list(F64_CASES).index(name)
    if c["n"] == "full":
        c["n"] = 128 * sms()
    return c


def in_gate(sizes, hidden):
    return len(sizes) == 4 and hidden == "tanh" and sizes[0] <= 32 and max(sizes[1:3]) <= 64 and sizes[3] <= 15


def arith_of(c):
    """The arithmetic of the case's forward / gradient launches."""
    if c["path"] == "tc" and c["obs_outlier"] is None and in_gate(c["sizes"], c["hidden"]):
        return "fp16x2"
    return "fp32"


# ---- problems -------------------------------------------------------------------------------------------------------
def problem(c):
    """Policy, observations, actions and rewards (= the advantages: gamma = lambda = 0, value network zero) in episodes
    of c["ep"] rows, the last one ragged."""
    rng = np.random.default_rng(c["seed"])
    sizes, dist, n = c["sizes"], c["dist"], c["n"]
    A = sizes[-1]
    flat = net(rng, sizes)
    obs = draw_obs(rng, [(sizes, flat)], n, c["hidden"])
    if c["obs_outlier"] is not None:
        obs[11] *= np.float32(c["obs_outlier"])
    log_std = np.linspace(-0.8, -0.2, A).astype(np.float32) if dist == "gaussian" else None
    if dist == "gaussian":
        mean = R.forward_kl(flat, sizes, obs, dist, np.zeros((n, A)), log_std, c["hidden"])["out"]
        act = (mean + np.exp(log_std.astype(np.float64)) * rng.standard_normal((n, A))).astype(np.float32)
    else:
        act = rng.integers(0, A, n).astype(np.float32)
    off = np.r_[np.arange(0, n, c["ep"]), n].astype(np.int64)
    batch = dict(obs=obs, act=act, rew=2.0 * rng.standard_normal(n) + 0.5,
                 last_obs=rng.standard_normal((off.size - 1, sizes[0])).astype(np.float32), ep_offsets=off,
                 ep_done=np.arange(off.size - 1) % 2 == 0)
    return dict(sizes=sizes, vs=sizes[:-1] + [1], dist=dist, flat=flat, log_std=log_std, batch=batch, n=n,
                hidden=c["hidden"])


def shard(batch, lo, hi):
    off = batch["ep_offsets"]
    s, t = int(off[lo]), int(off[hi])
    return dict(obs=batch["obs"][s:t], act=batch["act"][s:t], rew=batch["rew"][s:t], last_obs=batch["last_obs"][lo:hi],
                ep_offsets=(off[lo:hi + 1] - off[lo]).astype(np.int64), ep_done=batch["ep_done"][lo:hi])


def make_engine(pb, batch):
    from rl_replicas_b200.engine import VALUE, OnPolicyEngine
    e = OnPolicyEngine(pb["sizes"], pb["vs"], pb["dist"], batch["obs"].shape[0], batch["ep_done"].shape[0],
                       hidden_act=pb["hidden"])
    e.set_params(VALUE, np.zeros(e.n_value, np.float32))
    if pb["log_std"] is not None:
        e.set_log_std(pb["log_std"])
    e.set_adam(VALUE, None, None, 0)
    e.load_batch(batch)
    return e


STATE_VIEWS = ("cg_x", "cg_r", "cg_p", "cg_z", "cg_descent", "adv_raw", "adv_stats", "old_logp")
TS_FIELDS = ("step_size", "xhx", "loss_before", "new_loss", "kl", "accepted_index", "rejected", "cg_converged",
             "fvp_launches")


def trpo_kw(c, k):
    return dict(max_constraint=c["delta"], n_conjugate_gradients=k, max_backtracks=c["max_backtracks"],
                backtrack_ratio=c["ratio"], hvp_damping_coefficient=c["damping"])


def read_state(e, ts):
    from rl_replicas_b200.engine import OLD_POLICY, POLICY
    st = {k: e.view(k).cpu().numpy().copy() for k in STATE_VIEWS}
    st["grad"] = e.view("policy_grad").cpu().numpy()[:e.n_policy].copy()
    st["params"], st["old_params"] = e.get_params(POLICY), e.get_params(OLD_POLICY)
    st["slots"] = e.scalar_history()
    st["ts"] = {f: getattr(ts, f) for f in TS_FIELDS}
    return st


def run(engines, theta, c, k, n_global=0):
    """One TRPO update of every engine from theta (policy and old policy), n_conjugate_gradients = k; more than one
    engine: data-parallel ranks joined by an in-process all-reduce hook.  Returns rank 0's state after the update,
    with the other ranks' checked identical to it, and the fallback counter's increase."""
    from rl_replicas_b200.engine import OLD_POLICY, POLICY, OnPolicyEngine
    hp = OnPolicyEngine.hparams(gamma=0.0, gae_lambda=0.0, num_value_gradients=0, n_global_rows=n_global)
    for e in engines:  # theta None: continue from the engine's parameters
        if theta is not None:
            e.set_params(POLICY, theta)
            e.set_params(OLD_POLICY, theta)
    torch.cuda.synchronize()
    before = fallbacks()
    if len(engines) == 1:
        _, ts = engines[0].trpo_update(hp, **trpo_kw(c, k))
        states = [read_state(engines[0], ts)]
    else:
        W = len(engines)
        barrier, bufs, out, errors = threading.Barrier(W), [None] * W, [None] * W, []

        def hook(rank):
            def fn(t):
                torch.cuda.current_stream().synchronize()
                bufs[rank] = t
                barrier.wait()
                if rank == 0:
                    total = sum(bufs[1:], bufs[0].clone())
                    for b in bufs:
                        b.copy_(total)
                    torch.cuda.current_stream().synchronize()
                barrier.wait()
            return fn

        def work(r):
            try:
                with torch.cuda.stream(torch.cuda.Stream()):
                    out[r] = engines[r].trpo_update(hp, allreduce=hook(r), **trpo_kw(c, k))[1]
                    torch.cuda.current_stream().synchronize()
            except Exception as exc:  # pragma: no cover
                errors.append(exc)
                barrier.abort()

        threads = [threading.Thread(target=work, args=(r,)) for r in range(W)]
        for t in threads:
            t.start()
        for t in threads:
            t.join(timeout=300)
        assert not errors, errors
        states = [read_state(e, ts) for e, ts in zip(engines, out)]
        for s in states[1:]:  # every decision is taken from all-reduced values: identical on every rank
            assert s["ts"] == states[0]["ts"]
            for key in ("cg_x", "cg_r", "cg_p", "cg_z", "cg_descent", "grad", "params", "adv_stats"):
                np.testing.assert_array_equal(bits(s[key]), bits(states[0][key]), err_msg=key)
        # the reference sees the global batch: the ranks' per-row inputs in episode order
        for key in ("adv_raw", "old_logp"):
            states[0][key] = np.concatenate([s[key] for s in states])
    torch.cuda.synchronize()
    states[0]["fallbacks"] = fallbacks() - before
    return states[0]


def assert_same_state(a, b, what):
    for key in STATE_VIEWS + ("grad", "params", "old_params", "slots"):
        np.testing.assert_array_equal(bits(a[key]), bits(b[key]), err_msg=f"{what}: {key}")
    assert a["ts"] == b["ts"], what


# ---- the stages -------------------------------------------------------------------------------------------------------
class Ref:
    """The float64 reference of one update: the problem at theta with the engine's own per-row inputs."""

    def __init__(self, pb, theta, st):
        self.pb, self.theta = pb, theta
        self.args = (pb["sizes"], pb["batch"]["obs"], pb["batch"]["act"], pb["dist"])
        self.inputs = (st["adv_raw"], st["adv_stats"], st["old_logp"])
        self.n = pb["batch"]["obs"].shape[0]
        self.grad = R.policy_loss(theta, *self.args, "trpo_surrogate", pb["log_std"], *self.inputs, hidden=pb["hidden"],
                                  n_global=self.n)

    def F(self, v):
        s, obs, _, dist = self.args
        return R.fvp(self.theta, s, obs, dist, v, self.pb["log_std"], self.pb["hidden"])["fvp"]

    def evaluate(self, flat):
        return R.line_search_eval(flat, *self.args, self.theta, *self.inputs, self.pb["log_std"], self.pb["hidden"])


def gradient_errs(ref, st, arith):
    sizes = ref.pb["sizes"]
    errs = {f"grad.{k}": scaled_err(g, ref.grad["grads"][k], ref.grad["scales"][k])
            for k, g in R.split(st["grad"], sizes).items()}
    errs = {f"grad.{arith}": max(errs.values())}
    errs["loss_before"] = scal_err(st["ts"]["loss_before"] * ref.n, ref.grad["loss_sum"], ref.grad["loss_abs_sum"])
    return errs


def cg_errs(ref, states, c):
    """Iteration k of the engine (states[k]) against cg_iteration from its iterate k - 1 (states[0]: the initial state
    from the engine's gradient); returns errors and the iteration at which the engine stopped (None: it did not)."""
    errs = {"cg": 0.0}
    stopped = None
    for k in range(1, c["n_cg"] + 1):
        a, b = states[k - 1], states[k]
        if a["ts"]["cg_converged"]:  # stopped: every later iteration is a no-op
            for key in ("cg_x", "cg_r", "cg_p"):
                np.testing.assert_array_equal(bits(b[key]), bits(a[key]), err_msg=f"iteration {k}: {key}")
            assert b["ts"]["cg_converged"] == 1
            continue
        rdotr = float(np.float32(np.dot(a["cg_r"].astype(np.float64), a["cg_r"].astype(np.float64))))
        it = R.cg_iteration(ref.F, a["cg_x"], a["cg_r"], a["cg_p"], rdotr, c["damping"])
        # the iteration that meets the tolerance leaves p' = r' + mu p with r' and mu at rounding level: a direction no
        # later stage reads, so only x' and r' are compared there
        vs = ("x", "r") if b["ts"]["cg_converged"] else ("x", "r", "p")
        e = {f"it{k}.{v}": scaled_err(b[f"cg_{v}"], it[v], it["s" + v]) for v in vs}
        errs["cg"] = max(errs["cg"], *e.values())
        assert max(e.values()) < BAR["cg"], (k, e)
        # convergence: 10x off the tolerance on either side
        assert not TOL_CG / TOL_MARGIN <= it["rdotr"] <= TOL_CG * TOL_MARGIN, (k, it["rdotr"], "CG stops on a boundary")
        assert b["ts"]["cg_converged"] == int(it["rdotr"] < TOL_CG), (k, it["rdotr"])
        if b["ts"]["cg_converged"]:
            stopped = k
    return errs, stopped


def check_update(ref, st, c, arith, expect_fallbacks=0):
    """Step size, line search and final parameters of one update from the engine's x; returns (errors, decision)."""
    x, theta = st["cg_x"], ref.theta
    Fx = ref.F(x)
    errs = {"Fx": rel_err(st["cg_z"], Fx)}
    xhx, _ = R.step_size(x, Fx, c["damping"], c["delta"])
    ts = st["ts"]
    errs["xhx"] = abs(ts["xhx"] - xhx) / xhx
    _, step = R.step_size(x, Fx, c["damping"], c["delta"], f32_xhx=np.float32(ts["xhx"]))
    assert ts["step_size"] == float(step)
    np.testing.assert_array_equal(bits(st["cg_descent"]), bits(step * x), err_msg="descent")
    # the line search at the engine's steps; the float64 decision from the float64 evaluations
    nb, slots = c["max_backtracks"], st["slots"]
    loss_before = ref.grad["loss_sum"] / ref.n
    losses, kls = [], []
    errs[f"ls.loss.{arith}"] = errs[f"ls.kl.{arith}"] = 0.0
    margins = []
    for k in range(nb):
        ratio = np.float32(math.pow(c["ratio"], k))
        flat = (theta.astype(np.float64) - float(ratio) * st["cg_descent"].astype(np.float64)).astype(np.float32)
        ev = ref.evaluate(flat)
        losses.append(ev["loss_sum"] / ref.n)
        kls.append(ev["kl_sum"] / ref.n)
        errs[f"ls.loss.{arith}"] = max(errs[f"ls.loss.{arith}"],
                                       scal_err(slots[1 + k][0], ev["loss_sum"], ev["loss_abs_sum"]))
        errs[f"ls.kl.{arith}"] = max(errs[f"ls.kl.{arith}"], scal_err(slots[1 + k][6], ev["kl_sum"]))
        margins.append((ev["loss_abs_sum"] + ref.grad["loss_abs_sum"]) / ref.n)
        d = R.trpo_decisions(loss_before, losses, kls, c["delta"])
        if d["accepted"] >= 0:
            break
    # every decision at least 10x its bar away from its boundary
    for k in range(d["evaluated"]):
        assert abs(d["loss_margin"][k]) > TOL_MARGIN * BAR[f"ls.loss.{arith}"] * margins[k], (k, d)
        assert abs(d["kl_margin"][k]) > TOL_MARGIN * BAR[f"ls.kl.{arith}"] * kls[k], (k, d)
    assert ts["accepted_index"] == d["accepted"] and ts["rejected"] == int(d["rejected"]), (ts, d)
    assert not slots[1 + d["evaluated"]:1 + nb].any(), "slots after the accepted evaluation"
    assert ts["fvp_launches"] == c["n_cg"] + 1
    if d["rejected"]:
        np.testing.assert_array_equal(bits(st["params"]), bits(theta))
    else:
        ratio = np.float32(math.pow(c["ratio"], d["accepted"]))
        exact = theta.astype(np.float64) - float(ratio) * st["cg_descent"].astype(np.float64)
        want = exact.astype(np.float32)
        assert (np.abs(st["params"].astype(np.float64) - want) <= np.spacing(np.abs(want))).all(), "final parameters"
    np.testing.assert_array_equal(bits(st["old_params"]), bits(st["params"]))
    want = expect_fallbacks(d["evaluated"]) if callable(expect_fallbacks) else expect_fallbacks
    assert st["fallbacks"] == want, (st["fallbacks"], want)
    return errs, d


def report(label, errs):
    print(f"\n{label}: " + ", ".join(f"{k} {v:.1e}" for k, v in errs.items()))
    for k, v in errs.items():
        assert v < BAR[k], (label, k, v, BAR[k])


# ---- the cases --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(F64_CASES))
def test_trpo_stages(name, monkeypatch):
    c = cfg_of(name)
    monkeypatch.delenv("B200RL_FUSED_STEP", raising=False)
    if c["path"] == "notc":
        monkeypatch.setenv("B200RL_DISABLE_TC", "1")
    else:
        monkeypatch.delenv("B200RL_DISABLE_TC", raising=False)
    arith = arith_of(c)
    pb = problem(c)
    theta = pb["flat"]
    b, E = pb["batch"], pb["batch"]["ep_done"].size
    engines = [make_engine(pb, shard(b, 0, E - 1)), make_engine(pb, shard(b, E - 1, E))] if c["dp"] \
        else [make_engine(pb, b)]
    ng = pb["n"] if c["dp"] else 0
    K = c["n_cg"]
    states = {K: run(engines, theta, c, K, ng)}
    assert_same_state(run(engines, theta, c, K, ng), states[K], "run to run")
    for k in range(1, K):
        states[k] = run(engines, theta, c, k, ng)
    for e in engines:
        e.close()
    ref = Ref(pb, theta, states[K])
    for k in range(1, K + 1):  # the preamble and the gradient are the same in every run
        for key in ("adv_raw", "adv_stats", "old_logp", "grad"):
            np.testing.assert_array_equal(bits(states[k][key]), bits(states[K][key]), err_msg=key)
    g = states[K]["grad"]
    states[0] = dict(cg_x=np.zeros_like(g), cg_r=g, cg_p=g, ts=dict(cg_converged=0))
    errs = gradient_errs(ref, states[K], arith)
    e_cg, stopped = cg_errs(ref, states, c)
    errs.update(e_cg)
    if c["obs_outlier"] is not None:
        # every launch of the step on the outlier rows: the values, the old policy, the gradient, each F v and each
        # line-search evaluation
        expect = lambda evaluated: 3 + (K + 1) + evaluated
    else:
        expect = 0
    e_up, d = check_update(ref, states[K], c, arith, expect)
    errs.update(e_up)
    if stopped is not None:  # stopped at iteration j: the rest of the step is that of n_cg = j
        for key in ("cg_x", "cg_descent", "params"):
            np.testing.assert_array_equal(bits(states[K][key]), bits(states[stopped][key]), err_msg=key)
    assert stopped == c["converge"], (stopped, c["converge"])
    if c["accept"] is not None:
        assert d["accepted"] == c["accept"], d
    report(f"{name} {c['sizes']} {c['dist']} n={c['n']} path={c['path']} accepted={d['accepted']} "
           f"rejected={d['rejected']} cg_stop={stopped}", errs)


def test_consecutive_updates_on_one_engine(monkeypatch):
    """Three updates on one engine, a new batch loaded before each: accepted at k = 1, rejected, accepted at k = 0.
    Each is checked from the engine's parameters at its start, so state left over from the previous update (the
    accepted index, the CG / line-search flags, the scalar slots) shows as a wrong decision or a nonzero slot."""
    for k in ("B200RL_DISABLE_TC", "B200RL_FUSED_STEP"):
        monkeypatch.delenv(k, raising=False)
    plan = [("accept_1_kl", 1), ("reject", -1), ("accept_0", 0)]
    cs = [cfg_of(name) for name, _ in plan]
    pbs = [problem(c) for c in cs]
    e = make_engine(pbs[0], pbs[0]["batch"])
    from rl_replicas_b200.engine import POLICY
    theta = pbs[0]["flat"]
    for i, ((name, accept), c, pb) in enumerate(zip(plan, cs, pbs)):
        if i:
            e.load_batch(pb["batch"])
            theta = e.get_params(POLICY)
        st = run([e], theta if i == 0 else None, c, c["n_cg"])
        ref = Ref(pb, theta, st)
        errs = gradient_errs(ref, st, "fp16x2")
        e_up, d = check_update(ref, st, c, "fp16x2")
        errs.update(e_up)
        assert st["ts"]["cg_converged"] == 0
        assert d["accepted"] == accept, (name, d)
        report(f"update {i} ({name}) accepted={d['accepted']} rejected={d['rejected']}", errs)
    e.close()
