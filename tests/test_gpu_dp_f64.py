"""GPU: the data-parallel PPO and VPG updates against the float64 reference oracle/onpolicy_f64.py, stage by stage, with
every rank an engine in this process on one GPU (one host thread per rank).

Two transports join the ranks:
* "hook": an in-process all-reduce callback (AllReduce below) that sums the buffers the engines hand in, in rank order,
  float32 buffers in float32 and float64 buffers in float64, and writes the sum back to every rank.  It carries the
  advantage statistics, the fused step's one buffer per iteration (reduce_adam3 mode 1, callback, mode 2), the two-loop
  path's gradients with their scalar tails, the value loop's gradients, the final KL and the range flags.
* "peer": the one-shot exchange over peer-mapped memory (reduce_adam3 modes 3 and 4 with wait_peers_kernel), exchange
  buffers attached by raw pointer, every rank on its own stream; the small collectives still go through the hook.
  The single-launch form (mode 5) needs its whole grid resident at once, which ranks sharing one GPU cannot give each
  other, so every peer case pins B200RL_PEER_ONE_LAUNCH=0; mode 5 is left to tests/dist_check.py on several GPUs.

The reference runs on the global batch: the per-rank rows the engines hold (observations, actions) and the inputs the
engines computed for themselves (raw advantages, returns, old log-probs), concatenated in rank order, with the
all-reduced advantage statistics and n_global = the sum of the rank row counts.  So an error in one stage never reaches
the next one's check.

Scalar sums.  The single-GPU path keeps every per-launch scalar sum in float64.  Under data parallelism each rank's
sums travel as a float32 tail behind its gradient (adam.cu reduce_partials, mlp_tc3.cu reduce_adam3 modes 1 / 3), so a
slot carries, beyond the single-GPU bar, one float32 rounding of every rank's float64 partial sum S_r: 2^-24 sum_r |S_r|.
The hook then adds the float32 tails in float32, one rounding per addition: 2^-24 |S_0 + ... + S_j| for j = 1 .. W-1
(2^-24 |S| at two ranks).  Mode 4 adds the float32 tails in float64, which is exact here.  The row count (slot entry 5)
is exact while every rank holds fewer than 2^24 rows.  The final-KL slot (K) and the advantage statistics are
all-reduced in float64 and keep the single-GPU bar.

Largest errors measured on an H100 80GB HBM3 at 700 W, per path (the SUMMARY line each case prints): gradients against
their conditioning scale (bar 8e-6 fp16x2, 7e-6 fp32), scalar slots against the scale the single-GPU bar multiplies,
and the float32 tail's share of a slot's bar on that same scale.
    path (cases)                       policy grad  value grad  slots    slots / bar  float32 tail
    fused, hook (W = 2, 3, 4)          2.5e-7       1.0e-7      6.3e-8   7.7e-3       2.0e-7
    two-loop (tc2)                     8.0e-8       4.0e-8      5.2e-8   6.3e-3       1.2e-7
    fp32 kernel                        7.5e-8       5.0e-8      5.9e-8   8.2e-3       1.2e-7
    trainable log_std (log_std 1.9e-8) 6.2e-8       1.9e-8      5.0e-8   7.0e-3       1.2e-7
    VPG (W = 3)                        2.0e-8       2.5e-8      7.9e-8   9.8e-3       1.4e-7
    peer (W = 2, 3; after a trip)      1.5e-7       4.7e-8      4.4e-8   5.5e-3       6.0e-8
The float32 tail is at most 3 % of the single-GPU bar, so it never comes near deciding a check.  Parameters and moments
restate bit for bit from the exchanged gradient on every path."""
import math
import os
import socket
import threading
import time
from datetime import timedelta

import numpy as np
import pytest
import torch

from conftest import rel_err
from oracle import onpolicy as O
from oracle import onpolicy_f64 as R
from oracle.offpolicy_f64 import adam_moments_f32, adam_update_f32
from test_gpu_onpolicy_shapes import BAR, CLIP, bits, grad_errs, net, perturbed, sms

pytestmark = pytest.mark.gpu

U = 2.0 ** -24  # float32 unit roundoff
MARGIN = 1e-5  # smallest float64 distance of any row's PPO ratio from 1 +- clip (relative), asserted per case
LR = {"policy": 3e-4, "value": 1e-3}
B1 = 0.9


# ---- ranks ---------------------------------------------------------------------------------------------------------
class AllReduce:
    """all-reduce(sum) over `world` in-process ranks: rank 0 adds the buffers in rank order (in their own dtype) and
    writes the sum to every rank.  streams=True: the ranks run on their own streams, so every rank synchronises its
    stream before handing its buffer in, and rank 0 after writing the sums."""

    def __init__(self, world, streams=False):
        self.world, self.streams = world, streams
        self.barrier = threading.Barrier(world, timeout=30)
        self.bufs = [None] * world
        self.calls = 0

    def hook(self, rank):
        def fn(t):
            if self.streams:
                torch.cuda.current_stream().synchronize()
            self.bufs[rank] = t
            self.barrier.wait()
            if rank == 0:
                total = self.bufs[0].clone()
                for b in self.bufs[1:]:
                    total += b
                for b in self.bufs:
                    b.copy_(total)
                if self.streams:
                    torch.cuda.current_stream().synchronize()
                self.calls += 1
            self.barrier.wait()
        return fn


class Ranks:
    """W engines joined by the hook, or by the peer exchange (each rank on its own stream, buffers attached by raw
    pointer) with the hook for the small collectives."""

    def __init__(self, engines, peer):
        self.engines, self.peer, self.W = engines, peer, len(engines)
        self.streams = [torch.cuda.Stream() for _ in engines] if peer else None
        if peer:
            ptrs = [e.comm_export()[1] for e in engines]
            for r, e in enumerate(engines):
                e.comm_attach(r, ptrs)
        torch.cuda.synchronize()

    def run(self, fn):
        """fn(rank, engine, hook) on every rank in its own thread; returns the per-rank results.  A failing rank breaks
        the barrier, so the others fail too instead of waiting."""
        ar = AllReduce(self.W, streams=self.peer)
        out, errors = [None] * self.W, []

        def work(r):
            try:
                if self.peer:
                    with torch.cuda.stream(self.streams[r]):
                        out[r] = fn(r, self.engines[r], ar.hook(r))
                        torch.cuda.current_stream().synchronize()
                else:
                    out[r] = fn(r, self.engines[r], ar.hook(r))
            except BaseException as exc:  # pragma: no cover
                errors.append((r, exc))
                ar.barrier.abort()

        threads = [threading.Thread(target=work, args=(r,)) for r in range(self.W)]
        for t in threads:
            t.start()
        deadline = time.monotonic() + 300  # one deadline for all ranks
        for t in threads:
            t.join(timeout=max(0.0, deadline - time.monotonic()))
        assert not any(t.is_alive() for t in threads), "a rank is still running"
        assert not errors, errors
        torch.cuda.synchronize()
        return out

    def update(self, hp, algo="ppo"):
        return self.run(lambda r, e, hook: e.update(hp, algo, allreduce=hook))

    def close(self):
        for e in self.engines:
            e.close()


# ---- problems ------------------------------------------------------------------------------------------------------
def mean_fn(flat, sizes):
    layers = O.unflatten_layers(flat, sizes)
    return lambda o: O.mlp_forward(layers, o)[0]


def rank_batch(n, seed, obs_dim, A, discrete, mean):
    """a ragged block of episodes with n rows (n <= 8: one episode of n rows)"""
    from rl_replicas_b200 import synthetic
    lo = min(50, n)
    hi = max(lo + 1, min(400, n + 1))
    return synthetic.ragged_batch(n, obs_dim, A, discrete, seed=seed, min_len=lo, max_len=hi, mean_fn=mean)


def concat(batches):
    off, base = [np.zeros(1, np.int64)], 0
    for b in batches:
        off.append(b["ep_offsets"][1:] + base)
        base += b["obs"].shape[0]
    out = {k: np.concatenate([b[k] for b in batches]) for k in ("obs", "act", "rew", "last_obs", "ep_done")}
    out["ep_offsets"] = np.concatenate(off).astype(np.int64)
    return out


def logp(flat, pb, obs, act):
    return R.policy_loss(flat, pb["sizes"], obs, act, pb["dist"], "eval", pb["log_std"])["logp"]


def clear_clip_bounds(pb, batches, seed):
    """Redraw the actions of rows whose float64 PPO ratio (policy against old policy) lies within 1e-4 of a clip bound,
    so that the kernels' float32 ratios land on the reference's side of it.  The engine computes the old log-probs
    itself, so the rows are moved through their actions.  Another seed would not do: with the ratios spread past both
    bounds, about 2e-5 of all rows fall within 1e-5 of one, so a batch of 150 k rows (fused_uneven) has a few such
    rows whatever the seed.  The margin is asserted on the engine's own old log-probs all the same (check_update)."""
    rng = np.random.default_rng(seed)
    for b in batches:
        for _ in range(50):
            r = np.exp(logp(pb["pol"], pb, b["obs"], b["act"]) - logp(pb["old"], pb, b["obs"], b["act"]))
            near = np.flatnonzero(R.clip_margin(r, CLIP) < 10 * MARGIN)
            if near.size == 0:
                break
            if pb["dist"] == "categorical":
                b["act"][near] = (b["act"][near] + rng.integers(1, pb["sizes"][-1], near.size)) % pb["sizes"][-1]
            else:
                b["act"][near] += (0.05 * np.exp(pb["log_std"]) * rng.standard_normal((near.size, pb["sizes"][-1]))
                                   ).astype(np.float32)
        else:  # pragma: no cover
            raise AssertionError("could not move the rows off the clip bounds")


def dp_problem(ps, vs, dist, rows, seed, perturb=True):
    """Policy (moved off the old policy by `perturbed` when perturb), old policy, value network, log_std and one ragged
    block of episodes per rank with rows[r] rows."""
    rng = np.random.default_rng(seed)
    A = ps[-1]
    old, val = net(rng, ps), net(rng, vs)
    log_std = np.linspace(-0.7, -0.2, A).astype(np.float32) if dist == "gaussian" else None
    pb = dict(sizes=ps, vs=vs, dist=dist, flat=old, log_std=log_std)
    pol = perturbed(pb, seed + 1) if perturb else old.copy()
    if perturb and dist == "categorical" and A == 2:  # two logits: move their difference by 1.5 so the clip binds
        pol[-A:] += np.asarray([0.75, -0.75], np.float32)
    pb.update(pol=pol, old=old, val=val)
    batches = [rank_batch(n, seed + 10 + r, ps[0], A, dist == "categorical", mean_fn(old, ps)) for r, n in enumerate(rows)]
    if perturb:
        clear_clip_bounds(pb, batches, seed + 2)
    pb["batches"] = batches
    pb["rows"] = [b["obs"].shape[0] for b in batches]
    assert pb["rows"] == list(rows)
    pb["n_global"] = sum(pb["rows"])
    return pb


_OPEN_ENGINES = []  # closed by the clean_env fixture whatever the test's outcome


def make_engines(pb, train_log_std=False):
    from rl_replicas_b200.engine import OLD_POLICY, POLICY, VALUE, OnPolicyEngine
    engines = []
    for b in pb["batches"]:
        e = OnPolicyEngine(pb["sizes"], pb["vs"], pb["dist"], b["obs"].shape[0], b["ep_done"].shape[0],
                           train_log_std=train_log_std)
        tail = [pb["log_std"]] if train_log_std else []
        e.set_params(POLICY, np.concatenate([pb["pol"]] + tail))
        e.set_params(OLD_POLICY, np.concatenate([pb["old"]] + tail))
        e.set_params(VALUE, pb["val"])
        if pb["log_std"] is not None:
            e.set_log_std(pb["log_std"])
        e.set_adam(POLICY, None, None, 0)
        e.set_adam(VALUE, None, None, 0)
        e.load_batch(b)
        engines.append(e)
        _OPEN_ENGINES.append(e)
    return engines


def hparams(pb, K=1, Kv=1, max_kl=math.inf):
    from rl_replicas_b200.engine import OnPolicyEngine
    return OnPolicyEngine.hparams(max_kl_divergence=max_kl, num_policy_gradients=K, num_value_gradients=Kv,
                                  n_global_rows=pb["n_global"])


def state(e):
    """parameters and Adam moments of both networks"""
    from rl_replicas_b200.engine import POLICY, VALUE
    pm, pv, ps_ = e.get_adam(POLICY)
    vm, vv, vs_ = e.get_adam(VALUE)
    return dict(pol=e.get_params(POLICY), val=e.get_params(VALUE), pol_m=pm, pol_v=pv, val_m=vm, val_v=vv,
                pol_step=ps_, val_step=vs_)


def assert_same_bits(items, what):
    for r, x in enumerate(items[1:], 1):
        np.testing.assert_array_equal(bits(np.asarray(x)), bits(np.asarray(items[0])), err_msg=f"{what}: rank {r}")


def assert_same_state(states, keys=("pol", "val", "pol_m", "pol_v", "val_m", "val_v")):
    for k in keys:
        assert_same_bits([s[k] for s in states], k)


# ---- checks 1 - 4 of one update ------------------------------------------------------------------------------------
def tail_bar(parts, hook):
    """the float32 tail's share of a slot's bar (module docstring): parts = the per-rank float64 sums S_r"""
    t = U * sum(abs(p) for p in parts)
    if hook:
        acc = parts[0]
        for p in parts[1:]:
            acc += p
            t += U * abs(acc)
    return t


def check_update(pb, ranks, hp, algo, arith, before, stats, label, clip_binds=True, tls=False):
    """Checks 1-4 of one update with K = Kv = 1 that started from `before` (the state of every rank)."""
    W, ng, ps, vs, dist = ranks.W, pb["n_global"], pb["sizes"], pb["vs"], pb["dist"]
    ppo = algo == "ppo"
    K = 1
    Pp, Pv, A = before["pol"].size - (ps[-1] if tls else 0), before["val"].size, ps[-1]
    Pe = Pp + (A if tls else 0)
    # the engines' own inputs, rank by rank
    view = lambda e, k: e.view(k).cpu().numpy()
    adv = [view(e, "adv_raw") for e in ranks.engines]
    ret = [view(e, "ret") for e in ranks.engines]
    old_logp = [view(e, "old_logp") for e in ranks.engines] if ppo else [None] * W
    stats3 = [view(e, "adv_stats") for e in ranks.engines]
    slots = [e.scalar_history() for e in ranks.engines]
    pgrad = [view(e, "policy_grad")[:Pe] for e in ranks.engines]
    vgrad = [view(e, "value_grad")[:Pv] for e in ranks.engines]
    after = [state(e) for e in ranks.engines]
    errs = {}

    # 1. advantage statistics
    assert_same_bits(stats3, "adv_stats")
    s = stats3[0]
    s1 = sum(float(a.astype(np.float64).sum()) for a in adv)
    s2 = sum(float((a.astype(np.float64) ** 2).sum()) for a in adv)
    m1 = sum(float(np.abs(a.astype(np.float64)).sum()) for a in adv)
    assert abs(s[0] - s1) <= 1e-12 * m1 and abs(s[1] - s2) <= 1e-12 * s2, (s, s1, s2)
    assert s[2] == ng

    # the reference on the global batch
    obs = np.concatenate([b["obs"] for b in pb["batches"]])
    act = np.concatenate([b["act"] for b in pb["batches"]])
    adv_all, ret_all = np.concatenate(adv), np.concatenate(ret)
    olp_all = np.concatenate(old_logp) if ppo else None
    loss = "ppo_clip" if ppo else "vpg"
    p0 = before["pol"][:Pp]
    ls0 = before["pol"][Pp:] if tls else pb["log_std"]
    ref_p = R.policy_loss(p0, ps, obs, act, dist, loss, ls0, adv_all, s, olp_all, CLIP, n_global=ng)
    ref_v = R.value_loss(before["val"], vs, obs, ret_all, n_global=ng)
    if ppo:
        margin = float(R.clip_margin(ref_p["ratio"], CLIP).min())
        print(f"\n{label}: smallest clip margin {margin:.2e}")
        assert margin >= MARGIN, margin
        if clip_binds:
            assert (ref_p["ratio"] > 1 + CLIP).any() and (ref_p["ratio"] < 1 - CLIP).any()

    # 2. gradients, from the gradient views and from the first moments
    assert_same_bits(pgrad, "policy_grad")
    assert_same_bits(vgrad, "value_grad")
    assert_same_state(after)
    arith_p, arith_v = arith
    m_p0 = before["pol_m"]
    zero_m = not np.any(m_p0) and not np.any(before["val_m"])
    for src, gp, gv in (("view", pgrad[0], vgrad[0]),
                        ("exp_avg", after[0]["pol_m"].astype(np.float64) / (1 - B1), after[0]["val_m"].astype(np.float64) / (1 - B1))):
        if src == "exp_avg" and not zero_m:
            continue  # exp_avg / (1 - beta1) is the gradient only for a first step from zeroed moments
        e_p = grad_errs(gp[:Pp], ref_p, ps, f"{src}.policy.d")
        e_v = grad_errs(gv, ref_v, vs, f"{src}.value.d")
        if tls:
            e_p[f"{src}.dlog_std"] = float(np.max(np.abs(gp[Pp:].astype(np.float64) - ref_p["grad_log_std"]))
                                           / ref_p["scale_log_std"].max())
        for k, v in e_p.items():
            errs[k] = (v, BAR[arith_p])
        for k, v in e_v.items():
            errs[k] = (v, BAR[arith_v])

    # 3. scalar sums: slot 0 (policy launch), slot K (final KL, PPO), slot K + 1 (value launch)
    assert_same_bits(slots, "scalar slots")
    sl = slots[0]
    # the fused step's value chain sums the squared errors only (mlp_tc3.cu): its slot carries no row count
    assert sl[0][5] == ng and sl[K + 1][5] == (0 if stats[0].fused else ng)
    cut = np.cumsum([0] + pb["rows"])
    parts_p = [R.policy_loss(p0, ps, obs[a:b], act[a:b], dist, loss, ls0, adv_all[a:b], s,
                             olp_all[a:b] if ppo else None, CLIP, n_global=ng) for a, b in zip(cut[:-1], cut[1:])]
    parts_v = [R.value_loss(before["val"], vs, obs[a:b], ret_all[a:b], n_global=ng)["loss_sum"]
               for a, b in zip(cut[:-1], cut[1:])]
    hook = not (ranks.peer and stats[0].fused)  # the fused peer exchange (mode 4) adds the tails in float64

    tail_of_scale = {}  # the float32 tail's share of each slot's bar, against the scale the single-GPU bar multiplies

    def scalar(name, got, ref, scale, parts, arith_, tail=True):
        t = tail_bar(parts, hook) if tail else 0.0
        bar = BAR[arith_] * scale + t
        errs[name] = (abs(float(got) - ref) / bar, 1.0)
        scal_abs[name] = abs(float(got) - ref) / scale
        tail_of_scale[name] = t / scale

    sums = [("loss", 0, "loss_sum", "loss_abs_sum"), ("entropy", 2, "entropy_sum", None),
            ("logp", 3, "logp_sum", "logp_abs_sum"), ("logp2", 4, "logp2_sum", None)]
    if ppo:
        sums.append(("kl", 1, "kl_sum", "logp_abs_sum"))
    tails, scal_abs = {}, {}
    for name, k, key, sc in sums:
        parts = [q[key] for q in parts_p]
        tails[name] = tail_bar(parts, hook) / max(abs(ref_p[key]), 1e-300)
        scalar(f"slot0.{name}", sl[0][k], ref_p[key], abs(ref_p[key]) if sc is None else ref_p[sc], parts, arith_p)
    scalar("value.loss", sl[K + 1][0], ref_v["loss_sum"], ref_v["loss_sum"], parts_v, arith_v)
    tails["value.loss"] = tail_bar(parts_v, hook) / ref_v["loss_sum"]
    if ppo:  # the KL after the step, all-reduced in float64
        p1 = after[0]["pol"][:Pp]
        ls1 = after[0]["pol"][Pp:] if tls else pb["log_std"]
        lp1 = R.policy_loss(p1, ps, obs, act, dist, "eval", ls1)
        kl1 = float((olp_all.astype(np.float64) - lp1["logp"]).sum())
        scalar("slotK.kl", sl[K][1], kl1, lp1["logp_abs_sum"], [], arith_p, tail=False)
        assert sl[K][5] == ng

    # UpdateStats against the slots and n_global
    for r, st in enumerate(stats):
        assert st.policy_steps_applied == K and st.value_steps_applied == 1, r
        assert st.policy_loss_before == sl[0][0] / ng and st.entropy_before == sl[0][2] / ng
        assert st.value_loss_first == sl[K + 1][0] / ng and st.value_loss_mean == sl[K + 1][0] / ng / 1
        if ppo:
            assert st.kl_divergence == sl[st.policy_steps_applied][1] / ng
        mean = s[0] / s[2]
        assert st.adv_mean == mean
        assert abs(st.adv_std - math.sqrt((s[1] - s[2] * mean * mean) / (s[2] - 1.0))) <= 1e-14 * st.adv_std

    # 4. the step, restated in float32 from the exchanged gradient and the kernel's own moments
    step_p, step_v = before["pol_step"] + 1, before["val_step"] + 1
    assert after[0]["pol_step"] == step_p and after[0]["val_step"] == step_v
    for net_, g, lr, step in (("pol", pgrad[0], LR["policy"], step_p), ("val", vgrad[0], LR["value"], step_v)):
        m, v = adam_moments_f32(g, before[f"{net_}_m"], before[f"{net_}_v"])
        np.testing.assert_array_equal(bits(after[0][f"{net_}_m"]), bits(m), err_msg=f"{label} {net_} exp_avg")
        np.testing.assert_array_equal(bits(after[0][f"{net_}_v"]), bits(v), err_msg=f"{label} {net_} exp_avg_sq")
        p = adam_update_f32(before[net_], after[0][f"{net_}_m"], after[0][f"{net_}_v"], step, lr)
        np.testing.assert_array_equal(bits(after[0][net_]), bits(p), err_msg=f"{label} {net_} parameters")

    worst = max(errs, key=lambda k: errs[k][0] / errs[k][1])
    print(f"{label}: largest error / bar {errs[worst][0] / errs[worst][1]:.2e} ({worst} {errs[worst][0]:.1e}); "
          f"float32 tail / |sum|: " + ", ".join(f"{k} {v:.1e}" for k, v in tails.items()))
    print("  " + ", ".join(f"{k} {v:.1e}" for k, (v, b) in errs.items()))
    gmax = lambda pre: max((v for k, (v, b) in errs.items() if pre in k), default=float("nan"))
    print(f"SUMMARY {label} | policy grad {gmax('policy.d'):.1e} | value grad {gmax('value.d'):.1e} | "
          f"log_std grad {gmax('dlog_std'):.1e} | slots {max(scal_abs.values()):.1e} of scale, "
          f"{max(errs[k][0] for k in scal_abs):.1e} of bar | float32 tail {max(tail_of_scale.values()):.1e} of scale")
    bad = {k: v for k, v in errs.items() if not v[0] < v[1]}
    assert not bad, (label, bad)
    return after


# ---- case table ----------------------------------------------------------------------------------------------------
GAUSS = ([17, 64, 64, 6], [17, 64, 64, 1], "gaussian")
CASES = {
    # about 20 k rows per rank
    "fused_even": dict(nets=GAUSS, rows=lambda S: [20011, 19993], fused=1),
    # one 7-row episode; exactly one tile of 128 rows; 9 full tiles on every CTA
    "fused_uneven": dict(nets=GAUSS, rows=lambda S: [7, 128, 128 * 9 * S], fused=1),
    # ragged; rank 1 has fewer tiles than there are SMs
    "fused_categorical": dict(nets=([4, 64, 64, 2], [4, 64, 64, 1], "categorical"),
                              rows=lambda S: [12001, 1000, 128 * S + 1, 3307], fused=1),
    "two_loop": dict(nets=GAUSS, rows=lambda S: [6001, 2999], fused=0, env={"B200RL_FUSED_STEP": "0"}),
    # obs 33 is outside the tensor-core gate: the fp32 kernel (mlp_fused.cu) runs every launch
    "fp32_kernel": dict(nets=([33, 64, 64, 6], [33, 64, 64, 1], "gaussian"), rows=lambda S: [3001, 1500], fused=0,
                        arith=("fp32", "fp32")),
    # the exchanged policy vector is Pe = P + A: network parameters and log_std (the fp32 kernel's log_std columns)
    "train_log_std": dict(nets=GAUSS, rows=lambda S: [4101, 2500], fused=0, tls=True, arith=("fp32", "fp16x2")),
    "vpg": dict(nets=GAUSS, rows=lambda S: [3000, 77, 5000], fused=0, algo="vpg"),
    "peer_uneven": dict(nets=GAUSS, rows=lambda S: [10007, 7], fused=1, peer=True),
    "peer_three": dict(nets=GAUSS, rows=lambda S: [6000, 2500, 9001], fused=1, peer=True),
}


@pytest.fixture
def clean_env(monkeypatch):
    for k in ("B200RL_DISABLE_TC", "B200RL_FUSED_STEP", "B200RL_PEER_ONE_LAUNCH", "B200RL_PEER_EXCHANGE"):
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("B200RL_PEER_ONE_LAUNCH", "0")  # never mode 5 on one GPU (module docstring)
    yield monkeypatch
    # a failed case must not leave engines (and their peer-attached exchange buffers) to the next one
    while _OPEN_ENGINES:
        _OPEN_ENGINES.pop().close()
    torch.cuda.synchronize()


@pytest.mark.parametrize("name", list(CASES))
def test_dp_update_stage_by_stage(name, clean_env):
    c = CASES[name]
    for k, v in c.get("env", {}).items():
        clean_env.setenv(k, v)
    ps, vs, dist = c["nets"]
    algo, tls = c.get("algo", "ppo"), c.get("tls", False)
    pb = dp_problem(ps, vs, dist, c["rows"](sms()), seed=700 + 10 * list(CASES).index(name), perturb=algo == "ppo")
    ranks = Ranks(make_engines(pb, tls), c.get("peer", False))
    hp = hparams(pb)
    before = state(ranks.engines[0])
    stats = ranks.update(hp, algo)
    assert [st.fused for st in stats] == [c["fused"]] * ranks.W
    label = f"{name} W={ranks.W} rows={pb['rows']}"
    check_update(pb, ranks, hp, algo, c.get("arith", ("fp16x2", "fp16x2")), before, stats, label, tls=tls)
    ranks.close()


# ---- 5. KL early stop across ranks ---------------------------------------------------------------------------------
KL_ROWS = [5003, 3001]


def kl_problem():
    pb = dp_problem(*GAUSS, KL_ROWS, seed=900, perturb=False)
    pb["full"] = concat(pb["batches"])
    return pb


@pytest.mark.parametrize("peer", [False, True], ids=["hook", "peer"])
def test_dp_kl_early_stop(peer, clean_env):
    """The KL stop at steps 1, 7 and 9 of 12 (7 and 9 on both sides of the host's 8-iteration poll in
    run_fused_iterations): the same decision on every rank, the rule replayed on the engines' own slots, and both
    networks within 1e-5 of the float32 oracle on the concatenated batch."""
    K = 12
    pb = kl_problem()
    ng = pb["n_global"]
    ranks = Ranks(make_engines(pb), peer)
    ranks.update(hparams(pb, K, K))
    kls = ranks.engines[0].scalar_history()[:K, 1] / ng
    ranks.close()
    f32 = np.float32
    for stop in (1, 7, 9):
        lo, hi = f32(np.max(kls[:stop])), f32(kls[stop])
        assert hi > lo, (stop, kls)
        max_kl = (float(lo) + float(hi)) / 2 / 1.5
        assert lo < f32(1.5 * max_kl) < hi
        ranks = Ranks(make_engines(pb), peer)
        stats = ranks.update(hparams(pb, K, K, max_kl))
        states = [state(e) for e in ranks.engines]
        slots = [e.scalar_history() for e in ranks.engines]
        ranks.close()
        assert [st.policy_steps_applied for st in stats] == [stop] * ranks.W
        assert [st.value_steps_applied for st in stats] == [K] * ranks.W
        assert [st.fused for st in stats] == [1] * ranks.W
        fired = [i for i in range(K) if f32(slots[0][i, 1] / ng) > f32(1.5 * max_kl)]
        assert fired and fired[0] == stop, (fired, stop)
        assert_same_state(states)
        out = O.ppo_train(pb["full"], O.unflatten_layers(pb["pol"], pb["sizes"]), O.unflatten_layers(pb["val"], pb["vs"]),
                          "gaussian", pb["log_std"], O.AdamState(pb["pol"].size, LR["policy"]),
                          O.AdamState(pb["val"].size, LR["value"]), max_kl=max_kl, n_policy=K, n_value=K)
        assert out["policy_steps"] == stop
        ep, ev = rel_err(states[0]["pol"], out["policy_flat"]), rel_err(states[0]["val"], out["value_flat"])
        print(f"\nKL stop at {stop} ({'peer' if peer else 'hook'}): policy {ep:.1e}, value {ev:.1e} of the oracle")
        assert ep < 1e-5 and ev < 1e-5


# ---- 6. a range trip on one rank only --------------------------------------------------------------------------------
@pytest.mark.parametrize("peer", [False, True], ids=["hook", "peer"])
def test_dp_range_trip_on_one_rank(peer, clean_env):
    """One observation of rank 1 is 1e6 times the others: the fused step's fp16 operands leave their range there only.
    The range flags are all-reduced, so every rank redoes the update on the two-loop path (rank 0 from its snapshot),
    and the result is bit-identical to the same data-parallel update run with B200RL_FUSED_STEP=0.  On the peer path a
    clean update on the same engines then runs fused again: the aborted attempt kept the exchange's sequence numbers in
    step."""
    K = 2
    pb = dp_problem(*GAUSS, [4001, 3003], seed=950)
    clean_obs = pb["batches"][1]["obs"].copy()
    pb["batches"][1]["obs"][5] *= np.float32(1e6)
    runs = {}
    for label, fused in (("trip", True), ("two-loop", False)):
        if not fused:
            clean_env.setenv("B200RL_FUSED_STEP", "0")
        ranks = Ranks(make_engines(pb), peer and fused)
        stats = ranks.update(hparams(pb, K, K))
        assert [st.fused for st in stats] == [0] * ranks.W, label
        assert [st.policy_steps_applied for st in stats] == [K] * ranks.W
        runs[label] = [state(e) for e in ranks.engines]
        clean_env.delenv("B200RL_FUSED_STEP", raising=False)
        if fused:
            keep = ranks
        else:
            ranks.close()
    assert_same_state(runs["trip"])
    for k in ("pol", "val", "pol_m", "pol_v", "val_m", "val_v"):
        np.testing.assert_array_equal(bits(runs["trip"][0][k]), bits(runs["two-loop"][0][k]), err_msg=k)
    if peer:
        pb["batches"][1]["obs"] = clean_obs
        keep.engines[1].load_batch(pb["batches"][1])
        before = state(keep.engines[0])
        stats = keep.update(hparams(pb))
        assert [st.fused for st in stats] == [1] * keep.W
        check_update(pb, keep, hparams(pb), "ppo", ("fp16x2", "fp16x2"), before, stats,
                     "peer update after a range trip", clip_binds=False)
    keep.close()


# ---- 7. consecutive peer updates against the hook ------------------------------------------------------------------
def test_dp_consecutive_peer_updates_match_the_hook(clean_env):
    """Two updates of K = 3 on the peer path reuse both exchange-buffer parities within and across updates.  At two
    ranks a sum of two floats does not depend on the order of its terms, so parameters and moments equal the hook
    path's bit for bit; the scalar slots differ at most by the hook's one float32 rounding of each sum."""
    K = 3
    pb = dp_problem(*GAUSS, [5003, 3001], seed=980)
    runs = {}
    for peer in (False, True):
        ranks = Ranks(make_engines(pb), peer)
        hist = []
        for _ in range(2):
            stats = ranks.update(hparams(pb, K, K))
            assert [st.fused for st in stats] == [1] * ranks.W
            assert [st.policy_steps_applied for st in stats] == [K] * ranks.W
            states = [state(e) for e in ranks.engines]
            assert_same_state(states)
            hist.append((states[0], ranks.engines[0].scalar_history()))
        runs[peer] = hist
        ranks.close()
    worst = 0.0
    for (sh, slh), (sp, slp) in zip(runs[False], runs[True]):
        for k in ("pol", "val", "pol_m", "pol_v", "val_m", "val_v"):
            np.testing.assert_array_equal(bits(sp[k]), bits(sh[k]), err_msg=k)
        assert slh.shape == slp.shape
        rows = list(range(K)) + list(range(K + 1, 2 * K + 1))  # slot K (final KL) is all-reduced in float64
        np.testing.assert_array_equal(slp[K], slh[K])
        d = np.abs(slp[rows] - slh[rows])
        assert np.all(d <= U * np.abs(slh[rows])), d
        np.testing.assert_array_equal(slp[rows, 5], slh[rows, 5])
        worst = max(worst, float(np.max(d / np.maximum(U * np.abs(slh[rows]), 1e-300))))
    print(f"\nconsecutive peer updates: slots differ from the hook's by at most {worst:.2f} x 2^-24 |sum|")


# ---- 8. the public API: PPO(distributed=True) on a gloo group of two processes -------------------------------------
GLOO_K = 4


def gloo_problem():
    return dp_problem(*GAUSS, [5003, 3001], seed=990, perturb=False)


def _gloo_worker(rank, world, port, out):
    """One rank of PPO(..., distributed=True, process_group=pg) on cuda:0: _global_rows, _make_allreduce and its
    float32 / float64 buffers over gloo, the NCCL-free all-reduce per iteration (B200RL_PEER_EXCHANGE=0)."""
    import torch.distributed as dist
    from test_gpu_ppo import build, flat
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), B200RL_PEER_EXCHANGE="0")
    os.environ.pop("B200RL_FUSED_STEP", None)
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=timedelta(seconds=60))
    try:
        pg = dist.new_group(list(range(world)), backend="gloo")
        # gloo's all-reduce takes CUDA tensors of both dtypes the engine hands over
        for dt in (torch.float32, torch.float64):
            t = torch.full((3,), float(rank + 1), dtype=dt, device="cuda")
            dist.all_reduce(t, group=pg)
            assert t.is_cuda and t.tolist() == [3.0] * 3, (dt, t)
        pb = gloo_problem()
        ppo = build(pb["sizes"], pb["vs"], "gaussian", pb["pol"], pb["val"], pb["log_std"], distributed=True,
                    process_group=pg, num_policy_gradients=GLOO_K, num_value_gradients=GLOO_K,
                    max_kl_divergence=float("inf"))
        ppo.train_packed(pb["batches"][rank])
        st = ppo.last_update_stats
        out[rank] = dict(pol=flat(ppo.policy.network).tobytes(), val=flat(ppo.value_function.network).tobytes(),
                         peer=bool(ppo._engine.peer_exchange), fused=st.fused, steps=st.policy_steps_applied,
                         kl_divergence=st.kl_divergence, adv_std=st.adv_std, value_loss_mean=st.value_loss_mean)
        dist.barrier(group=pg)
    finally:
        dist.destroy_process_group()


def test_dp_public_api_on_gloo_matches_the_hook(clean_env):
    """PPO(distributed=True) on a gloo group of two spawned processes sharing this GPU: every rank's networks equal the
    in-process hook run's bit for bit (at two ranks a sum does not depend on the order of its terms), and so do the
    statistics the update reports."""
    import multiprocessing as mpc
    ctx = mpc.get_context("spawn")  # fork() from a multi-threaded process that holds a CUDA context is not safe
    with socket.socket() as sock:
        sock.bind(("127.0.0.1", 0))
        port = sock.getsockname()[1]
    with ctx.Manager() as mgr:
        out = mgr.dict()
        procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, out)) for r in range(2)]
        for p in procs:
            p.start()
        deadline = time.monotonic() + 300
        for p in procs:
            p.join(timeout=max(0.0, deadline - time.monotonic()))
        alive = [p for p in procs if p.is_alive()]
        for p in alive:
            p.terminate()
            p.join()
        assert not alive, "a rank did not finish"
        assert [p.exitcode for p in procs] == [0, 0]
        got = [dict(out[r]) for r in range(2)]
    pb = gloo_problem()
    ranks = Ranks(make_engines(pb), False)
    stats = ranks.update(hparams(pb, GLOO_K, GLOO_K))
    want = state(ranks.engines[0])
    for r, g in enumerate(got):
        assert not g["peer"] and g["fused"] == stats[0].fused == 1 and g["steps"] == GLOO_K, (r, g)
        np.testing.assert_array_equal(np.frombuffer(g["pol"], np.uint32), bits(want["pol"]), err_msg=f"rank {r} policy")
        np.testing.assert_array_equal(np.frombuffer(g["val"], np.uint32), bits(want["val"]), err_msg=f"rank {r} value")
        for k in ("kl_divergence", "adv_std", "value_loss_mean"):
            assert g[k] == getattr(stats[0], k), (r, k, g[k], getattr(stats[0], k))
    print(f"\ngloo public API: both ranks equal the hook run bit for bit ({GLOO_K} + {GLOO_K} steps, "
          f"rows {pb['rows']})")
