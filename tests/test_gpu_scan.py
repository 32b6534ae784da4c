"""GPU: b200rl_gae_scan (csrc/gae_scan.cu) against the float64 scan reference (oracle/onpolicy_f64.gae_scan), in both of
its kernels: the episode-parallel kernel (one warp per episode; the regime RL batches live in) and the tile kernel with
decoupled look-back (few or very long episodes).

Bars, per element, for adv and ret:  |got - ref64| <= 2^-24 |ref64| + 1e-12 S.  The first term is one float32 rounding of
the float64 recurrence, the second the float64 reassociation of a scan, relative to the same recurrence run over the
magnitudes of its terms (S).  Statistics: stats[2] == n, stats[0] / stats[1] equal the float64 sum / sum of squares of
the returned float32 advantages to 1e-12 (of the sum of magnitudes).  A NaN in the statistics is the tile kernel's
protocol-failure flag.  Every case prints its largest margin (error / bar; 1 = at the bar).  On large cases it sits just
under 1: that is the float32 rounding itself, which reaches 2^-24 |x| for x just above a power of two.

The launcher here keeps ONE workspace across launches, the way the engine does: the workspace is zeroed once and every
launch must leave it clean for the next, whichever kernel ran and whatever n was.  Outputs are prefilled with NaN and
followed by a sentinel tail, the workspace by a guard pattern; every launch is checked to write all n outputs and
nothing past them.
"""
import numpy as np
import pytest
import torch

from oracle import onpolicy_f64 as R

pytestmark = pytest.mark.gpu

F32 = np.float32
TAIL = 64      # sentinel floats after adv / ret
GUARD = 256    # pattern bytes after the workspace
SENTINEL = -7.25


def scan_kernel(n, n_ep):
    """The host's regime switch in b200rl_gae_scan (gae_scan.cu): which kernel a launch of this shape runs."""
    return "episode" if (n_ep >= 256 and n_ep <= n // 16 and n // n_ep <= 32768) else "tile"


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def episode_warps(n_ep):
    """Warps of the episode kernel's grid: min(ceil(n_ep / 8), 2 per SM) CTAs of 8 warps."""
    return min((n_ep + 7) // 8, 2 * sm_count()) * 8


def tile_grid_bound():
    """An upper bound of the tile kernel's persistent grid: resident CTAs of 288 threads, 2048 threads per SM."""
    return (2048 // 288) * sm_count()


# ---- batches ---------------------------------------------------------------------------------------------------------
def make_batch(lens, f64, seed, frac_not_done=0.5):
    """Random rewards (float64 or float32), nonzero values and last values, and a mix of done and not-done episodes."""
    rng = np.random.default_rng(seed)
    lens = np.asarray(lens, dtype=np.int64)
    assert lens.min() >= 1
    n, e = int(lens.sum()), lens.size
    rew = rng.standard_normal(n)
    if not f64:
        rew = rew.astype(F32)
    done = rng.random(e) >= frac_not_done
    if e >= 2:
        done[0], done[-1] = True, False
    else:
        done[:] = False
    return dict(rew=rew, values=rng.standard_normal(n, dtype=F32), last_values=rng.standard_normal(e, dtype=F32),
                off=np.concatenate([[0], np.cumsum(lens)]).astype(np.int64), done=done)


def lens_sum_to(rng, n_ep, total, lo, hi):
    """n_ep random lengths in [lo, hi] that sum to exactly `total`."""
    lens = rng.integers(lo, hi + 1, n_ep)
    while lens.sum() != total:
        i = int(rng.integers(n_ep))
        if lens.sum() < total and lens[i] < hi:
            lens[i] += 1
        elif lens.sum() > total and lens[i] > lo:
            lens[i] -= 1
    return lens


def tile_overlap_lens(rng, ks, tail):
    """Episodes such that tile t (2048 items; the last one `tail` items) is overlapped by exactly ks[t] episodes: the
    episode running into each tile continues from the tile before, ks[t] - 1 more start inside it."""
    sizes = [2048] * (len(ks) - 1) + [tail]
    cuts = []
    for t, (k, sz) in enumerate(zip(ks, sizes)):
        cuts += sorted((rng.choice(np.arange(1, sz), k - 1, replace=False) + 2048 * t).tolist())
    return np.diff([0] + cuts + [sum(sizes)])


def _ragged_1_64(seed=1, n_ep=6000):
    lens = np.random.default_rng(seed).integers(1, 65, n_ep)
    assert (lens == 1).any() and (lens == 2).any()
    return lens


def _ragged_200_3000():
    lens = np.random.default_rng(2).integers(200, 3001, 3000)
    off = np.concatenate([[0], np.cumsum(lens)])
    for m in (8, 256):  # episode starts and ends at every residue
        assert np.unique(off[:-1] % m).size == m and np.unique(off[1:] % m).size == m
    return lens


def _n_mod_8():
    lens = np.random.default_rng(3).integers(20, 80, 400)
    lens[-1] = 53
    lens[-2] += (3 - int(lens.sum())) % 8  # n % 8 == 3: the last episode runs through the final partial lane
    assert lens.sum() % 8 == 3
    return lens


EPISODE_CASES = {  # name -> (lengths, fraction of episodes not done); gamma 0.99, lambda 0.97
    "fixed_1024x1000": (lambda: [1000] * 1024, 0.1),
    "fixed_16384x1000": (lambda: [1000] * 16384, 0.1),
    "fixed_300x1001": (lambda: [1001] * 300, 0.3),
    "fixed_4096x999": (lambda: [999] * 4096, 0.3),
    "ragged_1_64": (_ragged_1_64, 0.5),
    "ragged_200_3000": (_ragged_200_3000, 0.5),
    "n_mod_8": (_n_mod_8, 0.5),
    "exactly_256_episodes": (lambda: np.random.default_rng(4).integers(20, 200, 256), 0.5),
    "exactly_n_over_16": (lambda: lens_sum_to(np.random.default_rng(5), 1000, 16000, 1, 31), 0.5),
}

TILE_CASES = {  # name -> (lengths, frac_not_done, gamma, lambda)
    "three_episodes_8M": (lambda: [3_000_001, 2_500_003, 2_900_005], 0.5, 0.99, 0.97),
    "tiles_48_49_partial_48": (lambda: tile_overlap_lens(np.random.default_rng(6), [48, 49, 48], 1001), 0.5, 0.99, 0.97),
    "tiles_49_48_partial_49": (lambda: tile_overlap_lens(np.random.default_rng(7), [49, 48, 49], 999), 0.5, 0.99, 0.97),
    "one_2M_episode_gamma_lambda_1": (lambda: [2_000_003], 1.0, 1.0, 1.0),
    "one_2M_episode_decaying": (lambda: [2_000_003], 1.0, 0.99, 0.97),
}


# ---- launcher --------------------------------------------------------------------------------------------------------
class Scan:
    """b200rl_gae_scan with one workspace for every launch (sized for n_max, zeroed once, followed by a guard)."""

    def __init__(self, n_max):
        from rl_replicas_b200 import _lib
        self.lib, self.check = _lib.load(), _lib.check
        self.wsb = int(self.lib.b200rl_gae_scan_workspace_bytes(n_max))
        self.ws = torch.zeros(self.wsb + GUARD, dtype=torch.uint8, device="cuda")
        self.guard = (torch.arange(GUARD, dtype=torch.int64) * 37 + 11).remainder(256).to(torch.uint8)
        self.ws[self.wsb:] = self.guard.cuda()

    @staticmethod
    def upload(b):
        return dict(rew=torch.from_numpy(np.ascontiguousarray(b["rew"])).cuda(), f64=b["rew"].dtype == np.float64,
                    v=torch.from_numpy(b["values"]).cuda(), lv=torch.from_numpy(b["last_values"]).cuda(),
                    off=torch.from_numpy(b["off"]).cuda(), done=torch.from_numpy(b["done"].astype(np.uint8)).cuda(),
                    n=int(b["off"][-1]), e=int(b["done"].size))

    def launch(self, x, gamma, lam):
        """Queues one launch on the current stream (inputs from upload()); returns its output buffers."""
        import ctypes as C
        p = lambda t: C.c_void_p(t.data_ptr())
        n, e = x["n"], x["e"]
        d = {}
        for k in ("adv", "ret"):
            d[k] = torch.full((n + TAIL,), float("nan"), dtype=torch.float32, device="cuda")
            d[k][n:] = SENTINEL
        d["stats"] = torch.full((3,), float("nan"), dtype=torch.float64, device="cuda")
        self.check(self.lib.b200rl_gae_scan(
            p(x["rew"]), int(x["f64"]), p(x["v"]), p(x["lv"]), p(x["off"]), p(x["done"]), n, e,
            gamma, lam, p(d["adv"]), p(d["ret"]), p(d["stats"]), p(self.ws), self.wsb,
            int(torch.cuda.current_stream().cuda_stream)), "gae_scan")
        d["n"] = n
        return d

    def finish(self, d):
        """Waits, checks that every output was written and nothing past them; returns host adv, ret, stats."""
        torch.cuda.synchronize()
        n = d["n"]
        out = []
        for k in ("adv", "ret"):
            t = d[k].cpu().numpy()
            assert np.isfinite(t[:n]).all(), f"{k}: {int((~np.isfinite(t[:n])).sum())} of {n} outputs not written"
            assert (t[n:] == F32(SENTINEL)).all(), f"{k}: written past n"
            out.append(t[:n])
        assert torch.equal(self.ws[self.wsb:].cpu(), self.guard), "workspace guard overwritten"
        return out[0], out[1], d["stats"].cpu().numpy()

    def run(self, b, gamma, lam):
        return self.finish(self.launch(self.upload(b), gamma, lam))


def check_scan(name, b, got, gamma, lam):
    """The bars of the module docstring; prints and returns the largest margins."""
    adv, ret, stats = got
    adv64, ret64, s_adv, s_ret = R.gae_scan(b["rew"], b["values"], b["last_values"], b["off"], b["done"], gamma, lam)
    margins = {}
    for k, x, ref, s in (("adv", adv, adv64, s_adv), ("ret", ret, ret64, s_ret)):
        err = np.abs(x.astype(np.float64) - ref)
        bar = 2.0 ** -24 * np.abs(ref) + 1e-12 * s
        m = np.where(bar > 0, err / np.where(bar > 0, bar, 1.0), np.where(err > 0, np.inf, 0.0))
        i = int(np.argmax(m))
        margins[k] = float(m[i])
        assert m[i] <= 1.0, (f"{name}: {k}[{i}] = {x[i]!r}, reference {ref[i]!r} (S = {s[i]:.3e}): "
                             f"{m[i]:.3g} x the bar; {int((m > 1).sum())} of {m.size} items over it")
    a = adv.astype(np.float64)
    assert stats[2] == adv.size, f"{name}: stats count {stats[2]} != n = {adv.size}"
    assert np.isfinite(stats[:2]).all(), f"{name}: statistics {stats[:2]} (NaN: the tile kernel flagged a failure)"
    s1, s2 = a.sum(), (a * a).sum()
    assert abs(stats[0] - s1) <= 1e-12 * np.abs(a).sum(), f"{name}: sum {stats[0]!r} != {s1!r}"
    assert abs(stats[1] - s2) <= 1e-12 * s2, f"{name}: sum of squares {stats[1]!r} != {s2!r}"
    print(f"{name}: n {adv.size} episodes {b['done'].size} gamma {gamma} lambda {lam} "
          f"margin adv {margins['adv']:.3f} ret {margins['ret']:.3f}")
    return margins


def episode_case(name, f64):
    lens_fn, nd = EPISODE_CASES[name]
    return make_batch(lens_fn(), f64, seed=sum(map(ord, name)) + f64, frac_not_done=nd), 0.99, 0.97


def tile_case(name, f64):
    lens_fn, nd, gamma, lam = TILE_CASES[name]
    return make_batch(lens_fn(), f64, seed=len(name) + f64, frac_not_done=nd), gamma, lam


def n_of(b):
    return int(b["off"][-1])


def e_of(b):
    return int(b["done"].size)


# ---- episode-parallel kernel ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("f64", [True, False], ids=["f64", "f32"])
@pytest.mark.parametrize("name", list(EPISODE_CASES))
def test_episode_kernel_matches_float64_reference(name, f64):
    b, gamma, lam = episode_case(name, f64)
    n, e = n_of(b), e_of(b)
    assert scan_kernel(n, e) == "episode"
    if name in ("fixed_16384x1000", "fixed_4096x999", "ragged_1_64", "ragged_200_3000"):
        assert e > episode_warps(e)  # grid-stride: warps take several episodes, the ring prefetches across them
    check_scan(f"{name}/{'f64' if f64 else 'f32'}", b, Scan(n).run(b, gamma, lam), gamma, lam)


@pytest.mark.parametrize("f64", [True, False], ids=["f64", "f32"])
def test_episode_kernel_gamma_lambda_edges(f64):
    b = make_batch(_ragged_1_64(seed=8, n_ep=700), f64, seed=9)
    assert scan_kernel(n_of(b), e_of(b)) == "episode"
    s = Scan(n_of(b))
    for gamma in (0.0, 0.99, 1.0):
        for lam in (0.0, 0.97, 1.0):
            check_scan(f"ragged_1_64x700/{'f64' if f64 else 'f32'}", b, s.run(b, gamma, lam), gamma, lam)


# ---- tile kernel ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("f64", [True, False], ids=["f64", "f32"])
@pytest.mark.parametrize("name", list(TILE_CASES))
def test_tile_kernel_matches_float64_reference(name, f64):
    b, gamma, lam = tile_case(name, f64)
    n, e = n_of(b), e_of(b)
    assert scan_kernel(n, e) == "tile"
    if name == "three_episodes_8M":
        assert (n + 2047) // 2048 > tile_grid_bound()  # every CTA walks several tiles
    check_scan(f"{name}/{'f64' if f64 else 'f32'}", b, Scan(n).run(b, gamma, lam), gamma, lam)


@pytest.mark.parametrize("gamma,lam", [(0.0, 0.0), (0.0, 1.0), (1.0, 0.0), (1.0, 1.0)])
def test_tile_kernel_gamma_lambda_edges(gamma, lam):
    b = make_batch([3, 4100, 1, 1, 2050, 17, 6000, 9], False, seed=10)
    assert scan_kernel(n_of(b), e_of(b)) == "tile"
    check_scan("short_tiles/f32", b, Scan(n_of(b)).run(b, gamma, lam), gamma, lam)


# ---- the regime switch ----------------------------------------------------------------------------------------------
BOUNDARY = {  # name -> (lengths, kernel the switch must pick)
    "n_ep_255": ([20] * 255, "tile"),
    "n_ep_256": ([20] * 256, "episode"),
    "n_4096_n_ep_256": ([16] * 256, "episode"),
    "n_4095_n_ep_256": ([16] * 255 + [15], "tile"),
    "len_32768_n_ep_256": ([32768] * 256, "episode"),
    "len_32769_n_ep_256": ([32769] * 256, "tile"),
}


def test_regime_switch_picks_the_mirrored_kernel():
    """The kernel actually launched (torch.profiler) is the one scan_kernel() predicts, on both sides of every bound of
    the switch, and both sides match the reference."""
    from torch.profiler import ProfilerActivity, profile
    runs = []
    with profile(activities=[ProfilerActivity.CUDA]) as prof:  # one session: the launches in order
        for name, (lens, want) in BOUNDARY.items():
            b = make_batch(lens, True, seed=12)
            assert scan_kernel(n_of(b), e_of(b)) == want, name
            runs.append((name, b, Scan(n_of(b)).run(b, 0.99, 0.97)))
    evs = sorted((ev for ev in prof.events()
                  if ev.device_type == torch.autograd.DeviceType.CUDA and "gae_scan" in ev.name),
                 key=lambda ev: ev.time_range.start)
    ran = ["episode" if "gae_scan_episode_kernel" in ev.name else "tile" for ev in evs]
    assert ran == [want for _, want in BOUNDARY.values()], f"scan kernels launched, in order: {[ev.name for ev in evs]}"
    for name, b, got in runs:
        check_scan(name, b, got, 0.99, 0.97)


# ---- the workspace contract: zeroed once, every launch leaves it clean -----------------------------------------------
REUSE_SEQUENCE = [  # alternates the kernels and the reward types; n grows and shrinks
    ("episode", "ragged_1_64", True),
    ("tile", "tiles_48_49_partial_48", False),
    ("episode", "fixed_300x1001", False),
    ("tile", "one_2M_episode_decaying", True),
    ("episode", "fixed_4096x999", True),
    ("tile", "tiles_49_48_partial_49", False),
    ("episode", "ragged_200_3000", False),
    ("tile", "one_2M_episode_gamma_lambda_1", False),
    ("episode", "n_mod_8", True),
]


def test_workspace_reused_across_kernels_and_sizes():
    cases = [(kind, name, *(episode_case if kind == "episode" else tile_case)(name, f64))
             for kind, name, f64 in REUSE_SEQUENCE]
    s = Scan(max(n_of(c[2]) for c in cases))
    first = None
    for kind, name, b, gamma, lam in cases:
        assert scan_kernel(n_of(b), e_of(b)) == kind, name
        got = s.run(b, gamma, lam)
        check_scan(f"reuse {name}", b, got, gamma, lam)
        if first is None:
            first = got
    _, name, b, gamma, lam = cases[0]
    again = s.run(b, gamma, lam)
    for x, y in zip(first, again):  # deterministic, and nothing carried over from the launches in between
        assert x.tobytes() == y.tobytes(), f"re-run of {name} after the sequence differs from its first run"


def test_tile_kernel_back_to_back_launches():
    """Three launches queued back to back on one workspace: each bumps the look-back epoch for the next."""
    b, gamma, lam = tile_case("tiles_48_49_partial_48", True)
    b2, _, _ = tile_case("one_2M_episode_decaying", True)
    for bb in (b, b2):
        s = Scan(n_of(bb))
        x = s.upload(bb)
        ds = [s.launch(x, gamma, lam) for _ in range(3)]
        outs = [s.finish(d) for d in ds]
        for k, got in enumerate(outs):
            check_scan(f"back-to-back {k}", bb, got, gamma, lam)
            for x, y in zip(outs[0], got):
                assert x.tobytes() == y.tobytes()


# ---- through the engine: one engine, batches that switch kernels -------------------------------------------------------
def _engine_batch(n, min_len, max_len, seed):
    from rl_replicas_b200 import synthetic
    b = synthetic.ragged_batch(n, 8, 2, False, seed=seed, min_len=min_len, max_len=max_len)
    b["ep_done"] = np.random.default_rng(seed).random(b["ep_done"].size) >= 0.3
    return b


def _check_engine(e, batch, hp, name):
    e.load_batch(batch)
    e.run_stage("preamble", hp)
    torch.cuda.synchronize()
    values, last_values = e.view("values").cpu().numpy(), e.view("last_values").cpu().numpy()
    assert np.abs(values).max() > 0 and np.abs(last_values).max() > 0
    b = dict(rew=np.asarray(batch["rew"], np.float64 if e.rewards_f64 else F32), values=values,
             last_values=last_values, off=batch["ep_offsets"], done=batch["ep_done"])
    got = (e.view("adv_raw").cpu().numpy(), e.view("ret").cpu().numpy(), e.view("adv_stats").cpu().numpy())
    check_scan(name, b, got, hp.gamma, hp.gae_lambda)
    return got


@pytest.mark.parametrize("f64", [True, False], ids=["f64", "f32"])
def test_engine_preamble_across_kernel_switches(f64):
    from rl_replicas_b200.engine import VALUE, OnPolicyEngine
    big = _engine_batch(20000, 1, 64, seed=13)
    small = _engine_batch(9000, 50, 400, seed=14)
    assert big["ep_done"].size >= 600 and scan_kernel(20000, big["ep_done"].size) == "episode"
    assert scan_kernel(9000, small["ep_done"].size) == "tile"
    rng = np.random.default_rng(15)
    ps, vs = [8, 32, 32, 2], [8, 32, 32, 1]
    e = OnPolicyEngine(ps, vs, "gaussian", 20000, big["ep_done"].size, rewards_f64=f64)
    flat = lambda sz: np.concatenate([np.concatenate([(rng.standard_normal((o, i)) / np.sqrt(i)).ravel(),
                                                      0.1 * rng.standard_normal(o)])
                                      for i, o in zip(sz[:-1], sz[1:])]).astype(F32)
    e.set_params(0, flat(ps))
    e.set_params(1, flat(ps))
    e.set_params(VALUE, flat(vs))
    hp = OnPolicyEngine.hparams(gamma=0.99, gae_lambda=0.97)
    tag = "f64" if f64 else "f32"
    first = _check_engine(e, big, hp, f"engine {tag} episode kernel")
    _check_engine(e, small, hp, f"engine {tag} tile kernel")
    again = _check_engine(e, big, hp, f"engine {tag} episode kernel again")
    for x, y in zip(first, again):
        assert x.tobytes() == y.tobytes()
    e.close()


def test_engine_load_batch_refuses_bad_offsets():
    from rl_replicas_b200._lib import B200RLError
    from rl_replicas_b200.engine import OnPolicyEngine
    e = OnPolicyEngine([8, 16, 2], [8, 16, 1], "gaussian", 1000, 100)
    good = _engine_batch(600, 5, 40, seed=16)
    e.load_batch(good)
    empty = dict(good, ep_offsets=good["ep_offsets"].copy())
    empty["ep_offsets"][3] = empty["ep_offsets"][2]  # episode 2 has no transition
    with pytest.raises(B200RLError, match="is empty"):
        e.load_batch(empty)
    for k, delta in ((0, 1), (-1, -1), (-1, 1)):  # offsets that do not start at 0 or do not end at n
        bad = dict(good, ep_offsets=good["ep_offsets"].copy())
        bad["ep_offsets"][k] += delta
        with pytest.raises(B200RLError, match="must start at 0 and end at n_rows"):
            e.load_batch(bad)
    e.close()


def test_stale_statistics_are_not_taken_for_look_back_records():
    """The per-episode statistics of an episode-kernel launch share workspace bytes with the look-back records of a
    later, larger tile-kernel launch, and each sum of squares lands in a record's tag slot.  Here every episode's sum of
    squares is exactly 1.0 (gamma = 0, one unit reward per episode, zero values): the tag a fresh workspace's first
    tile launch once gave its records, so stale slots read as published records and fed the look-back a wrong carry."""
    b = make_batch([16] * 4096, True, seed=17)
    b["rew"][:] = 0.0
    b["rew"][b["off"][:-1]] = 1.0
    b["values"][:] = 0.0
    b["last_values"][:] = 0.0
    long, gamma, lam = tile_case("one_2M_episode_decaying", True)
    assert scan_kernel(n_of(b), e_of(b)) == "episode" and scan_kernel(n_of(long), e_of(long)) == "tile"
    s = Scan(n_of(long))
    got = s.run(b, 0.0, 0.0)
    assert got[2][1] == e_of(b)
    check_scan("unit statistics", b, got, 0.0, 0.0)
    check_scan("tile launch after them", long, s.run(long, gamma, lam), gamma, lam)
