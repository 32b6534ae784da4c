"""CPU: prioritized experience replay's host side -- the oracle's sum tree and its layout against the library's,
Philox4x32-10 against its published known answers, the stratified draw against p_i / sum p (chi-square, seed pinned),
the beta schedule, the rows that receive the running max on appends (wrap included), the refusals, and the
LearnerGroup signature for prioritized DQN members.  The device side is tests/test_gpu_per.py."""
import numpy as np
import pytest
from scipy import stats

from oracle import per as OP
from test_dqn import make_dqn


def test_oracle_tree_sums_and_layout():
    from rl_replicas_b200 import _lib
    lib = _lib.load()
    rng = np.random.default_rng(0)
    for n in (1, 31, 32, 33, 1025, 2 ** 20 + 1):
        p = rng.random(n)
        levels = OP.tree_levels(p)
        assert len(levels[-1]) == 1 and len(levels) >= 2
        for child, parent in zip(levels[:-1], levels[1:]):
            pad = np.concatenate([child, np.zeros(-len(child) % 32)]).reshape(-1, 32)
            np.testing.assert_allclose(parent, pad.sum(1), rtol=1e-12)
        assert levels[-1][0] == pytest.approx(p.sum(), rel=1e-12)
        offs, total = OP.tree_offsets(n)
        assert len(offs) == len(levels) and all(o % 32 == 0 for o in offs)
        assert int(lib.b200rl_per_tree_floats(n)) == total
        assert abs(float(OP.root_f32(p)) - p.sum()) <= 1e-5 * p.sum()
    assert lib.b200rl_per_tree_floats(0) == -1 and lib.b200rl_per_tree_floats(2 ** 31) == -1


def test_philox_known_answers():
    """Random123's known-answer vectors for Philox4x32-10."""
    kats = [((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
            ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
            ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
             (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]
    for ctr, key, want in kats:
        got = OP.philox4x32_10(*ctr, *key)
        assert tuple(int(x) for x in got) == want


def test_sum_tree_never_returns_a_zero_leaf():
    p = np.array([0.0, 2.0, 0.0, 0.0, 1.0, 0.0])
    t = OP.SumTree(p)
    u = np.array([0.0, 1.999, 2.0, 2.5, 3.0 - 1e-12, 3.0, 3.5, 1e9])
    assert t.find(u).tolist() == [1, 1, 4, 4, 4, 4, 4, 4]


def test_stratified_draws_follow_the_priorities():
    """Chi-square of 200 steps x 256 draws over 50 leaves (a fifth of them zero) against B S p_i / sum p."""
    rng = np.random.default_rng(7)
    p = rng.random(50) ** 2 * 5.0
    p[rng.choice(50, 10, replace=False)] = 0.0
    S, B = 200, 256
    counts = np.zeros(50)
    for st in range(S):
        idx, _ = OP.stratified_draw(p.astype(np.float32), 1234, 3, st, B)
        counts += np.bincount(idx, minlength=50)
    assert counts[p == 0].sum() == 0
    nz = p > 0
    expected = S * B * p[nz] / p[nz].sum()
    chi2 = float(((counts[nz] - expected) ** 2 / expected).sum())
    pval = stats.chi2.sf(chi2, nz.sum() - 1)
    print(f"chi-square {chi2:.1f} on {nz.sum() - 1} degrees of freedom, p = {pval:.3f}")
    assert pval > 1e-3
    # stratification: every stratum [j M / B, (j + 1) M / B) holds exactly one u_j
    U = OP.per_uniforms(1234, 3, 0, B)
    assert ((U >= 0) & (U < 1)).all() and len(np.unique(U)) > B - 3


def test_beta_schedule():
    from rl_replicas_b200.replay_buffer import PrioritizedReplayBuffer
    rb = PrioritizedReplayBuffer(1000, beta_start=0.4, beta_anneal_steps=100)
    for t, want in ((0, 0.4), (50, 0.7), (100, 1.0), (10 ** 6, 1.0)):
        assert rb.beta(t) == pytest.approx(want, abs=1e-12)
        assert float(OP.beta_schedule(t, 0.4, 100)) == pytest.approx(want, abs=1e-12)


def _columns(n, seed=0):
    class Cols:
        def __init__(self):
            rng = np.random.default_rng(seed)
            self.cols = (rng.standard_normal((n, 3)).astype(np.float32), rng.integers(0, 2, n).astype(np.float32),
                         rng.standard_normal(n), rng.standard_normal((n, 3)).astype(np.float32), rng.random(n) < 0.1)

        def transition_columns(self):
            return self.cols
    return Cols()


def test_appends_mark_their_rows_for_the_running_max_with_wrap():
    """The physical rows each append wrote, merged while contiguous, are what the next refresh gives priority m."""
    from rl_replicas_b200.replay_buffer import PrioritizedReplayBuffer
    rb = PrioritizedReplayBuffer(100)
    rb.add_experience(_columns(30))
    assert rb._capacity == 100  # allocated at full size: rows never move
    assert rb._prio_dirty == []  # no tree yet: its first build gives every live row the initial max
    rb._tree, rb._prio_dirty = "built", []  # as after a refresh
    rb.add_experience(_columns(50))
    rb.add_experience(_columns(10))
    assert rb._prio_dirty == [(30, 60)]
    rb._prio_dirty = []
    rb.add_experience(_columns(25))  # 10 rows at the end, 15 wrapped to the front (overwriting the oldest)
    assert rb._prio_dirty == [(90, 25)] and rb.ring() == (15, 100, 100)
    rb.add_experience(_columns(250))  # more than the buffer: the newest 100 rows, everything rewritten
    assert rb._prio_dirty == [(90, 100)]


def test_refusals():
    from rl_replicas_b200.replay_buffer import PrioritizedReplayBuffer
    from test_offpolicy_group import td3 as make_td3
    for kw in (dict(alpha=-0.1), dict(beta_start=1.5), dict(beta_anneal_steps=0), dict(eps=0.0)):
        with pytest.raises(ValueError):
            PrioritizedReplayBuffer(100, **kw)
    rb = PrioritizedReplayBuffer(100)
    rb.add_experience(_columns(40))
    with pytest.raises(NotImplementedError, match="on the device"):
        rb.sample_minibatch(8)
    with pytest.raises(NotImplementedError, match="on the device"):
        rb.sample_indices(8)
    t = make_td3(0)
    with pytest.raises(ValueError, match="TD3 does not train on a PrioritizedReplayBuffer"):
        t.train(rb, 2, 8)
    d = make_dqn()
    d.replay_buffer = rb
    d.use_device_replay = False
    with pytest.raises(ValueError, match="use_device_replay"):
        d.train(rb, 2, 8)


def test_group_signature_for_prioritized_members():
    from rl_replicas_b200.algorithms import LearnerGroup
    from rl_replicas_b200.replay_buffer import PrioritizedReplayBuffer

    def member(seed, **kw):
        m = make_dqn(seed=seed)
        m.replay_buffer = PrioritizedReplayBuffer(1000, **kw)
        return m
    g = LearnerGroup()
    g.add(member(0, alpha=0.5))
    g.add(member(1, alpha=0.5))
    with pytest.raises(ValueError, match="prioritized replay alpha"):
        g.add(member(2, alpha=0.7))
    for attr, v in (("eps", 1e-3), ("beta_start", 0.5), ("beta_anneal_steps", 10)):
        with pytest.raises(ValueError, match=f"prioritized replay {attr}"):
            g.add(member(2, alpha=0.5, **{attr: v}))
    with pytest.raises(ValueError, match="prioritized replay"):
        g.add(make_dqn(seed=2))  # a uniform buffer
    u = LearnerGroup()
    u.add(make_dqn(seed=0))
    with pytest.raises(ValueError, match="prioritized replay"):
        u.add(member(1))


def test_group_refuses_members_sharing_a_prioritized_buffer():
    """Every member's priority update writes its own tree at the same time as the others': one shared tree would race."""
    from rl_replicas_b200.algorithms import LearnerGroup
    from rl_replicas_b200.replay_buffer import PrioritizedReplayBuffer
    shared = PrioritizedReplayBuffer(1000)
    a, b = make_dqn(seed=0), make_dqn(seed=1)
    a.replay_buffer = b.replay_buffer = shared
    g = LearnerGroup()
    g.add(a)
    with pytest.raises(ValueError, match="members 0 and 1 share one PrioritizedReplayBuffer"):
        g.add(b)
    b.replay_buffer = PrioritizedReplayBuffer(1000)
    g.add(b)
    b.replay_buffer = shared  # replaced after add(): train refuses before any work
    with pytest.raises(ValueError, match="share one PrioritizedReplayBuffer"):
        g.train(2, 8)
    u = LearnerGroup()  # uniform buffers may still be shared
    c, d = make_dqn(seed=0), make_dqn(seed=1)
    d.replay_buffer = c.replay_buffer
    u.add(c)
    u.add(d)
