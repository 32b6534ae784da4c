"""CPU: LearnerGroup's host side -- what it refuses (before any device call) and its per-member random streams."""
import random

import numpy as np
import pytest
import torch

from rl_replicas_b200 import synthetic
from test_sac import make_sac


def _layers(rng, sizes):
    return [(rng.standard_normal((o, i)).astype(np.float32), rng.standard_normal(o).astype(np.float32))
            for i, o in zip(sizes[:-1], sizes[1:])]


def td3(seed=0, twin=True, hidden=16):
    rng = np.random.default_rng(seed)
    qs = [_layers(rng, [5, hidden, 1]) for _ in range(2 if twin else 1)]
    return synthetic.offpolicy_learner(twin, _layers(rng, [3, hidden, 2]), qs)[0]


def test_refuses_members_that_cannot_share_an_engine():
    from rl_replicas_b200.algorithms import LearnerGroup
    cases = {
        "class": lambda a: td3(twin=False),
        "policy network": lambda a: td3(hidden=8),
        "gamma": lambda a: setattr(a, "gamma", 0.9),
        "polyak_rho": lambda a: setattr(a, "polyak_rho", 0.9),
        "target_noise_clip": lambda a: setattr(a, "target_noise_clip", 0.1),
        "policy_delay": lambda a: setattr(a, "policy_delay", 3),
        "use_device_rng": lambda a: setattr(a, "use_device_rng", True),
        "q_function_2 optimizer": lambda a: a.q_function_2.optimizer.param_groups[0].update(lr=3e-4),
        "policy optimizer": lambda a: a.policy.optimizer.param_groups[0].update(betas=(0.8, 0.999)),
    }
    for name, change in cases.items():
        g = LearnerGroup()
        g.add(td3(0))
        other = td3(1)
        other = change(other) or other
        with pytest.raises(ValueError, match=name):
            g.add(other)
        assert len(g) == 1


def test_refuses_sac_members_with_different_temperature_settings():
    from rl_replicas_b200.algorithms import LearnerGroup
    g = LearnerGroup()
    g.add(make_sac(seed=0, learn_alpha=True))
    for kw, name in ((dict(learn_alpha=False), "learn_alpha"), (dict(learn_alpha=True, alpha=0.5), "alpha"),
                     (dict(learn_alpha=True, target_entropy=-1.0), "target_entropy"),
                     (dict(learn_alpha=True, alpha_lr=1e-2), "alpha optimizer")):
        with pytest.raises(ValueError, match=name):
            g.add(make_sac(seed=1, **kw))
    a = make_sac(seed=2, learn_alpha=True)
    a.policy.log_std_min = -5.0
    with pytest.raises(ValueError, match="log_std bounds"):
        g.add(a)
    g.add(make_sac(seed=3, learn_alpha=True))  # different parameters, same settings
    assert len(g) == 2


def test_refuses_empty_groups_duplicates_and_too_many_members(tmp_path):
    from rl_replicas_b200.algorithms import LearnerGroup
    g = LearnerGroup()
    with pytest.raises(ValueError, match="no members"):
        g.train(5, 8)
    with pytest.raises(ValueError, match="no members"):
        g.learn(output_dirs=[])
    with pytest.raises(ValueError, match="TD3, DDPG or SAC"):
        g.add(object())
    a = td3(0)
    g.add(a)
    with pytest.raises(ValueError, match="already a member"):
        g.add(a)
    for k in range(1, 16):
        g.add(td3(k))
    with pytest.raises(ValueError, match="at most 16"):
        g.add(td3(16))
    with pytest.raises(ValueError, match="output_dirs"):
        g.learn(output_dirs=[str(tmp_path)])
    assert g._engine is None  # nothing above touched the device


def _draws(n):
    return ([random.random() for _ in range(n)], np.random.randint(0, 1000, n).tolist(), torch.randn(n).tolist())


@pytest.fixture
def restore_determinism():
    on = torch.are_deterministic_algorithms_enabled()
    yield
    torch.use_deterministic_algorithms(on)


def test_member_streams_replay_their_solo_sequences_and_leave_the_globals_alone(restore_determinism):
    from rl_replicas_b200.algorithms import LearnerGroup
    from rl_replicas_b200.utils import set_seed_for_libraries
    seeds = (0, 1, 2)
    solo = {}
    for s in seeds:  # what each member draws when it runs alone (built after seeding): three draws in a row
        set_seed_for_libraries(s)
        td3(s)
        solo[s] = [_draws(4) for _ in range(3)]
    g = LearnerGroup()
    for s in seeds:
        set_seed_for_libraries(s)
        g.add(td3(s))
    set_seed_for_libraries(123)
    before = (random.getstate(), np.random.get_state(), torch.get_rng_state())
    got = {s: [] for s in seeds}
    for _ in range(3):  # interleaved: member 0, 1, 2, then again
        for k, s in enumerate(seeds):
            with g.stream(k):
                got[s].append(_draws(4))
    assert got == solo
    assert random.getstate() == before[0]
    assert all(np.array_equal(a, b) for a, b in zip(np.random.get_state()[1:3], before[1][1:3]))
    assert torch.equal(torch.get_rng_state(), before[2])
    with pytest.raises(RuntimeError):  # a failure inside a member's work still restores the globals
        with g.stream(0):
            random.random()
            raise RuntimeError("boom")
    assert random.getstate() == before[0]
