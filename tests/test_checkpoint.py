"""Checkpoint parity + resume: save_model writes the reference's dictionary layout, load_model restores networks, Adam
state and step counters."""
import os
import types

import numpy as np
import pytest
import torch


def _ppo(seed, sizes_p=(5, 64, 64, 2), sizes_v=(5, 64, 64, 1)):
    from rl_replicas_b200.algorithms import PPO
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import GaussianPolicy
    from rl_replicas_b200.value_function import ValueFunction
    torch.manual_seed(seed)
    pnet, vnet = MLP(list(sizes_p)), MLP(list(sizes_v))
    policy = GaussianPolicy(pnet, torch.optim.Adam(pnet.parameters(), lr=3e-4),
                            torch.nn.Parameter(torch.full((sizes_p[-1],), -0.5)))
    algo = PPO(policy, ValueFunction(vnet, torch.optim.Adam(vnet.parameters(), lr=1e-3)), None, None)
    algo.current_total_steps = 0
    return algo


def _fake_adam_progress(optimizer, steps):
    """Populate Adam state the way `steps` real updates would leave it (any values: the test is about round-tripping)."""
    for group in optimizer.param_groups:
        for p in group["params"]:
            optimizer.state[p] = {"step": torch.tensor(float(steps)), "exp_avg": torch.randn_like(p),
                                  "exp_avg_sq": torch.rand_like(p)}


def test_ppo_checkpoint_round_trip(tmp_path):
    a = _ppo(0)
    _fake_adam_progress(a.policy.optimizer, 37)
    _fake_adam_progress(a.value_function.optimizer, 80)
    a.current_total_steps = 123456
    path = os.path.join(tmp_path, "model.pt")
    a.save_model(17, path)
    ckpt = torch.load(path, weights_only=False)
    assert set(ckpt) == {"epoch", "total_steps", "policy_state_dict", "policy_optimizer_state_dict",
                         "value_function_state_dict", "value_function_optimizer_state_dict"}  # ref ppo.py:296-306
    assert list(ckpt["policy_state_dict"]) == ["network.0.weight", "network.0.bias", "network.2.weight", "network.2.bias",
                                               "network.4.weight", "network.4.bias"]
    b = _ppo(1)
    assert b.load_model(path) == 17 and b.current_total_steps == 123456
    for ma, mb in ((a.policy, b.policy), (a.value_function, b.value_function), (a.policy, b.old_policy)):
        for pa, pb in zip(ma.network.parameters(), mb.network.parameters()):
            assert torch.equal(pa, pb)
    for oa, ob in ((a.policy.optimizer, b.policy.optimizer), (a.value_function.optimizer, b.value_function.optimizer)):
        for pa, pb in zip(oa.param_groups[0]["params"], ob.param_groups[0]["params"]):
            for k in ("step", "exp_avg", "exp_avg_sq"):
                assert torch.equal(torch.as_tensor(oa.state[pa][k]), torch.as_tensor(ob.state[pb][k]))
    # the engine-facing readers see the restored state (this is what the next train() uploads)
    from rl_replicas_b200.algorithms._onpolicy import describe_mlp, read_adam_state
    m, v, step = read_adam_state(b.policy.optimizer, describe_mlp(b.policy.network)[3])
    assert step == 37 and m.shape == v.shape


def _td3(seed, o=17, a=6, h=256):
    from rl_replicas_b200.algorithms import TD3
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.policies import DeterministicPolicy, RandomPolicy
    from rl_replicas_b200.q_function import QFunction
    from rl_replicas_b200.replay_buffer import ReplayBuffer
    torch.manual_seed(seed)
    pnet = MLP([o, h, h, a], torch.nn.ReLU, torch.nn.Tanh)
    qs = [MLP([o + a, h, h, 1], torch.nn.ReLU) for _ in range(2)]
    env = types.SimpleNamespace(action_space=types.SimpleNamespace(high=np.ones(a, np.float32), shape=(a,)),
                                spec=types.SimpleNamespace(id="stub"))
    algo = TD3(DeterministicPolicy(pnet, torch.optim.Adam(pnet.parameters(), lr=1e-3)), RandomPolicy(None),
               QFunction(qs[0], torch.optim.Adam(qs[0].parameters(), lr=1e-3)),
               QFunction(qs[1], torch.optim.Adam(qs[1].parameters(), lr=1e-3)), env, None, ReplayBuffer(), None)
    algo.current_total_steps = 0
    return algo


def test_td3_checkpoint_round_trip(tmp_path):
    a = _td3(0, h=32)
    for m in (a.policy, a.q_function_1, a.q_function_2):
        _fake_adam_progress(m.optimizer, 11)
    with torch.no_grad():
        for t in (a.target_policy, a.target_q_function_1, a.target_q_function_2):
            for p in t.network.parameters():
                p.add_(0.25)  # targets differ from the online networks, as after polyak averaging
    path = os.path.join(tmp_path, "model.pt")
    a.save_model(5, path)
    b = _td3(1, h=32)
    assert b.load_model(path) == 5
    pairs = ((a.policy, b.policy), (a.q_function_1, b.q_function_1), (a.q_function_2, b.q_function_2),
             (a.target_policy, b.target_policy), (a.target_q_function_1, b.target_q_function_1),
             (a.target_q_function_2, b.target_q_function_2))
    for ma, mb in pairs:
        for pa, pb in zip(ma.network.parameters(), mb.network.parameters()):
            assert torch.equal(pa, pb)
    assert not any(p.requires_grad for p in b.target_policy.network.parameters())
