"""Shared host logic of the on-policy trainers: introspect the user's modules, keep the native engine's device
state in sync with them, and mirror the reference's train() side effects (SURVEY.md section 8b):
  (1) policy.network / value_function.network parameters updated in place,
  (2) optimizer.state[p] = {step, exp_avg, exp_avg_sq} updated,
  (3) old_policy synced, (4) the logged scalars recorded.
"""
from __future__ import annotations

import logging
from typing import List, Optional, Tuple

import numpy as np
import torch
from torch import nn

from ..engine import OLD_POLICY, POLICY, VALUE, OnPolicyEngine
from ..networks import NoisyLinear, has_noisy_layers
from ..packing import pack_experience
from ..policies import CategoricalPolicy, GaussianPolicy

logger = logging.getLogger(__name__)

_ACT_NAMES = {nn.Tanh: "tanh", nn.ReLU: "relu", nn.Identity: "identity"}


def describe_mlp(module: nn.Module, allow_noisy: bool = False) -> Tuple[List[int], str, str, List[nn.Linear]]:
    """(sizes, hidden activation, output activation, Linear layers) of an MLP built like ref networks/mlp.py:24-31
    (``allow_noisy``: also with NoisyLinear layers, a NoisyMLP).  Anything else is refused loudly -- the engine has no
    generic-module fallback."""
    seq = getattr(module, "network", module)
    mods = list(seq.children()) if isinstance(seq, nn.Sequential) else None
    if not mods:
        raise NotImplementedError(f"the update engine supports MLP(Linear/activation pairs) networks only, got {type(module).__name__}")
    linears, acts = [], []
    for i, m in enumerate(mods):
        if i % 2 == 0:
            if isinstance(m, NoisyLinear) and allow_noisy:
                linears.append(m)
                continue
            if isinstance(m, NoisyLinear):
                raise NotImplementedError(f"layer {i} is a NoisyLinear: noisy layers are implemented for DQN, C51 and "
                                          "QR-DQN Q networks only")
            if not isinstance(m, nn.Linear) or m.bias is None:
                raise NotImplementedError(f"layer {i} must be nn.Linear with bias, got {type(m).__name__}")
            linears.append(m)
        else:
            if type(m) not in _ACT_NAMES:
                raise NotImplementedError(f"unsupported activation {type(m).__name__} (supported: Tanh, ReLU, Identity)")
            acts.append(_ACT_NAMES[type(m)])
    if len(acts) < len(linears):
        acts.append("identity")
    hidden = set(acts[:-1]) or {"tanh"}
    if len(hidden) != 1:
        raise NotImplementedError(f"hidden activations must all be the same, got {sorted(hidden)}")
    sizes = [linears[0].in_features] + [l.out_features for l in linears]
    for a, b in zip(linears[:-1], linears[1:]):
        if a.out_features != b.in_features:
            raise ValueError("inconsistent Linear sizes")
    return sizes, hidden.pop(), acts[-1], linears


def layer_params(layer) -> tuple:
    """A layer's parameters in the engine's flat order: (weight, bias) of an nn.Linear, (weight_mu, weight_sigma,
    bias_mu, bias_sigma) of a NoisyLinear."""
    if isinstance(layer, NoisyLinear):
        return layer.weight_mu, layer.weight_sigma, layer.bias_mu, layer.bias_sigma
    return layer.weight, layer.bias


def refuse_noisy(what: str, *modules) -> None:
    """Refuse networks with noisy layers in the algorithms that do not implement them."""
    for m in modules:
        if m is not None and has_noisy_layers(m):
            raise NotImplementedError(f"{what} does not take networks with noisy layers (NoisyLinear): they are "
                                      "implemented for DQN, C51 and QR-DQN Q networks only")


def flat_params(linears: List[nn.Linear]) -> np.ndarray:
    with torch.no_grad():
        return torch.cat([t.detach().reshape(-1).float().cpu() for l in linears for t in layer_params(l)]).numpy()


def write_flat(linears: List[nn.Linear], flat: np.ndarray) -> None:
    src = torch.from_numpy(np.ascontiguousarray(flat))
    o = 0
    with torch.no_grad():
        for l in linears:
            for t in layer_params(l):
                n = t.numel()
                t.copy_(src[o:o + n].view_as(t))
                o += n
    assert o == src.numel()


def adam_hparams(optimizer, linears: List[nn.Linear], what: str, extra=()):
    """(lr, beta1, beta2, eps) of a plain torch.optim.Adam over exactly this network's parameters, in order (followed by
    the tensors of ``extra``, e.g. a trainable log_std)."""
    if type(optimizer) is not torch.optim.Adam:
        raise NotImplementedError(f"{what}: the engine implements torch.optim.Adam, got {type(optimizer).__name__}")
    if len(optimizer.param_groups) != 1:
        raise NotImplementedError(f"{what}: exactly one param group is supported")
    g = optimizer.param_groups[0]
    want = [t for l in linears for t in layer_params(l)] + list(extra)
    if len(g["params"]) != len(want) or any(a is not b for a, b in zip(g["params"], want)):
        raise NotImplementedError(
            f"{what}: optimizer must hold exactly the network's parameters in order "
            "(for a Gaussian policy optionally followed by its log_std)")
    if g.get("weight_decay", 0) != 0 or g.get("amsgrad", False) or g.get("maximize", False):
        raise NotImplementedError(f"{what}: weight_decay / amsgrad / maximize are not supported")
    return float(g["lr"]), float(g["betas"][0]), float(g["betas"][1]), float(g["eps"])


def read_adam_state(optimizer, linears: List[nn.Linear], extra=()):
    ps = [t for l in linears for t in layer_params(l)] + list(extra)
    if not all(p in optimizer.state and "exp_avg" in optimizer.state[p] for p in ps):
        return None, None, 0
    m = torch.cat([optimizer.state[p]["exp_avg"].reshape(-1).float() for p in ps]).numpy()
    v = torch.cat([optimizer.state[p]["exp_avg_sq"].reshape(-1).float() for p in ps]).numpy()
    steps = {int(float(optimizer.state[p]["step"])) for p in ps}
    if len(steps) != 1:
        raise NotImplementedError("parameters of one optimizer have different step counts")
    return m, v, steps.pop()


def write_adam_state(optimizer, linears: List[nn.Linear], m: np.ndarray, v: np.ndarray, step: int, extra=()) -> None:
    if step == 0:
        return
    mt, vt = torch.from_numpy(m), torch.from_numpy(v)
    o = 0
    for p in [t for l in linears for t in layer_params(l)] + list(extra):
        n = p.numel()
        st = optimizer.state[p]
        st["step"] = torch.tensor(float(step))  # torch keeps the step as a float32 scalar tensor
        st["exp_avg"] = mt[o:o + n].view_as(p).clone()
        st["exp_avg_sq"] = vt[o:o + n].view_as(p).clone()
        o += n


class OnPolicyTrainerMixin:
    """Engine management shared by PPO / VPG / TRPO."""

    _engine: Optional[OnPolicyEngine] = None
    process_group = None
    distributed = False

    def _describe(self):
        psizes, pact, pout, self._plin = describe_mlp(self.policy.network)
        vsizes, vact, vout, self._vlin = describe_mlp(self.value_function.network)
        if pout != "identity" or vout != "identity":
            raise NotImplementedError("output activations other than Identity are not supported for on-policy nets")
        if pact != vact:
            raise NotImplementedError("policy and value networks must use the same hidden activation")
        if isinstance(self.policy, GaussianPolicy):
            dist = "gaussian"
        elif isinstance(self.policy, CategoricalPolicy):
            dist = "categorical"
        else:
            raise NotImplementedError(f"unsupported policy type {type(self.policy).__name__}")
        return psizes, vsizes, dist, pact

    def _trainable_log_std(self):
        """``[policy.log_std]`` when the user put it into the policy optimizer behind the network's parameters (then it
        is trained like in the reference, ref policies/gaussian_policy.py:25-37 + torch autograd), else ``[]``."""
        if not isinstance(self.policy, GaussianPolicy) or type(self.policy.optimizer) is not torch.optim.Adam:
            return []
        params = [p for g in self.policy.optimizer.param_groups for p in g["params"]]
        return [self.policy.log_std] if any(p is self.policy.log_std for p in params) else []

    def _ensure_engine(self, n_rows: int, n_episodes: int) -> OnPolicyEngine:
        psizes, vsizes, dist, act = self._describe()
        train_ls = bool(self._trainable_log_std())
        e = self._engine
        if (e is None or e.policy_sizes != psizes or e.value_sizes != vsizes or e.dist != dist
                or e.train_log_std != train_ls or e.max_rows < n_rows or e.max_episodes < n_episodes):
            if e is not None:
                e.close()
            cap_rows = max(n_rows, int(1.25 * n_rows) if e is not None else n_rows)
            cap_eps = max(n_episodes, 2 * n_episodes if e is not None else n_episodes)
            e = OnPolicyEngine(psizes, vsizes, dist, cap_rows, cap_eps, hidden_act=act, rewards_f64=True,
                               train_log_std=train_ls)
            self._engine = e
        return e

    def _push_state(self, e: OnPolicyEngine, with_old: bool) -> None:
        ls = self._trainable_log_std()
        tail = lambda policy: ([policy.log_std.detach().float().reshape(-1).numpy()] if ls else [])
        e.set_params(POLICY, np.concatenate([flat_params(self._plin)] + tail(self.policy)))
        if with_old:
            old_lin = describe_mlp(self.old_policy.network)[3]
            e.set_params(OLD_POLICY, np.concatenate([flat_params(old_lin)] + tail(self.old_policy)))
        e.set_params(VALUE, flat_params(self._vlin))
        if e.dist == "gaussian" and not ls:
            e.set_log_std(self.policy.log_std.detach().float().numpy())
        if type(self.policy.optimizer) is torch.optim.Adam:
            e.set_adam(POLICY, *read_adam_state(self.policy.optimizer, self._plin, ls))
        e.set_adam(VALUE, *read_adam_state(self.value_function.optimizer, self._vlin))

    def _pull_state(self, e: OnPolicyEngine, with_old: bool, policy_adam: bool = True) -> None:
        ls = self._trainable_log_std()
        flat = e.get_params(POLICY)
        n_net = flat.size - (ls[0].numel() if ls else 0)
        write_flat(self._plin, flat[:n_net])
        if ls:
            with torch.no_grad():
                ls[0].copy_(torch.from_numpy(flat[n_net:].copy()).view_as(ls[0]))
        write_flat(self._vlin, e.get_params(VALUE))
        if with_old:
            # ref ppo.py:183: old_policy.load_state_dict(policy.state_dict())  (log_std is part of the state dict)
            self.old_policy.load_state_dict(self.policy.state_dict())
        if policy_adam:
            write_adam_state(self.policy.optimizer, self._plin, *e.get_adam(POLICY), extra=ls)
        write_adam_state(self.value_function.optimizer, self._vlin, *e.get_adam(VALUE))

    def _global_rows(self, n_rows: int) -> int:
        """Rows over all ranks (the denominator of every mean).  The same collective tells the ranks whether any of them
        holds a fresh engine: then ALL of them (re)attach the NVLink gradient exchange (B200RL_PEER_EXCHANGE=0 keeps
        the NCCL all-reduce per iteration)."""
        if not self.distributed:
            return 0
        import os
        import torch.distributed as dist
        e = self._engine
        want = os.environ.get("B200RL_PEER_EXCHANGE", "1") != "0"
        fresh = int(want and e is not None and not e.peer_exchange and not getattr(e, "peer_refused", False))
        t = torch.tensor([n_rows, fresh], dtype=torch.int64, device="cuda")
        dist.all_reduce(t, group=self.process_group)
        if want and int(t[1].item()) > 0 and e is not None:
            if not e.enable_peer_exchange(self.process_group):
                e.peer_refused = True
                logger.warning("peer-memory gradient exchange unavailable: keeping the NCCL all-reduce per iteration")
        return int(t[0].item())

    def pack(self, experience):
        return pack_experience(experience)
