"""References of noisy DQN, C51 and QR-DQN (include/b200rl.h, "Noisy networks").  TEST INFRASTRUCTURE ONLY -- see
oracle/__init__.py.

* ``set_noise`` / ``train_f32``: float32.  Each NoisyLinear's eps_in / eps_out are set to the engine's draws (the
  online sample on the online network, the target sample on the target), then the existing float32 oracles
  (oracle/dqn.py, c51.py, qr.py) run the step on the module unchanged: torch's eager ``sigma * e + mu`` and autograd
  are the formulas the engine states.
* ``step_f64``: float64.  The weights are composed in float64, the existing float64 steps (oracle/dqn.py, c51.py,
  qr.py, dueling.py) run on them, and the chain rule dW_mu = dW, dW_sigma = dW e, db_mu = db, db_sigma = db f(eps_out)
  gives the gradient (and the per-entry gradient scale) of the noisy vector.

Layers are described as [(in, out, noisy)] in the engine's flat order; a draw vector holds eps_in, eps_out of every
noisy layer in that order.
"""
from __future__ import annotations

from typing import List, Sequence, Tuple

import numpy as np
import torch

from . import c51 as OC
from . import dqn as OD
from . import dueling as ODu
from . import qr as OQ

D = torch.float64


def noisy_layers(module: torch.nn.Module) -> list:
    """The NoisyLinear layers of ``module`` in the engine's flat order (module order)."""
    from rl_replicas_b200.networks import NoisyLinear
    return [m for m in module.modules() if isinstance(m, NoisyLinear)]


def layers_of(module: torch.nn.Module) -> List[Tuple[int, int, bool]]:
    """[(in, out, noisy)] of every Linear / NoisyLinear layer of ``module`` in flat order."""
    from rl_replicas_b200.networks import NoisyLinear
    return [(m.in_features, m.out_features, isinstance(m, NoisyLinear)) for m in module.modules()
            if isinstance(m, (torch.nn.Linear, NoisyLinear))]


def set_noise(module: torch.nn.Module, eps) -> None:
    """eps_in / eps_out of every NoisyLinear of ``module`` from one draw vector [E]."""
    eps = torch.as_tensor(np.asarray(eps, np.float32))
    o = 0
    with torch.no_grad():
        for m in noisy_layers(module):
            m.eps_in.copy_(eps[o:o + m.in_features])
            o += m.in_features
            m.eps_out.copy_(eps[o:o + m.out_features])
            o += m.out_features
    assert o == eps.numel(), (o, eps.numel())


def train_f32(oracle, minibatches, draws):
    """``oracle.train`` step by step with the engine's draws [S, 2, E]: step st's online sample on oracle.q, its target
    sample on oracle.q_targ.  Returns the oracle's logs over the S steps."""
    logs = {}
    for mb, d in zip(minibatches, draws):
        set_noise(oracle.q, d[0])
        set_noise(oracle.q_targ, d[1])
        for k, v in oracle.train([mb]).items():
            logs.setdefault(k, []).extend(v)
    return logs


def _f(x: torch.Tensor) -> torch.Tensor:
    return torch.copysign(x.abs().sqrt(), x)


def _noise_factors(layers, eps):
    """Per layer (f(eps_out), f(eps_in)) in float64, or None for a plain layer."""
    eps = torch.as_tensor(np.asarray(eps, np.float64))
    out, o = [], 0
    for n_in, n_out, noisy in layers:
        if noisy:
            fi, fo = _f(eps[o:o + n_in]), _f(eps[o + n_in:o + n_in + n_out])
            o += n_in + n_out
            out.append((fo, fi))
        else:
            out.append(None)
    assert o == eps.numel()
    return out


def compose_f64(flat, layers, eps) -> np.ndarray:
    """The composed (plain-layout) float64 parameter vector of a noisy vector ``flat`` under the draw ``eps``."""
    flat = torch.as_tensor(np.asarray(flat, np.float64))
    parts, o = [], 0
    for (n_in, n_out, noisy), fac in zip(layers, _noise_factors(layers, eps)):
        if noisy:
            fo, fi = fac
            W_mu = flat[o:o + n_out * n_in].view(n_out, n_in)
            W_s = flat[o + n_out * n_in:o + 2 * n_out * n_in].view(n_out, n_in)
            o += 2 * n_out * n_in
            b_mu, b_s = flat[o:o + n_out], flat[o + n_out:o + 2 * n_out]
            o += 2 * n_out
            parts += [(W_mu + W_s * torch.outer(fo, fi)).reshape(-1), b_mu + b_s * fo]
        else:
            parts.append(flat[o:o + n_out * n_in + n_out])
            o += n_out * n_in + n_out
    assert o == flat.numel()
    return torch.cat(parts).numpy()


def expand_f64(g, layers, eps) -> np.ndarray:
    """The chain rule from the composed layers' gradient ``g`` (plain layout) to the noisy vector's."""
    g = torch.as_tensor(np.asarray(g, np.float64))
    parts, o = [], 0
    for (n_in, n_out, noisy), fac in zip(layers, _noise_factors(layers, eps)):
        dW, db = g[o:o + n_out * n_in], g[o + n_out * n_in:o + n_out * n_in + n_out]
        o += n_out * n_in + n_out
        if noisy:
            fo, fi = fac
            parts += [dW, (dW.view(n_out, n_in) * torch.outer(fo, fi)).reshape(-1), db, db * fo]
        else:
            parts += [dW, db]
    assert o == g.numel()
    return torch.cat(parts).numpy()


def step_f64(kind: str, q_flat, targ_flat, eps_q, eps_t, mb, layers: Sequence[Tuple[int, int, bool]],
             sizes: Sequence[int], dueling_k: int = 0, hidden="relu", gamma=0.99, double_q=False, **head):
    """One noisy step in float64 (``kind`` "dqn", "c51" or "qr"; ``head``: n_atoms / v_min / v_max or n_quantiles):
    the float64 step of the plain or dueling network (``dueling_k``) on the composed weights, with grad and scale
    mapped to the noisy vector.  ``sizes`` as the plain / dueling step takes them."""
    q_c, t_c = compose_f64(q_flat, layers, eps_q), compose_f64(targ_flat, layers, eps_t)
    if dueling_k:
        fn = {"dqn": ODu.dqn_step_f64, "c51": ODu.c51_step_f64, "qr": ODu.qr_step_f64}[kind]
    else:
        fn = {"dqn": OD.dqn_step_f64, "c51": OC.c51_step_f64, "qr": OQ.qr_step_f64}[kind]
    args = {"dqn": (), "c51": (head.get("n_atoms"), head.get("v_min"), head.get("v_max")),
            "qr": (head.get("n_quantiles"),)}[kind]
    out = fn(q_c, t_c, mb, sizes, *args, hidden=hidden, gamma=gamma, double_q=double_q)
    out["grad"] = expand_f64(out["grad"], layers, eps_q)
    out["scale"] = np.abs(expand_f64(out["scale"], layers, eps_q))
    return out
