"""GPU parity of TRPO: Fisher-vector product kernel, device-side CG / line search, and TRPO.train end to end against
the reference's outputs (golden) and the numpy oracle."""
import numpy as np
import pytest
import torch

from conftest import batch_of, load_golden, rel_err
from oracle import onpolicy as O

pytestmark = pytest.mark.gpu


class Rec:
    def __init__(self):
        self.s = {}

    def record_scalar(self, tag, scalar, total_steps=None, tensorboard=False):
        self.s[tag] = float(scalar)


def build_trpo(g, **kw):
    from rl_replicas_b200.algorithms import TRPO
    from rl_replicas_b200.algorithms._onpolicy import describe_mlp, write_flat
    from rl_replicas_b200.networks import MLP
    from rl_replicas_b200.optimizers import ConjugateGradientOptimizer
    from rl_replicas_b200.policies import CategoricalPolicy, GaussianPolicy
    from rl_replicas_b200.value_function import ValueFunction
    ps, vs = [int(x) for x in g["policy_sizes"]], [int(x) for x in g["value_sizes"]]
    pnet, vnet = MLP(ps), MLP(vs)
    write_flat(describe_mlp(pnet)[3], g["policy_flat0"])
    write_flat(describe_mlp(vnet)[3], g["value_flat0"])
    opt = ConjugateGradientOptimizer(pnet.parameters())
    if "log_std" in g:
        policy = GaussianPolicy(pnet, opt, torch.nn.Parameter(torch.from_numpy(g["log_std"].astype(np.float32))))
    else:
        policy = CategoricalPolicy(pnet, opt)
    vf = ValueFunction(vnet, torch.optim.Adam(vnet.parameters(), lr=1e-3))
    t = TRPO(policy, vf, None, None, **kw)
    t.metrics_manager = Rec()
    t.current_total_steps = 0
    return t


def flat(m):
    return torch.nn.utils.parameters_to_vector(m.parameters()).detach().numpy()


@pytest.mark.parametrize("case", ["trpo_gaussian_small", "trpo_categorical_small"])
def test_trpo_train_matches_reference(case):
    g = load_golden(case)
    trpo = build_trpo(g, num_value_gradients=5)
    trpo.train_packed(batch_of(g))
    e, ts, st = trpo._engine, trpo.last_trpo_stats, trpo.last_update_stats
    # single Fisher-vector product vs the reference's double-backprop HVP of the same probe vector: tight.
    # (parameters were restored / moved by train; evaluate at theta_0 on a fresh engine)
    t2 = build_trpo(g, num_value_gradients=0)
    eng = t2._ensure_engine(g["obs"].shape[0], g["ep_done"].shape[0])
    t2._push_state(eng, with_old=True)
    eng.load_batch(batch_of(g))
    hv = eng.fvp(g["hvp_probe"], 1e-5)
    assert rel_err(hv, g["hvp_of_probe"]) < 1e-5
    # gradient, CG solution, descent step (documented looser bounds after 10 CG iterations, SURVEY 7.3-9)
    assert rel_err(e.view("policy_grad").cpu().numpy()[:g["grad0"].size], g["grad0"]) < 1e-5
    assert rel_err(e.view("cg_x").cpu().numpy(), g["cg_x"]) < 2e-3
    assert rel_err(e.view("cg_descent").cpu().numpy(), g["descent"]) < 2e-3
    assert ts.fvp_launches == 11 and not ts.rejected and ts.accepted_index >= 0
    assert rel_err(flat(trpo.policy.network), g["policy_flat_final"]) < 2e-3
    assert rel_err(flat(trpo.old_policy.network), flat(trpo.policy.network)) == 0.0
    assert rel_err(flat(trpo.value_function.network), g["value_flat_final"]) < 1e-5
    assert abs(ts.kl - g["final_kl"]) < 2e-2 * g["final_kl"]
    assert abs(ts.new_loss - g["final_loss"]) < 2e-2 * abs(g["final_loss"])
    m = trpo.metrics_manager.s
    assert abs(m["policy/loss"] - g["metric:policy/loss"]) < 1e-6
    assert abs(m["policy/avarage_entropy"] - g["metric:policy/avarage_entropy"]) < 1e-5
    assert abs(m["value_function/average_loss"] - g["metric:value_function/average_loss"]) < 1e-4 * g["metric:value_function/average_loss"]


def test_trpo_vs_oracle_and_rejection():
    """Against the numpy oracle on a seeded batch, plus the reject/restore branch (a KL limit no step can satisfy: the
    step must be rejected and the parameters restored bit-exactly)."""
    g = load_golden("trpo_gaussian_small")
    policy = O.unflatten_layers(g["policy_flat0"], [27, 64, 64, 8])
    out = O.trpo_policy_step(policy, "gaussian", g["log_std"], g["obs"], g["act"], g["adv"])
    trpo = build_trpo(g, num_value_gradients=0)
    trpo.train_packed(batch_of(g))
    ts = trpo.last_trpo_stats
    assert ts.accepted_index == out["accepted"]
    assert abs(ts.step_size - out["step_size"]) < 2e-3 * out["step_size"]
    assert rel_err(flat(trpo.policy.network), out["policy_flat"]) < 2e-3
    # rejection by construction: a negative KL limit, which no KL (a non-negative sum) can meet; the step size
    # sqrt(2 delta / xHx) is NaN and falls back to 1, the one evaluation fails and the parameters are restored
    t2 = build_trpo(g, num_value_gradients=0)
    t2.policy.optimizer.max_backtracks = 1
    t2.policy.optimizer.max_constraint = -1.0
    t2.train_packed(batch_of(g))
    ts2 = t2.last_trpo_stats
    assert ts2.rejected == 1 and ts2.accepted_index == -1 and ts2.step_size == 1.0
    np.testing.assert_array_equal(flat(t2.policy.network).view(np.uint32),
                                  g["policy_flat0"].astype(np.float32).view(np.uint32))


@pytest.mark.parametrize("sizes,dist", [([27, 64, 64, 8], "gaussian"), ([4, 64, 64, 2], "categorical"),
                                        ([17, 64, 32, 6], "gaussian"), ([9, 33, 20, 3], "categorical")])
@pytest.mark.parametrize("n", [50, 4097, 20011])
@pytest.mark.parametrize("v_scale", [1e-3, 1.0, 300.0])
def test_fvp_tensor_core_kernel_matches_oracle(sizes, dist, n, v_scale):
    """mlp_tc_fvp (forward + tangents + metric + backward on the tensor cores) against the numpy oracle's F v, for
    directions of very different magnitude (CG iterates span orders of magnitude); the fp32 re-run must not fire."""
    from gpu_helpers import fvp
    from rl_replicas_b200 import _lib
    rng = np.random.default_rng(n + sizes[0])
    layers = [(rng.standard_normal((o, i)).astype(np.float32) / np.sqrt(i), 0.1 * rng.standard_normal(o).astype(np.float32))
              for i, o in zip(sizes[:-1], sizes[1:])]
    flat_p = O.flatten_layers(layers)
    obs = rng.standard_normal((n, sizes[0])).astype(np.float32)
    log_std = np.full(sizes[-1], -0.5, np.float32) if dist == "gaussian" else None
    v = (v_scale * rng.standard_normal(flat_p.size)).astype(np.float32)
    before = int(_lib.load().b200rl_tc_fallback_count())
    got = fvp(sizes, flat_p, obs, dist, v, log_std)
    assert int(_lib.load().b200rl_tc_fallback_count()) == before
    want = O.fisher_vector_product(layers, dist, log_std, obs, v, damping=0.0)
    assert rel_err(got, want) < 1e-5


def test_fvp_row_outlier_is_redone_in_fp32():
    """One transition whose observation is 1e6 times the others drags every feature's scale up: all other rows lose
    their l-splits.  The precision guard notices (row max 2^17 below the column max) and the fp32 kernel redoes it."""
    from gpu_helpers import fvp
    from rl_replicas_b200 import _lib
    rng = np.random.default_rng(4)
    sizes, n = [27, 64, 64, 8], 3000
    layers = [(rng.standard_normal((o, i)).astype(np.float32) / np.sqrt(i), np.zeros(o, np.float32))
              for i, o in zip(sizes[:-1], sizes[1:])]
    flat_p = O.flatten_layers(layers)
    obs = rng.standard_normal((n, 27)).astype(np.float32)
    obs[5] *= 1e6
    log_std = np.full(8, -0.5, np.float32)
    v = rng.standard_normal(flat_p.size).astype(np.float32)
    before = int(_lib.load().b200rl_tc_fallback_count())
    got = fvp(sizes, flat_p, obs, "gaussian", v, log_std)
    want = O.fisher_vector_product(layers, "gaussian", log_std, obs, v, damping=0.0)
    assert int(_lib.load().b200rl_tc_fallback_count()) == before + 1
    assert rel_err(got, want) < 1e-5


def test_fvp_mixed_feature_magnitudes_stay_on_the_tensor_cores():
    """MuJoCo-style observations: features spanning 1e-3 .. 1e3.  Per-feature scales keep all of them at full
    precision; no re-run."""
    from gpu_helpers import fvp
    from rl_replicas_b200 import _lib
    rng = np.random.default_rng(5)
    sizes, n = [27, 64, 64, 8], 5000
    feat = (10.0 ** rng.uniform(-3, 3, 27)).astype(np.float32)
    layers = [(rng.standard_normal((o, i)).astype(np.float32) / np.sqrt(i), np.zeros(o, np.float32))
              for i, o in zip(sizes[:-1], sizes[1:])]
    layers[0] = ((layers[0][0] / feat[None, :]).astype(np.float32), layers[0][1])  # first layer undoes the feature scale
    flat_p = O.flatten_layers(layers)
    obs = (rng.standard_normal((n, 27)) * feat[None, :]).astype(np.float32)
    log_std = np.full(8, -0.5, np.float32)
    v = rng.standard_normal(flat_p.size).astype(np.float32)
    before = int(_lib.load().b200rl_tc_fallback_count())
    got = fvp(sizes, flat_p, obs, "gaussian", v, log_std)
    assert int(_lib.load().b200rl_tc_fallback_count()) == before
    want = O.fisher_vector_product(layers, "gaussian", log_std, obs, v, damping=0.0)
    assert rel_err(got, want) < 1e-5


@pytest.mark.parametrize("dist", ["gaussian", "categorical"])
def test_data_parallel_trpo_two_engines_one_gpu(dist):
    """b200rl_trpo_update_dp: two engines with half the episodes each and a test all-reduce hook against ONE engine on
    the whole batch.  Both ranks must hold bit-identical parameters and take the same line-search decision; against
    the single engine the surrogate gradient agrees at 1e-5 and the step at the conjugate-gradient bar of this file
    (2e-3: ten CG iterations amplify the different summation order of the reduced vectors)."""
    import threading

    import torch
    from rl_replicas_b200 import synthetic
    from rl_replicas_b200.engine import OLD_POLICY, POLICY, VALUE, OnPolicyEngine
    rng = np.random.default_rng(4)
    A = 6 if dist == "gaussian" else 5
    ps, vs = [17, 64, 64, A], [17, 64, 64, 1]
    mk = lambda sz: [(rng.standard_normal((o, i)).astype(np.float32) / np.sqrt(i), np.zeros(o, np.float32))
                     for i, o in zip(sz[:-1], sz[1:])]
    pl, vl = mk(ps), mk(vs)
    log_std = np.full(A, -0.5, np.float32) if dist == "gaussian" else None
    full = synthetic.ragged_batch(24000, 17, A, dist == "categorical", seed=6, min_len=50, max_len=400,
                                  mean_fn=(lambda o: O.mlp_forward(pl, o)[0]) if dist == "gaussian" else None)
    n = full["obs"].shape[0]
    Kv = 4

    def make(batch):
        e = OnPolicyEngine(ps, vs, dist, batch["obs"].shape[0], batch["ep_done"].shape[0])
        e.set_params(POLICY, O.flatten_layers(pl))
        e.set_params(OLD_POLICY, O.flatten_layers(pl))
        e.set_params(VALUE, O.flatten_layers(vl))
        if log_std is not None:
            e.set_log_std(log_std)
        e.set_adam(VALUE, None, None, 0)
        e.load_batch(batch)
        return e

    single = make(full)
    st1, ts1 = single.trpo_update(OnPolicyEngine.hparams(num_value_gradients=Kv))
    p1, v1 = single.get_params(POLICY), single.get_params(VALUE)
    g1 = single.view("policy_grad").cpu().numpy()[:single.n_policy].copy()

    barrier, bufs, calls = threading.Barrier(2), [None, None], [0]

    def hook(rank):
        def fn(t):
            torch.cuda.current_stream().synchronize()
            bufs[rank] = t
            barrier.wait()
            if rank == 0:
                total = bufs[0] + bufs[1]
                bufs[0].copy_(total)
                bufs[1].copy_(total)
                torch.cuda.current_stream().synchronize()
                calls[0] += 1
            barrier.wait()
        return fn

    engines = [make(synthetic.shard_batch(full, r, 2)) for r in range(2)]
    torch.cuda.synchronize()
    out, errors = [None, None], []

    def work(r):
        try:
            with torch.cuda.stream(torch.cuda.Stream()):
                out[r] = engines[r].trpo_update(OnPolicyEngine.hparams(n_global_rows=n, num_value_gradients=Kv),
                                                allreduce=hook(r))
                torch.cuda.current_stream().synchronize()
        except Exception as exc:  # pragma: no cover
            errors.append(exc)
            barrier.abort()

    threads = [threading.Thread(target=work, args=(r,)) for r in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=300)
    assert not errors, errors
    pd, vd = [e.get_params(POLICY) for e in engines], [e.get_params(VALUE) for e in engines]
    np.testing.assert_array_equal(pd[0], pd[1])
    np.testing.assert_array_equal(vd[0], vd[1])
    (sa, ta), (sb, tb) = out
    assert ta.accepted_index == tb.accepted_index == ts1.accepted_index and ta.rejected == tb.rejected == ts1.rejected == 0
    assert ta.fvp_launches == ts1.fvp_launches
    assert calls[0] >= 1 + 1 + ta.fvp_launches + 1 + Kv  # adv stats, gradient, every F v, >= 1 evaluation, value steps
    gd = engines[0].view("policy_grad").cpu().numpy()[:engines[0].n_policy]
    assert rel_err(gd, g1) < 1e-5
    assert abs(sa.policy_loss_before - st1.policy_loss_before) < 1e-5 * max(1.0, abs(st1.policy_loss_before))
    assert abs(sa.adv_std - st1.adv_std) < 1e-9 * st1.adv_std
    assert rel_err(pd[0], p1) < 2e-3 and rel_err(vd[0], v1) < 2e-5
    assert abs(ta.kl - ts1.kl) < 2e-2 * abs(ts1.kl) + 1e-7
    for e in engines + [single]:
        e.close()
