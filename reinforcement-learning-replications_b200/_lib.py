"""ctypes binding of libb200rl.so (C ABI declared in include/b200rl.h).

There is NO CPU fallback: if the library is missing or a call fails, this raises.
"""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B200RL_LIB") or os.path.join(HERE, "libb200rl.so")  # B200RL_LIB: an A/B build of the library

MAX_LAYERS = 4
MAX_LEARNERS = 16
N_SCALARS = 8
ACT = {"identity": 0, "tanh": 1, "relu": 2}
DIST = {"none": 0, "gaussian": 1, "categorical": 2}
LOSS = {"eval": 0, "ppo_clip": 1, "vpg": 2, "trpo_surrogate": 3, "mse": 4, "fvp": 5}
FLAG_FORWARD_ONLY, FLAG_NO_TC = 1, 2


class MlpDesc(C.Structure):
    _fields_ = [("n_layers", C.c_int32), ("sizes", C.c_int32 * (MAX_LAYERS + 1)), ("hidden_act", C.c_int32),
                ("out_act", C.c_int32)]

    @classmethod
    def make(cls, sizes, hidden_act="tanh", out_act="identity"):
        if not 2 <= len(sizes) <= MAX_LAYERS + 1:
            raise NotImplementedError(f"MLP with {len(sizes) - 1} Linear layers is outside the engine's range 1..{MAX_LAYERS}")
        d = cls()
        d.n_layers = len(sizes) - 1
        for i, s in enumerate(sizes):
            d.sizes[i] = int(s)
        d.hidden_act, d.out_act = ACT[hidden_act], ACT[out_act]
        return d


class LossGradArgs(C.Structure):
    _fields_ = [("mlp", MlpDesc), ("loss", C.c_int32), ("dist", C.c_int32), ("n_rows", C.c_int64),
                ("n_global", C.c_int64), ("clip_range", C.c_float), ("params", C.c_void_p), ("obs", C.c_void_p),
                ("actions", C.c_void_p), ("log_std", C.c_void_p), ("adv_raw", C.c_void_p), ("adv_stats", C.c_void_p),
                ("old_logp", C.c_void_p), ("target", C.c_void_p), ("row_out", C.c_void_p), ("partials", C.c_void_p),
                ("scalar_partials", C.c_void_p), ("skip_flag", C.c_void_p), ("out_full", C.c_void_p),
                ("old_out", C.c_void_p), ("direction", C.c_void_p), ("flags", C.c_int32),
                ("obs_absmax", C.c_void_p), ("target_absmax", C.c_void_p), ("train_log_std", C.c_int32)]


class OnPolicyConfig(C.Structure):
    _fields_ = [("policy", MlpDesc), ("value", MlpDesc), ("dist", C.c_int32), ("rewards_f64", C.c_int32),
                ("max_rows", C.c_int64), ("max_episodes", C.c_int64)]


class PpoHparams(C.Structure):
    _fields_ = [("gamma", C.c_double), ("gae_lambda", C.c_double), ("clip_range", C.c_double),
                ("max_kl_divergence", C.c_double), ("num_policy_gradients", C.c_int32),
                ("num_value_gradients", C.c_int32), ("policy_lr", C.c_double), ("policy_beta1", C.c_double),
                ("policy_beta2", C.c_double), ("policy_eps", C.c_double), ("value_lr", C.c_double),
                ("value_beta1", C.c_double), ("value_beta2", C.c_double), ("value_eps", C.c_double),
                ("n_global_rows", C.c_int64)]


class UpdateStats(C.Structure):
    _fields_ = [("policy_loss_before", C.c_double), ("entropy_before", C.c_double), ("logp_std_before", C.c_double),
                ("kl_divergence", C.c_double), ("value_loss_mean", C.c_double), ("policy_steps_applied", C.c_int32),
                ("value_steps_applied", C.c_int32), ("kernel_launches", C.c_int32), ("fused", C.c_int32),
                ("adv_mean", C.c_double), ("adv_std", C.c_double), ("value_loss_first", C.c_double),
                ("value_loss_last", C.c_double)]


class TrpoHparams(C.Structure):
    _fields_ = [("max_constraint", C.c_double), ("n_conjugate_gradients", C.c_int32), ("max_backtracks", C.c_int32),
                ("backtrack_ratio", C.c_double), ("hvp_damping_coefficient", C.c_double)]


class TrpoStats(C.Structure):
    _fields_ = [("step_size", C.c_double), ("xhx", C.c_double), ("loss_before", C.c_double), ("new_loss", C.c_double),
                ("kl", C.c_double), ("accepted_index", C.c_int32), ("rejected", C.c_int32), ("cg_converged", C.c_int32),
                ("fvp_launches", C.c_int32)]


class OffPolicyConfig(C.Structure):
    _fields_ = [("policy", MlpDesc), ("q", MlpDesc), ("n_q", C.c_int32), ("max_minibatch", C.c_int32),
                ("max_steps", C.c_int32), ("algo", C.c_int32), ("dueling_k", C.c_int32),
                ("noisy_layers", C.c_int32)]


class IqnConfig(C.Structure):
    _fields_ = [("n_cos", C.c_int32), ("n", C.c_int32), ("n_target", C.c_int32), ("k", C.c_int32)]


class D4pgConfig(C.Structure):
    _fields_ = [("n_atoms", C.c_int32), ("reserved", C.c_int32), ("v_min", C.c_double), ("v_max", C.c_double)]


class TqcConfig(C.Structure):
    _fields_ = [("n_quantiles", C.c_int32), ("n_drop_per_net", C.c_int32)]


class CqlConfig(C.Structure):
    _fields_ = [("n_actions", C.c_int32), ("lagrange", C.c_int32)]


class CqlHparams(C.Structure):
    _fields_ = [("weight", C.c_double), ("temperature", C.c_double), ("target_action_gap", C.c_double),
                ("alpha_lr", C.c_double), ("alpha_beta1", C.c_double), ("alpha_beta2", C.c_double),
                ("alpha_eps", C.c_double), ("backup_entropy", C.c_int32), ("reserved", C.c_int32)]


class RedqConfig(C.Structure):
    _fields_ = [("n_critics", C.c_int32), ("n_min", C.c_int32)]


class EdacConfig(C.Structure):
    _fields_ = [("n_critics", C.c_int32), ("reserved", C.c_int32), ("eta", C.c_double)]


class IqlConfig(C.Structure):
    _fields_ = [("value", MlpDesc)]


class IqlHparams(C.Structure):
    _fields_ = [("expectile", C.c_double), ("beta", C.c_double), ("max_weight", C.c_double),
                ("log_std_min", C.c_double), ("log_std_max", C.c_double), ("v_lr", C.c_double),
                ("v_beta1", C.c_double), ("v_beta2", C.c_double), ("v_eps", C.c_double)]


class SacHparams(C.Structure):
    _fields_ = [("alpha", C.c_double), ("target_entropy", C.c_double), ("alpha_lr", C.c_double),
                ("alpha_beta1", C.c_double), ("alpha_beta2", C.c_double), ("alpha_eps", C.c_double),
                ("log_std_min", C.c_double), ("log_std_max", C.c_double), ("learn_alpha", C.c_int32),
                ("reserved", C.c_int32)]


class DqnHparams(C.Structure):
    _fields_ = [("target_update_interval", C.c_int32), ("double_q", C.c_int32)]


class C51Hparams(C.Structure):
    _fields_ = [("n_atoms", C.c_int32), ("reserved", C.c_int32), ("v_min", C.c_double), ("v_max", C.c_double)]


class QrHparams(C.Structure):
    _fields_ = [("n_quantiles", C.c_int32), ("reserved", C.c_int32)]


class PerHparams(C.Structure):
    _fields_ = [("alpha", C.c_double), ("eps", C.c_double), ("beta_start", C.c_double),
                ("beta_anneal_steps", C.c_int64)]


class OffPolicyReplay(C.Structure):
    _fields_ = [("obs", C.c_void_p), ("act", C.c_void_p), ("rew", C.c_void_p), ("next_obs", C.c_void_p),
                ("done", C.c_void_p), ("rows", C.c_int64)]


class OffPolicyHparams(C.Structure):
    _fields_ = [("gamma", C.c_double), ("polyak_rho", C.c_double), ("target_noise_scale", C.c_double),
                ("target_noise_clip", C.c_double), ("action_limit", C.c_double), ("policy_delay", C.c_int32),
                ("use_target_noise", C.c_int32), ("policy_lr", C.c_double), ("policy_beta1", C.c_double),
                ("policy_beta2", C.c_double), ("policy_eps", C.c_double), ("q1_lr", C.c_double), ("q2_lr", C.c_double),
                ("q_beta1", C.c_double), ("q_beta2", C.c_double), ("q_eps", C.c_double)]


ALLREDUCE_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p)

# name -> (restype, argtypes); must list every symbol include/b200rl.h declares (tests/test_abi.py checks)
SIGNATURES = {
    "b200rl_last_error": (C.c_char_p, []),
    "b200rl_version": (C.c_int, []),
    "b200rl_launch_count": (C.c_int64, []),
    "b200rl_mlp_param_count": (C.c_int64, [C.POINTER(MlpDesc)]),
    "b200rl_mlp_grid": (C.c_int, [C.POINTER(MlpDesc), C.c_int64, C.c_int]),
    "b200rl_gae_scan_workspace_bytes": (C.c_size_t, [C.c_int64]),
    "b200rl_gae_scan": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                  C.c_int64, C.c_double, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_size_t, C.c_void_p]),
    "b200rl_mlp_loss_grad": (C.c_int, [C.POINTER(LossGradArgs), C.c_void_p]),
    "b200rl_absmax": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "b200rl_absmax_cols": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p]),
    "b200rl_tc_fallback_count": (C.c_int64, []),
    "b200rl_reduce_partials": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p,
                                         C.c_int, C.c_void_p, C.c_void_p]),
    "b200rl_adam_step": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_double,
                                   C.c_double, C.c_double, C.c_double, C.c_void_p, C.c_int, C.c_double, C.c_double,
                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200rl_onpolicy_create": (C.c_int, [C.POINTER(OnPolicyConfig), C.POINTER(C.c_void_p)]),
    "b200rl_onpolicy_destroy": (None, [C.c_void_p]),
    "b200rl_onpolicy_set_params": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_void_p]),
    "b200rl_onpolicy_get_params": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_void_p]),
    "b200rl_onpolicy_set_adam": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p]),
    "b200rl_onpolicy_get_adam": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int64,
                                           C.POINTER(C.c_int64), C.c_void_p]),
    "b200rl_onpolicy_set_train_log_std": (C.c_int, [C.c_void_p, C.c_int32]),
    "b200rl_onpolicy_set_log_std": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "b200rl_onpolicy_load_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                             C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_void_p]),
    "b200rl_ppo_update": (C.c_int, [C.c_void_p, C.POINTER(PpoHparams), C.c_void_p, C.c_void_p,
                                    C.POINTER(UpdateStats), C.c_void_p]),
    "b200rl_vpg_update": (C.c_int, [C.c_void_p, C.POINTER(PpoHparams), C.c_void_p, C.c_void_p,
                                    C.POINTER(UpdateStats), C.c_void_p]),
    "b200rl_trpo_update": (C.c_int, [C.c_void_p, C.POINTER(PpoHparams), C.POINTER(TrpoHparams), C.POINTER(UpdateStats),
                                     C.POINTER(TrpoStats), C.c_void_p]),
    "b200rl_trpo_update_dp": (C.c_int, [C.c_void_p, C.POINTER(PpoHparams), C.POINTER(TrpoHparams), C.c_void_p, C.c_void_p,
                                        C.POINTER(UpdateStats), C.POINTER(TrpoStats), C.c_void_p]),
    "b200rl_onpolicy_fvp": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_double, C.c_void_p]),
    "b200rl_onpolicy_device_view": (C.c_int, [C.c_void_p, C.c_char_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int64),
                                              C.POINTER(C.c_int32)]),
    "b200rl_offpolicy_create": (C.c_int, [C.POINTER(OffPolicyConfig), C.POINTER(C.c_void_p)]),
    "b200rl_offpolicy_destroy": (None, [C.c_void_p]),
    "b200rl_offpolicy_set_params": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_void_p]),
    "b200rl_offpolicy_get_params": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_void_p]),
    "b200rl_offpolicy_set_adam": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p]),
    "b200rl_offpolicy_get_adam": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int64,
                                            C.POINTER(C.c_int64), C.c_void_p]),
    "b200rl_offpolicy_state_floats": (C.c_int64, [C.c_void_p]),
    "b200rl_offpolicy_get_state": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(C.c_int64), C.c_void_p]),
    "b200rl_offpolicy_set_state": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(C.c_int64), C.c_void_p]),
    "b200rl_offpolicy_train": (C.c_int, [C.c_void_p, C.POINTER(OffPolicyHparams), C.c_int32, C.c_int32] +
                               [C.c_void_p] * 11 + [C.POINTER(C.c_int32), C.c_void_p]),
    "b200rl_offpolicy_train_gather": (C.c_int, [C.c_void_p, C.POINTER(OffPolicyHparams), C.c_int32, C.c_int32] +
                                      [C.c_void_p] * 5 + [C.c_int64] + [C.c_void_p] * 7 +
                                      [C.POINTER(C.c_int32), C.c_void_p]),
    "b200rl_offpolicy_train_gather_rng": (C.c_int, [C.c_void_p, C.POINTER(OffPolicyHparams), C.c_int32, C.c_int32] +
                                          [C.c_void_p] * 5 + [C.c_int64] * 3 + [C.c_uint64] * 2 + [C.c_void_p] * 5 +
                                          [C.POINTER(C.c_int32), C.c_void_p]),
    "b200rl_offpolicy_get_draws": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200rl_offpolicy_set_sac": (C.c_int, [C.c_void_p, C.POINTER(SacHparams)]),
    "b200rl_offpolicy_set_alpha": (C.c_int, [C.c_void_p, C.c_float, C.c_float, C.c_float, C.c_int64]),
    "b200rl_offpolicy_get_alpha": (C.c_int, [C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_float),
                                             C.POINTER(C.c_float), C.POINTER(C.c_int64)]),
    "b200rl_offpolicy_sac_outputs": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "b200rl_offpolicy_set_dqn": (C.c_int, [C.c_void_p, C.POINTER(DqnHparams)]),
    "b200rl_offpolicy_set_c51": (C.c_int, [C.c_void_p, C.POINTER(C51Hparams)]),
    "b200rl_offpolicy_set_qr": (C.c_int, [C.c_void_p, C.POINTER(QrHparams)]),
    "b200rl_offpolicy_create_group": (C.c_int, [C.POINTER(OffPolicyConfig), C.c_int32, C.POINTER(C.c_void_p)]),
    "b200rl_offpolicy_create_iqn": (C.c_int, [C.POINTER(OffPolicyConfig), C.POINTER(IqnConfig), C.c_int32,
                                              C.POINTER(C.c_void_p)]),
    "b200rl_offpolicy_create_d4pg": (C.c_int, [C.POINTER(OffPolicyConfig), C.POINTER(D4pgConfig), C.c_int32,
                                               C.POINTER(C.c_void_p)]),
    "b200rl_offpolicy_create_tqc": (C.c_int, [C.POINTER(OffPolicyConfig), C.POINTER(TqcConfig), C.c_int32,
                                              C.POINTER(C.c_void_p)]),
    "b200rl_offpolicy_get_policy_losses": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.POINTER(C.c_int32)]),
    "b200rl_offpolicy_train_gather_group": (C.c_int, [C.c_void_p, C.POINTER(OffPolicyHparams), C.c_int32, C.c_int32,
                                                      C.POINTER(OffPolicyReplay)] + [C.c_void_p] * 7 +
                                            [C.POINTER(C.c_int32), C.c_void_p]),
    "b200rl_offpolicy_train_gather_rng_group": (C.c_int, [C.c_void_p, C.POINTER(OffPolicyHparams), C.c_int32, C.c_int32,
                                                          C.POINTER(OffPolicyReplay)] + [C.c_void_p] * 9 +
                                                [C.POINTER(C.c_int32), C.c_void_p]),
    "b200rl_offpolicy_set_per": (C.c_int, [C.c_void_p, C.POINTER(PerHparams)]),
    "b200rl_offpolicy_train_prioritized": (C.c_int, [C.c_void_p, C.POINTER(OffPolicyHparams), C.c_int32, C.c_int32] +
                                           [C.c_void_p] * 5 + [C.c_int64, C.c_void_p, C.c_uint64, C.c_uint64] +
                                           [C.c_void_p] * 3),
    "b200rl_offpolicy_train_prioritized_group": (C.c_int, [C.c_void_p, C.POINTER(OffPolicyHparams), C.c_int32,
                                                           C.c_int32, C.POINTER(OffPolicyReplay)] + [C.c_void_p] * 6),
    "b200rl_offpolicy_get_per_draws": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32] + [C.c_void_p] * 4),
    "b200rl_offpolicy_set_nstep": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p]),
    "b200rl_offpolicy_get_nstep_draws": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32] + [C.c_void_p] * 4),
    "b200rl_offpolicy_set_noise_keys": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200rl_offpolicy_get_noisy_draws": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p]),
    "b200rl_offpolicy_get_iqn_draws": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p]),
    "b200rl_per_tree_floats": (C.c_int64, [C.c_int64]),
    "b200rl_per_tree_build": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p]),
    "b200rl_per_tree_set_range": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_void_p]),
    "b200rl_offpolicy_set_alpha_group": (C.c_int, [C.c_void_p] * 5),
    "b200rl_offpolicy_create_cql": (C.c_int, [C.POINTER(OffPolicyConfig), C.POINTER(CqlConfig), C.c_int32,
                                              C.POINTER(C.c_void_p)]),
    "b200rl_offpolicy_set_cql": (C.c_int, [C.c_void_p, C.POINTER(CqlHparams)]),
    "b200rl_offpolicy_set_alpha_prime_group": (C.c_int, [C.c_void_p] * 5),
    "b200rl_offpolicy_get_alpha_prime_group": (C.c_int, [C.c_void_p] * 5),
    "b200rl_offpolicy_cql_outputs": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "b200rl_offpolicy_set_cql_draws": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]),
    "b200rl_offpolicy_get_cql_draws": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]),
    "b200rl_offpolicy_get_alpha_group": (C.c_int, [C.c_void_p] * 5),
    "b200rl_offpolicy_create_iql": (C.c_int, [C.POINTER(OffPolicyConfig), C.POINTER(IqlConfig), C.c_int32,
                                              C.POINTER(C.c_void_p)]),
    "b200rl_offpolicy_set_iql": (C.c_int, [C.c_void_p, C.POINTER(IqlHparams)]),
    "b200rl_offpolicy_iql_outputs": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200rl_offpolicy_create_redq": (C.c_int, [C.POINTER(OffPolicyConfig), C.POINTER(RedqConfig), C.c_int32,
                                               C.POINTER(C.c_void_p)]),
    "b200rl_offpolicy_set_redq_subsets": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p]),
    "b200rl_offpolicy_get_redq_subsets": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p]),
    "b200rl_offpolicy_redq_outputs": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "b200rl_offpolicy_create_edac": (C.c_int, [C.POINTER(OffPolicyConfig), C.POINTER(EdacConfig), C.c_int32,
                                               C.POINTER(C.c_void_p)]),
    "b200rl_offpolicy_edac_outputs": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p]),
    "b200rl_discounted_cumsum": (C.c_int, [C.c_void_p, C.c_int64, C.c_double, C.c_void_p, C.c_void_p]),
    "b200rl_gae_f64": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_double, C.c_double, C.c_void_p,
                                 C.c_void_p]),
    "b200rl_normalize": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "b200rl_polyak": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_double, C.c_void_p]),
    "b200rl_onpolicy_comm_export": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p)]),
    "b200rl_ipc_open": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p)]),
    "b200rl_ipc_close": (C.c_int, [C.c_void_p]),
    "b200rl_onpolicy_comm_attach": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.POINTER(C.c_void_p)]),
    "b200rl_onpolicy_scalar_history": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(C.c_int32)]),
    "b200rl_onpolicy_run_stage": (C.c_int, [C.c_void_p, C.c_char_p, C.POINTER(PpoHparams), C.c_void_p]),
}

_lib = None


class B200RLError(RuntimeError):
    pass


def load() -> C.CDLL:
    """Load libb200rl.so and attach the signatures.  Raises if the library is absent (no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise B200RLError(
            f"{LIB_PATH} is missing: build it with `python __graft_entry__.py` (nvcc, sm_90a). "
            "There is no CPU fallback for the update path.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    _lib = lib
    return lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = load().b200rl_last_error()
        raise B200RLError(f"{what or 'libb200rl'} failed (rc={rc}): {msg.decode() if msg else '?'}")
