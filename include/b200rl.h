/*
 * b200rl.h -- C ABI of the H100-native (sm_90a) policy-gradient update engine (libb200rl.so).
 *
 * The reference (rl_replicas 0.0.7) is pure Python and has NO FFI / plugin layer: its drop-in seam is the Python
 * class API (SURVEY.md section 8b).  This header is the native boundary underneath our Python mirror of that API:
 * every entry point names the reference function(s) whose arithmetic it replaces (paths relative to
 * /root/reference/src/rl_replicas/).  INTEGRATION.md shows the ctypes stub a maintainer of the reference would add.
 *
 * Conventions
 *   - plain C types only: pointers + sizes; no torch / C++ types cross the boundary.
 *   - every function returns 0 on success, non-zero on failure; b200rl_last_error() describes the last failure of
 *     the calling thread.  CUDA errors are reported the same way (never swallowed, never a CPU fallback).
 *   - "device pointer" arguments must be 16-byte aligned and live on the current CUDA device.
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).  All launchers are asynchronous.
 *   - MLP parameters are ONE flat float32 vector in torch.nn.utils.parameters_to_vector order:
 *     W0 [out0,in0] row-major, b0 [out0], W1, b1, ...  (torch.nn.Linear layout, ref: networks/mlp.py:24-31).
 */
#ifndef B200RL_H
#define B200RL_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200RL_VERSION 100
#define B200RL_MAX_LAYERS 4   /* Linear layers per MLP */
#define B200RL_MAX_LEARNERS 16 /* learners in one off-policy group (b200rl_offpolicy_create_group) */
#define B200RL_N_SCALARS 8    /* per-launch scalar sums, see b200rl_mlp_loss_grad */

enum b200rl_activation { B200RL_ACT_IDENTITY = 0, B200RL_ACT_TANH = 1, B200RL_ACT_RELU = 2 };
enum b200rl_dist { B200RL_DIST_NONE = 0, B200RL_DIST_GAUSSIAN = 1, B200RL_DIST_CATEGORICAL = 2 };
enum b200rl_loss {
  B200RL_LOSS_EVAL = 0,           /* forward only: per-row output (value, or log-prob when dist != NONE) + scalar sums */
  B200RL_LOSS_PPO_CLIP = 1,       /* -mean(min(r A, clamp(r,1-c,1+c) A))        ref: algorithms/ppo.py:237-257 */
  B200RL_LOSS_VPG = 2,            /* -mean(logp A)                               ref: algorithms/vpg.py:194-207 */
  B200RL_LOSS_TRPO_SURROGATE = 3, /* -mean(r A)                                  ref: algorithms/trpo.py:154-165 */
  B200RL_LOSS_MSE = 4,            /* mean((out - target)^2)                      ref: algorithms/ppo.py:282-287 */
  B200RL_LOSS_FVP = 5             /* Fisher-vector product J^T M J v / N of mean KL(old || new) at theta_old:
                                     forward pass with tangents (J v), metric M of the distribution, then the ordinary
                                     backward pass (J^T); replaces the double backprop of
                                     optimizers/conjugate_gradient_optimizer.py:133-167 (trpo.py:167-175) */
};
#define B200RL_FLAG_FORWARD_ONLY 1 /* evaluate the loss terms of `loss` but run no backward pass (line search) */
#define B200RL_FLAG_NO_TC 2        /* force the fp32 CUDA-core kernel */

/* MLP description (ref: networks/mlp.py:15-31). */
typedef struct {
  int32_t n_layers;                     /* number of Linear layers, 1..B200RL_MAX_LAYERS */
  int32_t sizes[B200RL_MAX_LAYERS + 1]; /* widths: input, hidden..., output */
  int32_t hidden_act;                   /* enum b200rl_activation */
  int32_t out_act;
} b200rl_mlp_desc;

const char* b200rl_last_error(void);
int b200rl_version(void);
/* kernels launched by this library in this process so far (bench.py reports gpu_launches from it) */
int64_t b200rl_launch_count(void);
/* number of float32 parameters of the MLP (sum of out*in + out); -1 if the description is invalid */
int64_t b200rl_mlp_param_count(const b200rl_mlp_desc* mlp);
/* CTAs the fused MLP kernels use for n_rows rows on the current device (= rows of `partials`); -1 on error.
 * with_backward: 0 forward only with B200RL_LOSS_EVAL, 1 forward + backward, 2 Fisher-vector product, 3 forward-only
 * launches that set out_full / old_out / B200RL_FLAG_NO_TC or evaluate a loss other than EVAL (B200RL_FLAG_FORWARD_ONLY;
 * the larger of the tensor-core and the fp32 kernel's row counts),
 * 4 forward + backward on the fp32 kernel (B200RL_FLAG_NO_TC or train_log_std). */
int b200rl_mlp_grid(const b200rl_mlp_desc* mlp, int64_t n_rows, int with_backward);

/* ------------------------------------------------------------------------------------------------------------
 * gae_scan -- bootstrapped rewards, discounted returns, TD residuals, GAE  (one segmented reverse scan, float64 carry)
 *   replaces: utils.py:14-28 (discounted_cumulative_sums), :31-44 (gae), :74-87 (bootstrap_rewards_with_last_values)
 *             and the per-episode loops of algorithms/ppo.py:142-161.
 *   rewards     [n]     float32 (rewards_f64 = 0) or float64 (rewards_f64 = 1)
 *   values      [n]     V(obs_t)
 *   last_values [n_ep]  V(last_observation_e)
 *   ep_offsets  [n_ep+1] CSR offsets into the flat transition arrays (every episode has >= 1 step)
 *   ep_done     [n_ep]  1 = the episode ended (terminated or truncated) => no bootstrap (utils.py:81-82)
 *   adv_raw, ret [n]    outputs (float32 casts of the float64 recurrences, ppo.py:151,160)
 *   stats       [3]     float64: sum(adv_raw), sum(adv_raw^2), n   (for normalize_tensor, utils.py:90-92)
 *   workspace           b200rl_gae_scan_workspace_bytes(n) bytes of device memory, ZEROED ONCE by the caller at
 *                       allocation (cudaMemset); every launch leaves it ready for the next one (no per-call memset)
 * ------------------------------------------------------------------------------------------------------------ */
size_t b200rl_gae_scan_workspace_bytes(int64_t n);
int b200rl_gae_scan(const void* rewards, int rewards_f64, const float* values, const float* last_values,
                    const int64_t* ep_offsets, const uint8_t* ep_done, int64_t n, int64_t n_ep, double gamma,
                    double gae_lambda, float* adv_raw, float* ret, double* stats, void* workspace,
                    size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * mlp_loss_grad -- ONE fused kernel: MLP forward -> distribution log-prob -> loss -> dLoss/dOut -> MLP backward,
 * activations never leave the SM.  Per-CTA partial gradients go to `partials`; reduce with b200rl_reduce_adam.
 *   replaces: networks/mlp.py:33-41, policies/gaussian_policy.py:25-37, policies/categorical_policy.py:22-32,
 *             algorithms/ppo.py:237-257 (+ autograd backward at :234), :259-269 (approx KL), :282-287 (+ :277),
 *             algorithms/vpg.py:200-206, algorithms/trpo.py:154-165, utils.py:60-71 (compute_values, loss = EVAL),
 *             utils.py:90-92 (normalize_tensor, applied on load from adv_stats).
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct {
  b200rl_mlp_desc mlp;
  int32_t loss;            /* enum b200rl_loss */
  int32_t dist;            /* enum b200rl_dist */
  int64_t n_rows;          /* rows handled by this launch (this rank's shard) */
  int64_t n_global;        /* denominator of the mean (= n_rows on one GPU; sum over ranks otherwise) */
  float clip_range;        /* PPO clip epsilon */
  const float* params;     /* [P] device */
  const float* obs;        /* [n_rows, sizes[0]] device, row-major */
  const float* actions;    /* Gaussian: [n_rows, sizes[L]]; Categorical: [n_rows] (index as float, ppo.py:154) */
  const float* log_std;    /* Gaussian: [sizes[L]] */
  const float* adv_raw;    /* [n_rows] un-normalised advantages (policy losses) */
  const double* adv_stats; /* [3] global sum, sum of squares, count -> mean / unbiased std; NULL = use adv_raw as is */
  const float* old_logp;   /* [n_rows] (PPO / TRPO) */
  const float* target;     /* [n_rows] (MSE: discounted returns) */
  float* row_out;          /* optional [n_rows]: value (dist NONE) or log-prob (dist set); may be NULL */
  float* partials;         /* [grid, P] per-CTA partial gradients (losses other than EVAL) */
  double* scalar_partials; /* [grid, B200RL_N_SCALARS] per-CTA partial sums:
                              0 sum(loss terms)  1 sum(old_logp - logp)  2 sum(entropy)  3 sum(logp)  4 sum(logp^2)
                              5 rows processed   6 sum(KL(old || new)) when old_out is given   7 reserved */
  const int32_t* skip_flag; /* optional device flag: non-zero => the launch is a no-op (early stop) */
  float* out_full;         /* optional [n_rows, sizes[L]]: raw network outputs (means / logits) are written here */
  const float* old_out;    /* optional [n_rows, sizes[L]]: outputs of the old policy -> true KL(old || new) per row,
                              kl_divergence(old_dist, dist) of trpo.py:167-175 (Gaussian: same log_std for both) */
  const float* direction;  /* [P] the vector v of B200RL_LOSS_FVP, same flat layout as params */
  int32_t flags;           /* B200RL_FLAG_* */
  const float* obs_absmax; /* optional device array [sizes[0]]: per-feature max |obs| over the batch (scales of the fp16
                              tensor-core kernel; NULL = a pre-pass computes it on every launch, b200rl_absmax_cols) */
  const float* target_absmax; /* optional device scalar: max |target| (MSE backward); NULL = pre-pass */
  int32_t train_log_std;   /* Gaussian policy losses with a backward pass: also emit dLoss/dlog_std -- partial rows then
                              have P + sizes[L] columns (the gradient of log_std in the last sizes[L]).  Runs on the fp32
                              kernel.  policies/gaussian_policy.py:25-37 with log_std inside the optimizer */
} b200rl_mlp_loss_grad_args;

int b200rl_mlp_loss_grad(const b200rl_mlp_loss_grad_args* args, void* stream);

/* out[0] = max |x[i]| (+inf if x holds a NaN); `out` is a device float.  Callers that launch mlp_loss_grad many times
 * over the same observations / targets compute the hints once with this. */
int b200rl_absmax(const float* x, int64_t n, float* out, void* stream);
/* out[c] = max_r |x[r, c]| for a row-major [rows, cols] device array, cols <= 32 (the obs_absmax hint). */
int b200rl_absmax_cols(const float* x, int64_t rows, int32_t cols, float* out, void* stream);

/* Number of mlp_loss_grad launches (since process start) whose fp16 tensor-core pass left the fp16 range and were
 * recomputed by the fp32 kernel queued behind it.  Synchronises the device; diagnostics / tests only. */
int64_t b200rl_tc_fallback_count(void);

/* ------------------------------------------------------------------------------------------------------------
 * reduce_adam -- fixed-order reduction of the per-CTA partials into the flat gradient, then torch.optim.Adam's
 * single-tensor update on the flat parameter vector.
 *   replaces: optimizer.zero_grad()/loss.backward() accumulation + torch.optim.Adam.step() at
 *             algorithms/ppo.py:233-235, :276-278 (torch 2.5.1 _single_tensor_adam; no weight decay / amsgrad).
 *   b200rl_reduce_partials: grad[p] = sum_c partials[c,p]; scalars[k] = sum_c scalar_partials[c,k]  (c ascending).
 *     If grad_tail != 0 the scalar sums are ALSO written as float32 to grad[n_params .. n_params+B200RL_N_SCALARS)
 *     so that ONE all-reduce of [n_params + B200RL_N_SCALARS] floats carries gradient, loss and KL (SURVEY 8e).
 *     partials may be NULL (scalars only, for EVAL launches).
 *   b200rl_adam_step: m,v,params updated in place; `step` is the 1-based step number of THIS update (host-known).
 *     Early stop (ppo.py:176-181): kl_sum points at sum(old_logp - logp) of this step's forward pass (float64, or
 *     float32 when kl_is_f32); if kl_sum/n_global > kl_limit, or *stop_flag != 0, the update is skipped and
 *     *stop_flag is set; applied_counter (optional) counts applied updates.  If tail_src != NULL its
 *     B200RL_N_SCALARS float32 values (the all-reduced tail) are stored as float64 to tail_dst.
 * ------------------------------------------------------------------------------------------------------------ */
int b200rl_reduce_partials(const float* partials, const double* scalar_partials, int32_t grid, int64_t n_params,
                           float* grad, double* scalars, int grad_tail, const int32_t* skip_flag, void* stream);
int b200rl_adam_step(float* params, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n_params,
                     int64_t step, double lr, double beta1, double beta2, double eps, const void* kl_sum,
                     int kl_is_f32, double n_global, double kl_limit, int32_t* stop_flag, int32_t* applied_counter,
                     const float* tail_src, double* tail_dst, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * On-policy update engine: owns the device-resident batch, flat parameters, Adam state and workspaces of ONE
 * PPO / VPG / TRPO learner, and runs the whole per-epoch update (the reference's `train(experience)`).
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct b200rl_onpolicy b200rl_onpolicy;

typedef struct {
  b200rl_mlp_desc policy;
  b200rl_mlp_desc value;
  int32_t dist;            /* enum b200rl_dist */
  int32_t rewards_f64;     /* dtype of the rewards buffer handed to load_batch */
  int64_t max_rows;        /* capacity (transitions) */
  int64_t max_episodes;    /* capacity (episodes) */
} b200rl_onpolicy_config;

/* all-reduce(sum) hook for data-parallel runs: called from inside b200rl_ppo_update on the engine's stream order;
 * `buf` is a device pointer owned by the engine, dtype 0 = float32, 1 = float64.  NULL = single GPU. */
typedef int (*b200rl_allreduce_fn)(void* user, void* buf, int64_t count, int32_t dtype, void* stream);

typedef struct {
  double gamma, gae_lambda, clip_range, max_kl_divergence;
  int32_t num_policy_gradients, num_value_gradients;
  double policy_lr, policy_beta1, policy_beta2, policy_eps;
  double value_lr, value_beta1, value_beta2, value_eps;
  int64_t n_global_rows;   /* 0 = single GPU (use local rows) */
} b200rl_ppo_hparams;

typedef struct {
  double policy_loss_before;    /* ppo.py:166-168 */
  double entropy_before;        /* ppo.py:170,202 */
  double logp_std_before;       /* ppo.py:169,208 (unbiased) */
  double kl_divergence;         /* ppo.py:176-178,214 (last evaluated) */
  double value_loss_mean;       /* ppo.py:192,220 */
  int32_t policy_steps_applied; /* Adam steps actually taken by the policy loop */
  int32_t value_steps_applied;
  int32_t kernel_launches;      /* kernels launched by this update */
  int32_t fused;                /* 1 = the iterations ran on the fused policy + value step kernel (mlp_tc3.cu) */
  double adv_mean, adv_std;     /* normalize_tensor statistics actually used */
  double value_loss_first, value_loss_last;
} b200rl_update_stats;

int b200rl_onpolicy_create(const b200rl_onpolicy_config* cfg, b200rl_onpolicy** out);
void b200rl_onpolicy_destroy(b200rl_onpolicy* h);

/* which: 0 policy, 1 old_policy, 2 value.  Host <-> device copies of the flat parameter vectors. */
int b200rl_onpolicy_set_params(b200rl_onpolicy* h, int which, const float* host_flat, int64_t n, void* stream);
int b200rl_onpolicy_get_params(b200rl_onpolicy* h, int which, float* host_flat, int64_t n, void* stream);
/* which: 0 policy optimizer, 2 value optimizer; step = number of Adam steps already taken (optimizer.state[p]["step"]) */
int b200rl_onpolicy_set_adam(b200rl_onpolicy* h, int which, const float* exp_avg, const float* exp_avg_sq,
                             int64_t n, int64_t step, void* stream);
int b200rl_onpolicy_get_adam(b200rl_onpolicy* h, int which, float* exp_avg, float* exp_avg_sq, int64_t n,
                             int64_t* step, void* stream);
int b200rl_onpolicy_set_log_std(b200rl_onpolicy* h, const float* host_log_std, int64_t n, void* stream);
/* Trainable log_std (policies/gaussian_policy.py:25-37 when the user put log_std into the policy optimizer, after the
 * network's parameters): from then on the policy vectors of set / get_params (which 0 and 1) and set / get_adam (which 0)
 * are [network parameters | log_std], the PPO / VPG policy steps differentiate through it (on the fp32 kernel) and
 * Adam updates it; b200rl_onpolicy_set_log_std is then unused.  TRPO refuses it. */
int b200rl_onpolicy_set_train_log_std(b200rl_onpolicy* h, int32_t on);

/* Packed trajectory batch (SURVEY.md section 8a, a1).  src_on_device = 0: HOST buffers (pinned or pageable), copied
 * with cudaMemcpyAsync; 1: device buffers (device-to-device copy). */
int b200rl_onpolicy_load_batch(b200rl_onpolicy* h, const float* obs, const float* actions, const void* rewards,
                               const float* last_obs, const int64_t* ep_offsets, const uint8_t* ep_done,
                               int64_t n_rows, int64_t n_episodes, int src_on_device, void* stream);

/* The reference's PPO.train(experience) on the loaded batch (algorithms/ppo.py:139-223).  Asynchronous device work,
 * then one device->host read of the statistics (synchronises the stream). */
int b200rl_ppo_update(b200rl_onpolicy* h, const b200rl_ppo_hparams* hp, b200rl_allreduce_fn allreduce, void* user,
                      b200rl_update_stats* stats, void* stream);
/* The reference's VPG.train (algorithms/vpg.py:127-192): one policy step on -mean(logp A), then value steps. */
int b200rl_vpg_update(b200rl_onpolicy* h, const b200rl_ppo_hparams* hp, b200rl_allreduce_fn allreduce, void* user,
                      b200rl_update_stats* stats, void* stream);

/* The reference's TRPO.train (algorithms/trpo.py:130-226): surrogate gradient, ConjugateGradientOptimizer.step
 * (optimizers/conjugate_gradient_optimizer.py:59-98: n_cg Fisher-vector products + CG, step size, backtracking line
 * search, reject/restore), old-policy sync, value steps.  Single GPU (an all-reduce per FVP is not implemented). */
typedef struct {
  double max_constraint;          /* delta, default 0.01 */
  int32_t n_conjugate_gradients;  /* default 10 */
  int32_t max_backtracks;         /* default 15 */
  double backtrack_ratio;         /* default 0.8 */
  double hvp_damping_coefficient; /* default 1e-5 */
} b200rl_trpo_hparams;

typedef struct {
  double step_size;           /* sqrt(2 delta / (x^T H x + 1e-8)) */
  double xhx;
  double loss_before;         /* surrogate at theta_old */
  double new_loss, kl;        /* at the accepted (or last tried) parameters */
  int32_t accepted_index;     /* index k of the accepted ratio backtrack_ratio^k; -1 = none accepted */
  int32_t rejected;           /* 1 = line-search condition violated, parameters restored */
  int32_t cg_converged;       /* 1 = residual fell below 1e-10 before n_cg iterations */
  int32_t fvp_launches;
} b200rl_trpo_stats;

int b200rl_trpo_update(b200rl_onpolicy* h, const b200rl_ppo_hparams* hp, const b200rl_trpo_hparams* cg,
                       b200rl_update_stats* stats, b200rl_trpo_stats* trpo_stats, void* stream);
/* The same step data-parallel: every batch-derived sum (advantage statistics, surrogate gradient + scalar sums, every
 * Fisher-vector product, the scalar sums of every line-search evaluation, the value gradients) goes through `allreduce`
 * where it is formed; hp->n_global_rows = the global row count.  All ranks take identical CG / line-search decisions.
 * allreduce == NULL: b200rl_trpo_update. */
int b200rl_trpo_update_dp(b200rl_onpolicy* h, const b200rl_ppo_hparams* hp, const b200rl_trpo_hparams* cg,
                          b200rl_allreduce_fn allreduce, void* user, b200rl_update_stats* stats,
                          b200rl_trpo_stats* ts, void* stream);
/* One Fisher-vector product on the loaded batch at the current policy parameters: out = F v + damping * v (host
 * vectors of policy-parameter length); for tests against the reference's double-backprop Hessian-vector product. */
int b200rl_onpolicy_fvp(b200rl_onpolicy* h, const float* host_v, float* host_out, int64_t n, double damping,
                        void* stream);

/* Device views for tests / profiling (pointers stay owned by the engine):
 * name: "values","last_values","adv_raw","ret","old_logp","adv_stats","policy_grad","value_grad",
 *       "policy_params","old_policy_params","value_params", and after a TRPO update its conjugate-gradient state
 *       "cg_x","cg_r","cg_p","cg_descent" and "cg_z" (F x of the step-size product, without damping) */
int b200rl_onpolicy_device_view(b200rl_onpolicy* h, const char* name, void** ptr, int64_t* count, int32_t* dtype);

/* One-shot gradient exchange over peer-mapped device memory (data-parallel runs on ONE node: NVLink / NVSwitch).
 * Once attached, the fused PPO iterations no longer call `allreduce` for the gradient: every rank stores its reduced
 * [policy gradient | value gradient | scalar sums] into its exchange buffer and reads all ranks' buffers directly
 * (sum in rank order => bit-identical parameters on every rank); the callback still carries the three small
 * collectives per update (advantage statistics, final KL, range flags).
 *   comm_export: allocates the buffer on first use, returns its CUDA IPC handle (64 bytes) and local device pointer;
 *   ipc_open / ipc_close: map / unmap another rank's handle in this process (cudaIpcOpenMemHandle);
 *   comm_attach: peer_ptrs[r] = rank r's buffer as seen from THIS process (own buffer at [rank]); world <= 16.
 * Every rank must run the same sequence of updates (as with any collective). */
int b200rl_onpolicy_comm_export(b200rl_onpolicy* h, void* handle64, void** local_ptr);
int b200rl_ipc_open(const void* handle64, void** ptr);
int b200rl_ipc_close(void* ptr);
int b200rl_onpolicy_comm_attach(b200rl_onpolicy* h, int32_t rank, int32_t world, void* const* peer_ptrs);

/* Per-launch scalar sums of the LAST update, as read back by it (host copy, no device work): out[slot][k], k as in
 * b200rl_mlp_loss_grad_args.scalar_partials, already summed over CTAs (and ranks).  PPO: slot i = forward pass of
 * policy step i (so slot i+1, k=1, divided by the row count is the approximate KL after step i, ppo.py:176-178; slot
 * K = the forward-only pass after the last step), slots K+1.. = value steps (k=0: sum of squared errors).
 * *n_slots = slots available; at most max_slots are copied. */
int b200rl_onpolicy_scalar_history(b200rl_onpolicy* h, double* out, int32_t max_slots, int32_t* n_slots);

/* Profiling hook (not on the product path): runs ONE named stage of the update on the loaded batch -- "values",
 * "preamble", "scan", "old_logp", "policy_grad", "policy_grad_kernel", "value_grad", "value_grad_kernel", "fvp",
 * "pack_obs", "fused_step_kernel", "fused_step" --
 * so that bench.py can time single kernels with CUDA events and ncu can capture them.  Asynchronous.
 * Note: the fp16 tensor-core kernels keep one status ring per PROCESS on the device that was current at their first
 * launch: one process drives one GPU (the torchrun / one-rank-per-GPU model of SURVEY 8e). */
int b200rl_onpolicy_run_stage(b200rl_onpolicy* h, const char* stage, const b200rl_ppo_hparams* hp, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Stand-alone helpers behind rl_replicas.utils' public functions, for callers that use them outside train()
 * (device pointers; float64 where the reference computes in float64).
 *   b200rl_discounted_cumsum: out[t] = x[t] + discount * out[t+1]            ref: utils.py:14-28 (scipy lfilter, f64)
 *   b200rl_gae_f64: delta[t] = rewards[t] + gamma*values[t+1] - values[t], t < n (rewards / values hold n+1 entries),
 *                   out = discounted_cumsum(delta, gamma*gae_lambda)          ref: utils.py:31-44
 *                   values: float64, or float32 (values_f32 = 1: gamma*values is then a float32 product, as numpy
 *                   evaluates it for the float32 arrays compute_values returns)
 *   b200rl_normalize: out = (x - mean(x)) / std(x), unbiased std, no epsilon  ref: utils.py:90-92
 *   b200rl_polyak: target = f32(rho)*target + f32(1-rho)*param                ref: utils.py:47-57
 * ------------------------------------------------------------------------------------------------------------ */
int b200rl_discounted_cumsum(const double* x, int64_t n, double discount, double* out, void* stream);
int b200rl_gae_f64(const double* rewards, const void* values, int values_f32, int64_t n, double gamma,
                   double gae_lambda, double* out, void* stream);
int b200rl_normalize(const float* x, int64_t n, float* out, void* stream);
int b200rl_polyak(float* target, const float* param, int64_t n, double rho, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Off-policy update engine (DDPG / TD3, and SAC below): the reference's `train(replay_buffer, num_train_steps,
 * minibatch_size)` (algorithms/td3.py:214-358, algorithms/ddpg.py:195-293) on device.  Networks: 0 policy, 1 Q1, 2 Q2,
 * 3 target policy, 4 target Q1, 5 target Q2 (2 and 5 absent when n_q = 1, 3 absent for SAC).  Minibatch sampling (numpy RNG) and the
 * target-smoothing noise (torch CPU RNG) stay on the host so the reference's random streams are reproduced; ALL
 * minibatches of one train() call are handed over at once.
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct b200rl_offpolicy b200rl_offpolicy;

typedef struct {
  b200rl_mlp_desc policy;  /* [obs, hidden..., act]      (ref: policies/deterministic_policy.py); SAC: [obs, ..., 2 act] */
  b200rl_mlp_desc q;       /* [obs + act, hidden..., 1]  (ref: q_function.py:20-32) */
  int32_t n_q;             /* 1 = DDPG, 2 = TD3 (algo 0); SAC needs 2, DQN 1 */
  int32_t max_minibatch;   /* capacity: rows per minibatch */
  int32_t max_steps;       /* capacity: train steps per call */
  int32_t algo;            /* 0 = DDPG / TD3 (by n_q), 1 = SAC (see b200rl_offpolicy_set_sac), 2 = DQN (see
                            * b200rl_offpolicy_set_dqn), 3 = C51 (see b200rl_offpolicy_set_c51) */
} b200rl_offpolicy_config;

typedef struct {
  double gamma, polyak_rho;
  double target_noise_scale, target_noise_clip, action_limit; /* td3.py:328-332 */
  int32_t policy_delay;      /* td3.py:244 (DDPG: 1) */
  int32_t use_target_noise;  /* 1 = TD3 target smoothing, 0 = DDPG */
  double policy_lr, policy_beta1, policy_beta2, policy_eps;
  double q1_lr, q2_lr, q_beta1, q_beta2, q_eps;
} b200rl_offpolicy_hparams;

int b200rl_offpolicy_create(const b200rl_offpolicy_config* cfg, b200rl_offpolicy** out);
void b200rl_offpolicy_destroy(b200rl_offpolicy* h);
int b200rl_offpolicy_set_params(b200rl_offpolicy* h, int which, const float* host_flat, int64_t n, void* stream);
int b200rl_offpolicy_get_params(b200rl_offpolicy* h, int which, float* host_flat, int64_t n, void* stream);
/* which: 0 policy, 1 Q1, 2 Q2 optimizers */
int b200rl_offpolicy_set_adam(b200rl_offpolicy* h, int which, const float* exp_avg, const float* exp_avg_sq, int64_t n,
                              int64_t step, void* stream);
int b200rl_offpolicy_get_adam(b200rl_offpolicy* h, int which, float* exp_avg, float* exp_avg_sq, int64_t n,
                              int64_t* step, void* stream);
/* The whole learner state in one call, one copy and one synchronisation (what TD3.train / DDPG.train move per call):
 * blob = the parameters of every present network 0..5 in order, then exp_avg and exp_avg_sq of optimizers 0..2, EVERY
 * SEGMENT PADDED to a multiple of 64 floats (the padding carries no meaning); steps[3] =
 * the Adam step counts.  b200rl_offpolicy_state_floats = length of the blob.  Page-locked blobs copy by DMA. */
int64_t b200rl_offpolicy_state_floats(b200rl_offpolicy* h);
int b200rl_offpolicy_get_state(b200rl_offpolicy* h, float* blob, int64_t n_floats, int64_t* steps, void* stream);
int b200rl_offpolicy_set_state(b200rl_offpolicy* h, const float* blob, int64_t n_floats, const int64_t* steps,
                               void* stream);

/* HOST buffers: obs/next_obs [S,B,O], act [S,B,A], rew/done [S,B] float32 (done as 0/1), noise [S,B,A] raw N(0,1)
 * draws (NULL for DDPG).  Outputs (host): q1_values/q2_values [S,B] (the logged pre-update Q-values), q1_losses /
 * q2_losses [S], policy_losses [*n_policy_updates].  One upload, S steps without host synchronisation, one read-back. */
int b200rl_offpolicy_train(b200rl_offpolicy* h, const b200rl_offpolicy_hparams* hp, int32_t S, int32_t B,
                           const float* obs, const float* act, const float* rew, const float* next_obs,
                           const float* done, const float* noise, float* q1_values, float* q2_values, float* q1_losses,
                           float* q2_losses, float* policy_losses, int32_t* n_policy_updates, void* stream);

/* Same, with the minibatches gathered ON THE DEVICE from replay-buffer columns that already live in HBM
 * (d_obs / d_next_obs [rows,O], d_act [rows,A], d_rew / d_done [rows] float32): only the indices idx [S,B] (host,
 * int64, physical rows drawn by the host RNG exactly as replay_buffer.py:58 does) and the noise cross PCIe.
 *   replaces: replay_buffer.py:51-74 (sample_minibatch gather) + td3.py:222-228 (tensor conversion). */
int b200rl_offpolicy_train_gather(b200rl_offpolicy* h, const b200rl_offpolicy_hparams* hp, int32_t S, int32_t B,
                                  const float* d_obs, const float* d_act, const float* d_rew, const float* d_next_obs,
                                  const float* d_done, int64_t rows, const int64_t* idx, const float* noise,
                                  float* q1_values, float* q2_values, float* q1_losses, float* q2_losses,
                                  float* policy_losses, int32_t* n_policy_updates, void* stream);

/* Opt-in (SURVEY 8f-4): the same with the minibatch indices and the target-smoothing noise DRAWN ON THE DEVICE
 * (Philox4x32-10 keyed by `seed`, block `call`): nothing but the hyper-parameters crosses PCIe on the way in.  The
 * streams are not the reference's (numpy MT19937 / torch CPU generator): same distributions, different numbers.  The
 * replay ring: `ring_size` live rows, logical row u at physical (ring_start + u) % rows.
 *   replaces: replay_buffer.py:58 (np.random.randint) + td3.py:328 (torch.randn_like) for callers that opt in. */
int b200rl_offpolicy_train_gather_rng(b200rl_offpolicy* h, const b200rl_offpolicy_hparams* hp, int32_t S, int32_t B,
                                      const float* d_obs, const float* d_act, const float* d_rew,
                                      const float* d_next_obs, const float* d_done, int64_t rows, int64_t ring_start,
                                      int64_t ring_size, uint64_t seed, uint64_t call, float* q1_values,
                                      float* q2_values, float* q1_losses, float* q2_losses, float* policy_losses,
                                      int32_t* n_policy_updates, void* stream);
/* The draws of the last train_gather / train_gather_rng call: physical rows idx [S*B] (host int64), noise [S*B*A]
 * (host float32, or NULL) -- what a test replays through the oracle. */
int b200rl_offpolicy_get_draws(b200rl_offpolicy* h, int32_t S, int32_t B, int64_t* idx, float* noise, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Soft Actor-Critic on the same engine (config algo = 1, n_q = 2; Spinning Up sac/core.py, sac/sac.py).  The policy
 * network maps obs -> [mean | log_std] (2A outputs, Identity output layer); network 3 (target policy) is absent, so the
 * state blob holds networks 0, 1, 2, 4, 5.  Per train step, with draws eps' (for s') and eps (for s) and alpha:
 *   head(o, e): log_std = clamp(log_std, log_std_min, log_std_max), u = mean + exp(log_std) e, a = limit tanh(u),
 *               log pi = sum_j Normal(mean, std).log_prob(u) - sum_j 2 (log 2 - u - softplus(-2u))
 *               (limit = hparams.action_limit; the constant -A log(limit) is omitted, as in Spinning Up)
 *   critics:    y = r + gamma (1 - d) (min(Q1targ, Q2targ)(s', a') - alpha log pi'), a', log pi' = head(pi(s'), eps');
 *               one Adam step each on mean((Qi(s, a) - y)^2)
 *   policy:     one Adam step on mean(alpha log pi - min(Q1, Q2)(s, a_pi)), a_pi, log pi = head(pi(s), eps), with the
 *               critics just updated (torch.min's tie rule: equal values share the gradient)
 *   alpha:      learn_alpha = 1: one Adam step on -mean(log_alpha (log pi + target_entropy)), alpha = exp(log_alpha)
 *               from the next step on; learn_alpha = 0: alpha is the fixed value
 *   polyak:     Q1targ, Q2targ every step.  hparams.policy_delay / use_target_noise / target_noise_* do not apply.
 * train / train_gather take noise [S, 2, B, A] (per step the draw for s', then the one for s), required; train_gather_rng
 * draws it on the device and get_draws returns it in the same layout.  policy_losses has S entries.  SAC runs as a
 * CUDA graph, or as plain launches with B200RL_OFFPOLICY_GRAPH=0.
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct {
  double alpha;                 /* the fixed entropy coefficient (learn_alpha = 0) */
  double target_entropy;        /* H-bar, usually -A */
  double alpha_lr, alpha_beta1, alpha_beta2, alpha_eps; /* torch.optim.Adam over log_alpha */
  double log_std_min, log_std_max;                      /* -20, 2 */
  int32_t learn_alpha;          /* 0 or 1 */
  int32_t reserved;
} b200rl_sac_hparams;

/* Required once before the first train call of a SAC engine; part of the cached graph's key. */
int b200rl_offpolicy_set_sac(b200rl_offpolicy* h, const b200rl_sac_hparams* hp);
/* The temperature's state: float32 log_alpha, its Adam exp_avg / exp_avg_sq and step count. */
int b200rl_offpolicy_set_alpha(b200rl_offpolicy* h, float log_alpha, float exp_avg, float exp_avg_sq, int64_t step);
int b200rl_offpolicy_get_alpha(b200rl_offpolicy* h, float* log_alpha, float* exp_avg, float* exp_avg_sq, int64_t* step);
/* After a train call of S steps: mean log pi of each policy step and the alpha each step used (host [S] each). */
int b200rl_offpolicy_sac_outputs(b200rl_offpolicy* h, int32_t S, float* log_prob_means, float* alphas);

/* ------------------------------------------------------------------------------------------------------------
 * DQN on the same engine (config algo = 2, n_q = 1; Mnih et al. 2015, Double DQN: van Hasselt et al. 2016).  The
 * policy description must be zeroed; q = [obs, hidden..., n_actions] maps obs -> one value per action (n_actions >= 1).
 * Networks 1 (Q) and 4 (target Q) are present, so the state blob holds their parameters followed by optimizer 1's
 * exp_avg / exp_avg_sq; steps[3] keeps its layout (steps[1] is the Q optimizer's count, the others 0).  The action
 * column is one float32 per row holding the action index (act [S,B] for train, d_act [rows] for the gather paths).
 * Per train step, with t = the Q optimizer's step count after the step:
 *   v = Q_targ(s')[argmax_j Q(s')_j] (double_q = 1; Q at the start of the step) or max_j Q_targ(s')_j
 *       (torch's max / argmax: a NaN wins, ties go to the first index)
 *   y = r + gamma (1 - d) v;  one Adam step (optimizer 1) on F.smooth_l1_loss(Q(s)[a], y) (beta = 1, mean over B)
 *   target Q <- Q (exact copy) when t % target_update_interval == 0: the schedule follows each learner's own count,
 *       across calls and across get_state / set_state
 * hparams: only gamma and the q1_lr / q_beta1 / q_beta2 / q_eps Adam fields apply; every other field is ignored.
 * Outputs: q1_values [S,B] (Q(s)[a] before the update) and q1_losses [S]; *n_policy_updates = 0, and q2_values,
 * q2_losses and policy_losses may be NULL.  No noise is used: train / train_gather take noise = NULL, train_gather_rng
 * draws indices only.  A row whose action is not an integer in [0, n_actions) is never used as an index and adds nothing
 * to the update; the call then returns an error naming the learner and the step (the update has still run).  DQN
 * runs as a CUDA graph, or as plain launches with B200RL_OFFPOLICY_GRAPH=0, and in learner groups like the others.
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct {
  int32_t target_update_interval; /* >= 1: copy Q to the target every this many Q optimizer steps */
  int32_t double_q;               /* 0 = DQN target, 1 = Double DQN target */
} b200rl_dqn_hparams;

/* Required once before the first train call of a DQN engine; part of the cached graph's key. */
int b200rl_offpolicy_set_dqn(b200rl_offpolicy* h, const b200rl_dqn_hparams* hp);

/* ------------------------------------------------------------------------------------------------------------
 * C51 on the same engine (config algo = 3, n_q = 1; Bellemare, Dabney & Munos 2017): a DQN engine whose Q network maps
 * obs -> [n_actions x n_atoms] logits, row-major (action a owns columns a N .. a N + N - 1).  Everything the DQN
 * section says holds (networks, state blob, action column, hparams, target copies, outputs, invalid actions, graph,
 * groups; b200rl_offpolicy_set_dqn is required too) except the loss.  With N = n_atoms:
 *   support  dz = (v_max - v_min) / (N - 1), z_i = float32(v_min + i dz), both evaluated in double
 *   p(s, a)  = exp(log_softmax) of action a's N logits, x - max - log(sum exp(x - max)) in float32; every sum over
 *            atoms runs in index order; Q(s, a) = sum_i z_i p_i(s, a)
 *   a*       = argmax_a Q(s', a) with the expected values of Q (double_q = 1; at the start of the step) or of Q_targ
 *            (torch's argmax: a NaN wins, ties go to the first index)
 *   target   Tz_j = clamp(r + gamma (1 - d) z_j, v_min, v_max), b_j = (Tz_j - v_min) / dz,
 *            m_i = sum_j max(0, 1 - |b_j - i|) p_j(s', a*) from Q_targ (summed over j in index order)
 *   loss     one Adam step (optimizer 1) on mean_B(-sum_i m_i log p_i(s, a)); the gradient w.r.t. the action's logits is
 *            (p_i(s, a) sum_k m_k - m_i) / B, every other logit's 0
 * Outputs: q1_values [S,B] = Q(s, a) before the update, q1_losses [S] = the mean cross-entropy (summed in double).
 * The head is deterministic (no float atomics): a group's learners stay bit-identical to solo engines.  Prioritized
 * replay is not implemented for C51: b200rl_offpolicy_set_per and the train_prioritized calls refuse a C51 engine.
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct {
  int32_t n_atoms;  /* N, 2..256; the Q network's output width must be a multiple of N */
  int32_t reserved; /* ignored */
  double v_min, v_max; /* finite, v_min < v_max */
} b200rl_c51_hparams;

/* Required once before the first train call of a C51 engine and refused on other engines; writes the support into
 * every learner's arena; part of the cached graph's key. */
int b200rl_offpolicy_set_c51(b200rl_offpolicy* h, const b200rl_c51_hparams* hp);

/* ------------------------------------------------------------------------------------------------------------
 * QR-DQN on the same engine (Dabney, Rowland, Bellemare & Munos 2018): a DQN engine (config algo = 2) after
 * b200rl_offpolicy_set_qr, whose Q network maps obs -> [n_actions x n_quantiles] quantile locations, row-major (action a
 * owns columns a N .. a N + N - 1; theta_i(s, a) is the i-th).  Everything the DQN section says holds (networks, state
 * blob, action column, hparams, target copies, outputs, invalid actions, graph, groups, prioritized replay, n-step
 * returns; b200rl_offpolicy_set_dqn is required too) except the loss.  With N = n_quantiles, in float32:
 *   tau_i    = (float)(2i + 1) / (float)(2N)
 *   Q(s, a)  = (sum_i theta_i(s, a)) / N, summed over i in index order; q1_values logs it
 *   a*       = argmax_a Q(s', a) with the means of Q (double_q = 1; at the start of the step) or of Q_targ
 *            (torch's argmax: a NaN wins, ties go to the first index)
 *   target   T_j = r + (g (1 - d)) theta_j(s', a*) from Q_targ, g = gamma (n-step: the row's discount)
 *   loss     u_ij = T_j - theta_i(s, a), rho_i(u) = |tau_i - 1{u < 0}| h(u), h(u) = 0.5 u^2 if |u| < 1 else |u| - 0.5
 *            (kappa = 1); the row's L = (1/N) sum_i sum_j rho_i(u_ij), over j in index order, then over i in index
 *            order; one Adam step (optimizer 1) on (1/B) sum_b L_b, summed in double in a fixed order
 *   gradient w.r.t. the action's quantile i: -(sum_j |tau_i - 1{u_ij < 0}| clamp(u_ij, -1, 1)) / N times (1/B); every
 *            other output's 0
 * Prioritized replay: the loss is (1/B) sum_b w_b L_b and the gradient row b is scaled by w_b (with every w_b = 1 bit
 * for bit the unweighted step); the priority of row b is (L_b + eps)^alpha with its unweighted L_b from before the
 * Adam step, which takes the place of |delta| in the prioritized replay section (non-finite: counted, and the call
 * fails).  The head is deterministic (no float atomics): a group's learners stay bit-identical to solo engines.
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct {
  int32_t n_quantiles; /* N, 1..256; the Q network's output width must be a multiple of N */
  int32_t reserved;    /* ignored */
} b200rl_qr_hparams;

/* Makes the engine's loss head QR-DQN's for every later train call; refused on engines not created with algo = 2
 * (TD3 / DDPG, SAC, C51); part of the cached graph's key. */
int b200rl_offpolicy_set_qr(b200rl_offpolicy* h, const b200rl_qr_hparams* hp);

/* ------------------------------------------------------------------------------------------------------------
 * Learner groups: K independent off-policy learners (same config, same hyper-parameters, their own parameters, Adam
 * states, step counts, minibatches, noise, replay buffers and temperature) trained by one engine, every operation of a
 * step ONE launch for all K.  Each learner's arithmetic -- tile shapes, summation order, Adam's operation order -- is
 * that of a solo engine, so learner z of a group produces bit for bit what a solo engine fed learner z's inputs does.
 * Everything the engine owns for one learner lives in one arena; the K arenas lie at a fixed stride (a multiple of
 * 256 bytes), and a kernel finds learner z's buffers at + z * stride.
 *
 * b200rl_offpolicy_create is the group of one.  For K > 1 the calls above take and return a leading [K] axis, which
 * for K = 1 is exactly the solo layout: state_floats = K x the per-learner blob, get_state / set_state move
 * [K][blob] with steps[K][3]; train takes [K, S, B, ...] minibatches and [K, S, B, A] noise (SAC [K, S, 2, B, A]) and
 * returns values [K, S, B], losses [K, S] and policy_losses [K, S] (the first *n_policy_updates of each row; the
 * policy-delay schedule is shared); get_draws and sac_outputs likewise.  train_gather, train_gather_rng, set_alpha and
 * get_alpha are the group calls below with K = 1 and refuse K > 1; the per-network accessors (set_params, get_params,
 * set_adam, get_adam) refuse K > 1: a group's state moves as the blob.  A group runs as a CUDA graph, or as plain
 * launches with B200RL_OFFPOLICY_GRAPH=0.
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct {
  const float *obs, *act, *rew, *next_obs, *done; /* device replay columns, as for b200rl_offpolicy_train_gather */
  int64_t rows;
} b200rl_offpolicy_replay;

/* 1 <= n_learners <= B200RL_MAX_LEARNERS */
int b200rl_offpolicy_create_group(const b200rl_offpolicy_config* cfg, int32_t n_learners, b200rl_offpolicy** out);
/* replay[K]: each learner's own columns and row count; idx [K, S, B] physical rows of each learner's buffer */
int b200rl_offpolicy_train_gather_group(b200rl_offpolicy* h, const b200rl_offpolicy_hparams* hp, int32_t S, int32_t B,
                                        const b200rl_offpolicy_replay* replay, const int64_t* idx, const float* noise,
                                        float* q1_values, float* q2_values, float* q1_losses, float* q2_losses,
                                        float* policy_losses, int32_t* n_policy_updates, void* stream);
/* ring_start / ring_size / seed / call [K]: learner z's draws equal those of a solo engine with seed[z], call[z] */
int b200rl_offpolicy_train_gather_rng_group(b200rl_offpolicy* h, const b200rl_offpolicy_hparams* hp, int32_t S,
                                            int32_t B, const b200rl_offpolicy_replay* replay, const int64_t* ring_start,
                                            const int64_t* ring_size, const uint64_t* seed, const uint64_t* call,
                                            float* q1_values, float* q2_values, float* q1_losses, float* q2_losses,
                                            float* policy_losses, int32_t* n_policy_updates, void* stream);
/* [K] entries each */
int b200rl_offpolicy_set_alpha_group(b200rl_offpolicy* h, const float* log_alpha, const float* exp_avg,
                                     const float* exp_avg_sq, const int64_t* step);
int b200rl_offpolicy_get_alpha_group(b200rl_offpolicy* h, float* log_alpha, float* exp_avg, float* exp_avg_sq,
                                     int64_t* step);

/* ------------------------------------------------------------------------------------------------------------
 * Prioritized experience replay for DQN (Schaul et al. 2016, proportional).  Each learner's replay buffer has one
 * priority per physical row, held on the device in a sum tree (layout below); rows that are not live have priority 0.
 * Step st of a prioritized call, for each learner:
 *   draw:    M = the sum of the priorities; for j in 0..B-1, u_j = (j + U_j) * (M / B) with U_j = the top 24 bits of
 *            Philox4x32-10(counter (j, st, call, 0x9E5), key seed) times 2^-24 (a stream of its own, apart from the
 *            index and noise draws of train_gather_rng); idx_j = the leaf whose cumulative interval holds u_j.  A leaf
 *            of priority 0 is never drawn, even when rounding puts u_j at or past the last boundary.
 *   weights: w_j = (min_k p[idx_k] / p[idx_j])^beta (Schaul's (N P(j))^-beta over its largest value in the minibatch),
 *            beta = min(1, beta_start + (1 - beta_start) t / beta_anneal_steps), t = the Q optimizer's step count
 *            before the step (so the schedule carries across calls and get_state / set_state).
 *   update:  the DQN / Double DQN step with loss (1/B) sum_j w_j huber(delta_j) and output gradient
 *            w_j clamp(delta_j, -1, 1) / B (q1_losses logs this weighted loss); with every w_j = 1 it is bit for bit the
 *            unweighted step.
 *   priorities: for each row j in order (a leaf drawn twice keeps its last row's value), leaf idx_j <- (|delta_j| +
 *            eps)^alpha with delta_j from before the Adam step, and the running max m <- max(m, that value).  A row
 *            with an invalid action keeps its leaf as it was; a non-finite |delta_j| or priority leaves its leaf
 *            unchanged and is counted: the call then returns an error naming the learner and the step.  Interior
 *            nodes never hold a NaN.
 *   Step st + 1 draws from the tree step st left.
 * The draw, the weights and the gather of the five columns are one kernel, the priority update a second one beside the
 * backward pass: two launches per step more than train_gather_rng's steps, and no per-call draw or gather launches.
 *
 * Tree layout (float32, b200rl_per_tree_floats(leaves) floats): level 0 = the leaves (one per physical row), level
 * k + 1 = the sums of 32 consecutive nodes of level k, added in index order; every level padded with zeros to a
 * multiple of 32 floats, levels back to back; the last level is [root, running max m, 0 ...].  The buffer owns the
 * tree (zeroed, m = 1 at creation) and keeps it: b200rl_per_tree_set_range gives rows an append wrote priority m,
 * b200rl_per_tree_build recomputes every interior node from the leaves.  Interior nodes are always recomputed from
 * their children, never adjusted by differences: no drift, and groups stay bit-identical to solo engines.
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct {
  double alpha;              /* >= 0: priority = (|delta| + eps)^alpha */
  double eps;                /* > 0 */
  double beta_start;         /* in [0, 1] */
  int64_t beta_anneal_steps; /* >= 1 */
} b200rl_per_hparams;

/* Required before a prioritized call of a DQN engine (other engines are refused); part of the cached graph's key. */
int b200rl_offpolicy_set_per(b200rl_offpolicy* h, const b200rl_per_hparams* pp);
/* S prioritized DQN steps on device replay columns (as for train_gather) with `rows` physical rows and their tree
 * (rows leaves, device memory).  (seed, call) key the draws.  Outputs as for DQN: q1_values [S,B], q1_losses [S]. */
int b200rl_offpolicy_train_prioritized(b200rl_offpolicy* h, const b200rl_offpolicy_hparams* hp, int32_t S, int32_t B,
                                       const float* d_obs, const float* d_act, const float* d_rew,
                                       const float* d_next_obs, const float* d_done, int64_t rows, float* tree,
                                       uint64_t seed, uint64_t call, float* q1_values, float* q1_losses, void* stream);
/* The same for a learner group: replay[K], trees[K] (K distinct trees: learners never share one), seed[K], call[K];
 * outputs [K, S, B] and [K, S] */
int b200rl_offpolicy_train_prioritized_group(b200rl_offpolicy* h, const b200rl_offpolicy_hparams* hp, int32_t S,
                                             int32_t B, const b200rl_offpolicy_replay* replay, float* const* trees,
                                             const uint64_t* seed, const uint64_t* call, float* q1_values,
                                             float* q1_losses, void* stream);
/* Of the last prioritized call (host [K, S, B] each): the drawn rows, their weights and the new priorities they wrote
 * (NaN for a row that wrote none) -- what a test replays through the oracle.  Refused when the engine's last train
 * call that ran steps was not a prioritized one (it overwrote the drawn rows). */
int b200rl_offpolicy_get_per_draws(b200rl_offpolicy* h, int32_t S, int32_t B, int64_t* idx, float* weights,
                                   float* priorities, void* stream);
/* ------------------------------------------------------------------------------------------------------------
 * n-step returns for DQN and C51 (Rainbow's multi-step targets).  Each learner's replay buffer keeps, beside its five
 * columns, a float32 0/1 episode-end column over the same physical rows: row i is 1 when it was the last row of an
 * episode (a cut-off at the end of a sampling call counts) in the append that wrote it.  Every append ends on a marked
 * row, so the newest live row is always marked and a window never reads past the ring's head or into a row a ring
 * overwrite replaced.  For a drawn start row p0, with gamma = float32(hp.gamma), in float32 with every product and sum
 * rounded on its own (no contraction):
 *   p = p0;  R = rew[p];  g = gamma
 *   for k = 1 .. n-1:  if done[p] != 0 or ends[p] != 0: break
 *                      p = (p + 1) % rows  (the window may cross the wrap);  R = R + g rew[p];  g = g gamma
 *   the staged row: obs[p0], act[p0], rew := R, next_obs := next_obs[p], done := done[p], discount := g
 * The loss heads use discount where the one-step target uses gamma: DQN y = R + discount (1 - d) v (td_target's order),
 * C51 Tz_j = clamp(R + discount (1 - d) z_j, v_min, v_max); a prioritized step's priority is that of the n-step delta.
 * Double DQN takes its argmax at next_obs[p].  A window never reaches across an episode end: such a row bootstraps
 * from its own next_obs with a shorter horizon.  n = 1 is exactly the one-step update, on the one-step kernels.
 * On the gather paths one kernel walks the windows and stages all columns (in place of the five column gathers); on
 * the prioritized path the draw kernel does.  The host-staged b200rl_offpolicy_train refuses n > 1.
 * ------------------------------------------------------------------------------------------------------------ */
/* n_step 1..32 for the engine's next train calls (1 clears it); episode_ends[K] = each learner's device episode-end
 * column over the `rows` of the replay passed to the next call (required for n_step > 1; buffers that grow reallocate,
 * so set it before every call).  Refused on TD3, DDPG and SAC engines.  n_step is part of the cached graph's key, and so
 * are the columns on the prioritized path (its draw walks them inside the graph). */
int b200rl_offpolicy_set_nstep(b200rl_offpolicy* h, int32_t n_step, const float* const* episode_ends);
/* Of the last n-step call (host [K, S, B] each): each row's last window row, its return R and its discount g -- what a
 * test replays through the oracle.  Refused when the engine's last train call that ran steps was not an n-step one. */
int b200rl_offpolicy_get_nstep_draws(b200rl_offpolicy* h, int32_t S, int32_t B, int64_t* last_rows, float* returns,
                                     float* discounts, void* stream);

/* Floats of a tree over `leaves` rows (1 <= leaves < 2^31; -1 otherwise). */
int64_t b200rl_per_tree_floats(int64_t leaves);
/* Every interior node recomputed from the leaves (stream-ordered). */
int b200rl_per_tree_build(float* tree, int64_t leaves, void* stream);
/* Leaves start .. start + count - 1 (modulo leaves: the range may wrap) <- the running max m, ancestors recomputed. */
int b200rl_per_tree_set_range(float* tree, int64_t leaves, int64_t start, int64_t count, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200RL_H */
