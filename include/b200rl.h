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
  int32_t n_q;             /* 1 = DDPG, 2 = TD3 (algo 0); SAC and discrete SAC need 2, DQN 1 */
  int32_t max_minibatch;   /* capacity: rows per minibatch */
  int32_t max_steps;       /* capacity: train steps per call */
  int32_t algo;            /* 0 = DDPG / TD3 (by n_q), 1 = SAC (see b200rl_offpolicy_set_sac), 2 = DQN (see
                            * b200rl_offpolicy_set_dqn), 3 = C51 (see b200rl_offpolicy_set_c51), 4 = IQN (created by
                            * b200rl_offpolicy_create_iqn only; see "IQN" below), 5 = discrete SAC (see
                            * "Discrete SAC" below), 6 = D4PG (created by b200rl_offpolicy_create_d4pg only; see
                            * "D4PG" below), 7 = TQC (created by b200rl_offpolicy_create_tqc only; see "TQC" below),
                            * 8 = CQL (created by b200rl_offpolicy_create_cql only; see "CQL" below), 9 = IQL
                            * (created by b200rl_offpolicy_create_iql only; see "IQL" below), 10 = REDQ (created
                            * by b200rl_offpolicy_create_redq only; see "REDQ" below), 11 = EDAC (created by
                            * b200rl_offpolicy_create_edac only; see "EDAC" below) */
  int32_t dueling_k;       /* 0 = the Q network is a plain MLP; K >= 1 = a dueling Q network (algo 2 / 3 only; see
                            * "Dueling Q networks" below) */
  int32_t noisy_layers;    /* bit mask over the Q network's Linear layers in flat order: 0 = none; bit l = layer l is a
                            * noisy layer (algo 2 / 3 only; see "Noisy networks" below) */
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
/* which: 0 policy, 1 Q1, 2 Q2 optimizers (and 3 V on an IQL engine; 1..N the critics on a REDQ engine) */
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
 * Discrete SAC on the same engine (config algo = 5, n_q = 2; Christodoulou 2019, "Soft Actor-Critic for Discrete
 * Action Settings").  policy = [obs, hidden..., n] maps obs -> n logits (Identity output layer); q = [obs, hidden...,
 * n] maps obs -> one value per action for both critics and their targets (n >= 2, both widths equal).  Networks 0, 1,
 * 2, 4, 5 are present (no target policy), so the state blob, steps[3], set_alpha / get_alpha and sac_outputs keep
 * SAC's layout.  The action column is one float32 per row holding the action index (act [S,B] for train, d_act [rows]
 * for the gather paths), as for DQN.  Per train step on (s, a, r, s', d), with alpha = alpha[st] (the temperature at
 * the start of the step), in float32:
 *   log pi     log pi_j = (x_j - max x) - log(sum_k exp(x_k - max x)) of the logits x, every sum over actions in index
 *              order; pi_j = exp(log pi_j) (the log-softmax form: a vanishing probability gives pi log pi = 0)
 *   critics    V(s') = sum_j pi'_j (min(Q1targ, Q2targ)(s')_j - alpha log pi'_j), pi' the policy at s' at the start of
 *              the step; y = r + gamma (1 - d) V(s'); one Adam step each (optimizers 1, 2) on mean_B (Qk(s)[a] - y)^2,
 *              whose gradient w.r.t. critic k's outputs is 2 (Qk(s)[a] - y) / B in column a and 0 elsewhere
 *   policy     with the critics just updated (no gradient into them), m_j = min(Q1, Q2)(s)_j, c_j = alpha log pi_j - m_j:
 *              one Adam step (optimizer 0) on mean_B L, L = sum_j pi_j c_j; the logit gradient is
 *              pi_k (c_k - L) / B (the alpha term of d log pi cancels: sum_j pi_j = 1); pi is the policy at the start
 *              of the step
 *   alpha      learn_alpha = 1: one Adam step on -mean_B(log_alpha (E + target_entropy)), E = sum_j pi_j log pi_j from
 *              the policy step's pi(s); alpha = exp(log_alpha) from the next step on (target_entropy: 0.98 log n is
 *              the paper's choice); learn_alpha = 0: alpha is the fixed value
 *   polyak     Q1targ, Q2targ every step
 * b200rl_offpolicy_set_sac is required once before the first train call; its log_std_min / log_std_max are ignored.
 * hparams: gamma, polyak_rho and the Adam fields apply; policy_delay, use_target_noise, target_noise_* and
 * action_limit are ignored.  No noise is used: train / train_gather take noise = NULL, train_gather_rng draws indices
 * only, get_draws returns no noise.  Outputs: q1_values / q2_values [S,B] = Qk(s)[a] before the update, q1_losses /
 * q2_losses [S], policy_losses [S] (mean L, *n_policy_updates = S); sac_outputs gives mean E per step (in place of SAC's
 * mean log pi) and the alpha each step used.  A row whose action is not an integer in [0, n) is never used as an index,
 * adds nothing to either critic's loss or gradient and logs NaN; the call then returns an error naming the learner and
 * the step (the update has still run).  The heads reduce in a fixed order with no float atomics: a group's learners stay
 * bit-identical to solo engines.  Runs as a CUDA graph, or as plain launches with B200RL_OFFPOLICY_GRAPH=0.
 * Launches, with Lq and Lp the critics' and the policy's Linear layers: 1 per call (the temperature table), then per
 * step 10 Lq + 4 Lp + 4, one more with learn_alpha = 1 (forward passes: Q1, Q2 and pi at s, pi, Q1targ, Q2targ at s',
 * the updated Q1, Q2 at s; 2 critic heads; backward passes of 2 L - 1 launches, weight gradients and the dX chain
 * down to the first hidden layer, for both critics and the policy; 3 Adam steps; polyak; the policy head; the
 * temperature step): 46 per step at two hidden layers, 47 with a learned temperature.
 * Not implemented, and refused: dueling_k or noisy_layers != 0 at create; set_dqn, set_c51, set_qr, set_per, set_nstep,
 * set_noise_keys and the train_prioritized calls (prioritized replay, n-step returns, noisy, dueling and IQN networks).
 * ------------------------------------------------------------------------------------------------------------ */

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
 * Dueling Q networks (Wang et al. 2016) for DQN, QR-DQN and C51: config dueling_k = K >= 1 on an algo 2 or 3 engine.
 * The q description [obs, h1, h2, n K] (3 layers, hidden_act between layers, out_act identity) then describes
 *   trunk      h   = act(x W1^T + b1)                                    W1 [h1, obs]
 *   value      V   = act(h Wv^T + bv) Vo^T + vo                          Wv [h2, h1], Vo [K, h2]
 *   advantage  A   = act(h Wa^T + ba) Ao^T + ao                          Wa [h2, h1], Ao [n K, h2]
 *   output     Q[a, i] = V[i] + (A[a, i] - mean_i),  mean_i = (sum_b A[b, i]) / n        (action a owns columns
 *              a K .. a K + K - 1 of A and Q, the layout of a plain Q network's output)
 * in float32, the sum over actions b in index order and then one division by n; V[i] + (A[a, i] - mean_i) in that
 * order.  The flat parameter vector of networks 1 and 4 (set_params, get_params, the state blob, Adam) is W1, b1, Wv,
 * bv, Vo, vo, Wa, ba, Ao, ao: torch's parameters_to_vector of a module registering trunk, value and advantage in this
 * order; its length is P = h1 (obs + 1) + 2 h2 (h1 + 1) + K (h2 + 1) + n K (h2 + 1).  Q feeds the engine's loss head
 * unchanged: K = 1 for DQN, K = n_quantiles for QR-DQN (the quantile locations), K = n_atoms for C51 (the logits,
 * aggregated before the softmax).  Backward: dV[i] = sum_a dQ[a, i] and dA[a, i] = dQ[a, i] - (sum_b dQ[b, i]) / n,
 * both sums in index order; the trunk's input gradient dZv Wv + dZa Wa is one product whose k-sum runs over the value
 * stream's units, then the advantage stream's.  Every sum has a fixed order: results are deterministic and a group's
 * learners stay bit-identical to solo engines.  Prioritized replay, n-step returns, Double DQN, groups, the graph and
 * plain launches work as for a plain Q network.  Launches: a forward pass of a network takes 6 (5 GEMMs and the
 * aggregation) and the backward pass 9 (the aggregation's backward and 8 GEMMs), against 3 and 5 for a plain 3-layer
 * network; with the loss head, Adam and the target copy a step of DQN, QR-DQN or C51 takes 24 launches (30 with
 * double_q) where a plain 3-layer network's takes 14 (17), and a prioritized step adds its draw and priority update
 * (2) to either.
 * Refused at create: dueling_k < 0; dueling_k != 0 with algo 0 or 1; a q description that is not 3 layers, whose
 * output width is not a multiple of dueling_k, or whose out_act is not identity.
 * ------------------------------------------------------------------------------------------------------------ */

/* ------------------------------------------------------------------------------------------------------------
 * Noisy networks (Fortunato et al. 2018, factorized Gaussian noise) for DQN, QR-DQN and C51, plain or dueling: config
 * noisy_layers = a bit mask over the Q network's Linear layers in flat order (an MLP's layers 0 .. n_layers - 1; a
 * dueling network's trunk, value hidden, value out, advantage hidden, advantage out).  A noisy layer with `in` inputs
 * and `out` outputs has W_mu, W_sigma [out, in] and b_mu, b_sigma [out]; for one draw of eps_in [in] and eps_out [out],
 * each N(0, 1), in float32 with every product and sum rounded on its own (no contraction) and IEEE sqrt:
 *   f(x) = copysign(sqrt(|x|), x),  e_ij = f(eps_out_i) f(eps_in_j)
 *   W_ij = W_mu_ij + W_sigma_ij e_ij,  b_i = b_mu_i + b_sigma_i f(eps_out_i)
 * The flat parameter vector of networks 1 and 4 (set_params, get_params, the state blob, Adam, the target copy) holds
 * W_mu, W_sigma, b_mu, b_sigma for a noisy layer and W, b for a plain one, layer by layer: torch's parameters_to_vector
 * of a module whose noisy layers register weight_mu, weight_sigma, bias_mu, bias_sigma in this order.
 * Per train step and learner the online network draws one sample, which Q(s) and Double DQN's Q(s') share, and the
 * target network an independent one; the loss head runs unchanged on the composed layers, the backward pass gives
 * their dW and db, and dW_mu = dW, dW_sigma = dW e, db_mu = db, db_sigma = db f(eps_out) (e as the forward pass
 * rounded it); Adam updates mu and sigma, and the target copy copies both.  q1_values logs Q(s)[a] under the step's
 * online sample.
 * Draws: the network's E = sum(in + out) over its noisy layers values are eps_in, eps_out of each noisy layer in layer
 * order; values 4t .. 4t + 3 are the Box-Muller transform (as for train_gather_rng's noise) of Philox4x32-10(counter
 * (t, st, call, 0xA00 | r), key seed), st = the step of the call, r = 0 for the online network and 1 for the target
 * one.  (seed, call) come from b200rl_offpolicy_set_noise_keys, which every train call of such an engine needs afresh
 * (train, train_gather, train_gather_rng, train_prioritized and their group forms; a call without them is refused);
 * the keys live in device memory, so a cached graph is replayed across calls.
 * Launches: one kernel draws and composes both networks at the start of a step, one maps dW, db to the noisy gradient
 * before Adam: 2 per step more than the same network without noise (16 for a plain 3-layer DQN, QR-DQN or C51 step, 26
 * for a dueling one; 19 and 32 with double_q; a prioritized step adds its 2).  Every sum has a fixed order and no
 * float atomics are used: a group's learners stay bit-identical to solo engines.  Prioritized replay, n-step returns,
 * Double DQN, dueling networks, groups, the graph and plain launches work as without noise; C51 with prioritized
 * replay stays refused.
 * Refused at create: noisy_layers != 0 with algo 0 or 1 (n_q is 1 for every engine that takes it); bits at or beyond
 * the layer count.
 * ------------------------------------------------------------------------------------------------------------ */
/* seed[K], call[K]: the noise keys of the next train call, learner z's taken by its draws. */
int b200rl_offpolicy_set_noise_keys(b200rl_offpolicy* h, const uint64_t* seed, const uint64_t* call);
/* The raw N(0, 1) draws of the last train call's S steps: host eps [K, S, 2, E] (per step the online network's, then
 * the target's) -- what a test replays through the oracle. */
int b200rl_offpolicy_get_noisy_draws(b200rl_offpolicy* h, int32_t S, float* eps);

/* ------------------------------------------------------------------------------------------------------------
 * IQN on the same engine (config algo = 4, n_q = 1; Dabney, Ostrovski, Silver & Munos 2018): a DQN engine over an
 * implicit quantile network.  Everything the DQN section says holds (networks, state blob, action column, hparams,
 * target copies, outputs, invalid actions, graph, groups, prioritized replay, n-step returns;
 * b200rl_offpolicy_set_dqn is required too) except the network and the loss.  An IQN engine is created by
 * b200rl_offpolicy_create_iqn from a config with algo = 4 and the counts of a b200rl_iqn_config, which size its per-row
 * buffers; b200rl_offpolicy_create and create_group refuse algo 4.  With n_cos, N = n, N' = n_target and K = k (each
 * 1..256) and the q description [obs, d, h, n_actions] (3 layers, hidden_act between layers, out_act identity), in
 * float32:
 *   draws    step st of a call draws, per row b, N + N' + K fractions in the order online, target, argmax: draw
 *            t = b (N + N' + K) + j is word t % 4 of Philox4x32-10(counter (t / 4, st, call, 0xB00), key seed) = r, and
 *            tau = (2 (r >> 9) + 1) 2^-24, an odd multiple of 2^-24 in (0, 1), exact in float32.  (seed, call) come
 *            from b200rl_offpolicy_set_noise_keys, which every train call of an IQN engine needs afresh; the domain
 *            tag 0xB00 keeps these draws apart from the noisy networks' 0xA00.
 *   features x_i = cospi(float32(i tau)), i = 0 .. n_cos - 1: the product i tau rounded once, then CUDA's cospif (at
 *            most 1 ulp from cos(pi x)).  The draw kernel materialises them for the step's forward passes.
 *   network  on R = B M rows (M fractions per row, network row b M + i for fraction i of row b):
 *            psi = act(x W_psi^T + b_psi) [B, d], phi = act(cos W_phi^T + b_phi) [R, d] (two GEMMs),
 *            z[b M + i] = psi[b] * phi[b M + i] (one float32 product per element),
 *            Z = act(z W_h^T + b_h) W_out^T + b_out [R, n_actions] (two GEMMs).  Every GEMM is the engine's fp32
 *            product with its k-sum in index order.  The flat parameter vector of networks 1 and 4 is W_psi [d, obs],
 *            b_psi, W_phi [d, n_cos], b_phi, W_h [h, d], b_h, W_out [n_actions, h], b_out: torch's
 *            parameters_to_vector of a module registering the embedding, the tau embedding and the head in this order.
 *   passes   Q(s) with the N online fractions; Q_targ(s') once with the N' target and K argmax fractions of each row
 *            (psi(s') shared); with double_q, Q(s') with the K argmax fractions.
 *   a*       = argmax_a (sum_k Z(s', tau~_k, a)) / K over the argmax samples of Q (double_q = 1; at the start of the
 *            step) or of Q_targ, the sum over k in index order (torch's argmax: a NaN wins, ties go to the first index)
 *   target   T_j = r + (g (1 - d)) Z_targ(s', tau'_j, a*), g = gamma (n-step: the row's discount)
 *   loss     u_ij = T_j - theta_i, theta_i = Z(s, tau_i, a); rho_ij = |tau_i - 1{u_ij < 0}| h(u_ij), h(u) = 0.5 u^2 if
 *            |u| < 1 else |u| - 0.5 (kappa = 1); the row's L = (1/N') sum_i sum_j rho_ij, over j in index order, then
 *            over i in index order; one Adam step (optimizer 1) on (1/B) sum_b L_b, summed in double in a fixed order
 *   gradient dZ[b N + i, a] = -(sum_j |tau_i - 1{u_ij < 0}| clamp(u_ij, -1, 1)) / N' * w_b / B (w_b = 1 without
 *            prioritized replay), 0 in every other column; the GEMMs' dW and dX modes with the activation derivatives
 *            read from the layer outputs, and for the product dphi = dz * psi[b] and dpsi[b] = sum_i dz[b N + i] *
 *            phi[b N + i] (each product rounded, the sum over i in index order).  No input gradient.
 * q1_values logs (sum_i theta_i) / N.  Prioritized replay: the priority of row b is (L_b + eps)^alpha of its unweighted
 * L_b, as for QR-DQN (non-finite: counted, and the call fails).  The head and every sum have a fixed order and no float
 * atomics are used: a group's learners stay bit-identical to solo engines, learner z's draws being those of a solo
 * engine given z's keys.  Launches per step: the draw 1, each forward pass 5, the head 1, the backward pass 7 (4
 * weight-gradient GEMMs, 2 input-gradient GEMMs, the product's backward), Adam 1, the target copy 1: 21, 26 with
 * double_q; a prioritized step adds its draw and priority update (2).  Runs as a CUDA graph, or as plain launches with
 * B200RL_OFFPOLICY_GRAPH=0.
 * Refused at create: create_iqn with another algo, algo 4 through create / create_group, or with dueling_k or
 * noisy_layers; a count outside 1..256; a q description that is not 3 layers or whose out_act is not identity; too many actions for
 * the head's shared memory; max_minibatch x max(N, N' + K) above 65535 x 32 network rows.  b200rl_offpolicy_set_qr
 * refuses an IQN engine.
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct {
  int32_t n_cos;    /* cosine features of a fraction */
  int32_t n;        /* N: fractions per row for Q(s) */
  int32_t n_target; /* N': fractions per row for the target samples of Q_targ(s') */
  int32_t k;        /* K: fractions per row for the argmax over actions */
} b200rl_iqn_config;

/* An IQN engine of n_learners learners (1 = a solo engine; 1 <= n_learners <= B200RL_MAX_LEARNERS): cfg->algo = 4. */
int b200rl_offpolicy_create_iqn(const b200rl_offpolicy_config* cfg, const b200rl_iqn_config* iqn, int32_t n_learners,
                                b200rl_offpolicy** out);
/* The fractions of the last train call that ran steps: host taus [K, S, B, N + N' + K] (per row the online, target
 * and argmax ones; B that call's minibatch) -- what a test replays through the oracle. */
int b200rl_offpolicy_get_iqn_draws(b200rl_offpolicy* h, int32_t S, float* taus);

/* ------------------------------------------------------------------------------------------------------------
 * D4PG on the same engine (config algo = 6, n_q = 1; Barth-Maron et al. 2018, "Distributed Distributional
 * Deterministic Policy Gradients"): DDPG with a categorical critic, n-step returns and prioritized replay.  Created by
 * b200rl_offpolicy_create_d4pg from a config with algo = 6 and a b200rl_d4pg_config; b200rl_offpolicy_create and
 * create_group refuse algo 6.  Networks are DDPG's (0 policy, 1 critic, 3 target policy, 4 target critic), so the state
 * blob, steps[3], hparams and outputs keep DDPG's layout.  policy = [obs, ..., A] is DDPG's deterministic policy,
 * q = [obs + A, ..., N] maps [s | a] to N logits over the support.  With N = n_atoms, in float32:
 *   support  dz = (v_max - v_min) / (N - 1), z_i = float32(v_min + i dz), both evaluated in double (C51's)
 *   p(s, a)  = exp(log_softmax) of the N logits, x - max - log(sum exp(x - max)); Q(s, a) = sum_i z_i p_i(s, a), every
 *            sum over atoms in index order
 *   target   a' = mu_targ(s') (no smoothing: hparams.use_target_noise must be 0); Tz_j = clamp(r + g (1 - d) z_j,
 *            v_min, v_max), g = gamma (n-step: the row's discount), b_j = (Tz_j - v_min) / dz,
 *            m_i = sum_j max(0, 1 - |b_j - i|) p_j(s', a') from the target critic (C51's projection)
 *   critic   CE_b = -sum_i m_i log p_i(s, a); one Adam step (optimizer 1) on (1/B) sum_b w_b CE_b (w_b = 1 without
 *            prioritized replay); the logit gradient is w_b (p_i(s, a) sum_k m_k - m_i) / B
 *   policy   with the critic just updated: one Adam step (optimizer 0) on -(1/B) sum_b Q(s_b, mu(s_b)); the gradient
 *            w.r.t. the critic's logits is -(1/B) p_k (z_k - Q), backpropagated through the critic's action input
 *            columns into the policy (critic parameters frozen), as DDPG's is
 *   polyak   both targets, every policy step (hparams.policy_delay applies as for DDPG; D4PG uses 1)
 * Outputs: q1_values [S,B] = Q(s, a) before the update, q1_losses [S] = the weighted mean CE (summed in double),
 * policy_losses = -mean Q per policy step.  Prioritized replay (the section below): the draw gathers A action columns,
 * beta follows the critic optimizer's count, and the priority of row b is (KL_b + eps)^alpha with
 * KL_b = CE_b + sum_i m_i log m_i (0 log 0 = 0; a rounding-level negative KL counts as 0), from before the Adam step;
 * with every w_b = 1 loss and gradient are bit for bit the unweighted step's.  n-step returns as the section below
 * states them (set_nstep).  train_prioritized[_group] return no policy losses: b200rl_offpolicy_get_policy_losses reads
 * them.  The heads reduce in a fixed order with no float atomics: a group's learners stay bit-identical to solo engines.
 * Runs as a CUDA graph, or as plain launches with B200RL_OFFPOLICY_GRAPH=0.  Launches per step are DDPG's (the two
 * heads take the places of its two loss kernels); a prioritized step adds its draw and priority update (2).
 * Refused at create: create_d4pg with another algo, algo 6 through create / create_group; n_q != 1; dueling_k or
 * noisy_layers != 0; n_atoms outside 2..256; a non-finite support or v_min >= v_max; a critic that does not map
 * obs + A -> N.  set_c51, set_qr, set_dqn, set_sac and set_noise_keys refuse a D4PG engine.
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct {
  int32_t n_atoms;  /* N, 2..256: the critic's output width */
  int32_t reserved; /* ignored */
  double v_min, v_max; /* finite, v_min < v_max */
} b200rl_d4pg_config;

/* A D4PG engine of n_learners learners (1 = a solo engine; 1 <= n_learners <= B200RL_MAX_LEARNERS): cfg->algo = 6. */
int b200rl_offpolicy_create_d4pg(const b200rl_offpolicy_config* cfg, const b200rl_d4pg_config* d4pg,
                                 int32_t n_learners, b200rl_offpolicy** out);
/* The policy losses of the last train call that ran steps (host [K, S]; the first *n_policy_updates of each row):
 * what a prioritized call, which takes no policy-loss buffer, logged.  Refused on DQN engines. */
int b200rl_offpolicy_get_policy_losses(b200rl_offpolicy* h, int32_t S, float* policy_losses, int32_t* n_policy_updates);

/* ------------------------------------------------------------------------------------------------------------
 * TQC on the same engine (config algo = 7, n_q = 2; Kuznetsov, Shvechikov, Grishin & Vetrov 2020, "Controlling
 * Overestimation Bias with Truncated Mixture of Continuous Distributional Quantile Critics"): SAC with two quantile
 * critics and a truncated, pooled target.  Created by b200rl_offpolicy_create_tqc from a config with algo = 7 and a
 * b200rl_tqc_config; b200rl_offpolicy_create and create_group refuse algo 7.  Networks, the state blob, steps[3],
 * hparams, the noise layout [S, 2, B, A], set_sac (required), set_alpha / get_alpha and sac_outputs are SAC's; the
 * critics q = [obs + A, ..., M] map [s | a] to M quantile locations theta_n^m at tau_m = (2m + 1) / (2M) (float32,
 * QR-DQN's).  With N = 2 critics, d = n_drop_per_net, kN = N (M - d) and alpha = alpha[st], per step in float32:
 *   target   a', log pi' = head(pi(s'), eps') as for SAC; the 2M atoms theta_targ_n^m(s', a') of both target critics
 *            are sorted ascending (NaN last, as torch.sort) and the first kN kept, z_(1) <= ... <= z_(kN);
 *            y_i = r + gamma (1 - d_done) (z_(i) - alpha log pi') in SAC's order of operations.  The kept sequence of
 *            values is unique whatever the ties, so the target is deterministic.
 *   critics  per critic n (optimizers 1, 2): u_mi = y_i - theta_n^m(s, a), rho(u) = |tau_m - 1{u < 0}| h(u), h the
 *            Huber function at kappa = 1; the row loss L = (1 / (kN M)) sum_m sum_i rho(u_mi) (i ascending, then m in
 *            index order); one Adam step on (1/B) sum_b L_b (summed in double in a fixed order), whose gradient w.r.t.
 *            theta_n^m is -(sum_i |tau_m - 1{u_mi < 0}| clamp(u_mi, -1, 1)) / (kN M) / B
 *   policy   with the critics just updated: one Adam step (optimizer 0) on
 *            mean_B(alpha log pi - (1 / (2M)) sum_n sum_m theta_n^m(s, a_pi)); every output column of both critics
 *            carries -1 / (2 M B), backpropagated through their action columns into SAC's squash backward pass (critic
 *            parameters frozen)
 *   alpha, polyak  SAC's
 * Outputs: q{n}_values [S,B] = (sum_m theta_n^m(s, a)) / M before the update (index order), q{n}_losses [S] the critic
 * losses above, policy_losses [S], and sac_outputs' log-prob means and alphas as for SAC.  train, train_gather,
 * train_gather_rng and their group forms all work, as a CUDA graph or as plain launches with B200RL_OFFPOLICY_GRAPH=0.
 * The heads reduce in a fixed order with no float atomics: a group's learners stay bit-identical to solo engines.
 * Launches, with Lq and Lp the critics' and the policy's Linear layers: 1 per call (the temperature table), then per
 * step SAC's 12 Lq + 4 Lp + 7 (+1 with learn_alpha = 1) plus the target kernel: 56 per step at two hidden layers, 57
 * with a learned temperature.
 * Refused at create: create_tqc with another algo, algo 7 through create / create_group; n_q != 2; dueling_k or
 * noisy_layers != 0; n_quantiles outside 1..256; n_drop_per_net outside 0..n_quantiles - 1; critics that do not map
 * obs + A -> M.  set_dqn, set_c51, set_qr, set_per, set_nstep, set_noise_keys and the train_prioritized calls refuse a
 * TQC engine (prioritized replay and n-step returns are not implemented for it).
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct {
  int32_t n_quantiles;    /* M, 1..256: each critic's output width */
  int32_t n_drop_per_net; /* d, 0..M - 1: the largest d atoms per critic dropped from the pooled target */
} b200rl_tqc_config;

/* A TQC engine of n_learners learners (1 = a solo engine; 1 <= n_learners <= B200RL_MAX_LEARNERS): cfg->algo = 7. */
int b200rl_offpolicy_create_tqc(const b200rl_offpolicy_config* cfg, const b200rl_tqc_config* tqc, int32_t n_learners,
                                b200rl_offpolicy** out);

/* ------------------------------------------------------------------------------------------------------------
 * CQL on the same engine (config algo = 8, n_q = 2; Kumar, Zhou, Tucker & Levine 2020, "Conservative Q-Learning for
 * Offline Reinforcement Learning", CQL(H)): SAC whose critics also push down a log-sum-exp over sampled actions.
 * Created by b200rl_offpolicy_create_cql from a config with algo = 8 and a b200rl_cql_config; create and create_group
 * refuse algo 8.  Networks, the state blob, steps[3], set_sac (required), set_alpha / get_alpha, the noise layout
 * [S, 2, B, A] and sac_outputs are SAC's; set_cql is required too.  With N = n_actions, T = temperature, w = weight,
 * L = action_limit, A the action width, alpha = alpha[st] and per step in float32 (the policy and critics at the start
 * of the step):
 *   draws    per row i and j < N: u_ij = L (2 x_ij - 1) with x_ij uniform in [0, 1), log density lu = -A log(2L);
 *            a^n_ij, log pi^n_ij = head(pi(s'_i), eps^n_ij) and a^s_ij, log pi^s_ij = head(pi(s_i), eps^s_ij) with
 *            SAC's squash head, from the policy outputs the step computes anyway (the policy is not fanned out)
 *   target   y_i = r + gamma (1 - d) (min(Q1targ, Q2targ)(s', a') - [backup_entropy] alpha log pi')
 *   critic k c_ij = [Q_k(s_i, u_ij) - lu]_j ++ [Q_k(s_i, a^n_ij) - log pi^n_ij]_j ++ [Q_k(s_i, a^s_ij) - log pi^s_ij]_j
 *            (3N values, every one at s_i); P_i = T logsumexp_j(c_ij / T) (max first, then the sum in index order);
 *            gap_k = mean_i P_i - mean_i Q_k(s_i, a_i); w_eff = w, or alpha' w with the Lagrange step;
 *            loss_k = mean_i (Q_k(s_i, a_i) - y_i)^2 + w_eff gap_k [- alpha' tau]; samples and log densities are
 *            constants; d loss_k / d Q_k(s_i, sample j) = w_eff softmax_j(c_ij / T) / B and
 *            d loss_k / d Q_k(s_i, a_i) = 2 (Q_k - y_i) / B - w_eff / B; one Adam step per critic
 *   Lagrange (config lagrange = 1) alpha' = clamp(exp(log alpha'), 0, 1e6) at the start of the step; one Adam step on
 *            log alpha' for -1/2 sum_k alpha' (w gap_k - tau) (gaps of this step's pre-update critics) with alpha_lr /
 *            alpha_beta1 / alpha_beta2 / alpha_eps; step st reads alpha'[st] and writes alpha'[st + 1]
 *   policy, temperature, polyak   SAC's, in SAC's order (the policy step reads the critics just updated)
 * Each critic's forward and backward passes in the critic step run on R = (1 + 3N) B stacked rows: rows 0..B-1 are
 * [s_i | a_i], row B + i 3N + j is sample j of row i in the block order above; the data rows' forward results and the
 * order of the weight-gradient sums over them are SAC's, so weight = 0 reproduces a SAC engine bit for bit on the same
 * draws.  Draws: a call with host draws (train, train_gather) needs b200rl_offpolicy_set_cql_draws first with
 * [K][S][3][B][N][A] floats: x, then eps^s, then eps^n, each [B][N][A]; train_gather_rng draws them on the device
 * (Philox tag 0xC91, x with 24 bits) and get_cql_draws reads them back in that layout.
 * Outputs: SAC's (q{k}_losses the loss_k above) and cql_outputs' gaps [K][2][S] and alpha' [K][S] (1 without the
 * Lagrange step).  The heads reduce in a fixed order with no float atomics: a group's learners stay bit-identical to
 * solo engines.
 * Launches, with Lq and Lp the critics' and the policy's Linear layers: 1 per call (the temperature table), 1 more with
 * the Lagrange step (the alpha' table), then per step SAC's 12 Lq + 4 Lp + 7 (+1 with learn_alpha = 1) plus the staging
 * kernel and the two penalty heads (+1 with the Lagrange step): 58 per step at two hidden layers, 59 with a learned
 * temperature, 60 with both.  train_gather_rng adds one draw launch per call.
 * Refused at create: create_cql with another algo, algo 8 through create / create_group; n_q != 2; dueling_k or
 * noisy_layers != 0; n_actions outside 1..64; (1 + 3N) max_minibatch above 65535 x 32 rows.  Prioritized replay, n-step
 * returns and noisy layers are refused as for SAC.
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct {
  int32_t n_actions; /* N, 1..64: samples per row from each of the three proposals */
  int32_t lagrange;  /* 1 = learn alpha' against target_action_gap, 0 = a fixed weight */
} b200rl_cql_config;

typedef struct {
  double weight;            /* w >= 0 */
  double temperature;       /* T > 0 */
  double target_action_gap; /* tau (Lagrange only) */
  double alpha_lr, alpha_beta1, alpha_beta2, alpha_eps; /* the Adam settings of log alpha' (Lagrange only) */
  int32_t backup_entropy;   /* 1 = SAC's soft target, 0 = no entropy term in the backup */
  int32_t reserved;         /* zeroed by set_cql */
} b200rl_cql_hparams;

/* A CQL engine of n_learners learners (1 = a solo engine; 1 <= n_learners <= B200RL_MAX_LEARNERS): cfg->algo = 8. */
int b200rl_offpolicy_create_cql(const b200rl_offpolicy_config* cfg, const b200rl_cql_config* cql, int32_t n_learners,
                                b200rl_offpolicy** out);
/* Required once before the first train call; part of the cached graph's key. */
int b200rl_offpolicy_set_cql(b200rl_offpolicy* h, const b200rl_cql_hparams* hp);
/* {log alpha', exp_avg, exp_avg_sq} and the Adam step count of each of the K learners. */
int b200rl_offpolicy_set_alpha_prime_group(b200rl_offpolicy* h, const float* log_alpha_prime, const float* exp_avg,
                                           const float* exp_avg_sq, const int64_t* step);
int b200rl_offpolicy_get_alpha_prime_group(b200rl_offpolicy* h, float* log_alpha_prime, float* exp_avg,
                                           float* exp_avg_sq, int64_t* step);
/* gaps [K][2][S] and alpha' [K][S] of the last train call's steps. */
int b200rl_offpolicy_cql_outputs(b200rl_offpolicy* h, int32_t S, float* gaps, float* alpha_primes);
/* The host draws [K][S][3][B][N][A] of the next train / train_gather call, and the draws of the last call. */
int b200rl_offpolicy_set_cql_draws(b200rl_offpolicy* h, int32_t S, int32_t B, const float* draws);
int b200rl_offpolicy_get_cql_draws(b200rl_offpolicy* h, int32_t S, int32_t B, float* draws);

/* ------------------------------------------------------------------------------------------------------------
 * IQL on the same engine (config algo = 9, n_q = 2; Kostrikov, Nair & Levine 2021, "Offline Reinforcement Learning
 * with Implicit Q-Learning"): an expectile value network, an advantage-weighted policy and twin critics, none of which
 * is ever evaluated at an action outside the minibatch.  Created by b200rl_offpolicy_create_iql from a config with
 * algo = 9 and a b200rl_iql_config; create and create_group refuse algo 9.  Networks: 0 the policy [obs, ..., 2A]
 * (outputs [m | l]), 1 / 2 the critics [obs + A, ..., 1], 3 the value network V = iql->value [obs, ..., 1], 4 / 5 the
 * target critics; network 3 is trained (optimizer 3).  For an IQL engine the state blob is networks 0..5, then
 * exp_avg / exp_avg_sq of optimizers 0..3, each segment padded as above; steps is [K][4]; set_adam / get_adam take
 * which = 3.  Every other engine keeps its blob and steps[K][3].  With L = hparams.action_limit, tau = expectile,
 * beta, W = max_weight, per train step in float32 on a minibatch (s, a, r, s', d) of B rows (the reference
 * implementation's order: value, actor with the new V, critics with the new V, targets):
 *   target   q^_i = min(Q1targ, Q2targ)(s_i, a_i) (torch.min: a NaN propagates)
 *   value    (optimizer 3) u_i = q^_i - V(s_i), w_i = tau if u_i > 0 else 1 - tau; one Adam step on
 *            L_V = mean_i w_i u_i^2, whose gradient w.r.t. V(s_i) is -2 w_i u_i / B; V' = the updated network
 *   policy   (optimizer 0) mu = L tanh(m), log sigma = clamp(l, log_std_min, log_std_max);
 *            log pi(a | s) = sum_j Normal(mu_j, sigma_j).log_prob(a_j) (a Gaussian whose mean is bounded, not a squashed
 *            sample: a dataset action at +-L needs no atanh); e_i = min(exp(beta (q^_i - V'(s_i))), W), a constant (NaN
 *            stays NaN); one Adam step on L_pi = -mean_i e_i log pi(a_i | s_i), whose output gradients are
 *            -e_i (a_j - mu_j) / sigma_j^2 L (1 - tanh^2 m_j) / B (mean columns) and -e_i ((a_j - mu_j)^2 / sigma_j^2 - 1)
 *            / B inside the clamp, 0 outside it (log-std columns); beta = 0 is behaviour cloning
 *   critics  (optimizers 1, 2, the critics at the start of the step) y_i = r_i + gamma (1 - d_i) V'(s'_i); one Adam
 *            step each on mean_i (Q_k(s_i, a_i) - y_i)^2
 *   polyak   Q1targ, Q2targ with hparams.polyak_rho
 * Nothing is drawn: train / train_gather take noise = NULL, train_gather_rng draws the indices only, get_draws returns
 * no noise (its noise must be NULL).  hparams.use_target_noise must be 0 and policy_delay >= 1 (it does not apply).
 * V's learning rate comes with each call (b200rl_iql_hparams.v_lr, read by run, not part of the cached graph's key),
 * the rest of set_iql is part of the key.  Outputs: q{k}_values [S,B] (pre-update), q{k}_losses [S], policy_losses
 * [S] = L_pi, and iql_outputs' value losses L_V, value means mean_i V(s_i) (before the value step) and weight means
 * mean_i e_i, each [K][S].  The heads reduce in a fixed order with no float atomics (one CTA per head): a group's
 * learners stay bit-identical to solo engines.  train, train_gather, train_gather_rng and their group forms all work,
 * as a CUDA graph or as plain launches with B200RL_OFFPOLICY_GRAPH=0.
 * Launches, with Lq, Lp and Lv the critics', the policy's and the value network's Linear layers: per step
 * 8 Lq + 3 Lp + 5 Lv + 5 (8 forward passes, four weight-gradient backward passes without input gradients, the value,
 * policy and two critic heads, four Adam steps, polyak): 53 per step at two hidden layers.
 * Refused at create: create_iql with another algo, algo 9 through create / create_group; n_q != 2; dueling_k or
 * noisy_layers != 0; a policy that is not [obs, ..., 2A], critics that are not [obs + A, ..., 1], a value network that
 * is not [obs, ..., 1].  set_iql refuses tau outside (0, 1), beta < 0 or not finite, W <= 0 or not finite, log_std_min
 * >= log_std_max, and non-finite Adam settings; it refuses every other engine.  set_sac, set_cql, set_dqn, set_c51,
 * set_qr, set_per, set_nstep, set_noise_keys and the train_prioritized calls refuse an IQL engine.
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct {
  b200rl_mlp_desc value; /* V: [obs, hidden..., 1] */
} b200rl_iql_config;

typedef struct {
  double expectile;                  /* tau in (0, 1) */
  double beta;                       /* inverse temperature >= 0 (0 = behaviour cloning) */
  double max_weight;                 /* W > 0: the AWR weights are clamped to it */
  double log_std_min, log_std_max;   /* the policy's log-std clamp */
  double v_lr, v_beta1, v_beta2, v_eps; /* torch.optim.Adam over V (v_lr is read per call) */
} b200rl_iql_hparams;

/* An IQL engine of n_learners learners (1 = a solo engine; 1 <= n_learners <= B200RL_MAX_LEARNERS): cfg->algo = 9. */
int b200rl_offpolicy_create_iql(const b200rl_offpolicy_config* cfg, const b200rl_iql_config* iql, int32_t n_learners,
                                b200rl_offpolicy** out);
/* Required once before the first train call; part of the cached graph's key except v_lr. */
int b200rl_offpolicy_set_iql(b200rl_offpolicy* h, const b200rl_iql_hparams* hp);
/* value_losses, value_means and weight_means [K][S] of the last train call's steps. */
int b200rl_offpolicy_iql_outputs(b200rl_offpolicy* h, int32_t S, float* value_losses, float* value_means,
                                 float* weight_means);

/* ------------------------------------------------------------------------------------------------------------
 * REDQ on the same engine (config algo = 10, n_q = 2; Chen, Wang, Zhou & Ross 2021, "Randomized Ensembled Double
 * Q-Learning"): SAC's squashed-Gaussian policy over an ensemble of N critics whose target takes the min over a random
 * subset of M target critics.  Created by b200rl_offpolicy_create_redq from a config with algo = 10 and a
 * b200rl_redq_config {N, M}, 2 <= N <= 32, 1 <= M <= N; create and create_group refuse algo 10.
 * Networks: 0 the policy [obs, ..., 2A], 1..N the critics [obs + A, ..., 1], N+1..2N their targets.  Optimizers: 0
 * the policy, 1..N the critics.  The state blob is networks 0..2N in that order, then exp_avg / exp_avg_sq of
 * optimizers 0..N, each segment padded as above; steps is [K][1 + N]; set_params / get_params / set_adam / get_adam
 * take these indices.  Every other engine keeps its blob and steps[K][3] (IQL [K][4]).
 * Per train step st of a call of S steps, on a minibatch (s, a, r, s', d) of B rows, with G = hparams.policy_delay
 * >= 1 and alpha = alpha[st], in float32:
 *   subset   M distinct indices Mst of 0..N-1
 *   target   a', log pi' = head(pi(s'), eps') with SAC's head; only the M drawn target critics are evaluated;
 *            y = r + gamma (1 - d) (min_{i in Mst} Q'_i(s', a') - alpha log pi') (fminf: a NaN target critic loses
 *            to a number, as in SAC)
 *   critics  every Q_i takes one Adam step on mean_b (Q_i(s, a) - y)^2 (the reference's mse_loss * N: each critic's
 *            gradient is its own MSE's); the logged values are the values before the update
 *   policy   on steps with (st + 1) % G == 0 or st == S - 1 (ceil(S / G) per call): one Adam step on
 *            mean_b(alpha log pi - (1/N) sum_i Q_i(s, a_pi)), a_pi, log pi = head(pi(s), eps), with the critics
 *            just updated (SAC's order and the paper's Algorithm 1; the reference code evaluates this loss with the
 *            critics from before their Adam step); every critic output carries -1 / (N B), backpropagated through
 *            the critics' action columns (summed over the critics in index order) into SAC's squash backward pass
 *   alpha    learn_alpha = 1: SAC's temperature step on policy steps; alpha[st + 1] is its result there and alpha[st]
 *            on the other steps
 *   polyak   every step, all N target critics
 * All N critics share one Adam table row (hparams.q1_lr, which must equal q2_lr): a call is refused when the critics'
 * step counts differ.  Subsets: a train / train_gather call needs b200rl_offpolicy_set_redq_subsets first with
 * int32 [K][S][M]; train_gather_rng draws them on the device (a partial Fisher-Yates shuffle over Philox4x32-10 keyed
 * by (seed, call), tag 0x7ED; SAC's index and noise draws for the same key are unchanged); get_redq_subsets returns
 * the last call's.  Noise: SAC's [S, 2, B, A]; slot 1 (the draw for s) is read on policy steps only.
 * Outputs: the train call's q1 / q2 values and losses are critics 1 and 2; policy_losses has ceil(S / G) entries, as
 * do sac_outputs' log-prob means (its alphas have S); redq_outputs returns every critic's values [K][N][S][B] and
 * losses [K][N][S].  The heads reduce in a fixed order with no float atomics: a group's learners stay bit-identical to
 * solo engines.  train, train_gather, train_gather_rng and their group forms all work, as a CUDA graph or as plain
 * launches with B200RL_OFFPOLICY_GRAPH=0.
 * Launches, with Lq and Lp the critics' and the policy's Linear layers, independent of N and M: 1 per call (the
 * temperature table), then per step 4 Lq + Lp + 4, plus 2 Lq + 3 Lp + 3 (+1 with learn_alpha = 1) on a policy step:
 * 19 and 37 (38) at two hidden layers.  train_gather_rng adds one subset draw per call.
 * Refused at create: create_redq with another algo, algo 10 through create / create_group; n_q != 2; dueling_k or
 * noisy_layers != 0; N outside 2..32, M outside 1..N; a policy that is not [obs, ..., 2A] or critics that are not
 * [obs + A, ..., 1].  set_sac is required; set_dqn, set_c51, set_qr, set_per, set_nstep, set_noise_keys, set_cql,
 * set_iql and the train_prioritized calls refuse a REDQ engine; set_redq_subsets refuses every other engine.
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct {
  int32_t n_critics; /* N, 2..32 */
  int32_t n_min;     /* M, 1..N: target critics per step */
} b200rl_redq_config;

/* A REDQ engine of n_learners learners (1 = a solo engine; 1 <= n_learners <= B200RL_MAX_LEARNERS): cfg->algo = 10. */
int b200rl_offpolicy_create_redq(const b200rl_offpolicy_config* cfg, const b200rl_redq_config* redq,
                                 int32_t n_learners, b200rl_offpolicy** out);
/* The subsets int32 [K][S][M] of the next train / train_gather call (each M distinct members of 0..N-1), and the
 * subsets of the last call. */
int b200rl_offpolicy_set_redq_subsets(b200rl_offpolicy* h, int32_t S, const int32_t* subsets);
int b200rl_offpolicy_get_redq_subsets(b200rl_offpolicy* h, int32_t S, int32_t* subsets);
/* q_values [K][N][S][B] (before each step's update) and q_losses [K][N][S] of every critic in the last train call. */
int b200rl_offpolicy_redq_outputs(b200rl_offpolicy* h, int32_t S, float* q_values, float* q_losses);

/* ------------------------------------------------------------------------------------------------------------
 * EDAC and SAC-N on the same engine (config algo = 11, n_q = 2; An, Moon, Kim & Song 2021, "Uncertainty-Based Offline
 * Reinforcement Learning with Diversified Q-Ensemble"): SAC's squashed-Gaussian policy over an ensemble of N critics,
 * the target the min over all N target critics, and (eta > 0) a penalty that pushes the critics' action gradients
 * apart.  eta = 0 is SAC-N.  Created by b200rl_offpolicy_create_edac from a config with algo = 11 and a
 * b200rl_edac_config {N, eta}, 2 <= N <= 32, eta finite and >= 0 (fixed at create); create, create_group and
 * create_redq refuse algo 11.  The engine has REDQ's layout: networks 0 the policy, 1..N the critics, N+1..2N their
 * targets; optimizers 0..N; REDQ's state blob, steps[K][1 + N], set_params / get_params / set_adam / get_adam.
 * Per train step st of a call of S steps, on a minibatch (s, a, r, s', d) of B rows, with alpha = alpha[st], in float32:
 *   target   a', log pi' = head(pi(s'), eps') with SAC's head; y = r + gamma (1 - d) (min over all N target critics
 *            of Q'_i(s', a') - alpha log pi') (fminf, as SAC and REDQ)
 *   critics  every Q_i takes one Adam step on mean_b (Q_i(s, a) - y)^2 + eta D, both terms at the parameters from
 *            before the step, with
 *              D = (1 / (B (N - 1))) sum_b sum_{i != j} gh_i(b) . gh_j(b),  gh = g / (|g|_2 + 1e-10),
 *              g_i(b) = d Q_i(s_b, a_b) / d a at the dataset action
 *            (the authors' grad_loss); Adam steps on g_td + g_div, added in that order; the logged values are the
 *            values before the update and the logged losses the TD losses
 *   policy   every step: one Adam step on mean_b(alpha log pi - min_i Q_i(s, a_pi)), a_pi, log pi = head(pi(s), eps),
 *            with the critics just updated (SAC's and REDQ's order here; the authors' code evaluates this loss with the
 *            critics from before their update); per row the gradient goes to the first critic that attains the min
 *            (lowest index on ties; a NaN loses to a number), through its action columns into SAC's squash backward
 *   alpha    learn_alpha = 1: SAC's temperature step every step
 *   polyak   every step, all N target critics
 * The diversity gradient is computed without autograd (ReLU masks are piecewise constant): a ones-backward through the
 * critics gives g, edac_diversity_kernel gives u = d(eta D) / d g and D, a tangent forward of u through the masks and
 * the weight-gradient products give the parameter gradient of sum_b g . u; its bias and obs-column entries are exactly
 * 0.  That pass runs beside the target path and joins before the critics' Adam step.  With eta > 0 the critics' hidden
 * activation must be ReLU and their output identity.  All N critics share one Adam table row (hparams.q1_lr, which
 * must equal q2_lr); hparams.policy_delay must be >= 1 and is otherwise not read.  Noise: SAC's [S, 2, B, A].  Nothing else is drawn:
 * train_gather_rng draws SAC's indices and noise.  Outputs: the train call's q1 / q2 are critics 1 and 2, policy_losses
 * and sac_outputs have S entries, redq_outputs returns every critic's values and TD losses, and edac_outputs D per step.
 * The heads reduce in a fixed order with no float atomics: a group's learners stay bit-identical to solo engines.
 * train, train_gather, train_gather_rng and their group forms all work, as a CUDA graph or as plain launches with
 * B200RL_OFFPOLICY_GRAPH=0.
 * Launches, with Lq and Lp the critics' and the policy's Linear layers, independent of N: 1 per call (the temperature
 * table), then per step 6 Lq + 4 Lp + 7 (+1 with learn_alpha = 1), plus 3 Lq with eta > 0: 37 (38) and 46 (47) at two
 * hidden layers.
 * Refused at create: algo != 11; n_q != 2; dueling_k or noisy_layers != 0; N outside 2..32; a negative or non-finite
 * eta; a policy that is not [obs, ..., 2A] or critics that are not [obs + A, ..., 1]; with eta > 0, critics whose
 * hidden activation is not ReLU or whose output is not identity.  set_sac is required; set_redq_subsets,
 * get_redq_subsets, set_dqn, set_c51, set_qr, set_per, set_nstep, set_noise_keys, set_cql, set_iql and the
 * train_prioritized calls refuse an EDAC engine.
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct {
  int32_t n_critics; /* N, 2..32 */
  int32_t reserved;  /* 0 */
  double eta;        /* the diversity weight, finite and >= 0; 0 = SAC-N */
} b200rl_edac_config;

/* An EDAC engine of n_learners learners (1 = a solo engine; 1 <= n_learners <= B200RL_MAX_LEARNERS): cfg->algo = 11. */
int b200rl_offpolicy_create_edac(const b200rl_offpolicy_config* cfg, const b200rl_edac_config* edac,
                                 int32_t n_learners, b200rl_offpolicy** out);
/* diversity [K][S]: D of every step of the last train call (0 with eta = 0). */
int b200rl_offpolicy_edac_outputs(b200rl_offpolicy* h, int32_t S, float* diversity);

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

/* Required before a prioritized call of a DQN or D4PG engine (other engines are refused); part of the cached graph's
 * key. */
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
 * so set it before every call).  Refused on TD3, DDPG and SAC engines (D4PG engines take it).  n_step is part of the cached graph's key, and so
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
