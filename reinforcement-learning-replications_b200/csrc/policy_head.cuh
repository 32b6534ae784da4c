// Per-row distribution and loss math of the on-policy kernels (mlp_fused.cu, mlp_tc2.cu, mlp_tc3.cu, mlp_tc_fvp.cu):
// log-prob, entropy, d logp / d out, the PPO / VPG / TRPO surrogates, the value MSE, TRPO's true KL and its Fisher
// metric.  One thread evaluates one row.  The functions take pointers and sizes, so every kernel keeps
// its own layout: outputs, actions and tangents may sit in registers or shared memory; inputs read from global memory
// are passed as Ldg.  Loops over the action dimension run to the compile-time bound NA (15 in the tensor-core kernels,
// 16 in the fp32 kernel) and are guarded by a < A_out.
#pragma once
#include <cmath>

#include "common.cuh"

namespace b200rl {

constexpr float LOG_SQRT_2PI = 0.91893853320467274178f;  // log(sqrt(2 pi))
constexpr float ENT_CONST = 1.4189385332046727418f;      // 0.5 + 0.5 * log(2 pi)

// A read-only input in global memory, indexed like a pointer but loaded through the non-coherent cache (__ldg)
struct Ldg {
  const float* p;
  __device__ __forceinline__ float operator[](int i) const { return __ldg(p + i); }
};

// Per-action constants of Normal(mu, scale), scale = exp(log_std) (gaussian_policy.py:34)
struct NormalConsts {
  float var, log_scale, inv_2var, inv_var;
};
__device__ __forceinline__ NormalConsts normal_consts(const float* log_std, int a) {
  const float scale = expf(__ldg(log_std + a));
  const float var = scale * scale;  // Normal.log_prob: var = scale ** 2
  return {var, logf(scale), 1.f / (2.f * var), 1.f / var};
}

// The two ways the kernels divide by the variance.  They round differently, so each kernel keeps its own.
// VarDiv divides, as torch does: the fp32 kernel, which also recomputes the fp16 launches that leave fp16's range.
struct VarDiv {
  const float* var;
  __device__ __forceinline__ float over_var(float x, int a) const { return x / var[a]; }
  __device__ __forceinline__ float over_2var(float x, int a) const { return x / (2.f * var[a]); }
};
// VarRecip multiplies by 1/var and 1/(2 var) precomputed once per launch: one multiply per row instead of a division
// (the fp16 x 2 kernels).
struct VarRecip {
  const float* inv_var;
  const float* inv_2var;
  __device__ __forceinline__ float over_var(float x, int a) const { return x * inv_var[a]; }
  __device__ __forceinline__ float over_2var(float x, int a) const { return x * inv_2var[a]; }
};

// normalize_tensor (utils.py:90-92): mean and UNBIASED std of the advantages, no epsilon; 0 and 1 without statistics
__device__ __forceinline__ void adv_mean_std(const double* adv_stats, float& mean, float& std) {
  mean = 0.f;
  std = 1.f;
  if (adv_stats != nullptr) {
    const double s1 = adv_stats[0], s2 = adv_stats[1], cnt = adv_stats[2];
    const double m = s1 / cnt;
    mean = (float)m;
    std = (float)sqrt((s2 - cnt * m * m) / (cnt - 1.0));
  }
}

// Value loss (ppo.py:282-287): the row's squared error; dv = d mean((v - target)^2) / dv = 2 (v - target) / N
__device__ __forceinline__ float value_mse(float v, float target, float inv_n, float& dv) {
  const float diff = v - target;
  dv = (2.f * diff) * inv_n;
  return diff * diff;
}

// Diagonal Gaussian of mean mu: Normal.log_prob(x) and Normal.entropy summed over the actions, d logp / d mu per action
template <int NA, class X, class V>
__device__ __forceinline__ void gaussian_logp(X x, const float* mu, const float* log_scale, V v, int A_out,
                                              float& lp, float& ent, float* dlp) {
  float l = 0.f, e = 0.f;
#pragma unroll
  for (int a = 0; a < NA; ++a)
    if (a < A_out) {
      const float d = x[a] - mu[a];
      l += v.over_2var(-(d * d), a) - log_scale[a] - LOG_SQRT_2PI;  // torch Normal.log_prob
      e += ENT_CONST + log_scale[a];                                // torch Normal.entropy
      dlp[a] = v.over_var(d, a);
    }
  lp = l;
  ent = e;
}

// log(sum_a exp(x_a)), the largest x_a taken out first: the normalisation of Categorical(logits=x)
template <int NA, class X>
__device__ __forceinline__ float log_sum_exp(X x, int A_out) {
  float m = x[0];
#pragma unroll
  for (int a = 1; a < NA; ++a)
    if (a < A_out) m = fmaxf(m, x[a]);
  float se = 0.f;
#pragma unroll
  for (int a = 0; a < NA; ++a)
    if (a < A_out) se += expf(x[a] - m);
  return m + logf(se);
}

// Categorical(logits): log_prob of action ai, entropy, d logp / d logits per class
template <int NA>
__device__ __forceinline__ void categorical_logp(const float* logits, int ai, int A_out, float& lp, float& ent,
                                                 float* dlp) {
  const float lse = log_sum_exp<NA>(logits, A_out);
  float l = 0.f, e = 0.f;
#pragma unroll
  for (int a = 0; a < NA; ++a)
    if (a < A_out) {
      const float lg = logits[a] - lse;
      const float pa = expf(lg);
      e -= lg * pa;
      if (a == ai) l = lg;
      dlp[a] = (a == ai ? 1.f : 0.f) - pa;
    }
  lp = l;
  ent = e;
}

// kl_divergence(old_dist, dist) of one row (trpo.py:167-175).  Gaussian, same std: 0.5 ((mu_old - mu) / std)^2 summed.
template <int NA, class X, class V>
__device__ __forceinline__ float gaussian_kl(X mu_old, const float* mu, V v, int A_out) {
  float kl = 0.f;
#pragma unroll
  for (int a = 0; a < NA; ++a)
    if (a < A_out) {
      const float d = mu_old[a] - mu[a];
      kl += 0.5f * v.over_var(d * d, a);
    }
  return kl;
}
template <int NA, class X>
__device__ __forceinline__ float categorical_kl(X old_logits, const float* logits, int A_out) {
  const float lo = log_sum_exp<NA>(old_logits, A_out), ln = log_sum_exp<NA>(logits, A_out);
  float kl = 0.f;
#pragma unroll
  for (int a = 0; a < NA; ++a)
    if (a < A_out) {
      const float lpo = old_logits[a] - lo;
      kl += expf(lpo) * (lpo - (logits[a] - ln));
    }
  return kl;
}

// Fisher-vector product head: the metric of the distribution applied to the output tangent t = J v, over N:
// g = M t / N.  Gaussian with fixed std: M = diag(1/var).  Categorical: M = diag(p) - p p^T.
template <int NA, class V>
__device__ __forceinline__ void gaussian_metric(const float* t, V v, int A_out, float inv_n, float* g) {
#pragma unroll
  for (int a = 0; a < NA; ++a)
    if (a < A_out) g[a] = v.over_var(t[a], a) * inv_n;
}
template <int NA>
__device__ __forceinline__ void categorical_metric(const float* logits, const float* t, int A_out, float inv_n,
                                                   float* g) {
  const float lse = log_sum_exp<NA>(logits, A_out);
  float pt = 0.f;
#pragma unroll
  for (int a = 0; a < NA; ++a)
    if (a < A_out) pt += expf(logits[a] - lse) * t[a];
#pragma unroll
  for (int a = 0; a < NA; ++a)
    if (a < A_out) g[a] = expf(logits[a] - lse) * (t[a] - pt) * inv_n;
}

// Policy loss term of one row and coef = dLoss / dlogp of the row (the 1/N of the mean folded in):
// PPO clip (ppo.py:245-255), VPG (vpg.py:203), TRPO surrogate (trpo.py:161-163); 0 for any other loss
__device__ __forceinline__ float policy_loss(int loss, float lp, float oldlp, float adv, float inv_n, float clip_lo,
                                             float clip_hi, float& coef) {
  float term = 0.f;
  coef = 0.f;
  if (loss == B200RL_LOSS_PPO_CLIP) {
    const float ratio = expf(lp - oldlp);
    const float s1 = ratio * adv;
    const float s2 = fminf(fmaxf(ratio, clip_lo), clip_hi) * adv;
    term = -fminf(s1, s2);
    const bool pass = adv >= 0.f ? (ratio <= clip_hi) : (ratio >= clip_lo);
    coef = pass ? (-inv_n * adv) * ratio : 0.f;
  } else if (loss == B200RL_LOSS_VPG) {
    term = -(lp * adv);
    coef = -inv_n * adv;
  } else if (loss == B200RL_LOSS_TRPO_SURROGATE) {
    const float ratio = expf(lp - oldlp);
    term = -(ratio * adv);
    coef = (-inv_n * adv) * ratio;
  }
  return term;
}

// A policy row's share of scalar sums 0..4 (b200rl.h): loss term, old_logp - logp (with old_logp), entropy, logp, logp^2
__device__ __forceinline__ void add_policy_row_sums(double* sc, float term, float lp, float ent, float oldlp,
                                                    bool has_old) {
  sc[0] += (double)term;
  if (has_old) sc[1] += (double)(oldlp - lp);
  sc[2] += (double)ent;
  sc[3] += (double)lp;
  sc[4] += (double)lp * (double)lp;
}

}  // namespace b200rl
