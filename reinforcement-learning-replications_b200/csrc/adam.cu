// reduce_partials + adam_step.
//
// Replaces (reference: /root/reference/src/rl_replicas/): the gradient accumulation of loss.backward() and
// torch.optim.Adam.step() at algorithms/ppo.py:233-235 and :276-278 (torch 2.5.1 `_single_tensor_adam`, pinned in
// uv.lock:764-765; weight_decay = 0, amsgrad = False, maximize = False), plus the host-side early-stop test of
// algorithms/ppo.py:176-181, which moves onto the device so the 80-step loop never synchronises with the host.
#include "common.cuh"

namespace b200rl {

// grad[p] = sum over partial rows c of partials[c][p]; scalars[k] likewise.  The order is FIXED (independent of timing
// and of the launch geometry of the producer), so gradients are run-to-run identical: a block owns 32 parameters,
// warp w adds rows w, w+8, w+16, ... with four interleaved accumulators (independent loads in flight), and the eight
// warp sums are added in warp order.
constexpr int RP_WARPS = 8;
__global__ void __launch_bounds__(RP_WARPS * 32) reduce_partials_kernel(const float* __restrict__ partials,
                                                                        const double* __restrict__ scalar_partials,
                                                                        int grid, long long n_params,
                                                                        float* __restrict__ grad,
                                                                        double* __restrict__ scalars, int grad_tail,
                                                                        const int* __restrict__ skip_flag) {
  if (skip_flag != nullptr && *skip_flag != 0) return;
  __shared__ float part[RP_WARPS][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long p = (long long)blockIdx.x * 32 + lane;
  if (partials != nullptr) {
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
    if (p < n_params) {
      const float* q = partials + p;
      int c = warp;
      for (; c + 3 * RP_WARPS < grid; c += 4 * RP_WARPS) {
        s0 += q[(size_t)c * n_params];
        s1 += q[(size_t)(c + RP_WARPS) * n_params];
        s2 += q[(size_t)(c + 2 * RP_WARPS) * n_params];
        s3 += q[(size_t)(c + 3 * RP_WARPS) * n_params];
      }
      for (; c < grid; c += RP_WARPS) s0 += q[(size_t)c * n_params];
    }
    part[warp][lane] = (s0 + s1) + (s2 + s3);
    __syncthreads();
    if (warp == 0 && p < n_params) {
      float s = part[0][lane];
#pragma unroll
      for (int w = 1; w < RP_WARPS; ++w) s += part[w][lane];
      grad[p] = s;
    }
  }
  if (blockIdx.x == 0 && scalar_partials != nullptr) {  // scalars: 32 row classes x 8 scalars, then classes in order
    __shared__ double spart[RP_WARPS * 4][B200RL_N_SCALARS];
    const int k = lane & 7, cls = warp * 4 + (lane >> 3);
    double s = 0.0;
    for (int c = cls; c < grid; c += RP_WARPS * 4) s += scalar_partials[(size_t)c * B200RL_N_SCALARS + k];
    spart[cls][k] = s;
    __syncthreads();
    if (threadIdx.x < B200RL_N_SCALARS) {
      double t = 0.0;
      for (int c = 0; c < RP_WARPS * 4; ++c) t += spart[c][threadIdx.x];
      if (scalars != nullptr) scalars[threadIdx.x] = t;
      if (grad_tail) grad[n_params + threadIdx.x] = (float)t;  // piggy-backed on the gradient all-reduce
    }
  }
}

struct AdamArgs {
  float* params;
  const float* grad;
  float* m;
  float* v;
  long long n;
  float one_minus_b1, b2, one_minus_b2;
  float step_size;   // lr / (1 - beta1^t)
  float bc2_sqrt;    // sqrt(1 - beta2^t)
  float eps;
  const void* kl_sum;
  int kl_is_f32;
  double n_global, kl_limit;
  int* stop_flag;
  int* applied_counter;
  const float* tail_src;
  double* tail_dst;
  const float2* table;  // optional: {step_size, bc2_sqrt} read from device memory (CUDA-graph replays: the node's
  int table_idx;        // arguments stay fixed while the host refreshes the table before each launch)
};

// LANES (the off-policy engine's learner groups): learner blockIdx.z works on params / grad / m / v / table shifted by
// blockIdx.z * lane_stride bytes (one arena per learner, see offpolicy.cu); the arithmetic is the same for every learner.
template <bool LANES>
__global__ void __launch_bounds__(256) adam_step_kernel(const AdamArgs args, size_t lane_stride) {
  AdamArgs a = args;
  if (LANES) {
    const size_t off = blockIdx.z * lane_stride;
    a.params = reinterpret_cast<float*>(reinterpret_cast<char*>(a.params) + off);
    a.grad = reinterpret_cast<const float*>(reinterpret_cast<const char*>(a.grad) + off);
    a.m = reinterpret_cast<float*>(reinterpret_cast<char*>(a.m) + off);
    a.v = reinterpret_cast<float*>(reinterpret_cast<char*>(a.v) + off);
    a.table = reinterpret_cast<const float2*>(reinterpret_cast<const char*>(a.table) + off);
  }
  // early stop (ppo.py:176-181): the KL carried by this step's forward pass is the KL of the PREVIOUS update
  bool stop = false;
  if (a.stop_flag != nullptr) {
    stop = *a.stop_flag != 0;
    if (!stop && a.kl_sum != nullptr) {
      const double kl = a.kl_is_f32 ? (double)*static_cast<const float*>(a.kl_sum) : *static_cast<const double*>(a.kl_sum);
      stop = (float)(kl / a.n_global) > (float)a.kl_limit;
    }
  }
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (!stop && i < a.n) {
    float step_size = a.step_size, bc2_sqrt = a.bc2_sqrt;
    if (a.table != nullptr) {
      const float2 t = a.table[a.table_idx];
      step_size = t.x;
      bc2_sqrt = t.y;
    }
    const float g = a.grad[i];
    float m = a.m[i], v = a.v[i];
    m = m + a.one_minus_b1 * (g - m);                     // exp_avg.lerp_(grad, 1 - beta1)
    // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, 1 - beta2).  The compiler fuses a different product of this sum in
    // the LANES instantiation, so there the solo kernel's rounding is spelled out: a learner in a group must round
    // exactly as a solo learner does.
    if (LANES) v = __fmaf_rn(v, a.b2, __fmul_rn(__fmul_rn(g, g), a.one_minus_b2));
    else v = v * a.b2 + a.one_minus_b2 * (g * g);
    const float denom = sqrtf(v) / bc2_sqrt + a.eps;      // (exp_avg_sq.sqrt() / bias_correction2_sqrt).add_(eps)
    a.m[i] = m;
    a.v[i] = v;
    a.params[i] = a.params[i] - step_size * (m / denom);  // param.addcdiv_(exp_avg, denom, value=-step_size)
  }
  // every CTA evaluated `stop` from the same inputs; the flag is written by the LAST CTA only after all read it:
  // other CTAs never re-read it inside this launch, and later launches are stream-ordered behind this one.
  if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) {
    if (stop && a.stop_flag != nullptr) *a.stop_flag = 1;
    if (!stop && a.applied_counter != nullptr) *a.applied_counter += 1;
    if (a.tail_src != nullptr && a.tail_dst != nullptr)
      for (int k = 0; k < B200RL_N_SCALARS; ++k) a.tail_dst[k] = (double)a.tail_src[k];
  }
}

}  // namespace b200rl

using namespace b200rl;

extern "C" int b200rl_reduce_partials(const float* partials, const double* scalar_partials, int32_t grid,
                                      int64_t n_params, float* grad, double* scalars, int grad_tail,
                                      const int32_t* skip_flag, void* stream) {
  B200RL_REQUIRE(grid > 0 && n_params > 0, "reduce_partials: bad arguments");
  B200RL_REQUIRE((partials == nullptr && !grad_tail) || grad != nullptr, "reduce_partials: grad is NULL");
  const int blocks = partials == nullptr ? 1 : (int)((n_params + 31) / 32);
  reduce_partials_kernel<<<blocks, RP_WARPS * 32, 0, static_cast<cudaStream_t>(stream)>>>(partials, scalar_partials, grid,
                                                                                n_params, grad, scalars, grad_tail,
                                                                                skip_flag);
  B200RL_CUDA(cudaGetLastError());
  count_launch(1);
  return 0;
}

extern "C" int b200rl_adam_step(float* params, const float* grad, float* exp_avg, float* exp_avg_sq,
                                int64_t n_params, int64_t step, double lr, double beta1, double beta2, double eps,
                                const void* kl_sum, int kl_is_f32, double n_global, double kl_limit,
                                int32_t* stop_flag, int32_t* applied_counter, const float* tail_src,
                                double* tail_dst, void* stream) {
  B200RL_REQUIRE(params && grad && exp_avg && exp_avg_sq && n_params > 0 && step >= 1, "adam_step: bad arguments");
  AdamArgs a;
  a.params = params;
  a.grad = grad;
  a.m = exp_avg;
  a.v = exp_avg_sq;
  a.n = n_params;
  // host-side scalar math in double exactly like torch's Python-float arithmetic, then cast where torch casts
  const double bc1 = 1.0 - pow(beta1, (double)step);
  const double bc2 = 1.0 - pow(beta2, (double)step);
  a.one_minus_b1 = (float)(1.0 - beta1);
  a.b2 = (float)beta2;
  a.one_minus_b2 = (float)(1.0 - beta2);
  a.step_size = (float)(lr / bc1);
  a.bc2_sqrt = (float)sqrt(bc2);
  a.eps = (float)eps;
  a.kl_sum = kl_sum;
  a.kl_is_f32 = kl_is_f32;
  a.tail_src = tail_src;
  a.tail_dst = tail_dst;
  a.n_global = n_global;
  a.kl_limit = kl_limit;
  a.stop_flag = stop_flag;
  a.applied_counter = applied_counter;
  a.table = nullptr;
  a.table_idx = 0;
  const int blocks = (int)((n_params + 255) / 256);
  adam_step_kernel<false><<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(a, 0);
  B200RL_CUDA(cudaGetLastError());
  count_launch(1);
  return 0;
}

namespace b200rl {
// torch's host-side scalar math for step `step` (see b200rl_adam_step): {lr / (1 - beta1^t), sqrt(1 - beta2^t)}
void adam_scalars(int64_t step, double lr, double beta1, double beta2, float* step_size, float* bc2_sqrt) {
  *step_size = (float)(lr / (1.0 - pow(beta1, (double)step)));
  *bc2_sqrt = (float)sqrt(1.0 - pow(beta2, (double)step));
}
// Adam step whose two step-dependent scalars come from table[idx] in device memory (off-policy engine, graph replay);
// lanes > 1: one launch for `lanes` learners whose buffers (table included) lie lane_stride bytes apart
int adam_step_table(float* params, const float* grad, float* m, float* v, int64_t n, const float2* table, int idx,
                    double beta1, double beta2, double eps, cudaStream_t s, int lanes, size_t lane_stride) {
  AdamArgs a{};
  a.params = params;
  a.grad = grad;
  a.m = m;
  a.v = v;
  a.n = n;
  a.one_minus_b1 = (float)(1.0 - beta1);
  a.b2 = (float)beta2;
  a.one_minus_b2 = (float)(1.0 - beta2);
  a.eps = (float)eps;
  a.table = table;
  a.table_idx = idx;
  if (lanes == 1) adam_step_kernel<false><<<(int)((n + 255) / 256), 256, 0, s>>>(a, 0);
  else adam_step_kernel<true><<<dim3((unsigned)((n + 255) / 256), 1, (unsigned)lanes), 256, 0, s>>>(a, lane_stride);
  B200RL_CUDA(cudaGetLastError());
  count_launch(1);
  return 0;
}
}  // namespace b200rl
