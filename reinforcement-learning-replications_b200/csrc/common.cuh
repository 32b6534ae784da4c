// Shared helpers for libb200rl (sm_90a).
#pragma once
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <string>

#include "b200rl.h"

namespace b200rl {

void set_error(const char* fmt, ...);

#define B200RL_CUDA(expr)                                                                                  \
  do {                                                                                                     \
    cudaError_t _e = (expr);                                                                               \
    if (_e != cudaSuccess) {                                                                               \
      ::b200rl::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__);     \
      return 1;                                                                                            \
    }                                                                                                      \
  } while (0)

#define B200RL_REQUIRE(cond, ...)         \
  do {                                    \
    if (!(cond)) {                        \
      ::b200rl::set_error(__VA_ARGS__);   \
      return 2;                           \
    }                                     \
  } while (0)

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
inline int pad4(int x) { return (x + 3) & ~3; }

int device_sm_count();

// accumulator memory of the tensor-core kernels (tc_common.cuh) for a launch of `grid` CTAs on stream `s`
float* acc_mem(int grid, cudaStream_t s);
// grid of a tensor-core kernel: one CTA per 128-row tile, at most one per SM (-1: no device)
int tc_grid(int64_t n_rows);
// offsets of the weights and biases of a 3-Linear-layer network in its flat parameter vector (torch order: W1 b1 W2 b2
// W3 b3); returns the parameter count
int mlp3_offsets(const b200rl_mlp_desc& d, int w_off[3], int b_off[3]);

// global launch counter (bench.py reports gpu_launches from it)
void count_launch(int n = 1);
int64_t launches_total();

// Adam helpers shared with the off-policy engine (adam.cu)
void adam_scalars(int64_t step, double lr, double beta1, double beta2, float* step_size, float* bc2_sqrt);
int adam_step_table(float* params, const float* grad, float* m, float* v, int64_t n, const float2* table, int idx,
                    double beta1, double beta2, double eps, cudaStream_t s, int lanes = 1, size_t lane_stride = 0);

// TRPO vector kernels (trpo.cu)
int trpo_cg_init(const float* g, float* x, float* r, float* pv, int n, double* sc, int* flags, cudaStream_t s);
int trpo_cg_update(const float* z_raw, float damping, float* x, float* r, float* pv, int n, double* sc, int* flags,
                   cudaStream_t s);
int trpo_nan_to_zero(float* x, int n, cudaStream_t s);
int trpo_step_size(const float* x, const float* hx_raw, float damping, float delta, float* descent, const float* params,
                   float* prev, int n, double* sc, cudaStream_t s);
int trpo_ls_set_params(float* params, const float* prev, const float* descent, float ratio, int n, const int* flags,
                       cudaStream_t s);
int trpo_ls_check(const double* slot, double n_rows, float delta, double* sc, int* flags, int index, cudaStream_t s);
int trpo_ls_final(float* params, const float* prev, int n, float delta, const double* sc, int* flags, cudaStream_t s);
int trpo_set_scalar(double* dst, const double* slot, int k, double inv, cudaStream_t s);
int trpo_tail_to_slot(const float* tail, double* slot, cudaStream_t s);

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

}  // namespace b200rl
