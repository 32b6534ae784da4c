// Argument blocks and launchers of the fused policy + value step (mlp_tc3.cu), shared with the engine (engine.cu).
#pragma once
#include <cstdint>

#include "common.cuh"

namespace b200rl {

struct Tc3Net {  // one 3-Linear-layer network: widths and offsets into its flat parameter vector
  int n_out, h1, h2;
  int w_off[3], b_off[3];
};

struct Tc3Args {
  int n_in, dist;
  Tc3Net net[2];           // 0 policy, 1 value
  int P[2];                // parameter counts
  const float* params[2];
  long long n_rows;
  float inv_n, n_glob_f, clip_lo, clip_hi;
  const uint8_t* ximg;     // [tiles][16 KB] packed observation tiles (pack_obs_kernel)
  const float* xscale;     // [64] 2^ex_k, 2^-ex_k of the packed features
  const float* actions;
  const float* log_std;
  const float* adv_raw;
  const double* adv_stats;
  const float* old_logp;
  const float* target;        // discounted returns
  const float* target_absmax; // device scalar
  float* partials;            // [2 * grid][P0 + P1]
  double* scalar_partials;    // [2 * grid][16]: policy sums 0..7 (as b200rl_mlp_loss_grad), value sums 8..15
  const int* stop_flag;       // != 0: the policy loop has stopped early -> only the value chain runs
  const float* x_bad;         // raised (1.0f) by pack_obs_kernel: observations outside the fp16 range
  float* status;              // raised (1.0f) by this kernel on a range trip (floats: the flags ride an all-reduce)
  int run_policy, run_value;  // host-known: iteration index below the loop lengths
  float* acc_mem;             // accumulator memory, ACC_CTA_FLOATS per CTA (tc_common.cuh)
};

struct Ra3Seg {
  float *params, *m, *v;
  float one_minus_b1, b2, one_minus_b2, step_size, bc2_sqrt, eps;
};

constexpr int RA3_MAX_WORLD = 16;

struct Ra3Args {
  // 0 reduce + Adam, 1 reduce only (scalars appended to grad), 2 Adam only (scalars from grad's tail),
  // 3 reduce + publish into this rank's exchange buffer, 4 gather every rank's buffer over NVLink + Adam,
  // 5 = 3 + wait + 4 in one launch
  int mode;
  const float* partials;
  const double* scalar_partials;
  int rows;          // partial rows (2 * grid of the step kernel)
  long long P[2];
  float* grad;       // [P0 + P1 + 16]
  Ra3Seg seg[2];
  double *slot_p, *slot_v;  // scalar history slots of this iteration
  double n_global, kl_limit;
  int kl_limit_on;
  int* stop_flag;
  int *applied_p, *applied_v;
  int run_policy, run_value;
  // peer exchange (modes 3 / 4): every rank's buffer is [2 parities][xchg_stride floats] followed by 2 sequence words
  float* const* peers;       // device array [world] of the ranks' exchange buffers (peer-mapped device pointers)
  int world, rank;
  long long xchg_stride;
  unsigned seq;              // sequence number of this exchange (parity = seq & 1)
  unsigned* done_counter;    // device word, zero between launches
  int* comm_error;           // raised when a peer's flag did not arrive within the time-out
};

bool tc3_shape_ok(const b200rl_mlp_desc& pol, const b200rl_mlp_desc& val);
size_t tc3_ximg_bytes(int64_t n_rows);
int launch_pack_obs(const float* obs, int64_t n_rows, int n_in, const float* absmax, uint8_t* ximg, float* xscale,
                    float* bad_flag, cudaStream_t s);
int launch_mlp_tc3(const Tc3Args& k, cudaStream_t s);
int launch_reduce_adam3(const Ra3Args& a, cudaStream_t s);
int launch_wait_peers(const Ra3Args& a, cudaStream_t s);
bool ra3_one_wave(long long p_total);

}  // namespace b200rl
