// mlp_tc_fvp: TRPO's Fisher-vector product on the tensor cores (wgmma, sm_90a).
//
// Contract of B200RL_LOSS_FVP (see mlp_fused.cu, MODE 2, for the reference map: conjugate_gradient_optimizer.py:133-167
// double-backprops mean KL(old || new); at theta = theta_old that Hessian is the Fisher matrix (1/N) J^T M J):
//   forward           H1 = tanh(X W1^T + b1), H2 = tanh(H1 W2^T + b2), OUT = H2 W3^T + b3
//   tangent forward   T1 = (1 - H1^2) (X V1^T + vb1),  T2 = (1 - H2^2) (T1 W2^T + H1 V2^T + vb2),
//                     TOUT = T2 W3^T + H2 V3^T + vb3                       (V, vb = the direction vector v, J v = TOUT)
//   metric            dOut = M TOUT / N   (Gaussian, fixed std: M = diag(1/var); Categorical: M = diag(p) - p p^T)
//   backward          the ordinary backward pass of dOut  ->  J^T M J v / N  in the flat parameter layout
// Same machinery as mlp_tc2.cu (two fp16 splits per fp32 operand after an exact power-of-two pre-scale, 3 MMAs per
// chain product, M-stacked 2-MMA weight-gradient products, dZ written over H in place, range-checked with a predicated
// re-run -- here by the fp32 kernel), but ONE tile pipeline per CTA: the tangent activations T1 / T2 and the direction
// weights V need the shared memory the second slot uses there.
// Scales of the tangent operands come from bounds, not typical values (the direction's magnitude changes from one CG
// iteration to the next): |T1| <= n_in max|X| max|V1| + max|vb1| and so on; two products that accumulate into one
// accumulator memory region (T1 W2^T + H1 V2^T) must share ONE scale, so the pair (scale of T1, scale of V2) is chosen with
// e_T1 + e_W2 = 14 + e_V2 and both inside their ranges.
#include <cuda_fp16.h>

#include <cmath>

#include "common.cuh"
#include "policy_head.cuh"
#include "tc2_common.cuh"
#include "tc_common.cuh"

namespace b200rl {

constexpr int FV_ROWS = 128;
constexpr int FV_EPI_WARPS = 16;  // 4 lane groups x 4 column groups of 16 (8 warps with 32 columns each measured slower on B200)
constexpr int FV_EPI_THREADS = FV_EPI_WARPS * 32;
constexpr int FV_THREADS = FV_EPI_THREADS + 128;  // + the issuing warpgroup

// shared-memory map (bytes from the 1024-aligned base)
constexpr uint32_t FV_W1T = 32 * 128, FV_W = 64 * 128, FV_W3 = 16 * 128;  // one split each
constexpr uint32_t SF_XD = 0, SF_H1 = 2 * T2_ACT, SF_H2 = 4 * T2_ACT, SF_T1 = 6 * T2_ACT, SF_T2 = 8 * T2_ACT;
constexpr uint32_t SF_W1T = 10 * T2_ACT;
constexpr uint32_t SF_W2 = SF_W1T + 2 * FV_W1T;
constexpr uint32_t SF_W3 = SF_W2 + 2 * FV_W;
constexpr uint32_t SF_V1T = SF_W3 + 2 * FV_W3;
constexpr uint32_t SF_V2 = SF_V1T + 2 * FV_W1T;
constexpr uint32_t SF_V3 = SF_V2 + 2 * FV_W;
constexpr uint32_t SF_OPERANDS_END = SF_V3 + 2 * FV_W3;
constexpr uint32_t SF_BIAS = SF_OPERANDS_END;   // b1[64] b2[64] b3[16] | vb1[64] vb2[64] vb3[16] floats
constexpr uint32_t SF_DIST = SF_BIAS + 1152;    // 1/var[16] floats
constexpr uint32_t SF_SCALE = SF_DIST + 64;     // scale factors
constexpr uint32_t SF_RED = SF_SCALE + 128;     // block reduction scratch [20 warps][8] floats (read-out: [4][16] + 4 + 4)
constexpr uint32_t SF_BARS = SF_RED + 640;      // mbarriers ready, chain, off; bad flag
constexpr uint32_t SF_XS = SF_BARS + 64;        // per-feature observation scales [32] and inverses [32]
constexpr uint32_t SF_ROWMAX = SF_XS + 256;     // [128] largest scaled |obs| of each row (precision guard)
constexpr uint32_t SF_TOTAL = SF_ROWMAX + 512;
constexpr uint32_t FV_SMEM_BYTES = SF_TOTAL + 1024;
static_assert(FV_SMEM_BYTES <= 227 * 1024, "mlp_tc_fvp shared memory");

// accumulator columns
constexpr uint32_t ACC_Z1 = 0, ACC_ZB = 64, ACC_OUT = 128, ACC_TZ = 144, ACC_TOUT = 208;
constexpr uint32_t ACC_DW2 = 288, ACC_DW1 = 352, ACC_DW3 = 400, ACC_DB2 = 416;

enum {
  FS_X = 0, FS_G, FS_U1, FS_U2, FS_U3, FS_UT1, FS_UT2, FS_UT3, FS_T1, FS_T2, FS_UH2, FS_UH1, FS_OW3, FS_OW2, FS_OW1,
  FS_OB, FS_W1, FS_W2, FS_W3, FS_V1, FS_V2, FS_V3, FS_N
};

struct FvpArgs {
  int n_in, n_out, h1, h2;
  int w_off[3], b_off[3], P;
  int dist;
  long long n_rows;
  float inv_n, n_glob_f;
  const float* params;
  const float* direction;
  const float* obs;
  const float* log_std;
  float* partials;
  double* scalar_partials;
  const int* skip_flag;
  const float* obs_absmax;  // device [n_in]: per-feature max |obs|
  unsigned* status;
  unsigned seq;
  int total_rows;  // partial rows the consumer reduces (>= 2 * gridDim.x); the surplus is zeroed
  float* acc_mem;  // accumulator memory, ACC_CTA_FLOATS per CTA (tc_common.cuh)
};

__global__ void __launch_bounds__(FV_THREADS, 1) mlp_tc_fvp_kernel(const FvpArgs p) {
  extern __shared__ uint8_t smem_raw[];
  if (p.skip_flag != nullptr && *p.skip_flag != 0) return;

  const int tid = threadIdx.x, lane = tid & 31;
  float* const acc = p.acc_mem + (size_t)blockIdx.x * ACC_CTA_FLOATS;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);  // provably warp-uniform: role branches need no vote
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* sm = smem_raw + (base - raw);
  float* s_bias = reinterpret_cast<float*>(sm + SF_BIAS);
  float* s_vb = s_bias + 144;
  float* s_ivar = reinterpret_cast<float*>(sm + SF_DIST);
  float* s_scale = reinterpret_cast<float*>(sm + SF_SCALE);
  float* s_red = reinterpret_cast<float*>(sm + SF_RED);
  int* s_bad = reinterpret_cast<int*>(sm + SF_BARS + 48);
  const uint32_t bars = base + SF_BARS;  // ready +0, chain +8, off +16
  const int n_in = p.n_in, A_out = p.n_out, h1 = p.h1, h2 = p.h2;
  bool bad = false;

  // partial rows beyond this grid's 2 per CTA contribute nothing
  for (int row = 2 * (int)gridDim.x + (int)blockIdx.x; row < p.total_rows; row += (int)gridDim.x) {
    for (int i = tid; i < p.P; i += FV_THREADS) p.partials[(size_t)row * p.P + i] = 0.f;
    if (p.scalar_partials != nullptr && tid < B200RL_N_SCALARS) p.scalar_partials[(size_t)row * B200RL_N_SCALARS + tid] = 0.0;
  }

  // ---- setup: zero operand buffers; max |.| of the three weight matrices of params and of the direction ----
  for (uint32_t i = tid; i < SF_OPERANDS_END / 16; i += FV_THREADS) reinterpret_cast<uint4*>(sm)[i] = make_uint4(0, 0, 0, 0);
  if (tid == 0) *s_bad = 0;
  // per-feature observation scales (see mlp_tc2.cu): X_s[:,k] = X[:,k] 2^ex_k, 2^-ex_k folded into column k of W1 / V1
  float* s_xs = reinterpret_cast<float*>(sm + SF_XS);
  float* s_rowmax = reinterpret_cast<float*>(sm + SF_ROWMAX);
  if (tid < 32) {
    bool bx = false;
    const int e = tid < n_in ? fit_exp(__ldg(p.obs_absmax + tid), bx) : 0;
    s_xs[tid] = pow2i(e);
    s_xs[32 + tid] = pow2i(-e);
    if (bx) bad = true;
  }
  for (int i = tid; i < 128; i += FV_THREADS) s_rowmax[i] = 0.f;
  __syncthreads();
  {
    float mx[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};  // W1' W2 W3 V1' V2 V3 vb(all) unused
    auto scan = [&](const float* src, int n, float& m) {
      for (int idx = tid; idx < n; idx += FV_THREADS) {
        const float w = __ldg(src + idx);
        m = fmaxf(m, fabsf(w));
        if (w != w) bad = true;
      }
    };
    auto scan1 = [&](const float* src, float& m) {  // first layer: column k carries 2^-ex_k
      for (int idx = tid; idx < h1 * n_in; idx += FV_THREADS) {
        const float w = __ldg(src + idx) * s_xs[32 + idx % n_in];
        m = fmaxf(m, fabsf(w));
        if (w != w) bad = true;
      }
    };
    scan1(p.params + p.w_off[0], mx[0]);
    scan(p.params + p.w_off[1], h2 * h1, mx[1]);
    scan(p.params + p.w_off[2], A_out * h2, mx[2]);
    scan1(p.direction + p.w_off[0], mx[3]);
    scan(p.direction + p.w_off[1], h2 * h1, mx[4]);
    scan(p.direction + p.w_off[2], A_out * h2, mx[5]);
    scan(p.direction + p.b_off[0], h1, mx[6]);
    scan(p.direction + p.b_off[1], h2, mx[6]);
    scan(p.direction + p.b_off[2], A_out, mx[6]);
#pragma unroll
    for (int k = 0; k < 7; ++k) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mx[k] = fmaxf(mx[k], __shfl_xor_sync(0xffffffffu, mx[k], o));
      if (lane == 0) s_red[warp * 8 + k] = mx[k];
    }
  }
  __syncthreads();
  if (bad) *s_bad = 1;
  bad = false;
  if (tid == 0) {
    float mx[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int w = 0; w < FV_THREADS / 32; ++w)
      for (int k = 0; k < 7; ++k) mx[k] = fmaxf(mx[k], s_red[w * 8 + k]);
    bool b0 = false;
    const float xmax = 8192.f;  // every scaled observation feature is below 2^13
    const int ew1 = fit_exp(mx[0], b0), ew2 = fit_exp(mx[1], b0), ew3 = fit_exp(mx[2], b0);
    const int ev1 = fit_exp(mx[3], b0);
    const int ev2_max = fit_exp(mx[4], b0), ev3_max = fit_exp(mx[5], b0);
    // bounds of the tangents (|1 - H^2| <= 1, |H| <= 1) and the exponents that keep them below 2^14
    const float vbm = mx[6];
    const float B1 = (float)n_in * xmax * mx[3] + vbm;
    const float B2 = 64.f * (B1 * mx[1] + mx[4]) + vbm;
    const float B3 = 64.f * (B2 * mx[2] + mx[5]) + vbm;
    auto cap = [&](float b) { return (b > 0.f && b < INFINITY) ? 13 - ilogbf(b) : 0; };  // b * 2^e < 2^14
    if (!(B3 < INFINITY)) b0 = true;
    // common accumulator scales of the two-product sums
    const int c2 = min(cap(B1) + ew2, T2_H_EXP + ev2_max), c3 = min(cap(B2) + ew3, T2_H_EXP + ev3_max);
    const int et1 = c2 - ew2, ev2 = c2 - T2_H_EXP, et2 = c3 - ew3, ev3 = c3 - T2_H_EXP;
    s_scale[FS_U1] = pow2i(-ew1);
    s_scale[FS_U2] = pow2i(-(T2_H_EXP + ew2));
    s_scale[FS_U3] = pow2i(-(T2_H_EXP + ew3));
    s_scale[FS_UT1] = pow2i(-ev1);
    s_scale[FS_UT2] = pow2i(-c2);
    s_scale[FS_UT3] = pow2i(-c3);
    s_scale[FS_T1] = pow2i(et1);
    s_scale[FS_T2] = pow2i(et2);
    s_scale[FS_UH2] = pow2i(-ew3);
    s_scale[FS_UH1] = pow2i(-ew2);
    s_scale[FS_OW1] = 1.f;  // completed with the gradient scale once it is known (first tile, below); the column's
                            // 2^-ex_k is applied when the accumulator is read
    s_scale[FS_W1] = pow2i(ew1);
    s_scale[FS_W2] = pow2i(ew2);
    s_scale[FS_W3] = pow2i(ew3);
    s_scale[FS_V1] = pow2i(ev1);
    s_scale[FS_V2] = pow2i(ev2);
    s_scale[FS_V3] = pow2i(ev3);
    if (b0) *s_bad = 1;
  }
  __syncthreads();
  {
    auto put = [&](uint32_t buf, uint32_t stride, int r, int c, float x) {
      const __half hb = __float2half_rn(x);
      const __half lb = __float2half_rn(x - __half2float(hb));
      const uint32_t off = buf + (uint32_t)r * 128u + ((uint32_t)((c >> 3) ^ (r & 7)) << 4) + ((uint32_t)(c & 7) << 1);
      *reinterpret_cast<__half*>(sm + off) = hb;
      *reinterpret_cast<__half*>(sm + off + stride) = lb;
    };
    for (int pass = 0; pass < 2; ++pass) {  // params -> W buffers, direction -> V buffers
      const float* src = pass == 0 ? p.params : p.direction;
      const float s1 = s_scale[pass == 0 ? FS_W1 : FS_V1], s2 = s_scale[pass == 0 ? FS_W2 : FS_V2],
                  s3 = s_scale[pass == 0 ? FS_W3 : FS_V3];
      const uint32_t b1 = pass == 0 ? SF_W1T : SF_V1T, b2 = pass == 0 ? SF_W2 : SF_V2, b3 = pass == 0 ? SF_W3 : SF_V3;
      for (int idx = tid; idx < h1 * n_in; idx += FV_THREADS)  // first layer stored transposed: row = input
        put(b1, FV_W1T, idx % n_in, idx / n_in, (__ldg(src + p.w_off[0] + idx) * s_xs[32 + idx % n_in]) * s1);
      for (int idx = tid; idx < h2 * h1; idx += FV_THREADS)
        put(b2, FV_W, idx / h1, idx % h1, __ldg(src + p.w_off[1] + idx) * s2);
      for (int idx = tid; idx < A_out * h2; idx += FV_THREADS)
        put(b3, FV_W3, idx / h2, idx % h2, __ldg(src + p.w_off[2] + idx) * s3);
      float* bias = pass == 0 ? s_bias : s_vb;
      for (int i = tid; i < 64; i += FV_THREADS) {
        bias[i] = i < h1 ? __ldg(src + p.b_off[0] + i) : 0.f;
        bias[64 + i] = i < h2 ? __ldg(src + p.b_off[1] + i) : 0.f;
        if (!(fabsf(bias[i]) < INFINITY) || !(fabsf(bias[64 + i]) < INFINITY)) bad = true;
      }
      for (int i = tid; i < 16; i += FV_THREADS) {
        bias[128 + i] = i < A_out ? __ldg(src + p.b_off[2] + i) : 0.f;
        if (!(fabsf(bias[128 + i]) < INFINITY)) bad = true;
      }
    }
    if (p.dist == B200RL_DIST_GAUSSIAN)
      for (int a = tid; a < 16; a += FV_THREADS) s_ivar[a] = a < A_out ? normal_consts(p.log_std, a).inv_var : 1.f;
  }
  if (bad) *s_bad = 1;  // non-finite bias
  bad = false;
  if (tid == 0) {
    mbar_init(bars, FV_EPI_THREADS);
    mbar_init(bars + 8, 1);
    mbar_init(bars + 16, 1);
    fence_mbar_init();
  }
  fence_proxy_async_smem();
  __syncthreads();
  const long long num_tiles = (p.n_rows + FV_ROWS - 1) / FV_ROWS;
  const long long cta_tiles = (num_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x;

  if (warp >= FV_EPI_WARPS) {
    // =============================== MMA issuer warpgroup ============================================
    constexpr int K = K_MAJOR, MN = MN_MAJOR;
    const uint32_t ub = base;
    const Op2 XD_K = op2_kmajor(ub + SF_XD, T2_ACT), H1_K = op2_kmajor(ub + SF_H1, T2_ACT),
              H2_K = op2_kmajor(ub + SF_H2, T2_ACT), T1_K = op2_kmajor(ub + SF_T1, T2_ACT),
              T2_K = op2_kmajor(ub + SF_T2, T2_ACT), XD_K2 = op2_kmajor(ub + SF_XD + 64, T2_ACT);
    const Op2 H2_M = op2_mnmajor(ub + SF_H2, T2_ACT, T2_ACT), H1_M = op2_mnmajor(ub + SF_H1, T2_ACT, T2_ACT),
              XD_M0 = op2_mnmajor(ub + SF_XD, T2_ACT, T2_ACT), XD_M32 = op2_mnmajor(ub + SF_XD + 64, T2_ACT, T2_ACT);
    const Op2 W1T_M = op2_mnmajor(ub + SF_W1T, 32 * 128, FV_W1T), W2_K = op2_kmajor(ub + SF_W2, FV_W),
              W3_K = op2_kmajor(ub + SF_W3, FV_W3), W2_M = op2_mnmajor(ub + SF_W2, 64 * 128, FV_W),
              W3_M = op2_mnmajor(ub + SF_W3, 16 * 128, FV_W3);
    const Op2 V1T_M = op2_mnmajor(ub + SF_V1T, 32 * 128, FV_W1T), V2_K = op2_kmajor(ub + SF_V2, FV_W),
              V3_K = op2_kmajor(ub + SF_V3, FV_W3);
    uint32_t par = 0u;
    bool accum = false;
    for (long long k = 0; k < cta_tiles; ++k) {
#pragma unroll 1
      for (int stage = 0; stage < 6; ++stage) {
        mbar_wait(bars, par);
        par ^= 1u;
        // issue_chain3 <N, B major, k-steps[, accumulate]>, issue_stacked <N, k-steps, B splits>
        if (stage == 0) {  // Z1 = X W1^T ; TZ = X V1^T
          issue_chain3<64, MN, 2>(acc, ACC_Z1, XD_K, W1T_M);
          issue_chain3<64, MN, 2>(acc, ACC_TZ, XD_K, V1T_M);
          acc_commit(bars + 8);
        } else if (stage == 1) {  // Z2 = H1 W2^T ; TZ = T1 W2^T + H1 V2^T
          issue_chain3<64, K, 4>(acc, ACC_ZB, H1_K, W2_K);
          issue_chain3<64, K, 4>(acc, ACC_TZ, T1_K, W2_K);
          issue_chain3<64, K, 4, true>(acc, ACC_TZ, H1_K, V2_K);
          acc_commit(bars + 8);
        } else if (stage == 2) {  // OUT = H2 W3^T ; TOUT = T2 W3^T + H2 V3^T
          issue_chain3<16, K, 4>(acc, ACC_OUT, H2_K, W3_K);
          issue_chain3<16, K, 4>(acc, ACC_TOUT, T2_K, W3_K);
          issue_chain3<16, K, 4, true>(acc, ACC_TOUT, H2_K, V3_K);
          acc_commit(bars + 8);
        } else if (stage == 3) {  // dH2 = dOut W3 ; dW3^T += H2^T dOut (must retire before H2 becomes dZ2)
          issue_chain3<64, MN, 1>(acc, ACC_ZB, XD_K2, W3_M);
          issue_stacked<16, 8, 2>(acc, ACC_DW3, accum, H2_M, XD_M32);
          acc_commit(bars + 8);
        } else if (stage == 4) {  // dH1 = dZ2 W2 ; dW2 += dZ2^T H1 ; db2 += dZ2^T 1
          issue_chain3<64, MN, 4>(acc, ACC_ZB, H2_K, W2_M);
          issue_stacked<64, 8, 2>(acc, ACC_DW2, accum, H2_M, H1_M);
          issue_stacked<16, 8, 1>(acc, ACC_DB2, accum, H2_M, XD_M32);
          acc_commit(bars + 8);
        } else {  // dW1 += dZ1^T X, db1 through the ones column
          issue_stacked<48, 8, 2>(acc, ACC_DW1, accum, H1_M, XD_M0);
          acc_commit(bars + 16);
          accum = true;
        }
        __syncwarp();
      }
    }
  } else {
    // =============================== epilogue warps ==================================================
    const int q = warp & 3, half = warp >> 2;  // lane group, column group (16 columns each)
    const int r = 32 * q + lane;  // row of the tile == accumulator row
    const int cs = 16 * half;
    uint32_t ph_chain = 0, ph_off = 0;
    const float sH = pow2i(T2_H_EXP);
    float sG = 0.f;  // gradient scale: set from the first tile's dOut (every CTA owns its accumulators, so the scale
                     // may differ between CTAs; the partial rows leave the kernel in true units)
    double rows_done = 0.0;
    float db3[15];
#pragma unroll
    for (int a = 0; a < 15; ++a) db3[a] = 0.f;

    auto epi_arrive = [&]() {
      fence_proxy_async_smem();
      mbar_arrive(bars);
    };
    auto wait_chain = [&]() {
      mbar_wait(bars + 8, ph_chain);
      ph_chain ^= 1u;
    };
    // forward + tangent epilogue of a tanh layer: H = tanh(Z u + b) -> fp16 splits (and fp32 to accumulator memory when kept);
    // T = (1 - H^2) (TZ ut + vb) -> fp16 splits of the tangent buffer
    auto layer_epilogue = [&](uint32_t acc_z, const float* bias, const float* vbias, float unscale, float unscale_t,
                              float t_scale, uint32_t dst_h, uint32_t dst_t, bool keep_fp32) {
      {
        float z[16], w[16];
        acc_ld<16>(acc, r, acc_z + cs, z);
        acc_ld<16>(acc, r, ACC_TZ + cs, w);
#pragma unroll
        for (int j = 0; j < 16; ++j) z[j] = fmaf(z[j], unscale, bias[cs + j]);
        tanh16_scaled(z, 1.f);  // Z is finite: observations, weights and biases were all checked
        if (keep_fp32) acc_st<16>(acc, r, acc_z + cs, z);
#pragma unroll
        for (int ch = 0; ch < 2; ++ch) {
          float x[8], t[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float h = z[8 * ch + j];
            x[j] = h * sH;
            t[j] = (fmaf(w[8 * ch + j], unscale_t, vbias[cs + 8 * ch + j]) * fmaf(-h, h, 1.f)) * t_scale;
          }
          if (out_of_range8(t)) bad = true;
          store_chunk2(sm, dst_h, r, (cs >> 3) + ch, x);
          store_chunk2(sm, dst_t, r, (cs >> 3) + ch, t);
        }
      }
    };

    bool first = true;
    for (long long k = 0; k < cta_tiles; ++k) {
      const long long tile = blockIdx.x + k * gridDim.x;
      const long long row = tile * FV_ROWS + r;
      const bool valid = row < p.n_rows;
      {  // E0: observations
        float x0[8];
        const float* src = p.obs + row * n_in + 8 * half;
#pragma unroll
        for (int j = 0; j < 8; ++j) x0[j] = (valid && 8 * half + j < n_in) ? __ldg(src + j) : 0.f;
        if (!first) {
          mbar_wait(bars + 16, ph_off);
          ph_off ^= 1u;
        }
        first = false;
        float rmax = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          x0[j] *= s_xs[8 * half + j];
          rmax = fmaxf(rmax, fabsf(x0[j]));
        }
        atomicMax(reinterpret_cast<int*>(s_rowmax + r), __float_as_int(rmax));
        if (out_of_range8(x0)) bad = true;
        store_chunk2(sm, SF_XD, r, half, x0);
      }
#pragma unroll 1
      for (int layer = 0; layer < 2; ++layer) {  // one copy of the (large) layer epilogue: instruction-cache pressure
        epi_arrive();
        wait_chain();
        layer_epilogue(layer == 0 ? ACC_Z1 : ACC_ZB, s_bias + 64 * layer, s_vb + 64 * layer,
                       s_scale[layer == 0 ? FS_U1 : FS_U2], s_scale[layer == 0 ? FS_UT1 : FS_UT2],
                       s_scale[layer == 0 ? FS_T1 : FS_T2], layer == 0 ? SF_H1 : SF_H2, layer == 0 ? SF_T1 : SF_T2,
                       layer == 0);
      }
      epi_arrive();
      wait_chain();
      // ---- metric epilogue: dOut = M (J v) / N, one row per thread ----
      if (half == 0) {
        {  // precision guard (see mlp_tc2.cu)
          const float rm = s_rowmax[r];
          s_rowmax[r] = 0.f;
          if (valid && rm > 0.f && rm < 0.03125f) bad = true;
        }
        float o[16], t[16];
        acc_ld<16>(acc, r, ACC_OUT, o);
        acc_ld<16>(acc, r, ACC_TOUT, t);
        float dout[16];
#pragma unroll
        for (int a = 0; a < 16; ++a) dout[a] = 0.f;
        if (valid) {
          float tout[16];
          const float ut3 = s_scale[FS_UT3];
#pragma unroll
          for (int a = 0; a < 16; ++a) tout[a] = fmaf(t[a], ut3, s_vb[128 + a]);
          if (p.dist == B200RL_DIST_GAUSSIAN) {
            gaussian_metric<15>(tout, VarRecip{s_ivar, nullptr}, A_out, p.inv_n, dout);
          } else {
            float out[16];
            const float u3 = s_scale[FS_U3];
#pragma unroll
            for (int a = 0; a < 16; ++a) out[a] = fmaf(o[a], u3, s_bias[128 + a]);
            categorical_metric<15>(out, tout, A_out, p.inv_n, dout);
          }
          rows_done += 1.0;
        }
        if (k == 0) {
          // 2^eg maps this tile's max |dOut| to ~2^9: 2^6 of head room for later tiles and for the back-propagated
          // dZ, typical entries well inside fp16's normal range; anything larger trips the range check
          float m = 0.f;
#pragma unroll
          for (int a = 0; a < 15; ++a) m = fmaxf(m, fabsf(dout[a]));
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
          if (lane == 0) s_red[72 + q] = m;
          asm volatile("bar.sync 3, 128;" ::: "memory");
          m = fmaxf(fmaxf(s_red[72], s_red[73]), fmaxf(s_red[74], s_red[75]));
          int eg = (m > 0.f && m < INFINITY) ? 9 - ilogbf(m) : 0;
          eg = eg < -100 ? -100 : (eg > 100 ? 100 : eg);
          sG = pow2i(eg);
          if (tid == 0) {
            s_scale[FS_OW3] = pow2i(-(T2_H_EXP + eg));
            s_scale[FS_OW2] = pow2i(-(T2_H_EXP + eg));
            s_scale[FS_OW1] = s_scale[FS_OW1] * pow2i(-eg);
            s_scale[FS_OB] = pow2i(-eg);
          }
        }
        float x0[8], x1[8];
#pragma unroll
        for (int a = 0; a < 15; ++a) db3[a] += dout[a];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          x0[j] = dout[j] * sG;
          x1[j] = j < 7 ? dout[8 + j] * sG : 1.0f;  // ones column: db1 / db2 fall out of the dW products
        }
        if (out_of_range8(x0) || out_of_range8(x1)) bad = true;
        store_chunk2(sm, SF_XD, r, 4, x0);
        store_chunk2(sm, SF_XD, r, 5, x1);
      }
      epi_arrive();
      wait_chain();  // dH2 (and dW3)
      {
        const float unscale = s_scale[FS_UH2], hh = pow2i(-2 * T2_H_EXP);
        {
          float g[16];
          acc_ld<16>(acc, r, ACC_ZB + cs, g);
#pragma unroll
          for (int ch = 0; ch < 2; ++ch) {
            float x[8];
            load_chunk2(sm, SF_H2, r, (cs >> 3) + ch, x);
#pragma unroll
            for (int j = 0; j < 8; ++j)
              x[j] = (g[8 * ch + j] * unscale) * fmaf(-(x[j] * hh), x[j], 1.f);
            if (too_large8(x)) bad = true;
            store_chunk2(sm, SF_H2, r, (cs >> 3) + ch, x);
          }
        }
      }
      epi_arrive();
      wait_chain();  // dH1 (and dW2 / db2)
      {
        const float unscale = s_scale[FS_UH1];
        {
          float g[16], h[16];
          acc_ld<16>(acc, r, ACC_ZB + cs, g);
          acc_ld<16>(acc, r, ACC_Z1 + cs, h);
#pragma unroll
          for (int ch = 0; ch < 2; ++ch) {
            float x[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const float hv = h[8 * ch + j];
              x[j] = (g[8 * ch + j] * unscale) * (1.f - hv * hv);
            }
            if (too_large8(x)) bad = true;
            store_chunk2(sm, SF_H1, r, (cs >> 3) + ch, x);
          }
        }
      }
      epi_arrive();
    }

    // ---- per-CTA results ----
    if (!first) mbar_wait(bars + 16, ph_off);
    {
      float* dst = p.partials + ((size_t)blockIdx.x * 2 + (q >> 1)) * p.P;
      const int m = 32 * (q & 1) + lane;
      float v[16];
      // column groups 0, 1: dW2 (32 columns each); 2: dW1 + db1; 3: dW3^T, db2
      if (half < 2) {
#pragma unroll
        for (int c2 = 0; c2 < 2; ++c2) {
          const int cb = 2 * half + c2;
          acc_ld<16>(acc, r, ACC_DW2 + 16 * cb, v);
          const float u = s_scale[FS_OW2];
          if (m < h2)
#pragma unroll
            for (int j = 0; j < 16; ++j)
              if (16 * cb + j < h1) dst[p.w_off[1] + m * h1 + 16 * cb + j] = v[j] * u;
        }
      } else if (half == 2) {
#pragma unroll
        for (int cb = 0; cb < 3; ++cb) {
          acc_ld<16>(acc, r, ACC_DW1 + 16 * cb, v);
          if (m < h1) {
            if (cb < 2) {
              const float u = s_scale[FS_OW1];
#pragma unroll
              for (int j = 0; j < 16; ++j)
                if (16 * cb + j < n_in)
                  dst[p.w_off[0] + m * n_in + 16 * cb + j] = (v[j] * u) * s_xs[32 + 16 * cb + j];
            } else {
              dst[p.b_off[0] + m] = v[15] * s_scale[FS_OB];
            }
          }
        }
      } else {
        acc_ld<16>(acc, r, ACC_DW3, v);
        const float u = s_scale[FS_OW3];
        if (m < h2)
#pragma unroll
          for (int a = 0; a < 15; ++a)
            if (a < A_out) dst[p.w_off[2] + a * h2 + m] = v[a] * u;
        acc_ld<16>(acc, r, ACC_DB2, v);
        if (m < h2) dst[p.b_off[1] + m] = v[15] * s_scale[FS_OB];
      }
      if (half == 0) {
#pragma unroll
        for (int a = 0; a < 15; ++a) {
          float s = db3[a];
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
          if (lane == 0) s_red[q * 16 + a] = s;
        }
        const double rd = warp_sum(rows_done);
        if (lane == 0) s_red[64 + q] = (float)rd;  // <= 128 * tiles rows: exact in fp32
      }
    }
    asm volatile("bar.sync 2, %0;" ::"n"(FV_EPI_THREADS) : "memory");
    if (tid < A_out) {
      float s = 0.f;
      for (int w4 = 0; w4 < 4; ++w4) s += s_red[w4 * 16 + tid];
      p.partials[((size_t)blockIdx.x * 2) * p.P + p.b_off[2] + tid] = s;
      p.partials[((size_t)blockIdx.x * 2 + 1) * p.P + p.b_off[2] + tid] = 0.f;
    }
    if (p.scalar_partials != nullptr && tid < B200RL_N_SCALARS) {
      double t = 0.0;
      if (tid == 5)
        for (int w4 = 0; w4 < 4; ++w4) t += (double)s_red[64 + w4];
      p.scalar_partials[((size_t)blockIdx.x * 2) * B200RL_N_SCALARS + tid] = t;
      p.scalar_partials[((size_t)blockIdx.x * 2 + 1) * B200RL_N_SCALARS + tid] = 0.0;
    }
    if (bad) *s_bad = 1;
  }

  __syncthreads();
  if (tid == 0 && *s_bad != 0) *p.status = p.seq;  // redone by the fp32 kernel queued behind this launch
}

// ---- host side -------------------------------------------------------------------------------------------------
int tc2_take_slot(unsigned** status, unsigned* seq, float** scratch);
int launch_absmax_cols(const float* x, long long rows, int cols, float* out, cudaStream_t s);
int launch_fused_fallback(const b200rl_mlp_loss_grad_args* a, const unsigned* run_if, unsigned seq, int total_rows,
                          cudaStream_t s);

int launch_mlp_tc_fvp(const b200rl_mlp_loss_grad_args* a, int64_t n_glob, int total_rows, cudaStream_t s) {
  static bool configured = false;
  if (!configured) {
    B200RL_CUDA(cudaFuncSetAttribute(mlp_tc_fvp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FV_SMEM_BYTES));
    configured = true;
  }
  unsigned* status = nullptr;
  unsigned seq = 0;
  float* scratch = nullptr;
  if (tc2_take_slot(&status, &seq, &scratch)) return 1;
  FvpArgs k{};
  k.n_in = a->mlp.sizes[0];
  k.h1 = a->mlp.sizes[1];
  k.h2 = a->mlp.sizes[2];
  k.n_out = a->mlp.sizes[3];
  k.P = mlp3_offsets(a->mlp, k.w_off, k.b_off);
  k.dist = a->dist;
  k.n_rows = a->n_rows;
  k.inv_n = 1.0f / (float)n_glob;
  k.n_glob_f = (float)n_glob;
  k.params = a->params;
  k.direction = a->direction;
  k.obs = a->obs;
  k.log_std = a->log_std;
  k.partials = a->partials;
  k.scalar_partials = a->scalar_partials;
  k.skip_flag = a->skip_flag;
  k.status = status;
  k.seq = seq;
  k.total_rows = total_rows;
  if (a->obs_absmax == nullptr) {
    B200RL_CUDA(cudaMemsetAsync(scratch, 0, 32 * sizeof(float), s));
    if (launch_absmax_cols(a->obs, a->n_rows, k.n_in, scratch, s)) return 1;
    k.obs_absmax = scratch;
  } else {
    k.obs_absmax = a->obs_absmax;
  }
  const int grid = tc_grid(a->n_rows);
  B200RL_REQUIRE(grid > 0, "mlp_tc_fvp: no CUDA device");
  k.acc_mem = acc_mem(grid, s);
  B200RL_REQUIRE(k.acc_mem != nullptr, "mlp_tc_fvp: no accumulator memory (allocation failed, or the stream is being captured): %s",
                 cudaGetErrorString(cudaGetLastError()));
  mlp_tc_fvp_kernel<<<grid, FV_THREADS, FV_SMEM_BYTES, s>>>(k);
  B200RL_CUDA(cudaGetLastError());
  count_launch(1);
  return launch_fused_fallback(a, status, seq, total_rows, s);
}

}  // namespace b200rl
