// mlp_tc: the fused MLP step on the tensor cores (wgmma), sm_90a.
//
// Same contract and data flow as mlp_fused.cu (see there for the reference file:line map); this kernel is selected
// for the shapes the reference's on-policy recipes use: 3 Linear layers, hidden widths 64/64, tanh hidden,
// identity output, obs width <= 32, output width <= 15.  Everything else takes the fp32 kernel.
//
// Precision: the tensor cores have no fp32 MMA and plain TF32 violates the 1e-5 parity bar, so every fp32
// operand is split into THREE bf16 values x = h + m + l (24 mantissa bits) and every logical product is the six
// bf16 wgmma products  mm + hl + lh + hm + mh + hh  with fp32 accumulation -- 2^-24-grade relative error per
// product, which the golden / oracle parity tests hold to 1e-5.  bf16 (not tf32) because a SWIZZLE_128B buffer of 16-bit elements can
// be read BOTH K-major (activations as the A operand of the next layer) and MN-major (the same activations as an
// operand of the dW = dZ^T X product, whose reduction runs over the tile's rows); tf32 MN-major needs a different
// swizzle, i.e. a second copy of every activation .
//
// Per CTA: 128-row tiles, persistent over tiles (grid = min(#tiles, #SMs)), 8 epilogue warps + 1 MMA-issuing warpgroup.
//   shared memory  operand buffers, 64 bf16 columns x 128-byte rows, SWIZZLE_128B, three splits each:
//                  XD [128][64]: obs in cols 0..31, dOut in cols 32..46, ones in col 47 (bias gradients for free)
//                  H1, H2 [128][64]: activations, overwritten in place by dZ1 / dZ2 during the backward pass
//                  W1, W2 [64][64], W3 [16][64]: torch [out][in] order = K-major B operand in the forward pass and,
//                  unchanged, MN-major B operand of dX = dZ W in the backward pass
//   accumulator memory  Z1/H1, Z2/H2 (fp32, kept for tanh'), OUT, dH2, dH1 (M = 128) and the per-CTA gradient
//                  accumulators dW2, dW1, dW3^T, db2, db1 (M = 64) that persist across the CTA's tiles.
//   stages / tile  X -> [F1] -> tanh -> [F2] -> tanh -> [F3] -> log-prob/loss/dOut -> [dW3^T, dH2] -> dZ2 ->
//                  [dW2, db2, dH1] -> dZ1 -> [dW1, db1]; one acc_commit + mbarrier wait per bracketed stage.
#include <cuda_bf16.h>

#include <cmath>

#include "common.cuh"
#include "policy_head.cuh"
#include "tc_common.cuh"

namespace b200rl {

constexpr int TC_ROWS = 128;
constexpr int TC_EPI_WARPS = 8;
constexpr int TC_THREADS = TC_EPI_WARPS * 32 + 128;  // + the issuing warpgroup

// shared-memory map (bytes from the 1024-aligned base)
constexpr uint32_t ACT_BUF = 128 * 128;  // one split of a [128][64] bf16 buffer
constexpr uint32_t W_BUF = 64 * 128;     // one split of a [64][64] weight
constexpr uint32_t W3_BUF = 16 * 128;    // one split of the [16][64] output weight
constexpr uint32_t SM_XD = 0;
constexpr uint32_t SM_H1 = SM_XD + 3 * ACT_BUF;
constexpr uint32_t SM_H2 = SM_H1 + 3 * ACT_BUF;
constexpr uint32_t SM_W1 = SM_H2 + 3 * ACT_BUF;
constexpr uint32_t SM_W2 = SM_W1 + 3 * W_BUF;
constexpr uint32_t SM_W3 = SM_W2 + 3 * W_BUF;
constexpr uint32_t SM_OPERANDS_END = SM_W3 + 3 * W3_BUF;
constexpr uint32_t SM_BIAS = SM_OPERANDS_END;       // b1[64] b2[64] b3[16] floats
constexpr uint32_t SM_DIST = SM_BIAS + 1024;        // var[16], log_scale[16] floats
constexpr uint32_t SM_DB3 = SM_DIST + 256;          // [4 warps][16] floats
constexpr uint32_t SM_STAGE = SM_DB3 + 512;         // fp32 staging of the NEXT tile's observations [128][n_in<=32]
constexpr uint32_t SM_TOTAL = SM_STAGE + 128 * 32 * 4;
constexpr uint32_t TC_SMEM_BYTES = SM_TOTAL + 1024;  // + alignment slack

// accumulator column map
constexpr uint32_t ACC_Z1 = 0, ACC_Z2 = 64, ACC_OUT = 128, ACC_DH2 = 160, ACC_DH1 = 224, ACC_DW2 = 288, ACC_DW1 = 352,
                   ACC_DW3 = 384, ACC_DB2 = 400, ACC_DB1 = 416;

struct TcArgs {
  int n_in, n_out;
  int h1, h2;  // hidden widths (<= 64, zero-padded to the 64-wide buffers)
  int w_off[3], b_off[3], P;
  int loss, dist;
  long long n_rows;
  float inv_n, clip_lo, clip_hi;
  const float* params;
  const float* obs;
  const float* actions;
  const float* log_std;
  const float* adv_raw;
  const double* adv_stats;
  const float* old_logp;
  const float* target;
  float* row_out;
  float* partials;
  double* scalar_partials;
  const int* skip_flag;
  const unsigned* run_if;  // when set: run only if *run_if == seq (wide-range re-run of an mlp_tc2 launch)
  unsigned seq;
  int total_rows;          // partial rows the consumer reduces (> gridDim.x when standing in for mlp_tc2)
  float* acc_mem;              // accumulator memory, ACC_CTA_FLOATS per CTA (tc_common.cuh)
};

// byte offset of element (r, c) inside one split buffer (c < 64)
__device__ __forceinline__ uint32_t rel_rc(int r, int c) {
  return (uint32_t)r * 128u + ((uint32_t)((c >> 3) ^ (r & 7)) << 4) + ((uint32_t)(c & 7) << 1);
}

__device__ __forceinline__ void split2(float x0, float x1, uint32_t& h, uint32_t& m, uint32_t& l) {
  const __nv_bfloat162 hb = __floats2bfloat162_rn(x0, x1);
  const float2 hf = __bfloat1622float2(hb);
  const float r0 = x0 - hf.x, r1 = x1 - hf.y;
  const __nv_bfloat162 mb = __floats2bfloat162_rn(r0, r1);
  const float2 mf = __bfloat1622float2(mb);
  const __nv_bfloat162 lb = __floats2bfloat162_rn(r0 - mf.x, r1 - mf.y);
  h = *reinterpret_cast<const uint32_t*>(&hb);
  m = *reinterpret_cast<const uint32_t*>(&mb);
  l = *reinterpret_cast<const uint32_t*>(&lb);
}

// write 8 consecutive columns (one 16-byte chunk `ch`) of row r into the three split buffers starting at `buf`
__device__ __forceinline__ void store_chunk3(uint8_t* sm, uint32_t buf, uint32_t split_stride, int r, int ch,
                                             const float (&x)[8]) {
  uint4 h, m, l;
  split2(x[0], x[1], h.x, m.x, l.x);
  split2(x[2], x[3], h.y, m.y, l.y);
  split2(x[4], x[5], h.z, m.z, l.z);
  split2(x[6], x[7], h.w, m.w, l.w);
  const uint32_t off = buf + (uint32_t)r * 128u + ((uint32_t)(ch ^ (r & 7)) << 4);
  *reinterpret_cast<uint4*>(sm + off) = h;
  *reinterpret_cast<uint4*>(sm + off + split_stride) = m;
  *reinterpret_cast<uint4*>(sm + off + 2 * split_stride) = l;
}

__device__ __forceinline__ void cp_async16(uint32_t smem_dst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_dst), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit_wait_all() {
  asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
}

// the six split products, smallest terms first: (m,m) (h,l) (l,h) (h,m) (m,h) (h,h)
template <int N, int TA, int TB, bool M64, int KSTEPS>
__device__ __forceinline__ void issue6(float* acc, uint32_t acc_col, bool accumulate_first, const Op2 a, const Op2 b) {
  const uint32_t alo[6] = {a.lo + a.split_step, a.lo, a.lo + 2 * a.split_step, a.lo, a.lo + a.split_step, a.lo};
  const uint32_t blo[6] = {b.lo + b.split_step, b.lo + 2 * b.split_step, b.lo, b.lo + b.split_step, b.lo, b.lo};
  mma_product<N, true, TA, TB, M64>(acc, acc_col, alo, blo, 6, a.hi, b.hi, a.k_step, b.k_step, KSTEPS, accumulate_first);
}
// A (three splits) times an operand that is exact in bf16 (the ones column, split 0 only): three products
template <int N, int TA, int TB, bool M64, int KSTEPS>
__device__ __forceinline__ void issue3(float* acc, uint32_t acc_col, bool accumulate_first, const Op2 a, const Op2 b) {
  const uint32_t alo[3] = {a.lo + 2 * a.split_step, a.lo + a.split_step, a.lo}, blo[3] = {b.lo, b.lo, b.lo};
  mma_product<N, true, TA, TB, M64>(acc, acc_col, alo, blo, 3, a.hi, b.hi, a.k_step, b.k_step, KSTEPS, accumulate_first);
}

#ifdef B200RL_TC_TIMING
__device__ unsigned long long g_tc_t[16];
#define TC_T(i)                                   \
  do {                                            \
    if (tid == 0) {                               \
      const long long _n = clock64();             \
      tacc[i] += (unsigned long long)(_n - tlast); \
      tlast = _n;                                 \
    }                                             \
  } while (0)
#else
#define TC_T(i)
#endif

__device__ unsigned long long g_tc_fallbacks;  // launches of this kernel that actually re-ran an mlp_tc2 launch

template <bool BACKWARD>
__global__ void __launch_bounds__(TC_THREADS, 1) mlp_tc_kernel(const TcArgs p) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) unsigned long long mbar;
  __shared__ double s_sc[6][TC_EPI_WARPS];
  if (p.skip_flag != nullptr && *p.skip_flag != 0) return;  // early stop: whole launch is a no-op
  if (p.run_if != nullptr && *p.run_if != p.seq) return;    // the fp16 kernel's result stands
  if (p.run_if != nullptr && blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(&g_tc_fallbacks, 1ull);

  const int tid = threadIdx.x, lane = tid & 31;
  float* const acc = p.acc_mem + (size_t)blockIdx.x * ACC_CTA_FLOATS;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);  // provably warp-uniform: role branches need no vote
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;  // SWIZZLE_128B atoms are 1024-byte aligned
  uint8_t* sm = smem_raw + (base - raw);
  float* s_bias = reinterpret_cast<float*>(sm + SM_BIAS);
  float* s_dist = reinterpret_cast<float*>(sm + SM_DIST);
  float* s_db3 = reinterpret_cast<float*>(sm + SM_DB3);
  const int n_in = p.n_in, A_out = p.n_out, h1 = p.h1, h2 = p.h2;
  // partial rows beyond this grid (the consumer was sized for mlp_tc2's two rows per CTA) contribute nothing
  for (int row = (int)gridDim.x + (int)blockIdx.x; row < p.total_rows; row += (int)gridDim.x) {
    if (BACKWARD)
      for (int i = tid; i < p.P; i += TC_THREADS) p.partials[(size_t)row * p.P + i] = 0.f;
    if (p.scalar_partials != nullptr && tid < B200RL_N_SCALARS) p.scalar_partials[(size_t)row * B200RL_N_SCALARS + tid] = 0.0;
  }

  // ---- one-time setup: zero operand buffers, stage W (three bf16 splits), biases, distribution constants ----
  for (uint32_t i = tid; i < SM_OPERANDS_END / 16; i += TC_THREADS) reinterpret_cast<uint4*>(sm)[i] = make_uint4(0, 0, 0, 0);
  __syncthreads();
  {
    auto put = [&](uint32_t buf, uint32_t stride, int r, int c, float x) {
      const __nv_bfloat16 hb = __float2bfloat16_rn(x);
      const float r1 = x - __bfloat162float(hb);
      const __nv_bfloat16 mb = __float2bfloat16_rn(r1);
      const __nv_bfloat16 lb = __float2bfloat16_rn(r1 - __bfloat162float(mb));
      const uint32_t off = buf + rel_rc(r, c);
      *reinterpret_cast<__nv_bfloat16*>(sm + off) = hb;
      *reinterpret_cast<__nv_bfloat16*>(sm + off + stride) = mb;
      *reinterpret_cast<__nv_bfloat16*>(sm + off + 2 * stride) = lb;
    };
    for (int idx = tid; idx < h1 * n_in; idx += TC_THREADS)
      put(SM_W1, W_BUF, idx / n_in, idx % n_in, __ldg(p.params + p.w_off[0] + idx));
    for (int idx = tid; idx < h2 * h1; idx += TC_THREADS)
      put(SM_W2, W_BUF, idx / h1, idx % h1, __ldg(p.params + p.w_off[1] + idx));
    for (int idx = tid; idx < A_out * h2; idx += TC_THREADS)
      put(SM_W3, W3_BUF, idx / h2, idx % h2, __ldg(p.params + p.w_off[2] + idx));
    for (int i = tid; i < 64; i += TC_THREADS) {
      s_bias[i] = i < h1 ? __ldg(p.params + p.b_off[0] + i) : 0.f;
      s_bias[64 + i] = i < h2 ? __ldg(p.params + p.b_off[1] + i) : 0.f;
    }
    for (int i = tid; i < 16; i += TC_THREADS) s_bias[128 + i] = i < A_out ? __ldg(p.params + p.b_off[2] + i) : 0.f;
    if (p.dist == B200RL_DIST_GAUSSIAN)
      for (int a = tid; a < A_out; a += TC_THREADS) {
        const NormalConsts c = normal_consts(p.log_std, a);
        s_dist[a] = c.var;
        s_dist[16 + a] = c.log_scale;
      }
  }
  if (tid == 0) {
    mbar_init(smem_u32(&mbar), 1);
    fence_mbar_init();
  }
  fence_proxy_async_smem();
  __syncthreads();
  const uint32_t bar = smem_u32(&mbar);

  const long long num_tiles = (p.n_rows + TC_ROWS - 1) / TC_ROWS;
  constexpr int STAGES = BACKWARD ? 6 : 3;

  if (warp >= TC_EPI_WARPS) {
    // =============================== MMA issuer warp =================================================
    constexpr int K = K_MAJOR, MN = MN_MAJOR;
    // warp-uniform copy (ptxas keeps it in a uniform register: no per-instruction R2UR)
    const uint32_t ub = __shfl_sync(0xffffffffu, base, 0);
    const Op2 XD_K = op2_kmajor(ub + SM_XD, ACT_BUF), H1_K = op2_kmajor(ub + SM_H1, ACT_BUF),
              H2_K = op2_kmajor(ub + SM_H2, ACT_BUF), W1_K = op2_kmajor(ub + SM_W1, W_BUF),
              W2_K = op2_kmajor(ub + SM_W2, W_BUF), W3_K = op2_kmajor(ub + SM_W3, W3_BUF);
    const Op2 XD_K2 = op2_kmajor(ub + SM_XD + 64, ACT_BUF);  // cols 32..47 (dOut) as a K-major A operand
    // MN-major views: 64-element atoms along M / N are one buffer height (rows x 128 bytes) apart
    const Op2 H1_M = op2_mnmajor(ub + SM_H1, 128 * 128, ACT_BUF), H2_M = op2_mnmajor(ub + SM_H2, 128 * 128, ACT_BUF),
              XD_M0 = op2_mnmajor(ub + SM_XD, 128 * 128, ACT_BUF),        // X    (cols 0..31)
              XD_M32 = op2_mnmajor(ub + SM_XD + 64, 128 * 128, ACT_BUF),  // dOut (cols 32..47, col 47 = ones)
              W2_M = op2_mnmajor(ub + SM_W2, 64 * 128, W_BUF), W3_M = op2_mnmajor(ub + SM_W3, 16 * 128, W3_BUF);
    bool first = true;
    for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
#pragma unroll 1
      for (int s = 0; s < STAGES; ++s) {
        __syncthreads();  // operands of stage s are in shared memory (and the previous stage's MMAs have retired)
        // issue6 / issue3 <N, A major, B major, M = 64, k-steps>
        if (s == 0) {  // Z1 = X W1^T
          issue6<64, K, K, false, 2>(acc, ACC_Z1, false, XD_K, W1_K);
        } else if (s == 1) {  // Z2 = H1 W2^T
          issue6<64, K, K, false, 4>(acc, ACC_Z2, false, H1_K, W2_K);
        } else if (s == 2) {  // OUT = H2 W3^T
          issue6<16, K, K, false, 4>(acc, ACC_OUT, false, H2_K, W3_K);
        } else if (s == 3) {
          // dW3^T[i][o] += sum_r H2[r][i] dOut[r][o]   (both read MN-major: the reduction runs over rows)
          issue6<16, MN, MN, true, 8>(acc, ACC_DW3, !first, H2_M, XD_M32);
          // dH2 = dOut W3   (A: XD cols 32..47; B: W3 read MN-major, K = output index)
          issue6<64, K, MN, false, 1>(acc, ACC_DH2, false, XD_K2, W3_M);
        } else if (s == 4) {
          // dW2[o][i] += sum_r dZ2[r][o] H1[r][i] ; db2[o] += sum_r dZ2[r][o] * 1 ; dH1 = dZ2 W2
          issue6<64, MN, MN, true, 8>(acc, ACC_DW2, !first, H2_M, H1_M);
          issue3<16, MN, MN, true, 8>(acc, ACC_DB2, !first, H2_M, XD_M32);
          issue6<64, K, MN, false, 4>(acc, ACC_DH1, false, H2_K, W2_M);
        } else {
          // dW1[o][i] += sum_r dZ1[r][o] X[r][i] ; db1[o] += sum_r dZ1[r][o]
          issue6<32, MN, MN, true, 8>(acc, ACC_DW1, !first, H1_M, XD_M0);
          issue3<16, MN, MN, true, 8>(acc, ACC_DB1, !first, H1_M, XD_M32);
        }
        acc_commit(bar);
        __syncwarp();
      }
      first = false;
    }
  } else {
    // =============================== epilogue warps ==================================================
    const int q = warp & 3, half = warp >> 2;
    const int r = 32 * q + lane;                         // row of the tile == accumulator row
    const int c0 = 32 * half;                            // this warp's column half
    uint32_t phase = 0;

    float adv_mean, adv_std;
    adv_mean_std(p.adv_stats, adv_mean, adv_std);
    double sc[6] = {0, 0, 0, 0, 0, 0};
    float db3[16];
#pragma unroll
    for (int a = 0; a < 16; ++a) db3[a] = 0.f;

    // tanh layer epilogue: Z (accumulator memory) + bias -> tanh -> fp32 copy back to accumulator memory (for tanh') + bf16 splits to smem
    auto act_epilogue = [&](uint32_t acc_col, const float* bias, uint32_t dst_buf) {
#pragma unroll
      for (int sub = 0; sub < 2; ++sub) {  // 16 columns at a time keeps the live register set small
        const int cs = c0 + 16 * sub;
        float v[16];
        acc_ld<16>(acc, r, acc_col + cs, v);
#pragma unroll
        for (int j = 0; j < 16; ++j) v[j] = tanhf(v[j] + bias[cs + j]);
        if (BACKWARD) acc_st<16>(acc, r, acc_col + cs, v);
#pragma unroll
        for (int ch = 0; ch < 2; ++ch) {
          float x[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) x[j] = v[8 * ch + j];
          store_chunk3(sm, dst_buf, ACT_BUF, r, (cs >> 3) + ch, x);
        }
      }
    };
    // backward epilogue: dZ = dH * (1 - H^2), bf16 splits over the activation buffer (in place)
    auto dz_epilogue = [&](uint32_t acc_dh, uint32_t acc_h, uint32_t dst_buf) {
#pragma unroll
      for (int sub = 0; sub < 2; ++sub) {
        const int cs = c0 + 16 * sub;
        float g[16], h[16];
        acc_ld<16>(acc, r, acc_dh + cs, g);
        acc_ld<16>(acc, r, acc_h + cs, h);
#pragma unroll
        for (int ch = 0; ch < 2; ++ch) {
          float x[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float hv = h[8 * ch + j];
            x[j] = g[8 * ch + j] * (1.f - hv * hv);
          }
          store_chunk3(sm, dst_buf, ACT_BUF, r, (cs >> 3) + ch, x);
        }
      }
    };
    auto stage_done = [&]() {  // publish smem writes to the tensor core, hand over to the issuer, wait for its MMAs
      fence_proxy_async_smem();
      __syncthreads();
      mbar_wait(bar, phase);
      phase ^= 1u;
    };

    float pf_act[15], pf_adv = 0.f, pf_old = 0.f, pf_tgt = 0.f;
#pragma unroll
    for (int a = 0; a < 15; ++a) pf_act[a] = 0.f;
    const float* s_stage = reinterpret_cast<const float*>(sm + SM_STAGE);
    // stage one tile's observations (contiguous rows_here*n_in floats, 16-byte aligned) with cp.async; warps 4..7
    auto stage_obs = [&](long long t) {
      if (half == 1 && t < num_tiles) {
        const long long r0 = t * TC_ROWS;
        const long long rows_here = (p.n_rows - r0) < TC_ROWS ? (p.n_rows - r0) : TC_ROWS;
        const int n16 = (int)((rows_here * n_in * 4 + 15) / 16);  // the obs buffer is padded to 16 bytes by the engine
        const char* g = reinterpret_cast<const char*>(p.obs + r0 * n_in);
        for (int i = tid - 128; i < n16; i += 128) cp_async16(base + SM_STAGE + 16 * i, g + 16 * (size_t)i);
      }
      cp_async_commit_wait_all();
    };
    stage_obs(blockIdx.x);
    asm volatile("bar.sync 1, %0;" ::"n"(TC_EPI_WARPS * 32) : "memory");

#ifdef B200RL_TC_TIMING
    unsigned long long tacc[16];
    for (int i = 0; i < 16; ++i) tacc[i] = 0;
    long long tlast = clock64();
#endif
    for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const long long row = tile * TC_ROWS + r;
      const bool valid = row < p.n_rows;

      // ---- observations: staged as fp32 by cp.async (previous tile / prologue); one row per thread of warps 0..3
      //      converts its row to the three bf16 splits in cols 0..31 of XD ----
      if (half == 0) {
        const float* src = s_stage + r * n_in;
#pragma unroll
        for (int ch = 0; ch < 4; ++ch) {
          float x[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int c = 8 * ch + j;
            x[j] = (valid && c < n_in) ? src[c] : 0.f;
          }
          store_chunk3(sm, SM_XD, ACT_BUF, r, ch, x);
        }
        // loss inputs of this row: issue the loads now, consume them three stages later
        if (valid) {
          if (p.dist == B200RL_DIST_GAUSSIAN) {
#pragma unroll
            for (int a = 0; a < 15; ++a)
              if (a < A_out) pf_act[a] = __ldg(p.actions + row * A_out + a);
          } else if (p.dist == B200RL_DIST_CATEGORICAL) {
            pf_act[0] = __ldg(p.actions + row);
          }
          if (p.loss != B200RL_LOSS_EVAL && p.adv_raw != nullptr) pf_adv = __ldg(p.adv_raw + row);
          if (p.old_logp != nullptr) pf_old = __ldg(p.old_logp + row);
          if (p.loss == B200RL_LOSS_MSE) pf_tgt = __ldg(p.target + row);
        }
      }
      TC_T(0);
      stage_done();                                   // F1
      TC_T(1);
      act_epilogue(ACC_Z1, s_bias, SM_H1);
      TC_T(2);
      stage_done();                                   // F2
      TC_T(3);
      act_epilogue(ACC_Z2, s_bias + 64, SM_H2);
      TC_T(4);
      stage_done();                                   // F3
      TC_T(5);

      // warps 4..7 have no loss work: they fetch the next tile's observations into the staging buffer meanwhile
      stage_obs(tile + gridDim.x);

      // ---- distribution / loss epilogue (one thread per row: warps 0..3) ----
      if (half == 0) {
        float o[16];
        acc_ld<16>(acc, r, ACC_OUT, o);
        float out[16], dout[16];
#pragma unroll
        for (int a = 0; a < 16; ++a) {
          out[a] = o[a] + s_bias[128 + a];
          dout[a] = 0.f;
        }
        if (valid) {
          if (p.dist == B200RL_DIST_NONE) {
            const float vout = out[0];
            if (p.row_out) p.row_out[row] = vout;
            float term = 0.f;
            if (p.loss == B200RL_LOSS_MSE) term = value_mse(vout, pf_tgt, p.inv_n, dout[0]);
            sc[0] += (double)term;
            sc[5] += 1.0;
          } else {
            float lp, ent, dlp[16];
#pragma unroll
            for (int a = 0; a < 16; ++a) dlp[a] = 0.f;
            if (p.dist == B200RL_DIST_GAUSSIAN)
              gaussian_logp<15>(pf_act, out, s_dist + 16, VarDiv{s_dist}, A_out, lp, ent, dlp);
            else
              categorical_logp<15>(out, (int)pf_act[0], A_out, lp, ent, dlp);  // value.long()
            if (p.row_out) p.row_out[row] = lp;
            float adv = 0.f, oldlp = 0.f;
            if (p.loss != B200RL_LOSS_EVAL) {
              adv = pf_adv;
              if (p.adv_stats != nullptr) adv = (adv - adv_mean) / adv_std;  // utils.py:91
            }
            if (p.old_logp != nullptr) oldlp = pf_old;
            float coef;
            const float term = policy_loss(p.loss, lp, oldlp, adv, p.inv_n, p.clip_lo, p.clip_hi, coef);
#pragma unroll
            for (int a = 0; a < 15; ++a) dout[a] = coef * dlp[a];
            add_policy_row_sums(sc, term, lp, ent, oldlp, p.old_logp != nullptr);
            sc[5] += 1.0;
          }
        }
        if (BACKWARD) {
#pragma unroll
          for (int a = 0; a < 15; ++a) db3[a] += dout[a];
          dout[15] = 1.0f;  // ones column: db1 / db2 fall out of the dW tensor-core products
          float x0[8], x1[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            x0[j] = dout[j];
            x1[j] = dout[8 + j];
          }
          store_chunk3(sm, SM_XD, ACT_BUF, r, 4, x0);  // cols 32..39
          store_chunk3(sm, SM_XD, ACT_BUF, r, 5, x1);  // cols 40..47
        }
      }
      TC_T(6);
      if (BACKWARD) {
        stage_done();                                 // dW3^T, dH2
        TC_T(7);
        dz_epilogue(ACC_DH2, ACC_Z2, SM_H2);
        TC_T(8);
        stage_done();                                 // dW2, db2, dH1
        TC_T(9);
        dz_epilogue(ACC_DH1, ACC_Z1, SM_H1);
        TC_T(10);
        stage_done();                                 // dW1, db1
        TC_T(11);
      } else {
        // forward only: the next tile's F1 may not overwrite ACC_OUT/XD before everyone has read them
        asm volatile("bar.sync 1, %0;" ::"n"(TC_EPI_WARPS * 32) : "memory");
      }
    }

#ifdef B200RL_TC_TIMING
    if (tid == 0 && blockIdx.x == 0 && BACKWARD)
      for (int i = 0; i < 16; ++i) g_tc_t[i] = tacc[i];
#endif
    // ---- per-CTA results: gradient accumulators (M = 64 products: thread r < 16 of warp q holds row m = 16 q + r) ----
    if (BACKWARD && half == 0) {
      float* dst = p.partials + (size_t)blockIdx.x * p.P;
      const int m = 16 * q + lane;  // valid for lane < 16
      float v[32];
      for (int cb = 0; cb < 2; ++cb) {  // dW2 [64 o][64 i]
        acc_ld<32>(acc, r, ACC_DW2 + 32 * cb, v);
        if (lane < 16 && m < h2)
#pragma unroll
          for (int j = 0; j < 32; ++j)
            if (32 * cb + j < h1) dst[p.w_off[1] + m * h1 + 32 * cb + j] = v[j];
      }
      acc_ld<32>(acc, r, ACC_DW1, v);  // dW1 [64 o][32 i]
      if (lane < 16 && m < h1)
#pragma unroll
        for (int j = 0; j < 32; ++j)
          if (j < n_in) dst[p.w_off[0] + m * n_in + j] = v[j];
      float w[16];
      acc_ld<16>(acc, r, ACC_DW3, w);  // dW3^T [64 i][16 o]
      if (lane < 16 && m < h2)
#pragma unroll
        for (int a = 0; a < 15; ++a)
          if (a < A_out) dst[p.w_off[2] + a * h2 + m] = w[a];
      acc_ld<16>(acc, r, ACC_DB2, w);  // column 15 = sum_r dZ2[r][o]
      if (lane < 16 && m < h2) dst[p.b_off[1] + m] = w[15];
      acc_ld<16>(acc, r, ACC_DB1, w);
      if (lane < 16 && m < h1) dst[p.b_off[0] + m] = w[15];
      // db3: fixed-order reduction of the per-row accumulators
#pragma unroll
      for (int a = 0; a < 15; ++a) {
        float s = db3[a];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) s_db3[q * 16 + a] = s;
      }
    }
    asm volatile("bar.sync 1, %0;" ::"n"(TC_EPI_WARPS * 32) : "memory");
    if (BACKWARD && tid < A_out) {
      float s = 0.f;
      for (int w4 = 0; w4 < 4; ++w4) s += s_db3[w4 * 16 + tid];
      p.partials[(size_t)blockIdx.x * p.P + p.b_off[2] + tid] = s;
    }
    if (p.scalar_partials != nullptr) {
#pragma unroll
      for (int k = 0; k < 6; ++k) {
        const double v = warp_sum(sc[k]);
        if (lane == 0) s_sc[k][warp] = v;
      }
      asm volatile("bar.sync 1, %0;" ::"n"(TC_EPI_WARPS * 32) : "memory");
      if (tid < B200RL_N_SCALARS) {
        double t = 0.0;
        if (tid < 6)
          for (int w8 = 0; w8 < TC_EPI_WARPS; ++w8) t += s_sc[tid][w8];
        p.scalar_partials[(size_t)blockIdx.x * B200RL_N_SCALARS + tid] = t;
      }
    }
  }

  // ---- teardown ----
  __syncthreads();
}

#ifdef B200RL_TC_TIMING
extern "C" int b200rl_debug_tc_timing(unsigned long long* out16) {
  return (int)cudaMemcpyFromSymbol(out16, g_tc_t, sizeof(unsigned long long) * 16);
}
#endif

bool tc_shape_ok(const b200rl_mlp_desc& d) {
  return d.n_layers == 3 && d.sizes[1] >= 1 && d.sizes[1] <= 64 && d.sizes[2] >= 1 && d.sizes[2] <= 64 &&
         d.sizes[0] >= 1 && d.sizes[0] <= 32 &&
         d.sizes[3] >= 1 && d.sizes[3] <= 15 && d.hidden_act == B200RL_ACT_TANH && d.out_act == B200RL_ACT_IDENTITY;
}

static int launch_mlp_tc_impl(const b200rl_mlp_loss_grad_args* a, int64_t n_glob, const unsigned* run_if, unsigned seq,
                              int partial_rows, cudaStream_t s) {
  TcArgs k{};
  k.run_if = run_if;
  k.seq = seq;
  k.total_rows = partial_rows;
  k.n_in = a->mlp.sizes[0];
  k.n_out = a->mlp.sizes[3];
  k.h1 = a->mlp.sizes[1];
  k.h2 = a->mlp.sizes[2];
  k.P = mlp3_offsets(a->mlp, k.w_off, k.b_off);
  k.loss = a->loss;
  k.dist = a->dist;
  k.n_rows = a->n_rows;
  k.inv_n = 1.0f / (float)n_glob;
  k.clip_lo = (float)(1.0 - (double)a->clip_range);
  k.clip_hi = (float)(1.0 + (double)a->clip_range);
  k.params = a->params;
  k.obs = a->obs;
  k.actions = a->actions;
  k.log_std = a->log_std;
  k.adv_raw = a->adv_raw;
  k.adv_stats = a->adv_stats;
  k.old_logp = a->old_logp;
  k.target = a->target;
  k.row_out = a->row_out;
  k.partials = a->partials;
  k.scalar_partials = a->scalar_partials;
  k.skip_flag = a->skip_flag;
  const int grid = tc_grid(a->n_rows);
  B200RL_REQUIRE(grid > 0, "mlp_tc: no CUDA device");
  k.acc_mem = acc_mem(grid, s);
  B200RL_REQUIRE(k.acc_mem != nullptr, "mlp_tc: no accumulator memory (allocation failed, or the stream is being captured): %s",
                 cudaGetErrorString(cudaGetLastError()));
  if (a->loss != B200RL_LOSS_EVAL) {
    B200RL_CUDA(cudaFuncSetAttribute(mlp_tc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)TC_SMEM_BYTES));
    mlp_tc_kernel<true><<<grid, TC_THREADS, TC_SMEM_BYTES, s>>>(k);
  } else {
    B200RL_CUDA(cudaFuncSetAttribute(mlp_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)TC_SMEM_BYTES));
    mlp_tc_kernel<false><<<grid, TC_THREADS, TC_SMEM_BYTES, s>>>(k);
  }
  B200RL_CUDA(cudaGetLastError());
  count_launch(1);
  return 0;
}

int launch_mlp_tc(const b200rl_mlp_loss_grad_args* a, int64_t n_glob, cudaStream_t s) {
  return launch_mlp_tc_impl(a, n_glob, nullptr, 0u, 0, s);
}
// re-run of an mlp_tc2 launch whose values left the fp16 range: predicated on *run_if == seq
int launch_mlp_tc_fallback(const b200rl_mlp_loss_grad_args* a, int64_t n_glob, const unsigned* run_if, unsigned seq,
                           int partial_rows, cudaStream_t s) {
  return launch_mlp_tc_impl(a, n_glob, run_if, seq, partial_rows, s);
}

}  // namespace b200rl

namespace b200rl {
// device address of the counter, for kernels in other translation units (no relocatable device code in this build)
unsigned long long* tc_fallback_counter_ptr() {
  static unsigned long long* ptr = nullptr;
  if (ptr == nullptr) {
    void* q = nullptr;
    if (cudaGetSymbolAddress(&q, g_tc_fallbacks) == cudaSuccess) ptr = static_cast<unsigned long long*>(q);
  }
  return ptr;
}
}  // namespace b200rl

extern "C" int64_t b200rl_tc_fallback_count(void) {
  unsigned long long v = 0;
  if (cudaDeviceSynchronize() != cudaSuccess) return -1;
  if (cudaMemcpyFromSymbol(&v, b200rl::g_tc_fallbacks, sizeof(v)) != cudaSuccess) return -1;
  return (int64_t)v;
}
