// mlp_tc2: tensor-core kernel for the fused MLP step (wgmma, sm_90a).
//
// Same contract and data flow as mlp_fused.cu (see there for the reference file:line map).  Shape gate (tc_shape_ok,
// shared with mlp_tc_fvp.cu): 3 Linear layers, tanh hidden layers of width <= 64 -- zero-padded to 64 --, identity
// output, obs <= 32, out <= 15.
// Why two fp16 splits and not three bf16 ones (a first kernel split every operand into three bf16 values and ran six
// products per logical product).  The kernels were first written for B200 (tcgen05); the figures in this note were
// measured there with the per-stage clocks of tools/profile_step.py, not on H100:
//   * a tcgen05.mma of these small shapes cost 30..50 cycles on B200 whatever its size (instruction floor / SS-mode
//     operand feed), so the 282 MMAs per 128-row tile of that kernel -- not the math -- set its pace.  Here every
//     fp32 operand is split into TWO fp16 values x*2^e = h + l (22 mantissa bits, 3.0e-7 worst-case relative error
//     per product with the (l,l) term dropped) after an exact power-of-two pre-scale that parks it in fp16's normal
//     range.  A logical product is then 3 MMAs (h.l, l.h, h.h) on the forward/back-propagation chain and 2 MMAs for
//     the weight-gradient products, whose A operand (dZ^T) is read MN-major with BOTH splits stacked along M
//     (M = 128: rows 0..63 = h-split features, 64..127 = l-split features -- the second 64-element atom of an
//     MN-major operand sits one leading-byte-offset further, i.e. in the next split buffer).  101 MMAs per tile.
//   * with one tile in flight the epilogue warps spent 43% of their time on mbarriers (ncu source view): the
//     MMA -> tanh -> MMA chain is latency bound.  Two fp16 splits instead of three bf16 ones make TWO tiles fit in
//     shared memory (2 x 96 KB), so two tiles ("slots") are in flight per CTA.  All 16 epilogue warps work on one
//     epilogue job at a time, alternating between the slots in a fixed order, so the MMAs a job hands to the issuer
//     run under the other slot's next job; the issuer follows the same fixed order (no polling; K back-to-back MMAs
//     go out as one asm block).  The warp index is read through __shfl_sync so that ptxas can prove the role branch
//     warp-uniform: the issue path then stays in the uniform datapath (~6 instructions per MMA instead of 22 with a
//     vote + R2UR moves around every MMA) -- the issuer shares its scheduler with four epilogue warps, and those
//     four set the pace of every job.
// fp16 has a narrow exponent range: the scales come from the data (max |W| per layer computed per CTA, max |obs| and
// max |target| from a pre-pass or the caller) and every converted value is range-checked.  A launch that sees a
// value outside +-60000 after scaling raises its slot in a status ring and the host has already queued the
// fp32 kernel (mlp_fused.cu, unlimited range) behind it, predicated on that slot: it recomputes the launch.
// The two halves of the stacked accumulators are emitted as TWO partial rows per CTA (b200rl_mlp_grid reports
// 2 x CTAs), so the fixed-order reduction of b200rl_reduce_partials adds them -- no in-kernel combine.
#include <cuda_fp16.h>

#include <atomic>
#include <cmath>
#include <type_traits>

#include "common.cuh"
#include "policy_head.cuh"
#include "tc2_common.cuh"
#include "tc_common.cuh"

namespace b200rl {

constexpr int T2_ROWS = 128;
constexpr int T2_EPI_WARPS = 16;  // one pool: 4 warps per 32-row quarter of the tile, 16 columns each
constexpr int T2_EPI_THREADS = T2_EPI_WARPS * 32;
constexpr int T2_THREADS = T2_EPI_THREADS + 128;  // + the issuing warpgroup

// shared-memory map (bytes from the 1024-aligned base); every operand buffer = 2 fp16 splits, 128-byte rows, SW128
constexpr uint32_t T2_SLOT = 6 * T2_ACT;    // XD, H1, H2 of one slot
constexpr uint32_t T2_W1T = 32 * 128;       // one split of W1^T [32 in][64 out]
constexpr uint32_t T2_W = 64 * 128;         // one split of W2 [64 out][64 in]
constexpr uint32_t T2_W3 = 16 * 128;        // one split of W3 [16 out][64 in]
constexpr uint32_t S2_XD = 0;               // (slot-relative) obs cols 0..31 | dOut cols 32..46 | ones col 47
constexpr uint32_t S2_H1 = 2 * T2_ACT;      // (slot-relative) H1, overwritten in place by dZ1
constexpr uint32_t S2_H2 = 4 * T2_ACT;      // (slot-relative) H2, overwritten in place by dZ2
constexpr uint32_t S2_W1T = 2 * T2_SLOT;
constexpr uint32_t S2_W2 = S2_W1T + 2 * T2_W1T;
constexpr uint32_t S2_W3 = S2_W2 + 2 * T2_W;
constexpr uint32_t S2_OPERANDS_END = S2_W3 + 2 * T2_W3;
constexpr uint32_t S2_BIAS = S2_OPERANDS_END;  // b1[64] b2[64] b3[16] floats
constexpr uint32_t S2_DIST = S2_BIAS + 640;    // var[16], log_scale[16], 1/(2 var)[16], 1/var[16] floats
constexpr uint32_t S2_DB3 = S2_DIST + 256;     // [16 warps][16] floats: running sum_r dOut[r][a] per warp
constexpr uint32_t S2_SCALE = S2_DB3 + 1024;   // scale factors (floats)
constexpr uint32_t S2_RED = S2_SCALE + 64;     // block reduction scratch [20 warps][4] floats
constexpr uint32_t S2_SC = S2_RED + 320;       // [16 warps][7] doubles: running scalar sums per warp
constexpr uint32_t S2_BARS = S2_SC + 896;      // mbarriers: ready[2], chain[2], off[2]; bad flag
constexpr uint32_t S2_XS = S2_BARS + 64;       // per-feature observation scales 2^ex_k [32] and their inverses [32]
constexpr uint32_t S2_ROWMAX = S2_XS + 256;    // [2 slots][128] largest scaled |obs| of each row (precision guard)
constexpr uint32_t S2_TOTAL = S2_ROWMAX + 1024;
constexpr uint32_t T2_SMEM_BYTES = S2_TOTAL + 1024;  // + alignment slack
static_assert(T2_SMEM_BYTES <= 227 * 1024, "mlp_tc2 shared memory");

// accumulator column map (fp32).  Per slot (base = slot * 144): Z1 (kept as H1 for tanh'), ZB (Z2, then dH2, then
// dH1 -- each consumed by its epilogue before the next product overwrites it), OUT.  Shared stacked accumulators,
// row = feature (+64 for the l-split half): DW2, DW1 (cols 0..31 dW1, col 47 db1), DW3, DB2 (col 15).
constexpr uint32_t ACC_SLOT = 144, ACC_Z1 = 0, ACC_ZB = 64, ACC_OUT = 128;
constexpr uint32_t ACC_DW2 = 288, ACC_DW1 = 352, ACC_DW3 = 400, ACC_DB2 = 416;

// indices into the scale table in shared memory
enum { SC_X = 0, SC_G, SC_U1, SC_U2, SC_U3, SC_UH2, SC_UH1, SC_W1, SC_W2, SC_W3, SC_OW3, SC_OW2, SC_OW1, SC_OB, SC_N };

struct Tc2Args {
  int n_in, n_out;
  int h1, h2;  // hidden widths (<= 64; narrower layers are zero-padded to the 64-wide buffers, which keeps every
               // padded activation, gradient and weight-gradient entry exactly zero)
  int w_off[3], b_off[3], P;
  int loss, dist;
  long long n_rows;
  float inv_n, clip_lo, clip_hi;
  float n_glob_f;
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
  const float* obs_absmax;     // device [n_in]: per-feature max |obs|
  const float* target_absmax;  // device scalar (MSE) or NULL
  float* out_full;             // forward-only launches: raw network outputs [n_rows, n_out]
  const float* old_out;        // forward-only launches: outputs of the old policy -> true KL(old || new) in scalar 6
  int total_rows;              // partial rows the consumer reduces (at least two per CTA)
  unsigned* status;            // status-ring slot of this launch
  unsigned seq;                // value to store there when the launch must be redone by the wide-range kernel
  float* acc_mem;              // accumulator memory, ACC_CTA_FLOATS per CTA (tc_common.cuh)
};

#ifdef B200RL_TC_TIMING
__device__ unsigned long long g_tc2_t[24];
#define T2_T(i)                                   \
  do {                                            \
    if (tid == 0) {                               \
      const long long _n = clock64();             \
      tacc[i] += (unsigned long long)(_n - tlast); \
      tlast = _n;                                 \
    }                                             \
  } while (0)
#else
#define T2_T(i)
#endif

template <bool BACKWARD>
__global__ void __launch_bounds__(T2_THREADS, 1) mlp_tc2_kernel(const Tc2Args p) {
  extern __shared__ uint8_t smem_raw[];
  if (p.skip_flag != nullptr && *p.skip_flag != 0) return;  // early stop: whole launch is a no-op

  const int tid = threadIdx.x, lane = tid & 31;
  float* const acc = p.acc_mem + (size_t)blockIdx.x * ACC_CTA_FLOATS;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);  // provably warp-uniform: role branches need no vote
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;  // SWIZZLE_128B atoms are 1024-byte aligned
  uint8_t* sm = smem_raw + (base - raw);
  float* s_bias = reinterpret_cast<float*>(sm + S2_BIAS);
  float* s_dist = reinterpret_cast<float*>(sm + S2_DIST);
  float* s_db3 = reinterpret_cast<float*>(sm + S2_DB3);
  float* s_scale = reinterpret_cast<float*>(sm + S2_SCALE);
  float* s_red = reinterpret_cast<float*>(sm + S2_RED);
  double* s_sc = reinterpret_cast<double*>(sm + S2_SC);
  int* s_bad = reinterpret_cast<int*>(sm + S2_BARS + 48);
  const uint32_t bars = base + S2_BARS;  // ready[s] at +8s, chain[s] at +16+8s, off[s] at +32+8s
  const int n_in = p.n_in, A_out = p.n_out, h1 = p.h1, h2 = p.h2;
  bool bad = false;

  // ---- one-time setup: zero operand buffers; per-layer weight scales; stage W (two fp16 splits), biases ----
  for (uint32_t i = tid; i < S2_OPERANDS_END / 16; i += T2_THREADS) reinterpret_cast<uint4*>(sm)[i] = make_uint4(0, 0, 0, 0);
  if (tid == 0) *s_bad = 0;
  // Observation features are scaled one by one (MuJoCo-style observations mix magnitudes): X_s[:,k] = X[:,k] 2^ex_k
  // with the feature's own max at [2^12, 2^13), and the inverse factor is folded into column k of W1 -- exact.
  float* s_xs = reinterpret_cast<float*>(sm + S2_XS);
  float* s_rowmax = reinterpret_cast<float*>(sm + S2_ROWMAX);
  if (tid < 32) {
    bool bx = false;
    const int e = tid < n_in ? fit_exp(__ldg(p.obs_absmax + tid), bx) : 0;
    s_xs[tid] = pow2i(e);
    s_xs[32 + tid] = pow2i(-e);
    if (bx) bad = true;
  }
  for (int i = tid; i < 2 * 128; i += T2_THREADS) s_rowmax[i] = 0.f;
  __syncthreads();
  // the parameter vector is brought into the (still unused, later fully overwritten) H1 buffer of slot 0 with
  // independent coalesced loads: the passes below would otherwise pay one L2 round trip per element, serially
  float* s_par = reinterpret_cast<float*>(sm + S2_H1);
#pragma unroll 8
  for (int i = tid; i < p.P; i += T2_THREADS) s_par[i] = __ldg(p.params + i);
  __syncthreads();
  {
    float m1 = 0.f, m2 = 0.f, m3 = 0.f;
    for (int idx = tid; idx < h1 * n_in; idx += T2_THREADS) {
      const float w = (s_par[p.w_off[0] + idx]) * s_xs[32 + idx % n_in];
      m1 = fmaxf(m1, fabsf(w));
      if (w != w) bad = true;
    }
    for (int idx = tid; idx < h2 * h1; idx += T2_THREADS) {
      const float w = (s_par[p.w_off[1] + idx]);
      m2 = fmaxf(m2, fabsf(w));
      if (w != w) bad = true;
    }
    for (int idx = tid; idx < A_out * h2; idx += T2_THREADS) {
      const float w = (s_par[p.w_off[2] + idx]);
      m3 = fmaxf(m3, fabsf(w));
      if (w != w) bad = true;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, o));
      m2 = fmaxf(m2, __shfl_xor_sync(0xffffffffu, m2, o));
      m3 = fmaxf(m3, __shfl_xor_sync(0xffffffffu, m3, o));
    }
    if (lane == 0) {
      s_red[warp * 4 + 0] = m1;
      s_red[warp * 4 + 1] = m2;
      s_red[warp * 4 + 2] = m3;
    }
  }
  __syncthreads();
  if (bad) *s_bad = 1;  // NaN weight
  bad = false;
  if (tid == 0) {
    float m1 = 0.f, m2 = 0.f, m3 = 0.f;
    for (int w = 0; w < T2_THREADS / 32; ++w) {
      m1 = fmaxf(m1, s_red[w * 4 + 0]);
      m2 = fmaxf(m2, s_red[w * 4 + 1]);
      m3 = fmaxf(m3, s_red[w * 4 + 2]);
    }
    bool b0 = false;
    const int ew1 = fit_exp(m1, b0), ew2 = fit_exp(m2, b0), ew3 = fit_exp(m3, b0);
    // gradient scale: park typical |dLoss/dOut| * 2^eg near 2^3 (outliers stay far below the fp16 limit)
    int eg = 0;
    if (BACKWARD) {
      float typ;  // typical magnitude of N * dLoss/dOut
      if (p.loss == B200RL_LOSS_MSE) {
        const float tm = p.target_absmax != nullptr ? __ldg(p.target_absmax) : 1.f;
        typ = (tm > 0.f && tm < INFINITY) ? 0.25f * tm : 1.f;  // 2 * |v - target|, |diff| ~ a fraction of max|target|
      } else if (p.dist == B200RL_DIST_GAUSSIAN) {
        float smin = INFINITY;
        for (int a = 0; a < A_out; ++a) smin = fminf(smin, expf(__ldg(p.log_std + a)));
        typ = (smin > 0.f && smin < INFINITY) ? 1.f / smin : 1.f;  // |adv * ratio * z| / sigma
      } else {
        typ = 0.5f;
      }
      eg = 3 + ilogbf(p.n_glob_f) - ilogbf(typ);
      eg = eg < -100 ? -100 : (eg > 100 ? 100 : eg);
    }
    s_scale[SC_G] = pow2i(eg);
    s_scale[SC_U1] = pow2i(-ew1);
    s_scale[SC_U2] = pow2i(-(T2_H_EXP + ew2));
    s_scale[SC_U3] = pow2i(-(T2_H_EXP + ew3));
    s_scale[SC_UH2] = pow2i(-ew3);
    s_scale[SC_UH1] = pow2i(-ew2);
    s_scale[SC_W1] = pow2i(ew1);
    s_scale[SC_W2] = pow2i(ew2);
    s_scale[SC_W3] = pow2i(ew3);
    s_scale[SC_OW3] = pow2i(-(T2_H_EXP + eg));
    s_scale[SC_OW2] = pow2i(-(T2_H_EXP + eg));
    s_scale[SC_OW1] = pow2i(-eg);  // times 2^-ex_k of the column, applied when the accumulator is read
    s_scale[SC_OB] = pow2i(-eg);
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
    const float sw1 = s_scale[SC_W1], sw2 = s_scale[SC_W2], sw3 = s_scale[SC_W3];
    for (int idx = tid; idx < h1 * n_in; idx += T2_THREADS)  // W1 stored transposed: row = input, column = output
      put(S2_W1T, T2_W1T, idx % n_in, idx / n_in, ((s_par[p.w_off[0] + idx]) * s_xs[32 + idx % n_in]) * sw1);
    for (int idx = tid; idx < h2 * h1; idx += T2_THREADS)
      put(S2_W2, T2_W, idx / h1, idx % h1, (s_par[p.w_off[1] + idx]) * sw2);
    for (int idx = tid; idx < A_out * h2; idx += T2_THREADS)
      put(S2_W3, T2_W3, idx / h2, idx % h2, (s_par[p.w_off[2] + idx]) * sw3);
    for (int i = tid; i < 64; i += T2_THREADS) {
      s_bias[i] = i < h1 ? (s_par[p.b_off[0] + i]) : 0.f;
      s_bias[64 + i] = i < h2 ? (s_par[p.b_off[1] + i]) : 0.f;
      if (!(fabsf(s_bias[i]) < INFINITY) || !(fabsf(s_bias[64 + i]) < INFINITY)) bad = true;
    }
    for (int i = tid; i < 16; i += T2_THREADS) {
      s_bias[128 + i] = i < A_out ? (s_par[p.b_off[2] + i]) : 0.f;
      if (!(fabsf(s_bias[128 + i]) < INFINITY)) bad = true;
    }
    if (p.dist == B200RL_DIST_GAUSSIAN)
      for (int a = tid; a < A_out; a += T2_THREADS) {
        const NormalConsts c = normal_consts(p.log_std, a);
        s_dist[a] = c.var;
        s_dist[16 + a] = c.log_scale;
        s_dist[32 + a] = c.inv_2var;
        s_dist[48 + a] = c.inv_var;
      }
  }
  if (bad) *s_bad = 1;  // non-finite bias
  bad = false;
  if (tid == 0) {
    for (int s = 0; s < 2; ++s) {
      mbar_init(bars + 8 * s, T2_EPI_THREADS);   // ready[s]: every epilogue thread arrives once per job of slot s
      mbar_init(bars + 16 + 8 * s, 1);           // chain[s]: acc_commit
      mbar_init(bars + 32 + 8 * s, 1);           // off[s]:   acc_commit
    }
    fence_mbar_init();
  }
  fence_proxy_async_smem();
  __syncthreads();

  const long long num_tiles = (p.n_rows + T2_ROWS - 1) / T2_ROWS;
  // tiles of this CTA: blockIdx.x + k * gridDim.x; slot s takes k = s, s + 2, ...
  const long long cta_tiles = (num_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x;
  constexpr int STAGES = BACKWARD ? 6 : 3;

  if (warp >= T2_EPI_WARPS) {
    // =============================== MMA issuer warpgroup =================================================
    constexpr int K = K_MAJOR, MN = MN_MAJOR;
    const uint32_t ub = base, ubar = bars;  // warp-uniform by construction: from the shared-memory window
    // slot-0 views of the per-slot buffers (slot 1 = T2_SLOT further)
    const Op2 XD_K = op2_kmajor(ub + S2_XD, T2_ACT), H1_K = op2_kmajor(ub + S2_H1, T2_ACT),
              H2_K = op2_kmajor(ub + S2_H2, T2_ACT);
    const Op2 XD_K2 = op2_kmajor(ub + S2_XD + 64, T2_ACT);  // cols 32..47 (dOut) as a K-major A operand
    // MN-major views; as A operands (M = 128) the second atom is the l-split buffer, T2_ACT further
    const Op2 H2_M = op2_mnmajor(ub + S2_H2, T2_ACT, T2_ACT), H1_M = op2_mnmajor(ub + S2_H1, T2_ACT, T2_ACT),
              XD_M0 = op2_mnmajor(ub + S2_XD, T2_ACT, T2_ACT),        // X | dOut | ones (cols 0..47)
              XD_M32 = op2_mnmajor(ub + S2_XD + 64, T2_ACT, T2_ACT);  // dOut | ones (cols 32..47)
    // weights (shared by the slots)
    const Op2 W1T_M = op2_mnmajor(ub + S2_W1T, 32 * 128, T2_W1T), W2_K = op2_kmajor(ub + S2_W2, T2_W),
              W3_K = op2_kmajor(ub + S2_W3, T2_W3), W2_M = op2_mnmajor(ub + S2_W2, 64 * 128, T2_W),
              W3_M = op2_mnmajor(ub + S2_W3, 16 * 128, T2_W3);
    bool acc_dw3 = false, acc_dw2 = false, acc_dw1 = false;  // the first product into an accumulator overwrites it
    uint32_t par0 = 0u, par1 = 0u;
#ifdef B200RL_TC_TIMING
    unsigned long long iacc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#endif
    // The epilogue pool runs its jobs in a fixed order -- (slot 0, stage) then (slot 1, stage) -- and so does the
    // issuer: no polling (the slot only offsets the uniform descriptor bases: one copy of the issue code), and
    // products that accumulate into the shared gradient accumulators are issued in tile order, which makes a launch
    // bit-reproducible.
    auto serve = [&](const int S, const int stage) {
      const uint32_t so = (uint32_t)S * T2_SLOT;
      const uint32_t acol = (uint32_t)S * ACC_SLOT;
      const uint32_t bar_chain = ubar + 16 + 8 * S, bar_off = ubar + 32 + 8 * S;
      uint32_t& par = S == 0 ? par0 : par1;
#ifdef B200RL_TC_TIMING
      long long it0 = clock64();
#endif
      mbar_wait(ubar + 8 * S, par);  // every epilogue thread has delivered its share of the stage inputs
      par ^= 1u;
#ifdef B200RL_TC_TIMING
      long long it1 = clock64();
      iacc[6] += (unsigned long long)(it1 - it0);
#endif
      // issue_chain3 <N, B major, k-steps>, issue_stacked <N, k-steps, B splits>
      if (stage == 0) {  // Z1 = X W1^T
        issue_chain3<64, MN, 2>(acc, acol + ACC_Z1, op2_at(XD_K, so), W1T_M);
        acc_commit(bar_chain);
      } else if (stage == 1) {  // Z2 = H1 W2^T
        issue_chain3<64, K, 4>(acc, acol + ACC_ZB, op2_at(H1_K, so), W2_K);
        acc_commit(bar_chain);
      } else if (stage == 2) {  // OUT = H2 W3^T
        issue_chain3<16, K, 4>(acc, acol + ACC_OUT, op2_at(H2_K, so), W3_K);
        acc_commit(bar_chain);
      } else if (stage == 3) {
        // dH2 = dOut W3 (A: XD cols 32..47; B: W3 read MN-major, K = output index);
        // dW3^T[i][o] += sum_r H2[r][i] dOut[r][o]  -- must retire before the epilogue turns H2 into dZ2 in place
        issue_chain3<64, MN, 1>(acc, acol + ACC_ZB, op2_at(XD_K2, so), W3_M);
        issue_stacked<16, 8, 2>(acc, ACC_DW3, acc_dw3, op2_at(H2_M, so), op2_at(XD_M32, so));
        acc_dw3 = true;
        acc_commit(bar_chain);
      } else if (stage == 4) {
        // dH1 = dZ2 W2 ; dW2[o][i] += sum_r dZ2[r][o] H1[r][i] ; db2[o] += sum_r dZ2[r][o] * 1
        issue_chain3<64, MN, 4>(acc, acol + ACC_ZB, op2_at(H2_K, so), W2_M);
        issue_stacked<64, 8, 2>(acc, ACC_DW2, acc_dw2, op2_at(H2_M, so), op2_at(H1_M, so));
        issue_stacked<16, 8, 1>(acc, ACC_DB2, acc_dw2, op2_at(H2_M, so), op2_at(XD_M32, so));
        acc_dw2 = true;
        acc_commit(bar_chain);
      } else {
        // dW1[o][i] += sum_r dZ1[r][o] X[r][i] and, through the ones column, db1[o] += sum_r dZ1[r][o]
        issue_stacked<48, 8, 2>(acc, ACC_DW1, acc_dw1, op2_at(H1_M, so), op2_at(XD_M0, so));
        acc_dw1 = true;
        acc_commit(bar_off);
      }
      __syncwarp();
#ifdef B200RL_TC_TIMING
      iacc[stage] += (unsigned long long)(clock64() - it1);
#endif
    };
    for (long long kp = 0; kp < cta_tiles; kp += 2) {
#pragma unroll 1
      for (int stage = 0; stage < STAGES; ++stage) {
#pragma unroll 1
        for (int S = 0; S < 2; ++S)
          if (kp + S < cta_tiles) serve(S, stage);
      }
    }
#ifdef B200RL_TC_TIMING
    if (lane == 0 && blockIdx.x == 0 && BACKWARD)
      for (int i = 0; i < 8; ++i) g_tc2_t[16 + i] = iacc[i];
#endif
  } else {
    // =============================== epilogue warps: one pool of 16 ===================================
    // Two tiles ("slots") are in flight, but the epilogue warps are NOT bound to a slot: all 16 work on one epilogue
    // job at a time (16 columns each: 4 warps per 32-row quarter of the tile), alternating between the slots in a fixed order
    //   (slot 0, E0) (slot 1, E0) (slot 0, E1) (slot 1, E1) ... (slot 1, E5) | next pair of tiles
    // so the MMAs a job hands to the issuer run under the OTHER slot's next job.  (Binding 8 warps to each slot left
    // every epilogue latency bound -- 8 warps cannot fill the SM's issue slots -- and made both slots wait for their
    // MMAs at the same time; measured slower on B200.)  The one-row-per-thread loss
    // job needs only 4 warps; it rotates over the four column groups from tile to tile and the other 12 warps move on.
    const int q = warp & 3, part = warp >> 2;
    const int r = 32 * q + lane;                          // row of the tile == accumulator row
    const int cs = 16 * part;                             // this warp's 16 columns of a 64-column epilogue
    uint32_t ph_chain0 = 0, ph_chain1 = 0, ph_off0 = 0, ph_off1 = 0;
    bool first0 = true, first1 = true;
    const float sG = s_scale[SC_G];
    const float sH = pow2i(T2_H_EXP);
    // per-thread running sums over the rows this thread handled as a loss thread (one tile in four): reduced once, in
    // a fixed order, at the end of the kernel -- a warp reduction per tile would put ~130 dependent shuffles on the
    // latency-bound loss job
    double sc[6] = {0, 0, 0, 0, 0, 0};
    double sc_kl = 0.0;  // forward-only launches with old_out: sum of KL(old || new)
    float db3[15];
#pragma unroll
    for (int a = 0; a < 15; ++a) db3[a] = 0.f;

    float adv_mean, adv_std;
    adv_mean_std(p.adv_stats, adv_mean, adv_std);
    const float adv_inv_std = 1.f / adv_std;

#ifdef B200RL_TC_TIMING
    unsigned long long tacc[16];
    for (int i = 0; i < 16; ++i) tacc[i] = 0;
    long long tlast = clock64();
#endif
    auto job = [&](const int slot, const int stage, const long long k) {
      const uint32_t acol = (uint32_t)slot * ACC_SLOT;
      const uint32_t so = (uint32_t)slot * T2_SLOT;
      const uint32_t bar_ready = bars + 8 * slot, bar_chain = bars + 16 + 8 * slot, bar_off = bars + 32 + 8 * slot;
      const long long tile = blockIdx.x + k * gridDim.x;
      const long long row = tile * T2_ROWS + r;
      const bool valid = row < p.n_rows;
      const bool loss_warp = part == (int)(k & 3);  // rotates: every warp does the loss job of one tile in four
      auto arrive = [&]() {  // -> issuer: "this thread's share of the slot's next stage inputs is in shared memory"
        fence_proxy_async_smem();
        mbar_arrive(bar_ready);
      };
      auto wait_chain = [&]() {
        T2_T(2 * stage + 1);  // work since the last mark belongs to the previous job's tail (arrive)
        uint32_t& ph = slot == 0 ? ph_chain0 : ph_chain1;
        mbar_wait(bar_chain, ph);
        ph ^= 1u;
        T2_T(2 * stage);  // wait
      };
      if (stage == 0) {
        // ---- E0: observations (global fp32 -> scaled fp16 splits, cols 0..31 of XD; 8 columns per thread) ----
        float x[8];
        const float* src = p.obs + row * n_in + 8 * part;
#pragma unroll
        for (int j = 0; j < 8; ++j) x[j] = (valid && 8 * part + j < n_in) ? __ldg(src + j) : 0.f;
        bool& first = slot == 0 ? first0 : first1;
        if (BACKWARD && !first) {  // the slot's previous tile: dW1 still reads XD and H1 (dZ1)
          uint32_t& ph = slot == 0 ? ph_off0 : ph_off1;
          mbar_wait(bar_off, ph);
          ph ^= 1u;
        }
        first = false;
        float rmax = 0.f, nan_probe = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          x[j] *= s_xs[8 * part + j];
          rmax = fmaxf(rmax, fabsf(x[j]));  // drops NaNs ...
          nan_probe += x[j];                // ... so they are caught here
        }
        atomicMax(reinterpret_cast<int*>(s_rowmax + slot * 128 + r), __float_as_int(rmax));  // >= 0: int order
        if (!(rmax <= T2_RANGE) || nan_probe != nan_probe) bad = true;
        store_chunk2(sm, so + S2_XD, r, part, x);
        arrive();
      } else if (stage == 1 || stage == 2) {
        // ---- E1 / E2: Z (accumulator memory) * unscale + bias -> tanh -> [fp32 back to accumulator memory for tanh'] + fp16 splits ----
        wait_chain();
        const uint32_t col = acol + (stage == 1 ? ACC_Z1 : ACC_ZB) + cs;
        const float* bias = stage == 1 ? s_bias : s_bias + 64;
        const float unscale = s_scale[stage == 1 ? SC_U1 : SC_U2];
        const uint32_t dst = so + (stage == 1 ? S2_H1 : S2_H2);
        float z[16];
        acc_ld<16>(acc, r, col, z);
#pragma unroll
        for (int j = 0; j < 16; ++j) z[j] = fmaf(z[j], unscale, bias[cs + j]);
        tanh16_scaled(z, 1.f);  // |tanh| <= 1, and Z is finite: observations, weights and biases were all checked
        if (BACKWARD && stage == 1) acc_st<16>(acc, r, col, z);
#pragma unroll
        for (int ch = 0; ch < 2; ++ch) {
          float x[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) x[j] = z[8 * ch + j] * sH;
          store_chunk2(sm, dst, r, (cs >> 3) + ch, x);
        }
        arrive();
      } else if (stage == 3) {
        // ---- E3: distribution / loss epilogue, one row per thread, on this tile's loss warps ----
        float pf_act[15], pf_adv = 0.f, pf_old = 0.f, pf_tgt = 0.f;
#pragma unroll
        for (int a = 0; a < 15; ++a) pf_act[a] = 0.f;
        if (loss_warp && valid) {  // loss inputs of this row: issue the loads before waiting for F3
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
        wait_chain();  // every warp consumes the phase (a skipped parity wait could not be told from a completed one)
        if (loss_warp) {
          {  // precision guard: a row whose every feature sits 2^17 below its column's maximum has lost the l-splits
            const float rm = s_rowmax[slot * 128 + r];
            s_rowmax[slot * 128 + r] = 0.f;
            if (valid && rm > 0.f && rm < 0.03125f) bad = true;
          }
          float o[16];
          acc_ld<16>(acc, r, acol + ACC_OUT, o);
          float out[16], dout[16];
          const float u3 = s_scale[SC_U3];
#pragma unroll
          for (int a = 0; a < 16; ++a) {
            out[a] = fmaf(o[a], u3, s_bias[128 + a]);
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
              const VarRecip var{s_dist + 48, s_dist + 32};
              float lp, ent, dlp[16];
#pragma unroll
              for (int a = 0; a < 16; ++a) dlp[a] = 0.f;
              if (p.dist == B200RL_DIST_GAUSSIAN)
                gaussian_logp<15>(pf_act, out, s_dist + 16, var, A_out, lp, ent, dlp);
              else
                categorical_logp<15>(out, (int)pf_act[0], A_out, lp, ent, dlp);  // value.long()
              if (p.row_out) p.row_out[row] = lp;
              if (!BACKWARD) {
                if (p.out_full != nullptr) {
#pragma unroll
                  for (int a = 0; a < 15; ++a)
                    if (a < A_out) p.out_full[row * A_out + a] = out[a];
                }
                if (p.old_out != nullptr) {
                  const Ldg oo{p.old_out + row * A_out};
                  sc_kl += (double)(p.dist == B200RL_DIST_GAUSSIAN ? gaussian_kl<15>(oo, out, var, A_out)
                                                                    : categorical_kl<15>(oo, out, A_out));
                }
              }
              float adv = 0.f, oldlp = 0.f;
              if (p.loss != B200RL_LOSS_EVAL) {
                adv = pf_adv;
                if (p.adv_stats != nullptr) adv = (adv - adv_mean) * adv_inv_std;  // utils.py:91
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
            float x0[8], x1[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              x0[j] = dout[j] * sG;
              x1[j] = j < 7 ? dout[8 + j] * sG : 1.0f;  // ones column (col 47): db1 / db2 fall out of the dW products
            }
            if (out_of_range8(x0) || out_of_range8(x1)) bad = true;
            store_chunk2(sm, so + S2_XD, r, 4, x0);  // cols 32..39
            store_chunk2(sm, so + S2_XD, r, 5, x1);  // cols 40..47
          }
        }
        if (BACKWARD) arrive();
      } else if (stage == 4) {
        // ---- E4: dZ2 (scaled) = dH2_acc * 2^-ew3 * (1 - H2^2), H2 re-read from its fp16 splits, written in place ----
        wait_chain();  // dH2 (and dW3: H2 may be overwritten now)
        const float unscale = s_scale[SC_UH2], hh = pow2i(-2 * T2_H_EXP);
        float g[16];
        acc_ld<16>(acc, r, acol + ACC_ZB + cs, g);
#pragma unroll
        for (int ch = 0; ch < 2; ++ch) {
          float x[8];
          load_chunk2(sm, so + S2_H2, r, (cs >> 3) + ch, x);
#pragma unroll
          for (int j = 0; j < 8; ++j) x[j] = (g[8 * ch + j] * unscale) * fmaf(-(x[j] * hh), x[j], 1.f);
          if (too_large8(x)) bad = true;
          store_chunk2(sm, so + S2_H2, r, (cs >> 3) + ch, x);
        }
        arrive();
      } else {
        // ---- E5: dZ1 (scaled) = dH1_acc * 2^-ew2 * (1 - H1^2), H1 kept as fp32 in accumulator memory, written over H1 ----
        wait_chain();  // dH1 (and dW2 / db2: H1 may be overwritten now)
        const float unscale = s_scale[SC_UH1];
        float g[16], h[16];
        acc_ld<16>(acc, r, acol + ACC_ZB + cs, g);
        acc_ld<16>(acc, r, acol + ACC_Z1 + cs, h);
#pragma unroll
        for (int ch = 0; ch < 2; ++ch) {
          float x[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float hv = h[8 * ch + j];
            x[j] = (g[8 * ch + j] * unscale) * (1.f - hv * hv);
          }
          if (too_large8(x)) bad = true;
          store_chunk2(sm, so + S2_H1, r, (cs >> 3) + ch, x);
        }
        arrive();  // -> dW1 / db1, completion tracked by bar_off
      }
    };

    constexpr int NSTAGE = BACKWARD ? 6 : 4;  // forward only: E0, E1, E2 and the loss job (no arrival after it)
    for (long long kp = 0; kp < cta_tiles; kp += 2) {
#pragma unroll 1
      for (int stage = 0; stage < NSTAGE; ++stage) {
#pragma unroll 1
        for (int slot = 0; slot < 2; ++slot) {  // one copy of the job code: it is large and the I-cache is not
          if (kp + slot < cta_tiles) job(slot, stage, kp + slot);
          T2_T(2 * stage + 1);
        }
      }
    }
#ifdef B200RL_TC_TIMING
    if (tid == 0 && blockIdx.x == 0 && BACKWARD)
      for (int i = 0; i < 16; ++i) g_tc2_t[i] = tacc[i];
#endif

    // ---- per-CTA results ----
    if (BACKWARD) {  // the last dW1 of each slot that had a tile
      if (!first0) mbar_wait(bars + 32, ph_off0);
      if (!first1) mbar_wait(bars + 40, ph_off1);
    }
    asm volatile("bar.sync 2, %0;" ::"n"(T2_EPI_THREADS) : "memory");  // every MMA of the CTA has retired
    if (BACKWARD) {
      // stacked accumulators: rows 0..63 = h-split half (partial row 2b), rows 64..127 = l-split half (row 2b+1)
      float* dst = p.partials + ((size_t)blockIdx.x * 2 + (q >> 1)) * p.P;
      const int m = 32 * (q & 1) + lane;  // feature index
      float v[16];
      if (part < 2) {  // dW2 [h2 o][h1 i]: columns 32*part .. +31
#pragma unroll
        for (int cb = 0; cb < 2; ++cb) {
          const int cc = 32 * part + 16 * cb;
          acc_ld<16>(acc, r, ACC_DW2 + cc, v);
          const float u = s_scale[SC_OW2];
          if (m < h2)
#pragma unroll
            for (int j = 0; j < 16; ++j)
              if (cc + j < h1) dst[p.w_off[1] + m * h1 + cc + j] = v[j] * u;
        }
      } else if (part == 2) {  // dW1 [h1 o][n_in i] in cols 0..31, db1 in col 47
#pragma unroll
        for (int cb = 0; cb < 3; ++cb) {
          acc_ld<16>(acc, r, ACC_DW1 + 16 * cb, v);
          if (m < h1) {
            if (cb < 2) {
              const float u = s_scale[SC_OW1];
#pragma unroll
              for (int j = 0; j < 16; ++j)
                if (16 * cb + j < n_in)
                  dst[p.w_off[0] + m * n_in + 16 * cb + j] = (v[j] * u) * s_xs[32 + 16 * cb + j];
            } else {
              dst[p.b_off[0] + m] = v[15] * s_scale[SC_OB];
            }
          }
        }
      } else {  // dW3^T [h2 i][16 o] and db2 (col 15 = sum_r dZ2[r][o])
        acc_ld<16>(acc, r, ACC_DW3, v);
        const float u = s_scale[SC_OW3];
        if (m < h2)
#pragma unroll
          for (int a = 0; a < 15; ++a)
            if (a < A_out) dst[p.w_off[2] + a * h2 + m] = v[a] * u;
        acc_ld<16>(acc, r, ACC_DB2, v);
        if (m < h2) dst[p.b_off[1] + m] = v[15] * s_scale[SC_OB];
      }
    }
    // per-thread sums -> per-warp sums (tree) -> the 16 warps in order (below): fixed order => reproducible
    if (BACKWARD) {
#pragma unroll
      for (int a = 0; a < 15; ++a) {
        float t = db3[a];
#pragma unroll
        for (int o2 = 16; o2 > 0; o2 >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o2);
        if (lane == 0) s_db3[warp * 16 + a] = t;
      }
    }
    if (p.scalar_partials != nullptr) {
#pragma unroll
      for (int kk = 0; kk < 6; ++kk) {
        const double t = warp_sum(sc[kk]);
        if (lane == 0) s_sc[warp * 7 + kk] = t;
      }
      const double t = warp_sum(sc_kl);
      if (lane == 0) s_sc[warp * 7 + 6] = t;
    }
    asm volatile("bar.sync 2, %0;" ::"n"(T2_EPI_THREADS) : "memory");  // every warp's sums are in shared memory
    if (BACKWARD && tid < A_out) {  // db3: the 16 per-warp totals in warp order
      float t = 0.f;
      for (int w = 0; w < T2_EPI_WARPS; ++w) t += s_db3[w * 16 + tid];
      p.partials[((size_t)blockIdx.x * 2) * p.P + p.b_off[2] + tid] = t;
      p.partials[((size_t)blockIdx.x * 2 + 1) * p.P + p.b_off[2] + tid] = 0.f;
    }
    if (p.scalar_partials != nullptr && tid < B200RL_N_SCALARS) {
      double t = 0.0;
      if (tid < 7)
        for (int w = 0; w < T2_EPI_WARPS; ++w) t += s_sc[w * 7 + tid];
      p.scalar_partials[((size_t)blockIdx.x * 2) * B200RL_N_SCALARS + tid] = t;
      p.scalar_partials[((size_t)blockIdx.x * 2 + 1) * B200RL_N_SCALARS + tid] = 0.0;
      // rows the consumer reduces beyond this grid's two per CTA (sized for the fp32 re-run): zero
      for (int row = 2 * (int)gridDim.x + (int)blockIdx.x; row < p.total_rows; row += (int)gridDim.x)
        p.scalar_partials[(size_t)row * B200RL_N_SCALARS + tid] = 0.0;
    }
    if (bad) *s_bad = 1;
  }

  // ---- teardown ----
  __syncthreads();
  if (tid == 0 && *s_bad != 0) *p.status = p.seq;  // this launch is redone by the fp32 kernel queued behind it
}

// max |x| over a device array (pre-pass for the observation / target scale when the caller gave no hint)
__global__ void __launch_bounds__(256) absmax_kernel(const float* __restrict__ x, long long n, float* out) {
  float m = 0.f;
  bool nan = false;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    const float v = x[i];
    m = fmaxf(m, fabsf(v));
    nan |= (v != v);
  }
  if (nan) m = INFINITY;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(reinterpret_cast<int*>(out), __float_as_int(m));  // m >= 0: int order
}

// per-column max |x| of a row-major [rows, cols] array (cols <= 32): the per-feature observation scales
__global__ void __launch_bounds__(256) absmax_cols_kernel(const float* __restrict__ x, long long rows, int cols,
                                                          float* out) {
  const int c = threadIdx.x & 31, sub = threadIdx.x >> 5;
  float m = 0.f;
  bool nan = false;
  if (c < cols)
    for (long long r = (long long)blockIdx.x * 8 + sub; r < rows; r += (long long)gridDim.x * 8) {
      const float v = x[r * cols + c];
      m = fmaxf(m, fabsf(v));
      nan |= (v != v);
    }
  if (nan) m = INFINITY;
  if (c < cols && m > 0.f) atomicMax(reinterpret_cast<int*>(out + c), __float_as_int(m));
}

// ---- host side -------------------------------------------------------------------------------------------------
namespace {
constexpr int STATUS_SLOTS = 1024;
struct Tc2State {
  unsigned* status = nullptr;  // [STATUS_SLOTS]
  float* scratch = nullptr;    // [STATUS_SLOTS][40] absmax pre-pass results: 32 observation features, then the target
  std::atomic<unsigned> seq{1};
};
Tc2State g_tc2;

int tc2_configure() {  // once per process (one process drives one GPU): status ring, scratch, shared-memory opt-in
  B200RL_CUDA(cudaMalloc(reinterpret_cast<void**>(&g_tc2.status), STATUS_SLOTS * sizeof(unsigned)));
  B200RL_CUDA(cudaMemset(g_tc2.status, 0, STATUS_SLOTS * sizeof(unsigned)));
  B200RL_CUDA(cudaMalloc(reinterpret_cast<void**>(&g_tc2.scratch), STATUS_SLOTS * 40 * sizeof(float)));
  B200RL_CUDA(cudaFuncSetAttribute(mlp_tc2_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)T2_SMEM_BYTES));
  B200RL_CUDA(cudaFuncSetAttribute(mlp_tc2_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)T2_SMEM_BYTES));
  return 0;
}
}  // namespace

// next status-ring slot (shared by every fp16 tensor-core launch: mlp_tc2, mlp_tc_fvp).  A launch that must be redone
// stores its own sequence number in its slot and the predicated re-run queued right behind it on the same stream
// compares for equality, so a stale value from an earlier user of the slot can never fire it (0 is never handed out:
// the ring starts zeroed).
int tc2_take_slot(unsigned** status, unsigned* seq, float** scratch) {
  static const int configured = tc2_configure();  // thread-safe one-time initialisation
  if (configured != 0) {
    set_error("mlp_tc2: the one-time device setup (status ring, shared-memory opt-in) failed earlier in this process");
    return 1;
  }
  do {
    *seq = g_tc2.seq.fetch_add(1);
  } while (*seq == 0u);
  const unsigned slot = *seq % STATUS_SLOTS;
  *status = g_tc2.status + slot;
  *scratch = g_tc2.scratch + 40 * slot;
  return 0;
}

int launch_absmax_cols(const float* x, long long rows, int cols, float* out, cudaStream_t s) {
  if (rows > 0 && cols > 0) {
    absmax_cols_kernel<<<(int)std::min<long long>((rows + 7) / 8, 4LL * 132), 256, 0, s>>>(x, rows, cols, out);
    B200RL_CUDA(cudaGetLastError());
    count_launch(1);
  }
  return 0;
}

int launch_fused_fallback(const b200rl_mlp_loss_grad_args* a, const unsigned* run_if, unsigned seq, int total_rows,
                          cudaStream_t s);  // mlp_fused.cu: the fp32 kernel as the predicated re-run

bool tc_shape_ok(const b200rl_mlp_desc& d) {
  return d.n_layers == 3 && d.sizes[1] >= 1 && d.sizes[1] <= 64 && d.sizes[2] >= 1 && d.sizes[2] <= 64 &&
         d.sizes[0] >= 1 && d.sizes[0] <= 32 &&
         d.sizes[3] >= 1 && d.sizes[3] <= 15 && d.hidden_act == B200RL_ACT_TANH && d.out_act == B200RL_ACT_IDENTITY;
}

// total_rows: the partial rows the consumer reduces (b200rl_mlp_grid), at least two per CTA
int launch_mlp_tc2(const b200rl_mlp_loss_grad_args* a, int64_t n_glob, int total_rows, cudaStream_t s) {
  unsigned* status_slot = nullptr;
  unsigned seq = 0;
  float* scratch = nullptr;
  if (tc2_take_slot(&status_slot, &seq, &scratch)) return 1;
  Tc2Args k{};
  k.n_in = a->mlp.sizes[0];
  k.n_out = a->mlp.sizes[3];
  k.h1 = a->mlp.sizes[1];
  k.h2 = a->mlp.sizes[2];
  k.P = mlp3_offsets(a->mlp, k.w_off, k.b_off);
  k.loss = a->loss;
  k.dist = a->dist;
  k.n_rows = a->n_rows;
  k.inv_n = 1.0f / (float)n_glob;
  k.n_glob_f = (float)n_glob;
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
  k.status = status_slot;
  k.seq = seq;
  const bool backward = a->loss != B200RL_LOSS_EVAL && !(a->flags & B200RL_FLAG_FORWARD_ONLY);
  k.out_full = a->out_full;
  k.old_out = a->old_out;
  k.total_rows = total_rows;
  int launches = 0;
  // scale hints: use the caller's, else run the pre-pass (correct for any caller; the engine passes hints)
  const bool need_obs = a->obs_absmax == nullptr;
  const bool need_tgt = backward && a->loss == B200RL_LOSS_MSE && a->target_absmax == nullptr;
  if (need_obs || need_tgt) B200RL_CUDA(cudaMemsetAsync(scratch, 0, 40 * sizeof(float), s));
  if (need_obs) {
    if (launch_absmax_cols(a->obs, a->n_rows, k.n_in, scratch, s)) return 1;
  }
  if (need_tgt) {
    absmax_kernel<<<(int)std::min<long long>((a->n_rows + 255) / 256, 2LL * 132), 256, 0, s>>>(a->target, a->n_rows,
                                                                                              scratch + 32);
    ++launches;
  }
  k.obs_absmax = need_obs ? scratch : a->obs_absmax;
  k.target_absmax = need_tgt ? scratch + 32 : a->target_absmax;
  const int grid = tc_grid(a->n_rows);
  B200RL_REQUIRE(grid > 0, "mlp_tc2: no CUDA device");
  k.acc_mem = acc_mem(grid, s);
  B200RL_REQUIRE(k.acc_mem != nullptr, "mlp_tc2: no accumulator memory (allocation failed, or the stream is being captured): %s",
                 cudaGetErrorString(cudaGetLastError()));
  if (backward)
    mlp_tc2_kernel<true><<<grid, T2_THREADS, T2_SMEM_BYTES, s>>>(k);
  else
    mlp_tc2_kernel<false><<<grid, T2_THREADS, T2_SMEM_BYTES, s>>>(k);
  B200RL_CUDA(cudaGetLastError());
  count_launch(launches + 1);
  // wide-range re-run, predicated on this launch's status slot (a few microseconds when it does not fire)
  return launch_fused_fallback(a, status_slot, seq, total_rows, s);
}

}  // namespace b200rl

#ifdef B200RL_TC_TIMING
extern "C" int b200rl_debug_tc2_timing(unsigned long long* out16) {
  return (int)cudaMemcpyFromSymbol(out16, b200rl::g_tc2_t, sizeof(unsigned long long) * 24);
}
#endif

extern "C" int b200rl_absmax_cols(const float* x, int64_t rows, int32_t cols, float* out, void* stream) {
  using namespace b200rl;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200RL_REQUIRE(x != nullptr && out != nullptr && rows >= 0 && cols >= 1 && cols <= 32, "absmax_cols: bad argument");
  B200RL_CUDA(cudaMemsetAsync(out, 0, (size_t)cols * sizeof(float), s));
  return launch_absmax_cols(x, rows, cols, out, s);
}

extern "C" int b200rl_absmax(const float* x, int64_t n, float* out, void* stream) {
  using namespace b200rl;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200RL_REQUIRE(x != nullptr && out != nullptr && n >= 0, "absmax: bad argument");
  B200RL_CUDA(cudaMemsetAsync(out, 0, sizeof(float), s));
  if (n > 0) {
    absmax_kernel<<<(int)std::min<long long>((n + 255) / 256, 2LL * 132), 256, 0, s>>>(x, (long long)n, out);
    B200RL_CUDA(cudaGetLastError());
    count_launch(1);
  }
  return 0;
}
