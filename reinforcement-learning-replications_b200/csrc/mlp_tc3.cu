// mlp_tc3: ONE kernel per PPO iteration -- the policy step AND the value step over the same 128-row tile of the batch
// (wgmma, fp16 x 2 operand splitting as in mlp_tc2.cu; sm_90a).
//
// Why (reference: /root/reference/src/rl_replicas/algorithms/ppo.py:173-181 policy loop, :186-192 value loop): the two
// loops touch disjoint parameters and read the same fixed inputs (advantages and returns are computed before either
// loop, :142-161), so step i of both can share one pass over the batch.  Compared with two mlp_tc2 launches:
//   * the two networks share only the read-only observation tile, so each runs in CTAs of its own: CTA c G + slot
//     runs network c on the tiles of slot `slot`, the policy CTAs as the first wave and the value CTAs as the second.
//     Rows are independent in the forward / backward chain, so each 64-row half of a tile is one warpgroup that
//     issues its own m64 products and keeps the accumulator in registers: its epilogues work on the wgmma fragment
//     and hand their result to its next product in registers.  Two more warpgroups, one per m64 half of
//     the stacked A operands (the h and the l split), issue the weight-gradient products off the chains' critical
//     path, and keep their accumulators (88 floats a thread) in registers for the whole launch; they are stored once,
//     in grad_acc_off's layout, for the read-out.  mbarriers tell the gradient warpgroups when both chain halves have
//     delivered a stage's operands, and tell the chains when both have finished reading a buffer they are about to
//     overwrite.  dZ2, dZ1 and dOut have buffers of their own, so the gradient products run about one tile behind the
//     chains; the h-split warpgroup also brings the observations in;
//   * the chain epilogues move the fp16 pairs between the wgmma fragment and the swizzled activation buffers with
//     stmatrix / ldmatrix: 8 stmatrix.x4 per buffer written and 8 ldmatrix.x4 per buffer read back, instead of 32
//     st.shared / ld.shared.b32 each (same bytes at the same addresses).  Splitting each n64 chain product into two
//     n32 groups, to run the epilogue of one half under the product of the other, made the launch slower (more
//     shared-memory reads of A per product), and so did issuing the b3 running-sum loads before the OUT product
//     (126 registers instead of 122); neither is kept (README);
//   * Z2, OUT, dH2 and dH1 take their A operand from registers (wgmma RS form): the fp16 pairs an epilogue splits
//     for stmatrix are already the next product's A fragment, so the chain neither reads its own activations back
//     from shared memory nor synchronises its warpgroup before a product.  The buffers are still written, for the
//     gradient warpgroups and for dtanh, and deliver(3) / deliver(4) run under dH2 / dH1 (README);
//   * the observations are split into their fp16 pairs ONCE PER UPDATE by pack_obs_kernel (every step of the update
//     reads the same observations) into ready-made SWIZZLE_128B tile images [128 rows][h cols 0..31 | l cols 32..63];
//     the step kernel brings a tile image in with ONE 16 KB bulk copy (cp.async.bulk + mbarrier complete_tx) issued by
//     the producer warpgroup -- no epilogue touches the observations any more (E0 of mlp_tc2 is gone);
//   * the same producer copies each tile's per-row loss inputs (actions, adv_raw and old_logp, or the returns) into a
//     double-buffered shared area on the tile's mbarrier, and the advantage statistics are read once at set-up: the
//     loss head (E3) no longer waits on global memory in the middle of the chain;
//   * column 31 of the image is 1.0, so the bias gradients db1 / db2 still fall out of the weight-gradient products;
//   * two X buffers: the next tile's bulk copy goes into the buffer of the previous tile once its dW1 has retired;
//   * tanh'(H1) and tanh'(H2) are taken from the fp16 pairs in shared memory: no fp32 copy of H in registers;
//   * one reduction + Adam launch for both networks (reduce_adam3_kernel), one all-reduce per iteration.
// A range / precision trip (fp16 operands) raises a sticky flag; the engine then restores its snapshot and redoes the
// update on the two-loop path whose wide-range kernels have no such limits.
#include <cuda_fp16.h>

#include <cmath>

#include "common.cuh"
#include "policy_head.cuh"
#include "tc2_common.cuh"
#include "tc_common.cuh"
#include "tc3.cuh"

namespace b200rl {

constexpr int T3_ROWS = 128;
constexpr int T3_CHAIN_WARPS = 8;  // two chain warpgroups, one per 64-row half of the tile
constexpr int T3_THREADS = T3_CHAIN_WARPS * 32 + 256;  // + one weight-gradient warpgroup per m64 half of the A operand
constexpr int T3_WARPS = T3_THREADS / 32;

// ---- shared-memory map (bytes from the 1024-aligned base); one network per CTA ----
constexpr uint32_t S3_XB = 0;                        // X(k) in buffer k & 1
constexpr uint32_t S3_H1 = 2 * T2_ACT;               // fp16 pairs (h, then l): H1, H2, dZ2, dZ1
constexpr uint32_t S3_H2 = S3_H1 + 2 * T2_ACT;
constexpr uint32_t S3_DZ2 = S3_H2 + 2 * T2_ACT;
constexpr uint32_t S3_DZ1 = S3_DZ2 + 2 * T2_ACT;
constexpr uint32_t T3_W1T = 32 * 128, T3_W2 = 64 * 128, T3_W3 = 16 * 128;  // one split of each weight operand
constexpr uint32_t S3_DO = S3_DZ1 + 2 * T2_ACT;      // dOut: 16 columns h, then 16 columns l, at column 32 c
constexpr uint32_t S3_W = S3_DO + T2_ACT;            // W1T h,l | W2 h,l | W3 h,l
constexpr uint32_t S3_WNET = 2 * T3_W1T + 2 * T3_W2 + 2 * T3_W3;
constexpr uint32_t S3_OPERANDS_END = S3_W + S3_WNET;
constexpr uint32_t S3_BIAS = S3_OPERANDS_END;        // per net: b1[64] b2[64] b3[16] + pad = 160 floats
constexpr uint32_t S3_DIST = S3_BIAS + 2 * 640;      // var[16], log_scale[16], 1/(2 var)[16], 1/var[16]
constexpr uint32_t S3_SCALE = S3_DIST + 256;         // per net 16 floats
constexpr uint32_t S3_XS = S3_SCALE + 128;           // 2^ex_k [32], 2^-ex_k [32]
constexpr uint32_t S3_ADV = S3_XS + 256;             // advantage mean, 1 / std
constexpr uint32_t S3_RED = S3_ADV + 16;             // setup reduction scratch [16 warps][8] floats
constexpr uint32_t S3_BARS = S3_RED + 4 * 8 * T3_WARPS;  // 8 mbarriers (8 B each), bad flag at +120
// Per-row loss inputs of tile k in buffer k & 1, copied in with its observations (floats): policy: actions [128][A_out]
// (one column for a categorical policy) at 0, adv_raw at T3_LI_IN, old_logp at T3_LI_OLD; value: returns at T3_LI_IN.
constexpr uint32_t T3_LI_IN = 15 * T3_ROWS, T3_LI_OLD = 16 * T3_ROWS;
constexpr uint32_t T3_LI_BYTES = 17 * T3_ROWS * 4;
constexpr uint32_t S3_LOSS = S3_BARS + 128;
constexpr uint32_t S3_TOTAL = S3_LOSS + 2 * T3_LI_BYTES;
constexpr uint32_t T3_SMEM_BYTES = S3_TOTAL + 1024;  // + alignment slack
static_assert(T3_SMEM_BYTES <= 227 * 1024, "mlp_tc3 shared memory");
// end-of-kernel scratch, aliased onto the X buffers (every MMA has retired by then)
constexpr uint32_t S3_END_DB3 = 0;                   // [16 warps][16] floats
constexpr uint32_t S3_END_SC = 1024;                 // [16 warps][8] doubles

// ---- accumulator column map of the weight gradients (fp32) ----
// per net: DW2 (64) | DB2 (16, col 15 = db2) | DW1 (64: products with X's h columns, then with its l columns; col 31 =
// db1) | DW3 (32: products with dOut's h columns, then l).  The B operands of dW1 / dW3 hold their two splits side
// by side in one swizzle atom, so ONE product per k-step covers both; the halves are added when the accumulators
// are read, once per launch.  2 x 176 of the 512 columns; inside a product's columns the floats are fragment-major
// (grad_acc_off), not (row, column).
constexpr uint32_t ACC_GRAD_NET = 176;
// Running b3 sums: rows are tile rows, column 16 m + a holds sum class m (0..3) of output a (policy a < 15, value
// a = 15).  A row's output of tile k of network c goes to class (k + 2 c) & 3, and every class is added in tile order.
// The read-out then reduces class m with warp group m: the per-CTA sum is computed in the same order as when loss
// warps rotated over the tiles, so the b3 gradients do not depend on which thread evaluated a row.
constexpr uint32_t ACC_DB3 = 2 * ACC_GRAD_NET;
static_assert(ACC_DB3 + 4 * 16 <= ACC_COLS, "mlp_tc3 accumulator columns");
constexpr uint32_t ACC_DW2 = 0, ACC_DB2 = 64, ACC_DW1 = 80, ACC_DW3 = 144;

// Offset (floats into the CTA's accumulator block) of element (row, col) of the weight-gradient product with n columns
// that starts at accumulator column `pcol`.  Its n x 128 floats are fragment-major, not (row, column): the two m64
// halves' wgmma fragments one after the other, and in a fragment the 16-byte chunk j of issuing thread t (fragment
// elements 4 j .. 4 j + 3) is chunk 128 j + t.  A thread then loads and stores its fragment with n / 8 vector accesses,
// each of them 512 contiguous bytes per warp, and within the tile loop only the thread that wrote a float reads it.
__device__ __forceinline__ uint32_t grad_acc_off(uint32_t pcol, int n, int row, int col) {
  const int rr = row & 63;
  // wgmma D layout: thread t = 32 w + l holds rows 16 w + l / 4 (+ 8) and columns 8 j + 2 (l % 4) (+ 1)
  const int t = 32 * (rr >> 4) + 4 * (rr & 7) + ((col >> 1) & 3);
  const int e = 2 * ((rr >> 3) & 1) + (col & 1);
  return pcol * ACC_LANES + (uint32_t)((row >> 6) * 64 * n + 4 * (128 * (col >> 3) + t) + e);
}

#ifdef B200RL_TC3_TIMING
// CTA 0, chain warpgroup wg (64-row half): [10 wg + s - 1] cycles stage s (E1..E5) waited on an mbarrier,
// [10 wg + 4 + s] cycles of stage s in all (a stage ends when its result is stored, or delivered where it is handed to
// the gradient warpgroups; deliver(3) / deliver(4) come after the issue of dH2 / dH1); gradient warpgroup g (m64 half
// of A): [40 + 3 g + s - 3] cycles waited for the operands of stage s (3..5) (stage 4 of the observations' producer: also for the other half's dW3 to release the
// dOut buffer), [46 + 3 g + s - 3] cycles issuing its products, waiting for them and handing the buffers back;
// [52] tiles of the CTA, [53] set-up, [54] tile loop, [55] read-out
__device__ unsigned long long g_tc3_t[64];
#endif

enum { C3_G = 0, C3_U1, C3_U2, C3_U3, C3_UH2, C3_UH1, C3_W1, C3_W2, C3_W3, C3_OW3, C3_OW2, C3_OW1, C3_OB, C3_N };

__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// one contiguous span global -> shared, completion counted in bytes on the mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void bulk_copy_g2s(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}

// ------------------------------------------------------------------------------------------------------------------
// pack_obs: fp32 observations -> per-tile operand images.  Row r of a tile is 128 bytes: fp16 h-splits of the 32
// (zero-padded) scaled features, then their l-splits, 16-byte chunk j stored at chunk position j ^ (r & 7)
// (SWIZZLE_128B).  Feature k is scaled by 2^ex_k (its own maximum parked in [2^12, 2^13)); column 31 holds 1.0.
// The range / precision guards of mlp_tc2's E0 job run here, once per update.
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) pack_obs_kernel(const float* __restrict__ obs, long long n_rows, int n_in,
                                                       const float* __restrict__ absmax, uint8_t* __restrict__ ximg,
                                                       float* __restrict__ xscale, float* __restrict__ bad_flag) {
  __shared__ float s_xs[32];
  const int r = threadIdx.x;
  bool bad = false;
  if (r < 32) {
    const int e = r < n_in ? fit_exp(__ldg(absmax + r), bad) : 0;
    s_xs[r] = pow2i(e);
    if (blockIdx.x == 0) {
      xscale[r] = pow2i(e);
      xscale[32 + r] = pow2i(-e);
    }
  }
  __syncthreads();
  const long long tiles = (n_rows + T3_ROWS - 1) / T3_ROWS;
  for (long long t = blockIdx.x; t < tiles; t += gridDim.x) {
    const long long row = t * T3_ROWS + r;
    float x[32];
#pragma unroll
    for (int c = 0; c < 32; ++c) x[c] = 0.f;
    if (row < n_rows) {
      const float* src = obs + row * n_in;
      float rmax = 0.f, probe = 0.f;
#pragma unroll
      for (int c = 0; c < 31; ++c)
        if (c < n_in) {
          x[c] = __ldg(src + c) * s_xs[c];
          rmax = fmaxf(rmax, fabsf(x[c]));
          probe += x[c];
        }
      if (!(rmax <= T2_RANGE) || probe != probe) bad = true;
      // a row whose every feature sits 2^17 below its column's maximum has lost its l-splits
      if (rmax > 0.f && rmax < 0.03125f) bad = true;
      x[31] = 1.0f;
    }
    uint4 h[4], l[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      split2h(x[8 * j + 0], x[8 * j + 1], h[j].x, l[j].x);
      split2h(x[8 * j + 2], x[8 * j + 3], h[j].y, l[j].y);
      split2h(x[8 * j + 4], x[8 * j + 5], h[j].z, l[j].z);
      split2h(x[8 * j + 6], x[8 * j + 7], h[j].w, l[j].w);
    }
    uint8_t* dst = ximg + (size_t)t * T2_ACT + (size_t)r * 128;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      *reinterpret_cast<uint4*>(dst + ((j ^ (r & 7)) << 4)) = h[j];
      *reinterpret_cast<uint4*>(dst + (((4 + j) ^ (r & 7)) << 4)) = l[j];
    }
  }
  if (bad) *bad_flag = 1.0f;
}

// ------------------------------------------------------------------------------------------------------------------
// products
// ------------------------------------------------------------------------------------------------------------------
// D[64 x N] (+)= sum over TERMS of A_t B_t, KSTEPS k-steps of 16 each, as ONE group of wgmma m64nNk16: every k-step of
// every term back to back, one commit, one wait.  The fragment stays in the caller's registers.
template <int N, int TA, int TB, int TERMS, int KSTEPS>
__device__ __forceinline__ void wg_mma(float (&d)[N / 2], const uint32_t (&alo)[TERMS], const uint32_t (&blo)[TERMS],
                                       uint32_t a_hi, uint32_t b_hi, uint32_t a_k, uint32_t b_k, uint32_t accumulate) {
  wgmma_fence();
#pragma unroll
  for (int s = 0; s < TERMS; ++s)
#pragma unroll
    for (int k = 0; k < KSTEPS; ++k)
      wgmma_run<N, TA, TB>(d, ((uint64_t)a_hi << 32) | (alo[s] + (uint32_t)k * a_k),
                           ((uint64_t)b_hi << 32) | (blo[s] + (uint32_t)k * b_k), s == 0 && k == 0 ? accumulate : 1u);
  wgmma_commit();
  wgmma_wait_all();
}
// chain product of one 64-row half (A K-major, `a` already at the half's rows): (h,l) + (l,h) + (h,h), smallest terms
// first, overwriting the fragment
template <int N, int TB, int KSTEPS>
__device__ __forceinline__ void chain_mma(float (&d)[N / 2], const Op2 a, const Op2 b) {
  const uint32_t alo[3] = {a.lo, a.lo + a.split_step, a.lo}, blo[3] = {b.lo + b.split_step, b.lo, b.lo};
#pragma unroll
  for (int i = 0; i < N / 2; ++i) d[i] = 0.f;
  wg_mma<N, K_MAJOR, TB, 3, KSTEPS>(d, alo, blo, a.hi, b.hi, a.k_step, b.k_step, 0u);
}
// chain_mma with A from registers: ah[s] / al[s] = this thread's A fragment of k-step s in the h / l split (the previous
// epilogue's pairs, wgmma_f16_n64_rs).  The same terms in the same order, issued and committed but not waited for:
// until the caller's wgmma_wait_all, nothing may read or write d, ah or al.
template <int N, int TB, int KSTEPS>
__device__ __forceinline__ void chain_mma_rs(float (&d)[N / 2], const uint32_t (&ah)[KSTEPS][4],
                                             const uint32_t (&al)[KSTEPS][4], const Op2 b) {
#pragma unroll
  for (int i = 0; i < N / 2; ++i) d[i] = 0.f;
  wgmma_fence();
  auto desc = [&](uint32_t lo) { return ((uint64_t)b.hi << 32) | lo; };
#pragma unroll
  for (int k = 0; k < KSTEPS; ++k)
    wgmma_run_rs<N, TB>(d, ah[k], desc(b.lo + b.split_step + (uint32_t)k * b.k_step), k == 0 ? 0u : 1u);
#pragma unroll
  for (int k = 0; k < KSTEPS; ++k) wgmma_run_rs<N, TB>(d, al[k], desc(b.lo + (uint32_t)k * b.k_step), 1u);
#pragma unroll
  for (int k = 0; k < KSTEPS; ++k) wgmma_run_rs<N, TB>(d, ah[k], desc(b.lo + (uint32_t)k * b.k_step), 1u);
  wgmma_commit();
}
// Four 8 x 8 fp16 matrices between registers and shared memory; lane l gives the address of row l & 7 of matrix l >> 3
__device__ __forceinline__ void stmatrix_x4(uint32_t addr, const uint32_t (&r)[4]) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r[0]), "r"(r[1]),
               "r"(r[2]), "r"(r[3])
               : "memory");
}
__device__ __forceinline__ void ldmatrix_x4(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr)
               : "memory");
}
// This thread's fragment of the first m64 half of the weight-gradient product at column pcol, whatever its N:
// grad_acc_off's layout puts chunk j of the fragment 512 j floats further and the second half 64 N floats further.
__device__ __forceinline__ float* grad_frag(float* acc_cta, uint32_t pcol) {
  const int t = (int)(threadIdx.x & 127u);
  return acc_cta + grad_acc_off(pcol, 0, 16 * (t >> 5) + ((t & 31) >> 2), 2 * (t & 3));
}
// The products of one weight-gradient fragment `d` (both operands MN-major): TERMS terms (B split l, then h), KSTEPS
// k-steps each, A at descriptor low word `a_lo`; the first product overwrites on the first tile.
template <int N, int KSTEPS, int TERMS>
__device__ __forceinline__ void grad_products(float (&d)[N / 2], uint32_t a_lo, const Op2 a, const Op2 b, bool first) {
  // an opaque copy per product: products that share A would otherwise share its k-step descriptors, held live (and
  // spilled) next to the group's fragments
  uint32_t b_lo = b.lo;
  asm volatile("" : "+r"(a_lo), "+r"(b_lo));
#pragma unroll
  for (int s = 0; s < TERMS; ++s)
#pragma unroll
    for (int k = 0; k < KSTEPS; ++k)
      wgmma_run<N, MN_MAJOR, MN_MAJOR>(d, ((uint64_t)a.hi << 32) | (a_lo + (uint32_t)k * a.k_step),
                                       ((uint64_t)b.hi << 32) | (b_lo + (s + 1 < TERMS ? b.split_step : 0u) +
                                                                 (uint32_t)k * b.k_step),
                                       s == 0 && k == 0 ? (first ? 0u : 1u) : 1u);
}
// Stores this thread's fragment of m64 half `h` of the weight-gradient product with N columns at accumulator column
// `pcol` in grad_acc_off's layout: chunk j (fragment elements 4 j .. 4 j + 3) 512 j floats further.
template <int N>
__device__ __forceinline__ void grad_store(float* acc_cta, uint32_t pcol, int h, const float (&d)[N / 2]) {
  float* const frag = grad_frag(acc_cta, pcol) + 64 * N * h;
#pragma unroll
  for (int j = 0; j < N / 8; ++j)
    *reinterpret_cast<float4*>(frag + 512 * j) = make_float4(d[4 * j], d[4 * j + 1], d[4 * j + 2], d[4 * j + 3]);
}

// ------------------------------------------------------------------------------------------------------------------
// the step kernel
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(T3_THREADS, 1) mlp_tc3_kernel(const Tc3Args p) {
  extern __shared__ uint8_t smem_raw[];
  // Network c of this CTA (0 policy, 1 value) and its tile slot: with both networks launched, CTA c G + slot; with
  // one, CTA slot.  Both CTAs of a slot take tiles slot + k G and share accumulator block `slot` (disjoint columns).
  // Network-major order: the G policy CTAs (one per SM) make the first wave and the value CTAs the second, so every
  // SM runs one CTA of each network.  Interleaved, the SMs that drew a policy CTA for the first wave would have been
  // freed last and drawn half of the second wave's policy CTAs too.
  const bool two = p.run_policy != 0 && p.run_value != 0;
  const int G = two ? (int)(gridDim.x >> 1) : (int)gridDim.x;
  const int c = two ? (int)blockIdx.x / G : (p.run_policy != 0 ? 0 : 1);
  const int slot = (int)blockIdx.x - c * (two ? G : 0);
  // which network runs is the same for every thread of the grid
  const bool run_p = p.run_policy != 0 && (p.stop_flag == nullptr || *p.stop_flag == 0);
  const bool run_v = p.run_value != 0;
  if (!(c == 0 ? run_p : run_v)) return;
  if (*p.x_bad != 0.f) return;  // the packed observations left the fp16 range: the engine redoes the update (wide-range path)
  const int tid = threadIdx.x, lane = tid & 31;
  float* const acc = p.acc_mem + (size_t)slot * ACC_CTA_FLOATS;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);  // provably warp-uniform (see mlp_tc2.cu)
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* sm = smem_raw + (base - raw);
  float* s_bias = reinterpret_cast<float*>(sm + S3_BIAS);
  float* s_dist = reinterpret_cast<float*>(sm + S3_DIST);
  float* s_scale = reinterpret_cast<float*>(sm + S3_SCALE);
  float* s_xs = reinterpret_cast<float*>(sm + S3_XS);
  float* s_adv = reinterpret_cast<float*>(sm + S3_ADV);
  float* s_red = reinterpret_cast<float*>(sm + S3_RED);
  int* s_bad = reinterpret_cast<int*>(sm + S3_BARS + 120);
  const uint32_t bars = base + S3_BARS;
  const int n_in = p.n_in;
  bool bad = false;
#ifdef B200RL_TC3_TIMING
  unsigned long long tacc[64];
  for (int i = 0; i < 64; ++i) tacc[i] = 0;
  const long long t_kernel0 = clock64();
#endif

  // ---- one-time setup: scales; weights of this CTA's network as fp16 pairs; biases ----
  // Only the weight operands need zero padding (X tiles arrive whole by bulk copy, H, dZ and dOut are fully written by
  // their epilogues before any MMA reads them).  Both parameter vectors (44 KB) are first brought into the still unused
  // activation buffers with independent, coalesced loads: the two passes below (maxima, then conversion) would
  // otherwise pay an L2 round trip per element, one after the other (17 of the 18 us this set-up took on B200).  Every
  // CTA checks both networks' parameters, so a range trip is raised whichever networks run.
  for (uint32_t i = S3_W / 16 + tid; i < S3_OPERANDS_END / 16; i += T3_THREADS) reinterpret_cast<uint4*>(sm)[i] = make_uint4(0, 0, 0, 0);
  if (tid == 0) {
    *s_bad = 0;
    float adv_mean, adv_std;  // utils.py:91 (mean 0, std 1 without statistics)
    adv_mean_std(p.adv_stats, adv_mean, adv_std);
    s_adv[0] = adv_mean;
    s_adv[1] = 1.f / adv_std;
  }
  if (tid < 64) s_xs[tid] = __ldg(p.xscale + tid);
  float* s_par = reinterpret_cast<float*>(sm + S3_H1);
  static_assert(S3_W - S3_H1 >= 4 * (2 * 6000 + 64), "parameter staging area");
#pragma unroll 1
  for (int net = 0; net < 2; ++net) {
    const float* par = p.params[net];
    float* dst = s_par + (net == 0 ? 0 : p.P[0]);
#pragma unroll 8
    for (int i = tid; i < p.P[net]; i += T3_THREADS) dst[i] = (*(par + i));
  }
  __syncthreads();
#pragma unroll 1
  for (int net = 0; net < 2; ++net) {
    const Tc3Net& nn = p.net[net];
    const float* par = s_par + (net == 0 ? 0 : p.P[0]);
    float m1 = 0.f, m2 = 0.f, m3 = 0.f;
    for (int idx = tid; idx < nn.h1 * n_in; idx += T3_THREADS) {
      const float w = (*(par + nn.w_off[0] + idx)) * s_xs[32 + idx % n_in];
      m1 = fmaxf(m1, fabsf(w));
      if (w != w) bad = true;
    }
    for (int idx = tid; idx < nn.h2 * nn.h1; idx += T3_THREADS) {
      const float w = (*(par + nn.w_off[1] + idx));
      m2 = fmaxf(m2, fabsf(w));
      if (w != w) bad = true;
    }
    for (int idx = tid; idx < nn.n_out * nn.h2; idx += T3_THREADS) {
      const float w = (*(par + nn.w_off[2] + idx));
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
      s_red[warp * 8 + 4 * net + 0] = m1;
      s_red[warp * 8 + 4 * net + 1] = m2;
      s_red[warp * 8 + 4 * net + 2] = m3;
    }
  }
  __syncthreads();
  if (bad) *s_bad = 1;  // NaN weight
  bad = false;
  if (tid < 2) {
    const int net = tid;
    const Tc3Net& nn = p.net[net];
    float m1 = 0.f, m2 = 0.f, m3 = 0.f;
    for (int w = 0; w < T3_WARPS; ++w) {
      m1 = fmaxf(m1, s_red[w * 8 + 4 * net + 0]);
      m2 = fmaxf(m2, s_red[w * 8 + 4 * net + 1]);
      m3 = fmaxf(m3, s_red[w * 8 + 4 * net + 2]);
    }
    bool b0 = false;
    const int ew1 = fit_exp(m1, b0), ew2 = fit_exp(m2, b0), ew3 = fit_exp(m3, b0);
    float typ;  // typical magnitude of N * dLoss/dOut: the gradient scale parks it near 2^3
    if (net == 1) {
      const float tm = __ldg(p.target_absmax);
      typ = (tm > 0.f && tm < INFINITY) ? 0.25f * tm : 1.f;
    } else if (p.dist == B200RL_DIST_GAUSSIAN) {
      float smin = INFINITY;
      for (int a = 0; a < nn.n_out; ++a) smin = fminf(smin, expf(__ldg(p.log_std + a)));
      typ = (smin > 0.f && smin < INFINITY) ? 1.f / smin : 1.f;
    } else {
      typ = 0.5f;
    }
    int eg = 3 + ilogbf(p.n_glob_f) - ilogbf(typ);
    eg = eg < -100 ? -100 : (eg > 100 ? 100 : eg);
    float* sc = s_scale + 16 * net;
    sc[C3_G] = pow2i(eg);
    sc[C3_U1] = pow2i(-ew1);
    sc[C3_U2] = pow2i(-(T2_H_EXP + ew2));
    sc[C3_U3] = pow2i(-(T2_H_EXP + ew3));
    sc[C3_UH2] = pow2i(-ew3);
    sc[C3_UH1] = pow2i(-ew2);
    sc[C3_W1] = pow2i(ew1);
    sc[C3_W2] = pow2i(ew2);
    sc[C3_W3] = pow2i(ew3);
    sc[C3_OW3] = pow2i(-(T2_H_EXP + eg));
    sc[C3_OW2] = pow2i(-(T2_H_EXP + eg));
    sc[C3_OW1] = pow2i(-eg);  // times 2^-ex_k of the column, applied when the accumulator is read
    sc[C3_OB] = pow2i(-eg);
    if (b0) *s_bad = 1;
  }
  __syncthreads();
#pragma unroll 1
  for (int net = 0; net < 2; ++net) {
    const Tc3Net& nn = p.net[net];
    const float* par = s_par + (net == 0 ? 0 : p.P[0]);
    const uint32_t wb = S3_W;
    auto put = [&](uint32_t buf, uint32_t stride, int r, int c, float x) {
      const __half hb = __float2half_rn(x);
      const __half lb = __float2half_rn(x - __half2float(hb));
      const uint32_t off = buf + (uint32_t)r * 128u + ((uint32_t)((c >> 3) ^ (r & 7)) << 4) + ((uint32_t)(c & 7) << 1);
      *reinterpret_cast<__half*>(sm + off) = hb;
      *reinterpret_cast<__half*>(sm + off + stride) = lb;
    };
    const float* sc = s_scale + 16 * net;
    const float sw1 = sc[C3_W1], sw2 = sc[C3_W2], sw3 = sc[C3_W3];
    if (net == c) {
      for (int idx = tid; idx < nn.h1 * n_in; idx += T3_THREADS)  // W1 transposed: row = input, column = output
        put(wb, T3_W1T, idx % n_in, idx / n_in, ((*(par + nn.w_off[0] + idx)) * s_xs[32 + idx % n_in]) * sw1);
      for (int idx = tid; idx < nn.h2 * nn.h1; idx += T3_THREADS)
        put(wb + 2 * T3_W1T, T3_W2, idx / nn.h1, idx % nn.h1, (*(par + nn.w_off[1] + idx)) * sw2);
      for (int idx = tid; idx < nn.n_out * nn.h2; idx += T3_THREADS)
        put(wb + 2 * T3_W1T + 2 * T3_W2, T3_W3, idx / nn.h2, idx % nn.h2, (*(par + nn.w_off[2] + idx)) * sw3);
    }
    float* bb = s_bias + 160 * net;
    for (int i = tid; i < 64; i += T3_THREADS) {
      bb[i] = i < nn.h1 ? (*(par + nn.b_off[0] + i)) : 0.f;
      bb[64 + i] = i < nn.h2 ? (*(par + nn.b_off[1] + i)) : 0.f;
      if (!(fabsf(bb[i]) < INFINITY) || !(fabsf(bb[64 + i]) < INFINITY)) bad = true;
    }
    for (int i = tid; i < 16; i += T3_THREADS) {
      bb[128 + i] = i < nn.n_out ? (*(par + nn.b_off[2] + i)) : 0.f;
      if (!(fabsf(bb[128 + i]) < INFINITY)) bad = true;
    }
  }
  if (p.dist == B200RL_DIST_GAUSSIAN)
    for (int a = tid; a < p.net[0].n_out; a += T3_THREADS) {
      const NormalConsts nc = normal_consts(p.log_std, a);
      s_dist[a] = nc.var;
      s_dist[16 + a] = nc.log_scale;
      s_dist[32 + a] = nc.inv_2var;
      s_dist[48 + a] = nc.inv_var;
    }
  if (bad) *s_bad = 1;  // non-finite bias
  bad = false;
  if (tid == 0) {
    mbar_init(bars + 0, 1);  // xfull[b]: arrive.expect_tx by the producer + the copy's bytes
    mbar_init(bars + 8, 1);
    for (int i = 0; i < 3; ++i) {
      mbar_init(bars + 16 + 8 * i, 2);  // ready[s]: one arrive per chain warpgroup
      mbar_init(bars + 40 + 8 * i, 2);  // done[s]: one arrive per gradient warpgroup
    }
    fence_mbar_init();
  }
  fence_proxy_async_smem();
  __syncthreads();

  const long long num_tiles = (p.n_rows + T3_ROWS - 1) / T3_ROWS;
  const int cta_tiles = (int)((num_tiles - slot + G - 1) / G);  // tiles slot + k * G

  constexpr int K = K_MAJOR, MN = MN_MAJOR;
  const uint32_t ub = base;
  // mbarriers: xfull[b] at +8b; ready[s - 3] at +16 + 8 (s - 3) (both chain warpgroups have delivered the operands of
  // stage s); done[s - 3] at +40 + 8 (s - 3) (both gradient warpgroups' products of stage s have read their buffers)
  auto bar_ready = [&](int s) { return bars + 16u + 8u * (uint32_t)(s - 3); };
  auto bar_done = [&](int s) { return bars + 40u + 8u * (uint32_t)(s - 3); };
  // the per-thread sums of the chain rows this thread owned (read out below).  Policy: loss terms, old_logp - logp,
  // entropy, logp, logp^2; value: sc[0] = squared errors.  (The b3 sums live in accumulator memory, ACC_DB3.)
  double sc[5] = {0, 0, 0, 0, 0};
  int rows_done = 0;  // policy rows evaluated
#ifdef B200RL_TC3_TIMING
  long long t_loop0 = 0, t_loop_end = 0;
#endif

  if (warp >= T3_CHAIN_WARPS) {
    // ============ weight-gradient warpgroup g: rows 64 g .. 64 g + 63 of every stacked A operand (split h / l) ============
    // Issues its half of the stage 3..5 products of every tile into accumulators that stay in its registers for the
    // whole launch: dW3 n32, dW2 n64, db2 n16, dW1 n64 (88 floats).  Each product sees the same terms in the same order
    // as when the fragments went through L2 tile by tile.  Warpgroup 0 also brings the observation tiles in.
    // views at X buffer 0; the other is reached by adding a byte offset to the descriptors
    const Op2 X_M = op2_mnmajor(ub + S3_XB, T2_ACT, 64);         // B, N = 64: features h 0..31 (col 31 = ones) | l
    const Op2 X_M16 = op2_mnmajor(ub + S3_XB + 32, T2_ACT, 64);  // B, N = 16: h cols 16..31 (col 31 = ones)
    const Op2 DO_M = op2_at(op2_mnmajor(ub + S3_DO, T2_ACT, 32), c * 64);  // B, N = 32: dOut h | l
    const Op2 H1_M = op2_mnmajor(ub + S3_H1, T2_ACT, T2_ACT), H2_M = op2_mnmajor(ub + S3_H2, T2_ACT, T2_ACT);
    const Op2 DZ2_M = op2_mnmajor(ub + S3_DZ2, T2_ACT, T2_ACT), DZ1_M = op2_mnmajor(ub + S3_DZ1, T2_ACT, T2_ACT);
    const int g = (warp - T3_CHAIN_WARPS) >> 2;
    const bool producer = g == 0;
    const uint32_t ah = (uint32_t)g * (T2_ACT >> 4);  // this half's split of an A operand: descriptor low-word offset
    const uint32_t gcol = c * ACC_GRAD_NET;
    float w3[16], w2[32], b2[8], w1[32];
    // tile k of this CTA -> X buffer k & 1, and its per-row loss inputs -> loss-input buffer k & 1.  The engine pads
    // those columns to whole tiles, so the last tile's copies stay inside their allocations.
    const uint32_t act_bytes = T3_ROWS * 4u * (uint32_t)(p.dist == B200RL_DIST_GAUSSIAN ? p.net[0].n_out : 1);
    auto load_x = [&](int k) {
      const uint32_t b = (uint32_t)(k & 1), bar = bars + 8 * b;
      const long long tile = slot + (long long)k * G;
      const size_t row0 = (size_t)tile * T3_ROWS;
      const uint32_t li = ub + S3_LOSS + b * T3_LI_BYTES;
      uint32_t e;
      asm volatile("{\n\t.reg .pred q;\n\telect.sync _|q, 0xffffffff;\n\tselp.u32 %0, 1, 0, q;\n\t}" : "=r"(e));
      if (e && (warp & 3) == 0) {  // one thread of the warpgroup
        if (c == 0) {
          mbar_arrive_expect_tx(bar, T2_ACT + act_bytes + 2 * T3_ROWS * 4);
          bulk_copy_g2s(li, reinterpret_cast<const uint8_t*>(p.actions) + (size_t)tile * act_bytes, act_bytes, bar);
          bulk_copy_g2s(li + 4 * T3_LI_IN, p.adv_raw + row0, T3_ROWS * 4, bar);
          bulk_copy_g2s(li + 4 * T3_LI_OLD, p.old_logp + row0, T3_ROWS * 4, bar);
        } else {
          mbar_arrive_expect_tx(bar, T2_ACT + T3_ROWS * 4);
          bulk_copy_g2s(li + 4 * T3_LI_IN, p.target + row0, T3_ROWS * 4, bar);
        }
        bulk_copy_g2s(ub + S3_XB + b * T2_ACT, p.ximg + (size_t)tile * T2_ACT, T2_ACT, bar);
      }
      __syncwarp();
    };
    // every warp's share of the stage's products has retired: its buffers go back to the chains
    auto release = [&](int stage) {
      wgmma_commit();
      wgmma_wait_all();
      asm volatile("bar.sync %0, 128;" ::"r"(8 + g) : "memory");
      if ((tid & 127) == 0) mbar_arrive(bar_done(stage));
    };
    if (producer && cta_tiles > 0) load_x(0);
#pragma unroll 1
    for (int k = 0; k < cta_tiles; ++k) {
      const uint32_t xo = (uint32_t)(k & 1) * T2_ACT;
      const bool first = k == 0;  // the first tile's products overwrite the accumulators
      if (producer && k + 1 < cta_tiles) {
        // tile k + 1 goes to the buffers of tile k - 1, whose last readers (db2 and dW1 of both halves; the chains'
        // E3 for the loss inputs) are done once done[5] completes its tile k - 1 phase.  It cannot be a phase
        // further: its tile k phase needs this warpgroup's own tile k arrival.
        if (k > 0) mbar_wait(bar_done(5), (uint32_t)((k - 1) & 1));
        load_x(k + 1);
      }
#ifdef B200RL_TC3_TIMING
      long long it0 = clock64(), it1;
#define TC3_GSPLIT(s)                                                   \
  it1 = clock64();                                                      \
  tacc[40 + 3 * g + (s) - 3] += (unsigned long long)(it1 - it0);
#define TC3_GEND(s)                                                     \
  it0 = clock64();                                                      \
  tacc[46 + 3 * g + (s) - 3] += (unsigned long long)(it0 - it1);
#else
#define TC3_GSPLIT(s)
#define TC3_GEND(s)
#endif
      // dW3^T[i][o] += sum_r H2[r][i] dOut[r][o]
      mbar_wait(bar_ready(3), (uint32_t)(k & 1));
      TC3_GSPLIT(3)
      wgmma_fence();
      grad_products<32, 8, 1>(w3, H2_M.lo + ah, H2_M, DO_M, first);
      release(3);
      TC3_GEND(3)
      // dW2[o][i] += sum_r dZ2[r][o] H1[r][i] ; db2[o] += sum_r dZ2[r][o] * 1 (ones column of X)
      mbar_wait(bar_ready(4), (uint32_t)(k & 1));
      TC3_GSPLIT(4)
      wgmma_fence();
      grad_products<64, 8, 2>(w2, DZ2_M.lo + ah, DZ2_M, H1_M, first);
      grad_products<16, 8, 1>(b2, DZ2_M.lo + ah, DZ2_M, op2_at(X_M16, xo), first);
      release(4);
      TC3_GEND(4)
      // dW1[o][i] += sum_r dZ1[r][o] X[r][i]; column 31 (ones) collects db1
      mbar_wait(bar_ready(5), (uint32_t)(k & 1));
      TC3_GSPLIT(5)
      wgmma_fence();
      grad_products<64, 8, 1>(w1, DZ1_M.lo + ah, DZ1_M, op2_at(X_M, xo), first);
      release(5);
      TC3_GEND(5)
#undef TC3_GSPLIT
#undef TC3_GEND
    }
    if (cta_tiles > 0) {  // once per launch: the fragments into the CTA's accumulator block, read out below
      grad_store<32>(acc, gcol + ACC_DW3, g, w3);
      grad_store<64>(acc, gcol + ACC_DW2, g, w2);
      grad_store<16>(acc, gcol + ACC_DB2, g, b2);
      grad_store<64>(acc, gcol + ACC_DW1, g, w1);
    }
#ifdef B200RL_TC3_TIMING
    if ((tid & 127) == 0 && blockIdx.x == 0) {
      for (int s = 0; s < 3; ++s) {
        g_tc3_t[40 + 3 * g + s] = tacc[40 + 3 * g + s];
        g_tc3_t[46 + 3 * g + s] = tacc[46 + 3 * g + s];
      }
      if (producer) g_tc3_t[52] = (unsigned long long)cta_tiles;
    }
#endif
  } else {
    // ========================= chain warpgroup wg: rows 64 wg .. 64 wg + 63 of the tile =========================
    // Z1 -> E1 -> Z2 -> E2 -> OUT -> E3 -> dH2 -> E4 -> dH1 -> E5 with the accumulator in this warpgroup's registers.
    // Fragment element i of a thread is row r0 + 8 ((i >> 1) & 1), column 8 (i >> 2) + 2 q + (i & 1) (wgmma D layout).
    // dZ2 and dZ1 have buffers of their own, so the gradient products of a tile can run while the chains go on to the
    // next one: a chain only waits for the previous tile's readers of a buffer it is about to overwrite.
    const int wg = warp >> 2;
    const int quad = lane >> 2, q = lane & 3;
    const int r0 = 64 * wg + 16 * (warp & 3) + quad;  // == quad (mod 8): the swizzle phase of both fragment rows
    const uint32_t rows = (uint32_t)wg * (64u * 128u);  // this half in a K-major buffer
    // Z1's A, X, comes from shared memory (the bulk copy puts it there); the later products take A from registers
    const Op2 X_K = op2_at(op2_kmajor(ub + S3_XB, 64), rows);  // A: X, h at +0, l at +64 bytes
    const Op2 W1T_M = op2_mnmajor(ub + S3_W, 32 * 128, T3_W1T);
    const Op2 W2_K = op2_kmajor(ub + S3_W + 2 * T3_W1T, T3_W2), W2_M = op2_mnmajor(ub + S3_W + 2 * T3_W1T, 64 * 128, T3_W2);
    const Op2 W3_K = op2_kmajor(ub + S3_W + 2 * T3_W1T + 2 * T3_W2, T3_W3),
              W3_M = op2_mnmajor(ub + S3_W + 2 * T3_W1T + 2 * T3_W2, 16 * 128, T3_W3);
    const float* scl = s_scale + 16 * c;
    const float* bias = s_bias + 160 * c;
    const float sH = pow2i(T2_H_EXP), hh = pow2i(-2 * T2_H_EXP);
    const int A_out = p.net[0].n_out;

    // A packed pair of fragment elements (4 j + 2 r, +1: row r0 + 8 r, columns 8 j + 2 q, +1) is this thread's share of
    // the 8 x 8 fp16 matrix (rows 8 r .. 8 r + 7 of the warp's 16, 16-byte chunk j), as stmatrix / ldmatrix lay it out,
    // and a row of that matrix is one 16-byte chunk of a SWIZZLE_128B buffer.  One .x4 access moves matrices
    // (j, 0), (j, 1), (j + 1, 0), (j + 1, 1) for even j, i.e. fragment elements 4 j .. 4 j + 7; lane l gives the address
    // of row l & 7 of matrix l >> 3: at `buf` + mat_off(j), chunk (j + (l >> 4)) ^ (l & 7) = j ^ ((l >> 4) ^ (l & 7)).
    // The four registers of one .x4 access (j = 2 s) are also the wgmma A fragment of k-step s, in the order a0..a3:
    // the chain's next product takes them from registers (chain_mma_rs) instead of reading the buffer back.
    const uint32_t mat_row = base + (uint32_t)(64 * wg + 16 * (warp & 3) + 8 * ((lane >> 3) & 1) + (lane & 7)) * 128u;
    const uint32_t mat_chunk = (uint32_t)((lane >> 4) ^ (lane & 7)) << 4;
    auto mat_off = [&](uint32_t buf, int j) -> uint32_t { return mat_row + buf + (((uint32_t)j << 4) ^ mat_chunk); };
    uint32_t ph[4][4], pl[4][4];  // the fragment's fp16 pairs, h and l split: [k-step of the next product][a0..a3]
    auto split_pairs = [&](const float (&x)[32]) {
#pragma unroll
      for (int s = 0; s < 4; ++s)
#pragma unroll
        for (int m = 0; m < 4; ++m) split2h(x[8 * s + 2 * m], x[8 * s + 2 * m + 1], ph[s][m], pl[s][m]);
    };
    auto store_pairs = [&](uint32_t buf) {
#pragma unroll
      for (int s = 0; s < 4; ++s) {
        stmatrix_x4(mat_off(buf, 2 * s), ph[s]);
        stmatrix_x4(mat_off(buf + T2_ACT, 2 * s), pl[s]);
      }
    };
    // E1 / E2: Z * unscale + bias -> tanh(.) * 2^14
    auto act = [&](float (&z)[32], float unscale, const float* bs) {
#pragma unroll
      for (int g = 0; g < 2; ++g) {
        float t[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          const int e = 16 * g + i;
          t[i] = fmaf(z[e], unscale, bs[8 * (e >> 2) + 2 * q + (e & 1)]);
        }
        tanh16_scaled(t, sH);
#pragma unroll
        for (int i = 0; i < 16; ++i) z[16 * g + i] = t[i];
      }
    };
    // E4 / E5: dZ (scaled) = dH * unscale * (1 - H^2), H read back from its fp16 pair in `buf`.
    // (1 - H^2) * 2^28 = fma(-Hs, Hs, 2^28) with Hs = H * 2^14 as stored; 2^-28 is folded into the unscale factor
    auto dtanh = [&](float (&g)[32], float unscale, uint32_t buf) {
      const float one28 = 268435456.f;
      float m = 0.f;
#pragma unroll
      for (int j = 0; j < 8; j += 2) {
        uint32_t hw[4], lw[4];
        ldmatrix_x4(mat_off(buf, j), hw);
        ldmatrix_x4(mat_off(buf + T2_ACT, j), lw);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&hw[i]));
          const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&lw[i]));
          const float x0 = a.x + b.x, x1 = a.y + b.y;
          float& g0 = g[4 * j + 2 * i];
          float& g1 = g[4 * j + 2 * i + 1];
          g0 = (g0 * unscale) * fmaf(-x0, x0, one28);
          g1 = (g1 * unscale) * fmaf(-x1, x1, one28);
          m = fmaxf(m, fmaxf(fabsf(g0), fabsf(g1)));
        }
      }
      if (!(m <= T2_RANGE)) bad = true;  // magnitude only: the inputs were checked
    };
    // this warpgroup's shared-memory writes -> visible to the gradient warpgroups' products of stage s (the barrier also
    // orders H1 / H2 before dtanh reads them back).  deliver(3) and deliver(4) run under the chain's next product, whose
    // registers and operands they do not touch.
    auto deliver = [&](int s) {
      fence_proxy_async_smem();
      asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
      if ((tid & 127) == 0) mbar_arrive(bar_ready(s));
    };
#ifdef B200RL_TC3_TIMING
    long long t_mark = 0;
#endif
    auto wait = [&](int s, uint32_t bar, uint32_t parity) {
#ifdef B200RL_TC3_TIMING
      const long long w0 = clock64();
#endif
      mbar_wait(bar, parity);
#ifdef B200RL_TC3_TIMING
      tacc[10 * wg + s - 1] += (unsigned long long)(clock64() - w0);
#endif
    };
    auto stage_end = [&](int s) {
#ifdef B200RL_TC3_TIMING
      const long long t = clock64();
      tacc[10 * wg + 4 + s] += (unsigned long long)(t - t_mark);
      t_mark = t;
#endif
    };

#ifdef B200RL_TC3_TIMING
    t_loop0 = clock64();
    t_mark = t_loop0;
#endif
    {
#pragma unroll 1
      for (int k = 0; k < cta_tiles; ++k) {
        const long long tile = slot + (long long)k * G;
        const uint32_t xo = (uint32_t)(k & 1) * T2_ACT;
        float d[32];
        // ---- Z1 = X W1^T -> E1 -> H1 ----
        wait(1, bars + 8 * (uint32_t)(k & 1), (uint32_t)((k >> 1) & 1));  // the tile's observations have arrived
        chain_mma<64, MN, 2>(d, op2_at(X_K, xo), W1T_M);
        act(d, scl[C3_U1], bias);
        split_pairs(d);
        // dW3, dW2 and db2 of the last tile have read H2, dOut, dZ2 and H1 (the chains' own products, in order)
        if (k > 0) wait(1, bar_done(4), (uint32_t)((k - 1) & 1));
        // H1 and H2 are written for the gradient warpgroups (deliver(4), deliver(3)) and for this warp's own dtanh; no
        // chain product reads them back, so no warpgroup barrier follows
        store_pairs(S3_H1);
        stage_end(1);
        // ---- Z2 = H1 W2^T -> E2 -> H2 ----
        chain_mma_rs<64, K, 4>(d, ph, pl, W2_K);
        wgmma_wait_all();
        act(d, scl[C3_U2], bias + 64);
        split_pairs(d);
        store_pairs(S3_H2);
        stage_end(2);
        // ---- OUT = H2 W3^T -> E3: loss head, one row per owner thread (lanes q = 0, 1 own rows r0, r0 + 8) ----
        const int orow = r0 + 8 * q;
        const long long row = tile * T3_ROWS + orow;
        const bool owner = q < 2, valid = owner && row < p.n_rows;
        // this row's running b3 sums of its class (ACC_DB3); a class starts at zero on its first tile, k < 4
        float* const s3p = acc + (ACC_DB3 + 16u * (uint32_t)((k + 2 * c) & 3)) * ACC_LANES + orow;
        float o[8];
        chain_mma_rs<16, K, 4>(o, ph, pl, W3_K);
        wgmma_wait_all();
        // the row's loss inputs, copied in with the tile's observations (xfull[k & 1], waited for above)
        const float* li = reinterpret_cast<const float*>(sm + S3_LOSS + (uint32_t)(k & 1) * T3_LI_BYTES);
        float pf_act[15], pf_in = 0.f, pf_old = 0.f;  // pf_in: the advantage (policy) or the return (value)
#pragma unroll
        for (int a = 0; a < 15; ++a) pf_act[a] = 0.f;
        if (valid) {
          if (c == 0) {
            if (p.dist == B200RL_DIST_GAUSSIAN) {
#pragma unroll
              for (int a = 0; a < 15; ++a)
                if (a < A_out) pf_act[a] = li[orow * A_out + a];
            } else {
              pf_act[0] = li[orow];
            }
            pf_old = li[T3_LI_OLD + orow];
          }
          pf_in = li[T3_LI_IN + orow];
        }
        float out[16];  // the owner's output row, gathered from its quad
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
          for (int qq = 0; qq < 4; ++qq)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const float v0 = __shfl_sync(0xffffffffu, o[4 * j + e], (lane & ~3) | qq);
              const float v1 = __shfl_sync(0xffffffffu, o[4 * j + 2 + e], (lane & ~3) | qq);
              out[8 * j + 2 * qq + e] = q == 0 ? v0 : v1;
            }
        float x0[8], x1[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) x0[j] = x1[j] = 0.f;
        if (owner) {
          const float u3 = scl[C3_U3], sG = scl[C3_G];
          if (c == 0) {
            float dout[16];
#pragma unroll
            for (int a = 0; a < 16; ++a) {
              out[a] = fmaf(out[a], u3, bias[128 + a]);
              dout[a] = 0.f;
            }
            if (valid) {
              float lp, ent, dlp[16];
#pragma unroll
              for (int a = 0; a < 16; ++a) dlp[a] = 0.f;
              if (p.dist == B200RL_DIST_GAUSSIAN)
                gaussian_logp<15>(pf_act, out, s_dist + 16, VarRecip{s_dist + 48, s_dist + 32}, A_out, lp, ent, dlp);
              else
                categorical_logp<15>(out, (int)pf_act[0], A_out, lp, ent, dlp);  // value.long()
              const float adv = (pf_in - s_adv[0]) * s_adv[1];
              float coef;
              const float term = policy_loss(B200RL_LOSS_PPO_CLIP, lp, pf_old, adv, p.inv_n, p.clip_lo, p.clip_hi, coef);
#pragma unroll
              for (int a = 0; a < 15; ++a) dout[a] = coef * dlp[a];
              add_policy_row_sums(sc, term, lp, ent, pf_old, true);
            }
#pragma unroll
            for (int a = 0; a < 15; ++a) s3p[a * ACC_LANES] = (k >= 4 ? s3p[a * ACC_LANES] : 0.f) + dout[a];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              x0[j] = dout[j] * sG;
              x1[j] = j < 7 ? dout[8 + j] * sG : 0.f;
            }
          } else {
            float s3 = k >= 4 ? s3p[15 * ACC_LANES] : 0.f;
            if (valid) {
              float dout;
              sc[0] += (double)value_mse(fmaf(out[0], u3, bias[128]), pf_in, p.inv_n, dout);
              s3 += dout;
              x0[0] = dout * sG;
            }
            s3p[15 * ACC_LANES] = s3;
          }
          if (out_of_range8(x0) || out_of_range8(x1)) bad = true;
        }
        if (owner) {
          // 16 columns h, then 16 columns l, at fp16 columns 32 c .. 32 c + 31 of the dOut buffer
          uint4 h0, l0, h1, l1;
          split2h(x0[0], x0[1], h0.x, l0.x);
          split2h(x0[2], x0[3], h0.y, l0.y);
          split2h(x0[4], x0[5], h0.z, l0.z);
          split2h(x0[6], x0[7], h0.w, l0.w);
          split2h(x1[0], x1[1], h1.x, l1.x);
          split2h(x1[2], x1[3], h1.y, l1.y);
          split2h(x1[4], x1[5], h1.z, l1.z);
          split2h(x1[6], x1[7], h1.w, l1.w);
          uint8_t* rowp = sm + S3_DO + (uint32_t)orow * 128u;
          const uint32_t sw = (uint32_t)(orow & 7), c4 = 4u * (uint32_t)c;
          *reinterpret_cast<uint4*>(rowp + (((c4 + 0u) ^ sw) << 4)) = h0;
          *reinterpret_cast<uint4*>(rowp + (((c4 + 1u) ^ sw) << 4)) = h1;
          *reinterpret_cast<uint4*>(rowp + (((c4 + 2u) ^ sw) << 4)) = l0;
          *reinterpret_cast<uint4*>(rowp + (((c4 + 3u) ^ sw) << 4)) = l1;
        }
        // ---- dH2 = dOut W3 -> E4 -> dZ2 ----
        // The warp's 16 dOut rows were written by its own owner lanes: read back as the A fragment of the one k-step
        // (chunks 4 c, 4 c + 1 of the h split, 4 c + 2, 4 c + 3 of the l split) after a warp-level barrier only
        __syncwarp();
        {
          uint32_t doh[1][4], dol[1][4];
          ldmatrix_x4(mat_off(S3_DO, 4 * c), doh[0]);
          ldmatrix_x4(mat_off(S3_DO, 4 * c + 2), dol[0]);
          chain_mma_rs<64, MN, 1>(d, doh, dol, W3_M);
          deliver(3);
          stage_end(3);
          wgmma_wait_all();
        }
        dtanh(d, scl[C3_UH2] * hh, S3_H2);
        split_pairs(d);
        store_pairs(S3_DZ2);
        // ---- dH1 = dZ2 W2 -> E5 -> dZ1 ----
        chain_mma_rs<64, MN, 4>(d, ph, pl, W2_M);
        deliver(4);
        stage_end(4);
        wgmma_wait_all();
        dtanh(d, scl[C3_UH1] * hh, S3_H1);
        if (k > 0) wait(5, bar_done(5), (uint32_t)((k - 1) & 1));  // dW1 of the last tile has read dZ1
        split_pairs(d);
        store_pairs(S3_DZ1);
        deliver(5);
        stage_end(5);
      }
    }
#ifdef B200RL_TC3_TIMING
    t_loop_end = clock64();
    if ((tid & 127) == 0 && blockIdx.x == 0)
      for (int i = 0; i < 10; ++i) g_tc3_t[10 * wg + i] = tacc[10 * wg + i];
#endif
    // the valid rows this thread owned, counted here rather than in a register of the loop
    if (c == 0 && q < 2)
      for (int k = 0; k < cta_tiles; ++k) rows_done += (slot + (long long)k * G) * T3_ROWS + r0 + 8 * q < p.n_rows;
  }

  asm volatile("bar.sync 7, %0;" ::"n"(T3_THREADS) : "memory");  // every product has retired and its accumulators
                                                                 // are stored
  // ---- per-CTA results: this network's entries of partial rows 2 slot and 2 slot + 1 (the other CTA of the slot
  // writes the other network's) ----
  {
    // stacked accumulators: rows 0..63 = h-split half (partial row 2b), rows 64..127 = l-split half (row 2b + 1);
    // 8 jobs (dW2 x 4 column blocks, dW1 x 2, dW3, db2); warp `part` takes jobs part, part + 4
    const int qw = warp & 3, part = warp >> 2;
    const int r = 32 * qw + lane;
    float* dst_row = p.partials + ((size_t)slot * 2 + (qw >> 1)) * (size_t)(p.P[0] + p.P[1]);
    const int m = 32 * (qw & 1) + lane;  // feature index
    float v[16], w[16];
    const Tc3Net& nn = p.net[c];
    float* dst = dst_row + (c == 0 ? 0 : p.P[0]);
    const float* scn = s_scale + 16 * c;
    const bool have = cta_tiles > 0;
    const uint32_t gcol = c * ACC_GRAD_NET;
#pragma unroll 1
    for (int jb = part; jb < 8; jb += 4) {
      // the job's product (first column, N), the job's columns in it, and those of its second half where the
      // operand's l columns went to their own block
      const uint32_t pcol = gcol + (jb < 4 ? ACC_DW2 : (jb < 6 ? ACC_DW1 : (jb == 6 ? ACC_DW3 : ACC_DB2)));
      const int pn = jb < 6 ? 64 : (jb == 6 ? 32 : 16);
      const int col = jb < 4 ? 16 * jb : (jb < 6 ? 16 * (jb - 4) : 0);
      const int col2 = jb < 4 ? col : (jb < 6 ? col + 32 : (jb == 6 ? 16 : col));
      if (have) {
        // col and col2 are multiples of 8: column col + j of row r sits grad_acc_off(0, pn, 0, j) after column col
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          v[j] = acc[grad_acc_off(pcol, pn, r, col) + grad_acc_off(0, pn, 0, j)];
          w[j] = acc[grad_acc_off(pcol, pn, r, col2) + grad_acc_off(0, pn, 0, j)];
        }
      } else {
#pragma unroll
        for (int j = 0; j < 16; ++j) v[j] = w[j] = 0.f;  // a CTA without tiles: accumulator memory was never written
      }
      if (jb < 4) {  // dW2 [h2 o][h1 i]: columns 16 jb .. +15
        const float u = scn[C3_OW2];
        if (m < nn.h2)
#pragma unroll
          for (int j = 0; j < 16; ++j)
            if (16 * jb + j < nn.h1) dst[nn.w_off[1] + m * nn.h1 + 16 * jb + j] = v[j] * u;
      } else if (jb < 6) {  // dW1 [h1 o][n_in i] in columns 0..30, db1 in column 31
        const int c0 = 16 * (jb - 4);
        const float u = scn[C3_OW1];
        if (m < nn.h1) {
#pragma unroll
          for (int j = 0; j < 16; ++j)
            if (c0 + j < n_in)
              dst[nn.w_off[0] + m * n_in + c0 + j] = ((v[j] + w[j]) * u) * s_xs[32 + c0 + j];
          if (jb == 5) dst[nn.b_off[0] + m] = (v[15] + w[15]) * scn[C3_OB];
        }
      } else if (jb == 6) {  // dW3^T [h2 i][16 o]
        const float u = scn[C3_OW3];
        if (m < nn.h2)
#pragma unroll
          for (int a = 0; a < 15; ++a)
            if (a < nn.n_out) dst[nn.w_off[2] + a * nn.h2 + m] = (v[a] + w[a]) * u;
      } else {  // db2 (column 15 = sum_r dZ2[r][o] * ones)
        if (m < nn.h2) dst[nn.b_off[1] + m] = v[15] * scn[C3_OB];
      }
    }
  }
  // per-thread sums -> per-warp sums (tree) -> the warps in order: fixed order => reproducible.  The scratch aliases
  // the X buffers (idle now).
  float* e_db3 = reinterpret_cast<float*>(sm + S3_XB + S3_END_DB3);
  double* e_sc = reinterpret_cast<double*>(sm + S3_XB + S3_END_SC);
  {
    // b3: warp 4 m + j takes class m of rows 32 j .. 32 j + 31 (see ACC_DB3); a class without tiles was never written
    const int m = warp >> 2, rr = 32 * (warp & 3) + lane;
#pragma unroll
    for (int a = 0; a < 16; ++a) {
      const int cn = a == 15 ? 1 : 0;
      const bool have = cn == c && ((m - 2 * cn) & 3) < cta_tiles;
      float t = have ? acc[(ACC_DB3 + 16 * m + a) * ACC_LANES + rr] : 0.f;
#pragma unroll
      for (int o2 = 16; o2 > 0; o2 >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o2);
      if (lane == 0) e_db3[warp * 16 + a] = t;
    }
  }
#pragma unroll
  for (int kk = 0; kk < 5; ++kk) {
    const double t = warp_sum(sc[kk]);
    if (lane == 0) e_sc[warp * 8 + kk] = t;
  }
  {
    const double t = warp_sum((double)rows_done);
    if (lane == 0) e_sc[warp * 8 + 5] = t;
  }
  __syncthreads();
  const size_t Ptot = (size_t)(p.P[0] + p.P[1]);
  if (tid < 16) {  // b3 gradients: the 16 per-warp totals in warp order; policy a = 0..14, value in slot 15
    const int cn = tid == 15 ? 1 : 0, a = tid == 15 ? 0 : tid;
    if (cn == c && a < p.net[cn].n_out) {
      float t = 0.f;
      for (int w = 0; w < T3_WARPS; ++w) t += e_db3[w * 16 + tid];
      const size_t off = (cn == 0 ? 0 : (size_t)p.P[0]) + p.net[cn].b_off[2] + a;
      p.partials[((size_t)slot * 2) * Ptot + off] = t;
      p.partials[((size_t)slot * 2 + 1) * Ptot + off] = 0.f;
    }
  }
  // scalar sums: policy 0..7, value 8..15, written by the CTA of their network; a network that does not run gets
  // zeros from the CTA of the one that does
  const bool other_runs = c == 0 ? run_v : run_p;
  if (tid >= 32 && tid < 32 + 2 * B200RL_N_SCALARS && ((tid - 32) / B200RL_N_SCALARS == c || !other_runs)) {
    const int s = tid - 32;
    double t = 0.0;
    if (s / B200RL_N_SCALARS == c) {
      if (s < 6) {
        for (int w = 0; w < T3_CHAIN_WARPS; ++w) t += e_sc[w * 8 + s];
      } else if (s == 8) {
        for (int w = 0; w < T3_CHAIN_WARPS; ++w) t += e_sc[w * 8 + 0];
      }
    }
    p.scalar_partials[((size_t)slot * 2) * (2 * B200RL_N_SCALARS) + s] = t;
    p.scalar_partials[((size_t)slot * 2 + 1) * (2 * B200RL_N_SCALARS) + s] = 0.0;
  }
  if (bad) *s_bad = 1;
#ifdef B200RL_TC3_TIMING
  if (tid == 0 && blockIdx.x == 0) {
    g_tc3_t[53] = (unsigned long long)(t_loop0 - t_kernel0);      // setup
    g_tc3_t[54] = (unsigned long long)(t_loop_end - t_loop0);     // tile loop (chain warpgroup 0)
    g_tc3_t[55] = (unsigned long long)(clock64() - t_loop_end);   // read-out
  }
#endif

  // ---- teardown ----
  __syncthreads();
  if (tid == 0 && *s_bad != 0) *p.status = 1.0f;  // sticky: the engine redoes the update on the wide-range path
}

// ------------------------------------------------------------------------------------------------------------------
// reduce_adam3: fixed-order reduction of the per-CTA partial rows of BOTH networks (as b200rl_reduce_partials) and
// torch.optim.Adam's single-tensor update of both parameter vectors (as b200rl_adam_step), early-stop test included
// (ppo.py:176-181), in ONE launch.  mode 0: reduce + Adam (single GPU); mode 1: reduce only, scalars appended to the
// flat gradient as float32 (the buffer ONE all-reduce carries); mode 2: Adam only, scalars read back from that tail.
// A block owns 32 parameters; every block derives the stop decision from the same inputs in the same order.
//
// Data-parallel runs on one node replace "mode 1, NCCL all-reduce, mode 2" by a one-shot exchange over peer-mapped
// memory (NVLink / NVSwitch): mode 3 reduces and stores this rank's [gradient | scalars] into its exchange buffer,
// the last block to finish publishes the sequence number (release, system scope); mode 4 waits for every rank's
// sequence number (acquire; wait_peers_kernel, one warp), reads ALL ranks' buffers -- its own included -- and adds them in rank order, so every
// rank applies bit-identical updates, then runs Adam.  22 KB per rank: latency bound (~2 us per peer read over NVLink on B200).
// Buffers alternate between two parities: a rank can only be one exchange ahead of its slowest peer (it needs that
// peer's next sequence number to finish its own), so the buffer it overwrites was read by everybody.
// mode 5 = modes 3 and 4 in ONE launch (the blocks wait for the sequence numbers themselves): a data-parallel iteration
// is then two launches, like a single-GPU one.  It needs every block resident at once (ra3_one_wave).
// ------------------------------------------------------------------------------------------------------------------
constexpr int RA3_WARPS = 8;

// One float from every rank's exchange buffer.  The loads are issued back to back (a peer read over NVLink took ~2 us on B200:
// a loop with one load per trip would pay that once per rank) and added in rank order, the same sum on every rank.
template <typename Acc>
__device__ __forceinline__ Acc ra3_gather(float* const* peers, int world, long long offset) {
  float x[RA3_MAX_WORLD];
#pragma unroll
  for (int r = 0; r < RA3_MAX_WORLD; ++r) {
    x[r] = 0.f;
    if (r < world) asm volatile("ld.relaxed.sys.global.f32 %0, [%1];" : "=f"(x[r]) : "l"(peers[r] + offset) : "memory");
  }
  Acc t = (Acc)0;
#pragma unroll
  for (int r = 0; r < RA3_MAX_WORLD; ++r)
    if (r < world) t += (Acc)x[r];
  return t;
}

__global__ void __launch_bounds__(RA3_WARPS * 32, 3) reduce_adam3_kernel(const Ra3Args a) {
  __shared__ float part[RA3_WARPS][32];
  __shared__ double spart[RA3_WARPS * 4][2 * B200RL_N_SCALARS];
  __shared__ double s_scal[2 * B200RL_N_SCALARS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long Ptot = a.P[0] + a.P[1];
  const long long pidx = (long long)blockIdx.x * 32 + lane;
  const bool stopped_before = a.stop_flag != nullptr && *a.stop_flag != 0;
  const bool run_p = a.run_policy != 0 && !stopped_before, run_v = a.run_value != 0;
  const unsigned parity = a.seq & 1u;
  if (a.mode == 4) {  // every rank's buffer of this exchange has arrived (wait_peers_kernel ran before this launch)
    if (threadIdx.x < 2 * B200RL_N_SCALARS)
      s_scal[threadIdx.x] = ra3_gather<double>(a.peers, a.world, parity * a.xchg_stride + Ptot + threadIdx.x);
  } else if (a.mode != 2) {
    // scalar sums: 32 row classes x 16 scalars, then the classes in order (same in every block)
    const int k = lane & 15, cls = warp * 4 + (lane >> 4) * 2;  // two classes per half-warp pass
    for (int half = 0; half < 2; ++half) {
      double s = 0.0;
      for (int c = cls + half; c < a.rows; c += RA3_WARPS * 4) s += a.scalar_partials[(size_t)c * (2 * B200RL_N_SCALARS) + k];
      spart[cls + half][k] = s;
    }
    __syncthreads();
    if (threadIdx.x < 2 * B200RL_N_SCALARS) {
      double t = 0.0;
      for (int c = 0; c < RA3_WARPS * 4; ++c) t += spart[c][threadIdx.x];
      s_scal[threadIdx.x] = t;
    }
  } else {
    if (threadIdx.x < 2 * B200RL_N_SCALARS) s_scal[threadIdx.x] = (double)a.grad[Ptot + threadIdx.x];
  }
  __syncthreads();
  float g = 0.f;
  if (a.mode == 4) {
    if (warp == 0 && pidx < Ptot) {
      g = ra3_gather<float>(a.peers, a.world, parity * a.xchg_stride + pidx);
      if (a.grad != nullptr) a.grad[pidx] = g;
    }
  } else if (a.mode != 2) {
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
    if (pidx < Ptot) {
      const float* qp = a.partials + pidx;
      int c = warp;
      for (; c + 3 * RA3_WARPS < a.rows; c += 4 * RA3_WARPS) {
        s0 += qp[(size_t)c * Ptot];
        s1 += qp[(size_t)(c + RA3_WARPS) * Ptot];
        s2 += qp[(size_t)(c + 2 * RA3_WARPS) * Ptot];
        s3 += qp[(size_t)(c + 3 * RA3_WARPS) * Ptot];
      }
      for (; c < a.rows; c += RA3_WARPS) s0 += qp[(size_t)c * Ptot];
    }
    part[warp][lane] = (s0 + s1) + (s2 + s3);
    __syncthreads();
    if (warp == 0 && pidx < Ptot) {
      g = part[0][lane];
#pragma unroll
      for (int w = 1; w < RA3_WARPS; ++w) g += part[w][lane];
      if (a.grad != nullptr) a.grad[pidx] = g;
    }
  } else if (warp == 0 && pidx < Ptot) {
    g = a.grad[pidx];
  }
  if (a.mode == 1) {
    if (blockIdx.x == 0 && threadIdx.x < 2 * B200RL_N_SCALARS) a.grad[Ptot + threadIdx.x] = (float)s_scal[threadIdx.x];
    return;
  }
  if (a.mode == 3 || a.mode == 5) {
    float* mine = a.peers[a.rank] + parity * a.xchg_stride;
    if (warp == 0 && pidx < Ptot) mine[pidx] = g;
    if (blockIdx.x == 0 && threadIdx.x < 2 * B200RL_N_SCALARS) mine[Ptot + threadIdx.x] = (float)s_scal[threadIdx.x];
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
      const unsigned prev = atomicAdd(a.done_counter, 1u);
      if (prev == gridDim.x - 1) {  // every block's part of the buffer is written: publish
        *a.done_counter = 0u;
        __threadfence_system();
        unsigned* flag = reinterpret_cast<unsigned*>(a.peers[a.rank] + 2 * a.xchg_stride) + parity;
        asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(flag), "r"(a.seq) : "memory");
      }
    }
    if (a.mode == 3) return;
    // mode 5: the same launch goes on to gather.  Lane r of warp 0 waits for rank r's sequence number -- this rank's own
    // included, which is what tells a block that the OTHER blocks of this grid have written their parts (every block is
    // resident: the host checked that the grid fits the device in one wave, so the spinning blocks cannot starve the
    // publishing one).
    if (warp == 0 && lane < a.world) {
      const unsigned* flag = reinterpret_cast<const unsigned*>(a.peers[lane] + 2 * a.xchg_stride) + parity;
      const long long t0 = clock64();
      unsigned seen;
      for (;;) {
        asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(seen) : "l"(flag) : "memory");
        if (seen == a.seq) break;
        if (clock64() - t0 > 20000000000LL) {  // ~10 s: a rank died or never launched
          *a.comm_error = 1;
          break;
        }
        __nanosleep(64);
      }
    }
    __syncthreads();
    if (threadIdx.x < 2 * B200RL_N_SCALARS)
      s_scal[threadIdx.x] = ra3_gather<double>(a.peers, a.world, parity * a.xchg_stride + Ptot + threadIdx.x);
    if (warp == 0 && pidx < Ptot) {
      g = ra3_gather<float>(a.peers, a.world, parity * a.xchg_stride + pidx);
      if (a.grad != nullptr) a.grad[pidx] = g;
    }
    __syncthreads();
  }
  // early stop (ppo.py:176-181): the KL carried by this step's forward pass is the KL after the PREVIOUS update
  bool stop = !run_p;
  if (run_p && a.kl_limit_on) stop = (float)(s_scal[1] / a.n_global) > (float)a.kl_limit;
  if (warp == 0 && pidx < Ptot) {
    const int sidx = pidx < a.P[0] ? 0 : 1;
    const bool apply = sidx == 0 ? (run_p && !stop) : run_v;
    if (apply) {
      const Ra3Seg& sg = a.seg[sidx];
      const long long i = sidx == 0 ? pidx : pidx - a.P[0];
      float m = sg.m[i], v = sg.v[i];
      m = m + sg.one_minus_b1 * (g - m);                      // exp_avg.lerp_(grad, 1 - beta1)
      v = v * sg.b2 + sg.one_minus_b2 * (g * g);              // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, 1 - beta2)
      const float denom = sqrtf(v) / sg.bc2_sqrt + sg.eps;    // (exp_avg_sq.sqrt() / bias_correction2_sqrt).add_(eps)
      sg.m[i] = m;
      sg.v[i] = v;
      sg.params[i] = sg.params[i] - sg.step_size * (m / denom);  // param.addcdiv_(exp_avg, denom, value=-step_size)
    }
  }
  if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) {
    if (run_p) {
      for (int k = 0; k < B200RL_N_SCALARS; ++k) a.slot_p[k] = s_scal[k];
      if (stop) *a.stop_flag = 1;
      else *a.applied_p += 1;
    }
    if (run_v) {
      for (int k = 0; k < B200RL_N_SCALARS; ++k) a.slot_v[k] = s_scal[B200RL_N_SCALARS + k];
      *a.applied_v += 1;
    }
  }
}

// One warp waits until every rank has published the sequence number of this exchange.  A separate, tiny launch: while
// it spins it holds next to nothing of its SM, and the gather + Adam launch behind it needs no polling at all.
__global__ void __launch_bounds__(32) wait_peers_kernel(float* const* peers, int world, long long xchg_stride,
                                                        unsigned seq, int* comm_error) {
  if ((int)threadIdx.x >= world) return;
  const unsigned* flag = reinterpret_cast<const unsigned*>(peers[threadIdx.x] + 2 * xchg_stride) + (seq & 1u);
  const long long t0 = clock64();
  unsigned seen;
  do {
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(seen) : "l"(flag) : "memory");
    if (seen != seq && clock64() - t0 > 20000000000LL) {  // ~10 s: a rank died or never launched
      *comm_error = 1;
      break;
    }
  } while (seen != seq);
}

// ---- host side -------------------------------------------------------------------------------------------------
int launch_wait_peers(const Ra3Args& a, cudaStream_t s) {
  wait_peers_kernel<<<1, 32, 0, s>>>(a.peers, a.world, a.xchg_stride, a.seq, a.comm_error);
  B200RL_CUDA(cudaGetLastError());
  count_launch(1);
  return 0;
}

int tc3_configure() {
  static const int rc = []() -> int {
    return (int)cudaFuncSetAttribute(mlp_tc3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)T3_SMEM_BYTES);
  }();
  if (rc != 0) set_error("mlp_tc3: cudaFuncSetAttribute failed (%s)", cudaGetErrorString((cudaError_t)rc));
  return rc;
}

size_t tc3_ximg_bytes(int64_t n_rows) { return (size_t)((n_rows + T3_ROWS - 1) / T3_ROWS) * T2_ACT; }

bool tc3_shape_ok(const b200rl_mlp_desc& pol, const b200rl_mlp_desc& val) {
  auto ok = [](const b200rl_mlp_desc& d) {
    return d.n_layers == 3 && d.hidden_act == B200RL_ACT_TANH && d.out_act == B200RL_ACT_IDENTITY && d.sizes[0] >= 1 &&
           d.sizes[0] <= 31 && d.sizes[1] >= 1 && d.sizes[1] <= 64 && d.sizes[2] >= 1 && d.sizes[2] <= 64 &&
           d.sizes[3] >= 1 && d.sizes[3] <= 15;
  };
  return ok(pol) && ok(val) && pol.sizes[0] == val.sizes[0] && val.sizes[3] == 1;
}

int launch_pack_obs(const float* obs, int64_t n_rows, int n_in, const float* absmax, uint8_t* ximg, float* xscale,
                    float* bad_flag, cudaStream_t s) {
  const int64_t tiles = (n_rows + T3_ROWS - 1) / T3_ROWS;
  if (tiles <= 0) return 0;
  const int grid = (int)std::min<int64_t>(tiles, 8LL * 132);
  pack_obs_kernel<<<grid, 128, 0, s>>>(obs, n_rows, n_in, absmax, ximg, xscale, bad_flag);
  B200RL_CUDA(cudaGetLastError());
  count_launch(1);
  return 0;
}

int launch_mlp_tc3(const Tc3Args& k, cudaStream_t s) {
  if (tc3_configure()) return 1;
  const int grid = tc_grid(k.n_rows);  // tile slots: one accumulator block and one pair of partial rows each
  B200RL_REQUIRE(grid > 0, "mlp_tc3: no CUDA device");
  Tc3Args kk = k;
  kk.acc_mem = acc_mem(grid, s);
  B200RL_REQUIRE(kk.acc_mem != nullptr, "mlp_tc3: no accumulator memory (allocation failed, or the stream is being captured): %s",
                 cudaGetErrorString(cudaGetLastError()));
  // one CTA per (slot, network): 2 slot + c when both networks run
  mlp_tc3_kernel<<<(k.run_policy && k.run_value) ? 2 * grid : grid, T3_THREADS, T3_SMEM_BYTES, s>>>(kk);
  B200RL_CUDA(cudaGetLastError());
  count_launch(1);
  return 0;
}

// mode 5 spins inside the grid: only when all of its blocks are resident together
bool ra3_one_wave(long long p_total) {
  static const int per_sm = []() -> int {
    int n = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, reduce_adam3_kernel, RA3_WARPS * 32, 0) != cudaSuccess) {
      (void)cudaGetLastError();
      return 0;
    }
    return n;
  }();
  const int sms = device_sm_count();
  return sms > 0 && (p_total + 31) / 32 <= (long long)per_sm * sms;
}

int launch_reduce_adam3(const Ra3Args& a, cudaStream_t s) {
  const long long Ptot = a.P[0] + a.P[1];
  reduce_adam3_kernel<<<(int)((Ptot + 31) / 32), RA3_WARPS * 32, 0, s>>>(a);
  B200RL_CUDA(cudaGetLastError());
  count_launch(1);
  return 0;
}

}  // namespace b200rl

#ifdef B200RL_TC3_TIMING
extern "C" int b200rl_debug_tc3_timing(unsigned long long* out64, int reset) {
  if (reset) {
    unsigned long long z[64] = {0};
    return (int)cudaMemcpyToSymbol(b200rl::g_tc3_t, z, sizeof(z));
  }
  return (int)cudaMemcpyFromSymbol(out64, b200rl::g_tc3_t, sizeof(unsigned long long) * 64);
}
#endif
