// Hand-written sm_90a primitives of the tensor-core kernels: warpgroup MMA (wgmma) on shared-memory descriptors, or
// with A from registers, the per-CTA accumulator memory the kernels address by (row, column), mbarrier and proxy fences.
// PTX spellings follow the CUDA 12.9 ISA.
//
// Work split.  The epilogue warps of a kernel hold one row of a 128-row tile per thread and read or write
// accumulators by (row, column); one warpgroup (four warps) issues the products.  A product
// D[M x N] (+)= sum_t A_t B_t runs as wgmma m64nNk16 over each 64-row half of M, with the accumulator fragment in the
// issuing warpgroup's registers: it is loaded from the accumulator memory when the product accumulates, and stored
// back when the product is done.  The issuing warpgroup then arrives once on the stage's mbarrier (acc_commit).
//
// Accumulator memory.  An H100 SM has 227 KB of shared memory for a block and the kernels' operand buffers fill most
// of it, so the fp32 accumulators (up to 512 columns x 128 rows = 256 KB per CTA) live in a per-launch global buffer
// of gridDim.x such blocks, column-major (ACC_LANES floats per column).  It is written and read back by the same CTA
// within a tile's stages, so it stays in the 50 MB L2.
#pragma once
#include <cstdint>

namespace b200rl {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- mbarrier -------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// Blocks until the phase with the given parity has completed.  try_wait suspends in hardware for a bounded time;
// the loop re-arms it.  `spin_guard` bounds the total wait so a protocol bug traps instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
#pragma unroll 1  // inlined at ~20 sites of the tensor-core kernels: keep the spin loop small (instruction cache)
  for (uint32_t it = 0; it < (1u << 22); ++it) {  // ~16 s at the 4 us suspend hint
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}"
        : "=r"(done)
        : "r"(bar), "r"(parity), "r"(4000u)  // suspend-time hint (ns): sleep in hardware instead of spinning
        : "memory");
    if (done) return;
  }
  __trap();
}

// ---- proxy fence ----------------------------------------------------------------------------------------------
// generic-proxy shared-memory writes (operand buffers) -> visible to wgmma, which reads through the async proxy
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- accumulator memory ----------------------------------------------------------------------------------------
// Accumulator memory is ordinary global memory: the mbarrier arrive / wait pairs (release / acquire) and the named
// barriers order it between the issuing warpgroup and the epilogue warps.
constexpr uint32_t ACC_COLS = 512, ACC_LANES = 128;
constexpr size_t ACC_CTA_FLOATS = (size_t)ACC_COLS * ACC_LANES;

// `acc` below is the CTA's block: acc_mem + blockIdx.x * ACC_CTA_FLOATS.

// N consecutive columns from `col` of accumulator row `row`.  The epilogue threads hold one row each, so a warp reading
// one column of its 32 rows touches one 128-byte line.
template <int N>
__device__ __forceinline__ void acc_ld(const float* acc, int row, uint32_t col, float (&v)[N]) {
  const float* p = acc + col * ACC_LANES + row;
#pragma unroll
  for (int j = 0; j < N; ++j) v[j] = p[j * ACC_LANES];
}
template <int N>
__device__ __forceinline__ void acc_st(float* acc, int row, uint32_t col, const float (&v)[N]) {
  float* p = acc + col * ACC_LANES + row;
#pragma unroll
  for (int j = 0; j < N; ++j) p[j * ACC_LANES] = v[j];
}

// The issuing warpgroup's products are complete and stored: one arrive on `bar` (count 1) for the whole warpgroup.
// Named barrier 8 is reserved for the issuing warpgroup (the epilogue warps use 1..3).
__device__ __forceinline__ void acc_commit(uint32_t bar) {
  __threadfence_block();
  asm volatile("bar.sync 8, 128;" ::: "memory");
  if ((threadIdx.x & 127u) == 0) mbar_arrive(bar);
}

// ---- descriptors ----------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor (wgmma), SWIZZLE_128B:
//   [0,14) start address >> 4   [16,30) leading byte offset >> 4   [32,46) stride byte offset >> 4
//   [49,52) base offset = 0     [62,64) layout type (1 = SWIZZLE_128B)
// K-major: 128-byte rows, 8-row groups `sbo` = 1024 bytes apart.  MN-major: `lbo` = distance between 64-element
// atoms along M / N, `sbo` = distance between 8-row groups along K.
__host__ __device__ constexpr uint64_t make_smem_desc_sw128(uint32_t addr_bytes, uint32_t lbo_bytes,
                                                            uint32_t sbo_bytes) {
  return (uint64_t)((addr_bytes >> 4) & 0x3FFFu) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16) |
         ((uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32) | (1ull << 62);
}

// One operand of a split product: 32-bit halves of the descriptor of split 0 / k-step 0, the low-word advance per
// split (buffer stride >> 4) and per k-step (bytes >> 4).  All fields are warp-uniform.
struct Op2 {
  uint32_t lo, hi, split_step, k_step;
};
__device__ __forceinline__ Op2 op2_kmajor(uint32_t addr, uint32_t split_bytes) {  // K along the 128-byte rows
  const uint64_t d = make_smem_desc_sw128(addr, 16, 1024);
  return Op2{(uint32_t)d, (uint32_t)(d >> 32), split_bytes >> 4, 32u >> 4};
}
// K along the rows; `atom_stride` = byte distance between 64-element atoms along M/N (the next split buffer when the
// operand is read with M = 128 "stacked")
__device__ __forceinline__ Op2 op2_mnmajor(uint32_t addr, uint32_t atom_stride, uint32_t split_bytes) {
  const uint64_t d = make_smem_desc_sw128(addr, atom_stride, 1024);
  return Op2{(uint32_t)d, (uint32_t)(d >> 32), split_bytes >> 4, 2048u >> 4};
}
__device__ __forceinline__ Op2 op2_at(Op2 o, uint32_t byte_off) {  // same view, `byte_off` further (slot select)
  o.lo += byte_off >> 4;
  return o;
}

// ---- wgmma -----------------------------------------------------------------------------------------------------
// D[64 x N] (+)= A[64 x 16] B[16 x N], fp32 accumulate in registers; TA / TB: operand read MN-major (transposed).
template <int TA, int TB>
__device__ __forceinline__ void wgmma_f16_n16(float (&d)[8], uint64_t a, uint64_t b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, %11, %12;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB)
      : "memory");
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_f16_n32(float (&d)[16], uint64_t a, uint64_t b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, %19, %20;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB)
      : "memory");
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_f16_n48(float (&d)[24], uint64_t a, uint64_t b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %26, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n48k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23}, %24, %25, p, 1, 1, %27, %28;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
      : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB)
      : "memory");
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_f16_n64(float (&d)[32], uint64_t a, uint64_t b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, %35, %36;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB)
      : "memory");
}

// D[64 x N] (+)= A[64 x 16] B[16 x N] with A from registers (K-major, fp16): a[0..3] = this thread's packed pairs of
// rows m0 and m0 + 8 (m0 = 16 warp + lane / 4) at columns 2 (lane % 4) + {0, 1}, then of the same rows at 8 columns
// further.  That is the layout of fragment elements 8 s .. 8 s + 7 of an f32 accumulator, so columns 16 s .. 16 s + 15
// of one product can be k-step s of the next.  The RS form has no transpose for A; TB: B read MN-major.
template <int TB>
__device__ __forceinline__ void wgmma_f16_n16_rs(float (&d)[8], const uint32_t (&a)[4], uint64_t b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7}, {%8,%9,%10,%11}, %12, p, 1, 1, %14;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(scale_d), "n"(TB)
      : "memory");
}
template <int TB>
__device__ __forceinline__ void wgmma_f16_n64_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32,%33,%34,%35}, %36, p, 1, 1, %38;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(scale_d), "n"(TB)
      : "memory");
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

template <int N, int TA, int TB>
__device__ __forceinline__ void wgmma_run(float (&d)[N / 2], uint64_t a, uint64_t b, uint32_t scale_d) {
  if constexpr (N == 16) wgmma_f16_n16<TA, TB>(d, a, b, scale_d);
  else if constexpr (N == 32) wgmma_f16_n32<TA, TB>(d, a, b, scale_d);
  else if constexpr (N == 48) wgmma_f16_n48<TA, TB>(d, a, b, scale_d);
  else wgmma_f16_n64<TA, TB>(d, a, b, scale_d);
}
template <int N, int TB>
__device__ __forceinline__ void wgmma_run_rs(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t b, uint32_t scale_d) {
  static_assert(N == 16 || N == 64, "register-A wgmma shape without a wrapper");
  if constexpr (N == 16) wgmma_f16_n16_rs<TB>(d, a, b, scale_d);
  else wgmma_f16_n64_rs<TB>(d, a, b, scale_d);
}

// Operand majors (template arguments TA / TB of the products): K-major, or MN-major (read transposed).
constexpr int K_MAJOR = 0, MN_MAJOR = 1;

// Accumulator columns acc_col .. acc_col + N - 1 (+)= sum over `terms` of A_t B_t, each `ksteps` k-steps of 16
// (descriptor low words advance by a_k / b_k per k-step; the high words are shared); the first product overwrites
// unless `acc_first`.  M = 128 runs as two m64nNk16 halves (A's low word advanced to rows 64..127).  Executed by all
// 128 threads of the issuing warpgroup.
template <int N, int TA, int TB, int T>
__device__ __forceinline__ void mma_product(float* acc_cta, uint32_t acc_col, const uint32_t (&alo)[T],
                                            const uint32_t (&blo)[T], int terms, uint32_t a_hi, uint32_t b_hi,
                                            uint32_t a_k, uint32_t b_k, int ksteps, bool acc_first) {
  static_assert(N == 16 || N == 32 || N == 48 || N == 64, "wgmma shape without a wrapper");
  const int t = (int)(threadIdx.x & 127u), w = t >> 5, l = t & 31;
  // rows 64..127 of A: the next 64-element atom (MN-major: one leading byte offset further) or 64 rows of 128 bytes
  const uint32_t a_half = TA == MN_MAJOR ? ((alo[0] >> 16) & 0x3FFFu) : (64u * 128u) >> 4;
  float* acc = acc_cta + acc_col * ACC_LANES;
#pragma unroll 1
  for (int h = 0; h < 2; ++h) {
    // this thread's fragment (wgmma D layout): rows m0 and m0 + 8, columns 2 (l % 4) + 8 j + {0, 1}.  One base
    // pointer, the rest immediate offsets: per-element offsets would be loop-invariant and kept live across the issuer.
    const int m0 = 16 * w + (l >> 2) + 64 * h;
    float* frag = acc + 2 * (l & 3) * ACC_LANES + m0;
    float d[N / 2];
#pragma unroll
    for (int i = 0; i < N / 2; ++i)
      d[i] = acc_first ? frag[(8 * (i >> 2) + (i & 1)) * ACC_LANES + 8 * ((i >> 1) & 1)] : 0.f;
    wgmma_fence();
    uint32_t scale = acc_first ? 1u : 0u;
#pragma unroll
    for (int s = 0; s < T; ++s) {
      if (s >= terms) break;
      uint32_t a = alo[s] + (uint32_t)h * a_half, b = blo[s];
#pragma unroll 1
      for (int k = 0; k < ksteps; ++k) {
        wgmma_run<N, TA, TB>(d, ((uint64_t)a_hi << 32) | a, ((uint64_t)b_hi << 32) | b, scale);
        scale = 1u;
        a += a_k;
        b += b_k;
      }
    }
    wgmma_commit();
    wgmma_wait_all();
#pragma unroll
    for (int i = 0; i < N / 2; ++i) frag[(8 * (i >> 2) + (i & 1)) * ACC_LANES + 8 * ((i >> 1) & 1)] = d[i];
  }
}

}  // namespace b200rl
