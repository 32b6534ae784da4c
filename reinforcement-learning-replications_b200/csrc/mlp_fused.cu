// mlp_fused: MLP forward -> distribution log-prob -> loss -> dLoss/dOut -> MLP backward in ONE persistent kernel.
//
// Replaces (reference: /root/reference/src/rl_replicas/): networks/mlp.py:33-41, policies/gaussian_policy.py:25-37,
// policies/categorical_policy.py:22-32, algorithms/ppo.py:237-257 + autograd backward (:234), :259-269, :282-287
// (+ :277), algorithms/vpg.py:200-206, algorithms/trpo.py:154-165, utils.py:60-71 and utils.py:90-92 (on load).
//
// It is also the wide-range re-run of the fp16 tensor-core kernels (mlp_tc2.cu, mlp_tc_fvp.cu): every launch of theirs
// queues this kernel behind it, predicated on the launch's status slot, and it recomputes a launch whose values left
// fp16's range.
//
// Data flow (fp32 CUDA-core path; the tensor-core kernels keep the same flow):
//   * grid = min(#tiles, #SMs) persistent CTAs, tile = 64 rows, static round-robin tile -> CTA map (deterministic).
//   * all weights live in shared memory for the whole launch, in both [out][in] and [in][out] order, so every
//     tile product is the SAME k-major inner loop  C[m][n] += A[k][m] * B[k][n]  with float4 shared loads:
//        forward      C = X_l^T-major x W^T     (k = input feature)
//        dX           C = dZ^T-major  x W       (k = output feature)
//        dW           C = dZ row-major x X row-major   (k = row of the tile)
//     which is why each activation is kept in shared memory in row-major AND feature-major form.
//   * activations never touch HBM; per-CTA weight gradients accumulate in shared memory across the CTA's tiles and
//     are written once as partials[cta][P]; b200rl_reduce_partials sums them in a fixed order.
//   * HBM reads per row: obs (4*O) + actions (4*A) + adv_raw (4) + old_logp (4) [policy] or target (4) [value].
#include <atomic>
#include <cmath>
#include <cstdlib>

#include "common.cuh"
#include "policy_head.cuh"

namespace b200rl {

constexpr int TM_MAX = 64;         // rows per tile (64, or 32 / 16 when the network needs more shared memory)
constexpr int MLP_THREADS = 256;   // 8 warps
constexpr int MAXL = B200RL_MAX_LAYERS;

struct MlpLayout {
  int tm;  // rows per tile
  int L;
  int n[MAXL + 1];   // widths
  int ld[MAXL + 1];  // pad4(width)
  int hidden_act, out_act;
  int w_off[MAXL], b_off[MAXL];  // offsets into the flat parameter vector
  int P;
  // shared-memory offsets, in floats (all multiples of 4)
  int s_wrm[MAXL];   // W   [n_out][ld[l]]      (dX: k = output feature)
  int s_wt[MAXL];    // W^T [n_in][ld[l+1]]     (forward: k = input feature)
  int s_bias[MAXL];  // [ld[l+1]]
  int s_dw;          // [P] gradient accumulators
  int s_xrm[MAXL + 1];  // activation l, row-major  [TM][ld[l]]
  int s_xt[MAXL + 1];   // activation l, feature-major [n[l]][TM]; reused for dZ_l^T during the backward pass
  int s_dz[2];          // dZ row-major ping-pong [TM][ldz]
  int ldz;
  int s_dist;           // per-action constants (Gaussian): var[A], log_scale[A]
  // Fisher-vector product only: direction weights V^T [n_in][ld[l+1]], direction bias, tangents (feature-major)
  int s_vt[MAXL], s_vb[MAXL];
  int s_tt[MAXL + 1];   // tangent of activation l, feature-major [n[l]][TM]
  int s_trm;            // tangent of the output, row-major [TM][ld[L]]
  int total_floats;
};

static int build_layout_tm(const b200rl_mlp_desc& d, bool backward, bool fvp, int TM, MlpLayout* out) {
  B200RL_REQUIRE(d.n_layers >= 1 && d.n_layers <= MAXL, "mlp: n_layers %d out of range 1..%d", d.n_layers, MAXL);
  MlpLayout L{};
  L.tm = TM;
  L.L = d.n_layers;
  L.hidden_act = d.hidden_act;
  L.out_act = d.out_act;
  int p = 0;
  for (int l = 0; l <= L.L; ++l) {
    B200RL_REQUIRE(d.sizes[l] >= 1 && d.sizes[l] <= 1024, "mlp: layer width %d out of range", d.sizes[l]);
    L.n[l] = d.sizes[l];
    L.ld[l] = pad4(d.sizes[l]);
  }
  for (int l = 0; l < L.L; ++l) {
    L.w_off[l] = p;
    p += L.n[l + 1] * L.n[l];
    L.b_off[l] = p;
    p += L.n[l + 1];
  }
  L.P = p;
  int s = 0;
  auto take = [&](int nfloats) {
    int o = s;
    s += pad4(nfloats);
    return o;
  };
  for (int l = 0; l < L.L; ++l) {
    L.s_wrm[l] = take(L.n[l + 1] * L.ld[l]);
    L.s_wt[l] = take(L.n[l] * L.ld[l + 1]);
    L.s_bias[l] = take(L.ld[l + 1]);
  }
  L.s_dw = backward ? take(L.P) : 0;
  for (int l = 0; l <= L.L; ++l) {
    L.s_xrm[l] = take(TM * L.ld[l]);
    L.s_xt[l] = take(L.ld[l] * TM);
  }
  L.ldz = 4;
  for (int l = 1; l <= L.L; ++l) L.ldz = L.ld[l] > L.ldz ? L.ld[l] : L.ldz;
  if (backward) {
    L.s_dz[0] = take(TM * L.ldz);
    L.s_dz[1] = take(TM * L.ldz);
  }
  L.s_dist = take(2 * L.ld[L.L]);
  if (fvp) {
    for (int l = 0; l < L.L; ++l) {
      L.s_vt[l] = take(L.n[l] * L.ld[l + 1]);
      L.s_vb[l] = take(L.ld[l + 1]);
    }
    for (int l = 1; l <= L.L; ++l) L.s_tt[l] = take(L.ld[l] * TM);
    L.s_trm = take(TM * L.ld[L.L]);
  }
  L.total_floats = s;
  *out = L;
  return 0;
}

// shared memory a block may use on sm_90 (dynamic + static)
constexpr size_t SMEM_LIMIT = 227 * 1024;
// static shared memory of mlp_fused_kernel<tm, mode> (defined below); 0 if it cannot be queried
static size_t fused_static_smem(int tm, int mode);

// largest tile height whose shared-memory footprint (the layout plus the kernel's static arrays) fits
int build_layout(const b200rl_mlp_desc& d, bool backward, MlpLayout* out, bool fvp = false) {
  for (int tm = TM_MAX; tm >= 16; tm >>= 1) {
    if (build_layout_tm(d, backward, fvp, tm, out)) return 2;
    const size_t st = fused_static_smem(tm, fvp ? 2 : (backward ? 1 : 0));
    if ((size_t)out->total_floats * sizeof(float) + st <= SMEM_LIMIT) return 0;
  }
  return 0;  // caller reports the size
}

struct FusedArgs {
  MlpLayout lay;
  int loss, dist;
  long long n_rows;
  float inv_n;      // 1 / n_global (float, like autograd's 1/N)
  float clip_lo, clip_hi;
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
  float* out_full;
  const float* old_out;
  const float* direction;
  const unsigned* run_if;  // when set: run only if *run_if == seq (re-run of a tensor-core launch that left fp16's range)
  unsigned seq;
  int total_rows;          // partial rows the consumer reduces (> gridDim.x when standing in for / sized like a tensor-core launch)
  int train_log_std;       // Gaussian: partial rows carry dLoss/dlog_std in columns P .. P + A - 1 (row stride P + A)
};

__device__ unsigned long long g_tc_fallbacks;  // re-runs of a tensor-core launch that fired (b200rl_tc_fallback_count)

__device__ __forceinline__ float apply_act(float z, int kind) {
  if (kind == B200RL_ACT_TANH) return tanhf(z);
  if (kind == B200RL_ACT_RELU) return fmaxf(z, 0.f);
  return z;
}
__device__ __forceinline__ float act_prime_from_output(float a, int kind) {
  if (kind == B200RL_ACT_TANH) return 1.f - a * a;
  if (kind == B200RL_ACT_RELU) return a > 0.f ? 1.f : 0.f;
  return 1.f;
}

// C[m][n] = sum_k A[k*lda + m] * B[k*ldb + n] (+ sum_k A2[k*lda2 + m] * B2[k*ldb2 + n]), m < 4*M4, n < 4*N4;
// 4x4 register tile per thread.
template <class Epi>
__device__ __forceinline__ void tile_gemm(const float* __restrict__ A, int lda, const float* __restrict__ B, int ldb,
                                          int K, int M4, int N4, Epi epi, const float* __restrict__ A2 = nullptr,
                                          int lda2 = 0, const float* __restrict__ B2 = nullptr, int ldb2 = 0,
                                          int K2 = 0) {
  const int ntiles = M4 * N4;
  for (int t = threadIdx.x; t < ntiles; t += MLP_THREADS) {
    const int mi = t % M4, ni = t / M4;
    const float* a = A + 4 * mi;
    const float* b = B + 4 * ni;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
#pragma unroll 4
    for (int k = 0; k < K; ++k) {
      const float4 av = *reinterpret_cast<const float4*>(a + (size_t)k * lda);
      const float4 bv = *reinterpret_cast<const float4*>(b + (size_t)k * ldb);
      const float ar[4] = {av.x, av.y, av.z, av.w};
      const float br[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(ar[i], br[j], acc[i][j]);
    }
    if (K2 > 0) {
      const float* a2 = A2 + 4 * mi;
      const float* b2 = B2 + 4 * ni;
#pragma unroll 4
      for (int k = 0; k < K2; ++k) {
        const float4 av = *reinterpret_cast<const float4*>(a2 + (size_t)k * lda2);
        const float4 bv = *reinterpret_cast<const float4*>(b2 + (size_t)k * ldb2);
        const float ar[4] = {av.x, av.y, av.z, av.w};
        const float br[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(ar[i], br[j], acc[i][j]);
      }
    }
    epi(4 * mi, 4 * ni, acc);
  }
}

// MODE 0: forward only (EVAL / line search), 1: forward + backward, 2: Fisher-vector product (forward with tangents,
// metric, backward)
template <int TM, int MODE>
__global__ void __launch_bounds__(MLP_THREADS, 1) mlp_fused_kernel(const FusedArgs p) {
  constexpr bool BACKWARD = MODE != 0;
  constexpr bool FVP = MODE == 2;
  extern __shared__ __align__(16) float smem[];
  const MlpLayout& Y = p.lay;
  const int tid = threadIdx.x;
  if (p.skip_flag != nullptr && *p.skip_flag != 0) return;  // early stop: the whole launch is a no-op
  if (p.run_if != nullptr) {
    if (*p.run_if != p.seq) return;  // the tensor-core result stands
    if (blockIdx.x == 0 && tid == 0) atomicAdd(&g_tc_fallbacks, 1ull);
  }
  // the consumer reduces total_rows partial rows: those beyond this grid are zero
  for (int row = (int)gridDim.x + (int)blockIdx.x; row < p.total_rows; row += (int)gridDim.x) {
    if (BACKWARD)
      for (int i = tid; i < Y.P; i += MLP_THREADS) p.partials[(size_t)row * Y.P + i] = 0.f;
    if (p.scalar_partials != nullptr && tid < B200RL_N_SCALARS) p.scalar_partials[(size_t)row * B200RL_N_SCALARS + tid] = 0.0;
  }
  const int L = Y.L;

  // ---- stage the weights once per launch: W, W^T and bias ----
  for (int l = 0; l < L; ++l) {
    const int nin = Y.n[l], nout = Y.n[l + 1];
    const float* w = p.params + Y.w_off[l];
    float* wrm = smem + Y.s_wrm[l];
    float* wt = smem + Y.s_wt[l];
    for (int idx = tid; idx < nin * nout; idx += MLP_THREADS) {
      const int o = idx / nin, i = idx - o * nin;
      const float x = __ldg(w + idx);
      wrm[o * Y.ld[l] + i] = x;
      wt[i * Y.ld[l + 1] + o] = x;
    }
    // pad columns of W^T feed accumulators that are discarded, but keep them finite
    for (int idx = tid; idx < nin * (Y.ld[l + 1] - nout); idx += MLP_THREADS) {
      const int i = idx / (Y.ld[l + 1] - nout), c = nout + idx % (Y.ld[l + 1] - nout);
      wt[i * Y.ld[l + 1] + c] = 0.f;
    }
    for (int idx = tid; idx < nout * (Y.ld[l] - nin); idx += MLP_THREADS) {
      const int o = idx / (Y.ld[l] - nin), c = nin + idx % (Y.ld[l] - nin);
      wrm[o * Y.ld[l] + c] = 0.f;
    }
    for (int o = tid; o < Y.ld[l + 1]; o += MLP_THREADS)
      smem[Y.s_bias[l] + o] = o < nout ? __ldg(p.params + Y.b_off[l] + o) : 0.f;
  }
  if (FVP) {
    for (int l = 0; l < L; ++l) {
      const int nin = Y.n[l];
      float* vt = smem + Y.s_vt[l];
      for (int idx = tid; idx < nin * Y.ld[l + 1]; idx += MLP_THREADS) vt[idx] = 0.f;
    }
    __syncthreads();
    for (int l = 0; l < L; ++l) {
      const int nin = Y.n[l], nout = Y.n[l + 1];
      float* vt = smem + Y.s_vt[l];
      for (int idx = tid; idx < nin * nout; idx += MLP_THREADS) {
        const int o = idx / nin, i = idx - o * nin;
        vt[i * Y.ld[l + 1] + o] = __ldg(p.direction + Y.w_off[l] + idx);
      }
      for (int o = tid; o < Y.ld[l + 1]; o += MLP_THREADS)
        smem[Y.s_vb[l] + o] = o < nout ? __ldg(p.direction + Y.b_off[l] + o) : 0.f;
    }
  }
  if (BACKWARD)
    for (int i = tid; i < Y.P; i += MLP_THREADS) smem[Y.s_dw + i] = 0.f;
  const int A_out = Y.n[L];
  if (p.dist == B200RL_DIST_GAUSSIAN) {
    for (int a = tid; a < A_out; a += MLP_THREADS) {
      const NormalConsts c = normal_consts(p.log_std, a);
      smem[Y.s_dist + a] = c.var;
      smem[Y.s_dist + Y.ld[L] + a] = c.log_scale;
    }
  }
  // pad columns of the row-major activations are only ever read into discarded accumulators; zero them once
  for (int l = 0; l <= L; ++l)
    for (int idx = tid; idx < TM * Y.ld[l]; idx += MLP_THREADS) smem[Y.s_xrm[l] + idx] = 0.f;
  if (BACKWARD)
    for (int idx = tid; idx < 2 * TM * Y.ldz; idx += MLP_THREADS) smem[Y.s_dz[0] + idx] = 0.f;

  float adv_mean, adv_std;
  adv_mean_std(p.adv_stats, adv_mean, adv_std);
  __syncthreads();

  double sc[7] = {0, 0, 0, 0, 0, 0, 0};  // loss terms, old_logp - logp, entropy, logp, logp^2, rows, KL(old||new)
  float dls[16];  // this thread's share of dLoss/dlog_std (train_log_std)
#pragma unroll
  for (int a = 0; a < 16; ++a) dls[a] = 0.f;
  const long long num_tiles = (p.n_rows + TM - 1) / TM;
  const int n0 = Y.n[0], ld0 = Y.ld[0];

  for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const long long r0 = tile * TM;
    const int rows_here = (int)((p.n_rows - r0) < TM ? (p.n_rows - r0) : TM);

    // ---- observations tile: one contiguous, coalesced read; stored row-major and feature-major ----
    {
      const float* src = p.obs + r0 * n0;
      float* xrm = smem + Y.s_xrm[0];
      float* xt = smem + Y.s_xt[0];
      const int cnt = rows_here * n0;
      for (int idx = tid; idx < TM * n0; idx += MLP_THREADS) {
        const int r = idx / n0, f = idx - r * n0;
        const float x = idx < cnt ? __ldg(src + idx) : 0.f;
        xrm[r * ld0 + f] = x;
        xt[f * TM + r] = x;
      }
    }
    __syncthreads();

    // ---- forward ----
    for (int l = 0; l < L; ++l) {
      const int nout = Y.n[l + 1], ldo = Y.ld[l + 1];
      const int kind = (l == L - 1) ? Y.out_act : Y.hidden_act;
      const float* bias = smem + Y.s_bias[l];
      float* orm = smem + Y.s_xrm[l + 1];
      float* ot = smem + Y.s_xt[l + 1];
      tile_gemm(smem + Y.s_xt[l], TM, smem + Y.s_wt[l], ldo, Y.n[l], TM / 4, ldo / 4,
                [&](int m0, int c0, float (&acc)[4][4]) {
#pragma unroll
                  for (int j = 0; j < 4; ++j) {
                    const int c = c0 + j;
                    if (c < nout) {
                      const float b = bias[c];
                      float h[4];
#pragma unroll
                      for (int i = 0; i < 4; ++i) {
                        h[i] = apply_act(acc[i][j] + b, kind);
                        orm[(m0 + i) * ldo + c] = h[i];
                      }
                      *reinterpret_cast<float4*>(ot + c * TM + m0) = make_float4(h[0], h[1], h[2], h[3]);
                    }
                  }
                });
      __syncthreads();
      if (FVP) {
        // tangent (J v) propagation: T_{l+1} = act'(H_{l+1}) * (T_l W^T + X_l V^T + v_b);  T_0 = 0
        const float* vb = smem + Y.s_vb[l];
        float* tt = smem + Y.s_tt[l + 1];
        float* trm = smem + Y.s_trm;
        const bool last = (l == L - 1);
        tile_gemm(smem + Y.s_xt[l], TM, smem + Y.s_vt[l], ldo, Y.n[l], TM / 4, ldo / 4,
                  [&](int m0, int c0, float (&acc)[4][4]) {
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                      const int c = c0 + j;
                      if (c < nout) {
                        float t[4];
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                          t[i] = (acc[i][j] + vb[c]) * act_prime_from_output(orm[(m0 + i) * ldo + c], kind);
                          if (last) trm[(m0 + i) * ldo + c] = t[i];
                        }
                        *reinterpret_cast<float4*>(tt + c * TM + m0) = make_float4(t[0], t[1], t[2], t[3]);
                      }
                    }
                  },
                  l > 0 ? smem + Y.s_tt[l] : nullptr, TM, smem + Y.s_wt[l], ldo, l > 0 ? Y.n[l] : 0);
        __syncthreads();
      }
    }

    // ---- distribution / loss epilogue: one thread per row ----
    if (tid < TM) {
      const int r = tid;
      const long long row = r0 + r;
      const bool valid = r < rows_here;
      const float* out = smem + Y.s_xrm[L] + r * Y.ld[L];
      float* dzrm = BACKWARD ? smem + Y.s_dz[L & 1] + r * Y.ldz : nullptr;
      float* dzt = smem + Y.s_xt[L];
      if (valid && FVP) {
        // dOut = M (J v) / N, written row-major and then feature-major
        const float* t = smem + Y.s_trm + r * Y.ld[L];
        if (p.dist == B200RL_DIST_GAUSSIAN)
          gaussian_metric<16>(t, VarDiv{smem + Y.s_dist}, A_out, p.inv_n, dzrm);
        else
          categorical_metric<16>(out, t, A_out, p.inv_n, dzrm);
        for (int a = 0; a < A_out; ++a) dzt[a * TM + r] = dzrm[a];
        sc[5] += 1.0;
      } else if (valid) {
        if (p.dist == B200RL_DIST_NONE) {
          const float vout = out[0];
          if (p.row_out) p.row_out[row] = vout;
          float term = 0.f;
          if (p.loss == B200RL_LOSS_MSE) {
            float dv;
            term = value_mse(vout, __ldg(p.target + row), p.inv_n, dv);
            if (BACKWARD) {
              const float g = dv * act_prime_from_output(vout, Y.out_act);
              dzrm[0] = g;
              dzt[r] = g;
            }
          }
          sc[0] += (double)term;
          sc[5] += 1.0;
        } else {
          const VarDiv var{smem + Y.s_dist};
          float lp, ent, dlp[16];
          if (p.dist == B200RL_DIST_GAUSSIAN)
            gaussian_logp<16>(Ldg{p.actions + row * A_out}, out, smem + Y.s_dist + Y.ld[L], var, A_out, lp, ent, dlp);
          else
            categorical_logp<16>(out, (int)__ldg(p.actions + row), A_out, lp, ent, dlp);  // value.long()
          if (p.row_out) p.row_out[row] = lp;
          if (p.out_full)
            for (int a = 0; a < A_out; ++a) p.out_full[row * A_out + a] = out[a];
          if (p.old_out) {
            const Ldg oo{p.old_out + row * A_out};
            sc[6] += (double)(p.dist == B200RL_DIST_GAUSSIAN ? gaussian_kl<16>(oo, out, var, A_out)
                                                              : categorical_kl<16>(oo, out, A_out));
          }
          float adv = 0.f, oldlp = 0.f;
          if (p.loss != B200RL_LOSS_EVAL) {
            adv = __ldg(p.adv_raw + row);
            if (p.adv_stats != nullptr) adv = (adv - adv_mean) / adv_std;  // utils.py:91
          }
          if (p.old_logp != nullptr) oldlp = __ldg(p.old_logp + row);
          float coef;
          const float term = policy_loss(p.loss, lp, oldlp, adv, p.inv_n, p.clip_lo, p.clip_hi, coef);
          if (BACKWARD) {
            for (int a = 0; a < A_out; ++a) {
              const float g = coef * dlp[a] * act_prime_from_output(out[a], Y.out_act);
              dzrm[a] = g;
              dzt[a * TM + r] = g;
            }
            if (p.train_log_std) {
              // d logp / d log_std_a = (act_a - mu_a)^2 / var_a - 1   (Normal.log_prob with scale = exp(log_std),
              // gaussian_policy.py:34); the entropy does not enter the losses (ppo.py:245-255, vpg.py:203)
              const float* act = p.actions + row * A_out;
#pragma unroll
              for (int a = 0; a < 16; ++a)
                if (a < A_out) dls[a] += coef * ((__ldg(act + a) - out[a]) * dlp[a] - 1.f);
            }
          }
          add_policy_row_sums(sc, term, lp, ent, oldlp, p.old_logp != nullptr);
          sc[5] += 1.0;
        }
      } else if (BACKWARD) {
        for (int a = 0; a < A_out; ++a) {
          dzrm[a] = 0.f;
          dzt[a * TM + r] = 0.f;
        }
      }
    }
    __syncthreads();

    // ---- backward ----
    if (BACKWARD) {
      for (int l = L; l >= 1; --l) {
        const int nl = Y.n[l], nprev = Y.n[l - 1], ldprev = Y.ld[l - 1];
        const float* dz = smem + Y.s_dz[l & 1];
        // dW_l[o][i] += sum_r dZ[r][o] * X_{l-1}[r][i]
        float* dw = smem + Y.s_dw + Y.w_off[l - 1];
        tile_gemm(dz, Y.ldz, smem + Y.s_xrm[l - 1], ldprev, TM, Y.ld[l] / 4, ldprev / 4,
                  [&](int o0, int i0, float (&acc)[4][4]) {
#pragma unroll
                    for (int i = 0; i < 4; ++i)
#pragma unroll
                      for (int j = 0; j < 4; ++j)
                        if (o0 + i < nl && i0 + j < nprev) dw[(o0 + i) * nprev + i0 + j] += acc[i][j];
                  });
        // db_l[o] += sum_r dZ[r][o]
        for (int o = tid; o < nl; o += MLP_THREADS) {
          float s = 0.f;
#pragma unroll 8
          for (int r = 0; r < TM; ++r) s += dz[r * Y.ldz + o];
          smem[Y.s_dw + Y.b_off[l - 1] + o] += s;
        }
        if (l > 1) {
          // dX_{l-1} = dZ_l x W_l ; dZ_{l-1} = dX_{l-1} * act'(X_{l-1})
          const float* xprev = smem + Y.s_xrm[l - 1];
          float* dzo = smem + Y.s_dz[(l - 1) & 1];
          float* dzt = smem + Y.s_xt[l - 1];
          const int kind = Y.hidden_act;
          tile_gemm(smem + Y.s_xt[l], TM, smem + Y.s_wrm[l - 1], ldprev, nl, TM / 4, ldprev / 4,
                    [&](int m0, int c0, float (&acc)[4][4]) {
#pragma unroll
                      for (int j = 0; j < 4; ++j) {
                        const int c = c0 + j;
                        if (c < nprev) {
                          float g[4];
#pragma unroll
                          for (int i = 0; i < 4; ++i) {
                            g[i] = acc[i][j] * act_prime_from_output(xprev[(m0 + i) * ldprev + c], kind);
                            dzo[(m0 + i) * Y.ldz + c] = g[i];
                          }
                          *reinterpret_cast<float4*>(dzt + c * TM + m0) = make_float4(g[0], g[1], g[2], g[3]);
                        }
                      }
                    });
        }
        __syncthreads();
      }
    }
  }

  // ---- per-CTA results ----
  if (BACKWARD) {
    const int n_ls = p.train_log_std ? Y.n[Y.L] : 0;
    float* dst = p.partials + (size_t)blockIdx.x * (Y.P + n_ls);
    for (int i = tid; i < Y.P; i += MLP_THREADS) dst[i] = smem[Y.s_dw + i];
    if (n_ls > 0) {  // per-thread sums -> warp tree -> the warps in order: fixed order, reproducible
      __shared__ float s_ls[MLP_THREADS / 32][16];
      const int lane = tid & 31, warp = tid >> 5;
#pragma unroll
      for (int a = 0; a < 16; ++a) {
        float t = dls[a];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
        if (lane == 0) s_ls[warp][a] = t;
      }
      __syncthreads();
      if (tid < n_ls) {
        float t = 0.f;
        for (int w = 0; w < MLP_THREADS / 32; ++w) t += s_ls[w][tid];
        dst[Y.P + tid] = t;
      }
    }
  }
  if (p.scalar_partials != nullptr) {
    __shared__ double s_sc[7][MLP_THREADS / 32];
    const int lane = tid & 31, warp = tid >> 5;
#pragma unroll
    for (int k = 0; k < 7; ++k) {
      const double v = warp_sum(sc[k]);
      if (lane == 0) s_sc[k][warp] = v;
    }
    __syncthreads();
    if (tid < B200RL_N_SCALARS) {
      double t = 0.0;
      if (tid < 7)
        for (int w = 0; w < MLP_THREADS / 32; ++w) t += s_sc[tid][w];
      p.scalar_partials[(size_t)blockIdx.x * B200RL_N_SCALARS + tid] = t;
    }
  }
}

static size_t fused_static_smem(int tm, int mode) {
  // bytes + 1 once known, 0 before: threads that query concurrently store the same value
  static std::atomic<size_t> cache[3][3];
  const int t = tm == 64 ? 0 : (tm == 32 ? 1 : 2);
  const size_t c = cache[t][mode].load(std::memory_order_relaxed);
  if (c != 0) return c - 1;
  static const void* const fns[3][3] = {
      {(const void*)mlp_fused_kernel<64, 0>, (const void*)mlp_fused_kernel<64, 1>, (const void*)mlp_fused_kernel<64, 2>},
      {(const void*)mlp_fused_kernel<32, 0>, (const void*)mlp_fused_kernel<32, 1>, (const void*)mlp_fused_kernel<32, 2>},
      {(const void*)mlp_fused_kernel<16, 0>, (const void*)mlp_fused_kernel<16, 1>, (const void*)mlp_fused_kernel<16, 2>}};
  cudaFuncAttributes fa;
  if (cudaFuncGetAttributes(&fa, fns[t][mode]) != cudaSuccess) {
    (void)cudaGetLastError();  // no device: nothing launches, and the grid query reports that
    return 0;
  }
  cache[t][mode].store(fa.sharedSizeBytes + 1, std::memory_order_relaxed);
  return fa.sharedSizeBytes;
}

static int fused_grid(const MlpLayout& lay, int64_t n_rows) {
  const int64_t tiles = (n_rows + lay.tm - 1) / lay.tm;
  const int sms = device_sm_count();
  if (sms <= 0) return -1;
  return (int)(tiles < sms ? (tiles < 1 ? 1 : tiles) : sms);
}

// fp16 x 2 tensor-core kernels (mlp_tc2.cu, mlp_tc_fvp.cu): two partial rows per CTA
bool tc_shape_ok(const b200rl_mlp_desc& d);
int launch_mlp_tc2(const b200rl_mlp_loss_grad_args* a, int64_t n_glob, int total_rows, cudaStream_t s);
int launch_mlp_tc_fvp(const b200rl_mlp_loss_grad_args* a, int64_t n_glob, int total_rows, cudaStream_t s);

// The tensor-core kernels are in use for this network: its shape is in their gate, and B200RL_DISABLE_TC=1 (fp32
// kernels only, for A/B parity runs) is not set.  Read on every call so tests can flip it.
bool use_tc(const b200rl_mlp_desc& d) {
  const char* e = getenv("B200RL_DISABLE_TC");
  if (e != nullptr && e[0] == '1') return false;
  return tc_shape_ok(d);
}

// Partial rows of a tensor-core launch: its own two per CTA, or the grid of its fp32 re-run (with that layout) if that
// is larger.  The consumer reduces this many rows whichever of the two kernels wrote them.
static int tc_total_rows(const b200rl_mlp_desc& mlp, int64_t n_rows, bool backward, bool fvp) {
  MlpLayout lay;
  if (build_layout(mlp, backward, &lay, fvp)) return -1;
  const int g = tc_grid(n_rows), f = fused_grid(lay, n_rows);
  if (g <= 0 || f <= 0) return -1;
  return 2 * g > f ? 2 * g : f;
}

}  // namespace b200rl

using namespace b200rl;

extern "C" int64_t b200rl_mlp_param_count(const b200rl_mlp_desc* mlp) {
  if (!mlp || mlp->n_layers < 1 || mlp->n_layers > MAXL) return -1;
  int64_t p = 0;
  for (int l = 0; l < mlp->n_layers; ++l) {
    if (mlp->sizes[l] < 1 || mlp->sizes[l + 1] < 1) return -1;
    p += (int64_t)mlp->sizes[l + 1] * mlp->sizes[l] + mlp->sizes[l + 1];
  }
  return p;
}

// with_backward: 0 forward only (EVAL), 1 forward + backward, 2 Fisher-vector product, 3 forward only with out_full /
// old_out / NO_TC / a loss other than EVAL, 4 forward + backward on the fp32 kernel (NO_TC or train_log_std)
extern "C" int b200rl_mlp_grid(const b200rl_mlp_desc* mlp, int64_t n_rows, int with_backward) {
  if (!mlp) return -1;
  const bool backward = with_backward == 1 || with_backward == 2 || with_backward == 4, fvp = with_backward == 2;
  if (with_backward >= 0 && with_backward <= 3 && use_tc(*mlp)) return tc_total_rows(*mlp, n_rows, backward, fvp);
  MlpLayout lay;
  if (build_layout(*mlp, backward, &lay, fvp)) return -1;
  return fused_grid(lay, n_rows);
}

namespace b200rl {
// the fp32 kernel, optionally as the predicated re-run of a tensor-core launch (run_if / seq / total_rows)
static int launch_fused(const b200rl_mlp_loss_grad_args* a, const unsigned* run_if, unsigned seq, int total_rows,
                        cudaStream_t s) {
  const bool fvp = a->loss == B200RL_LOSS_FVP;
  const bool forward_only = (a->flags & B200RL_FLAG_FORWARD_ONLY) != 0 || a->loss == B200RL_LOSS_EVAL;
  const bool backward = !forward_only;
  FusedArgs k{};
  if (build_layout(a->mlp, backward, &k.lay, fvp)) return 2;
  k.run_if = run_if;
  k.seq = seq;
  k.total_rows = total_rows;
  const int mode = fvp ? 2 : (backward ? 1 : 0);
  const size_t smem_bytes = (size_t)k.lay.total_floats * sizeof(float);
  const size_t static_bytes = fused_static_smem(k.lay.tm, mode);
  B200RL_REQUIRE(smem_bytes + static_bytes <= SMEM_LIMIT,
                 "mlp_loss_grad: network needs %zu bytes of shared memory (%zu for its layout + %zu static; > 227 KiB); "
                 "too large for the fused kernel",
                 smem_bytes + static_bytes, smem_bytes, static_bytes);
  const int64_t n_glob = a->n_global > 0 ? a->n_global : a->n_rows;
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
  k.out_full = a->out_full;
  k.old_out = a->old_out;
  k.direction = a->direction;
  k.train_log_std = (a->train_log_std != 0 && backward && a->dist == B200RL_DIST_GAUSSIAN) ? 1 : 0;
  const int grid = fused_grid(k.lay, a->n_rows);
  B200RL_REQUIRE(grid > 0, "mlp_loss_grad: no CUDA device");
#define B200RL_LAUNCH_FUSED(TMV, MODEV)                                                                       \
  do {                                                                                                         \
    B200RL_CUDA(cudaFuncSetAttribute(mlp_fused_kernel<TMV, MODEV>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                     (int)smem_bytes));                                                        \
    mlp_fused_kernel<TMV, MODEV><<<grid, MLP_THREADS, smem_bytes, s>>>(k);                                     \
  } while (0)
#define B200RL_LAUNCH_TM(TMV)                      \
  do {                                             \
    if (mode == 2) B200RL_LAUNCH_FUSED(TMV, 2);    \
    else if (mode == 1) B200RL_LAUNCH_FUSED(TMV, 1); \
    else B200RL_LAUNCH_FUSED(TMV, 0);              \
  } while (0)
  if (k.lay.tm == 64) B200RL_LAUNCH_TM(64);
  else if (k.lay.tm == 32) B200RL_LAUNCH_TM(32);
  else B200RL_LAUNCH_TM(16);
#undef B200RL_LAUNCH_TM
#undef B200RL_LAUNCH_FUSED
  B200RL_CUDA(cudaGetLastError());
  count_launch(1);
  return 0;
}

int launch_fused_fallback(const b200rl_mlp_loss_grad_args* a, const unsigned* run_if, unsigned seq, int total_rows,
                          cudaStream_t s) {
  return launch_fused(a, run_if, seq, total_rows, s);
}

}  // namespace b200rl

extern "C" int64_t b200rl_tc_fallback_count(void) {
  unsigned long long v = 0;
  if (cudaDeviceSynchronize() != cudaSuccess) return -1;
  if (cudaMemcpyFromSymbol(&v, g_tc_fallbacks, sizeof(v)) != cudaSuccess) return -1;
  return (int64_t)v;
}

extern "C" int b200rl_mlp_loss_grad(const b200rl_mlp_loss_grad_args* a, void* stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200RL_REQUIRE(a != nullptr, "mlp_loss_grad: NULL args");
  const bool fvp = a->loss == B200RL_LOSS_FVP;
  const bool forward_only = (a->flags & B200RL_FLAG_FORWARD_ONLY) != 0 || a->loss == B200RL_LOSS_EVAL;
  const bool backward = !forward_only;
  B200RL_REQUIRE(!(fvp && forward_only), "mlp_loss_grad: FVP cannot be forward-only");
  FusedArgs k{};
  if (build_layout(a->mlp, backward, &k.lay, fvp)) return 2;
  const int L = k.lay.L;
  B200RL_REQUIRE(a->n_rows >= 0, "mlp_loss_grad: negative n_rows");
  if (a->n_rows == 0) {  // an empty shard (data-parallel ranks may hold none): every partial row is zero
    const int rows = b200rl_mlp_grid(&a->mlp, 0, fvp ? 2 : (backward ? 1 : 0));
    B200RL_REQUIRE(rows > 0, "mlp_loss_grad: no CUDA device");
    if (backward) B200RL_REQUIRE(a->partials, "mlp_loss_grad: partials is NULL");
    if (backward)
      B200RL_CUDA(cudaMemsetAsync(a->partials, 0,
                                  (size_t)rows * (k.lay.P + (a->train_log_std ? k.lay.n[L] : 0)) * sizeof(float), s));
    if (a->scalar_partials)
      B200RL_CUDA(cudaMemsetAsync(a->scalar_partials, 0, (size_t)rows * B200RL_N_SCALARS * sizeof(double), s));
    return 0;
  }
  B200RL_REQUIRE(a->params && a->obs, "mlp_loss_grad: params/obs is NULL");
  B200RL_REQUIRE(a->loss >= B200RL_LOSS_EVAL && a->loss <= B200RL_LOSS_FVP, "mlp_loss_grad: bad loss %d", a->loss);
  if (a->dist == B200RL_DIST_NONE) {
    B200RL_REQUIRE(a->loss == B200RL_LOSS_EVAL || a->loss == B200RL_LOSS_MSE,
                   "mlp_loss_grad: dist NONE supports only EVAL / MSE");
    B200RL_REQUIRE(k.lay.n[L] == 1, "mlp_loss_grad: value head must have one output, got %d", k.lay.n[L]);
    B200RL_REQUIRE(a->loss != B200RL_LOSS_MSE || a->target, "mlp_loss_grad: MSE needs target");
    B200RL_REQUIRE(!a->out_full && !a->old_out, "mlp_loss_grad: out_full / old_out need a distribution");
  } else {
    B200RL_REQUIRE(a->dist == B200RL_DIST_GAUSSIAN || a->dist == B200RL_DIST_CATEGORICAL, "mlp_loss_grad: bad dist");
    B200RL_REQUIRE(a->loss != B200RL_LOSS_MSE, "mlp_loss_grad: MSE needs dist NONE");
    B200RL_REQUIRE(fvp || a->actions, "mlp_loss_grad: actions is NULL");
    B200RL_REQUIRE(k.lay.n[L] <= 16, "mlp_loss_grad: at most 16 action dimensions, got %d", k.lay.n[L]);
    B200RL_REQUIRE(a->dist != B200RL_DIST_GAUSSIAN || a->log_std, "mlp_loss_grad: Gaussian needs log_std");
    if (a->loss != B200RL_LOSS_EVAL && !fvp) B200RL_REQUIRE(a->adv_raw, "mlp_loss_grad: policy loss needs adv_raw");
    if (a->loss == B200RL_LOSS_PPO_CLIP || a->loss == B200RL_LOSS_TRPO_SURROGATE)
      B200RL_REQUIRE(a->old_logp, "mlp_loss_grad: PPO/TRPO loss needs old_logp");
    if (fvp) B200RL_REQUIRE(a->direction, "mlp_loss_grad: FVP needs the direction vector");
  }
  if (backward) B200RL_REQUIRE(a->partials, "mlp_loss_grad: partials is NULL");
  const int64_t n_glob = a->n_global > 0 ? a->n_global : a->n_rows;
  // The tensor-core kernels take a launch in their shape gate unless it sets NO_TC.  They produce raw outputs / the
  // true KL on mlp_tc2's forward-only variant only, and dLoss/dlog_std not at all (FVP launches ignore train_log_std).
  const bool wants_out = a->out_full != nullptr || a->old_out != nullptr;
  const bool tc = use_tc(a->mlp) && !(a->flags & B200RL_FLAG_NO_TC) && (forward_only || !wants_out);
  if (tc && (fvp || !a->train_log_std)) {
    const int rows = tc_total_rows(a->mlp, a->n_rows, backward, fvp);
    B200RL_REQUIRE(rows > 0, "mlp_loss_grad: no CUDA device");
    return fvp ? launch_mlp_tc_fvp(a, n_glob, rows, s) : launch_mlp_tc2(a, n_glob, rows, s);
  }
  // a forward-only launch in the gate writes the partial rows b200rl_mlp_grid reports for the tensor-core path
  const int rows = forward_only && use_tc(a->mlp) ? tc_total_rows(a->mlp, a->n_rows, false, false) : 0;
  return launch_fused(a, nullptr, 0u, rows, s);
}
