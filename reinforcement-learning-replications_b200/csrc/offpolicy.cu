// Off-policy update engine: DDPG / TD3 train() on device-resident minibatches.
//
// Replaces (reference: /root/reference/src/rl_replicas/): algorithms/td3.py:214-358 (train, train_policy,
// compute_targets, train_q_function), algorithms/ddpg.py:195-293, q_function.py:20-32, policies/
// deterministic_policy.py:23-32, utils.py:47-57 (polyak_average), and the torch.optim.Adam steps inside them.
//
// Regime: minibatch B ~ 100-256 rows, 256-wide ReLU MLPs (~70k parameters each): ~0.5 GFLOP per train step, i.e.
// launch-latency bound, not throughput bound (SURVEY 7.3-8).  The design therefore minimises host involvement:
// ALL `num_train_steps` minibatches (and the target-smoothing noise) are uploaded once, every step runs as a fixed
// sequence of small fp32 kernels with no host synchronisation, and losses / Q-values are read back once at the end.
// GEMMs are one generic 32x32x32 shared-memory-tiled fp32 kernel in three operand arrangements (forward NT, dX NN,
// dW TN) with the activation derivative fused into the operand load, so activations are never rewritten; torch.cat of
// [s | a] is a split operand, the target-smoothing noise an epilogue.  File map: tile function and elementwise kernels;
// the engine (one state slab); enqueue_steps = the S steps as a four-stream dependency graph (captured once, replayed,
// or issued as plain launches with B200RL_OFFPOLICY_GRAPH=0); the three entry points
// train (host-staged minibatches), train_gather (host-drawn indices, device gather), train_gather_rng (device draws).
// Learner groups (create_group): K learners in K arenas at a fixed stride, every kernel above with a LANES
// instantiation that serves all of them in one launch; a K = 1 engine runs the solo instantiations.
// SAC (config algo = 1) is a second step program on the same engine: its head / soft-loss / temperature kernels and
// enqueue_sac_steps, run as a captured graph or as plain launches like the TD3 / DDPG steps.
// DQN (config algo = 2) is a third: a per-row Huber loss head on discrete actions (dqn_loss_kernel), a target copy
// gated by a per-learner step table (dqn_target_copy_kernel) and enqueue_dqn_steps; networks 1 and 4 only.
// C51 (config algo = 3) is DQN's step program with a categorical head over return distributions (c51_loss_kernel).
// QR-DQN (set_qr on a DQN engine) is DQN's step program with a quantile Huber head (qr_loss_kernel), prioritized replay
// and n-step returns included.
// Dueling Q networks (config dueling_k, DQN / QR-DQN / C51): dueling_forward / dueling_backward take the place of
// net_forward / net_backward for networks 1 and 4 -- the same GEMMs plus dueling_forward_kernel / dueling_backward_kernel
// between the last layer and the loss head; nothing else in the step program differs.
// Noisy networks (config noisy_layers, DQN / QR-DQN / C51, plain or dueling): noisy_compose_kernel draws both networks'
// weight noise and composes their layers into the plain layout the GEMMs read at the start of each step, and
// noisy_expand_kernel maps the composed layers' gradient to the noisy vector's before Adam.
// IQN (config algo = 4) is DQN's step program over an implicit quantile network: iqn_draw_kernel draws the step's
// fractions and their cosine features, iqn_forward / iqn_backward run the network on one row per fraction, and
// iqn_loss_kernel is the loss head.
// Prioritized replay for DQN (train_prioritized): a 32-way sum tree per replay buffer, drawn from, weighed and gathered
// by per_draw_kernel and updated by per_update_kernel inside the same step program.
// n-step returns for DQN / C51 (set_nstep): nstep_gather_kernel (or per_draw_kernel's NSTEP instantiation) walks each
// drawn row's window and stages its return and discount; the loss heads' NSTEP instantiations read the per-row discount
// in place of gamma.
// D4PG (config algo = 6, create_d4pg) is DDPG's step program (enqueue_steps) with a categorical critic over [s | a]:
// c51_loss_kernel (act = NULL, n = 1) as the critic's head, d4pg_policy_loss_kernel as the policy's, and DQN's
// prioritized draw / priority update and n-step staging.
// TQC (config algo = 7, create_tqc) is SAC's step program (enqueue_sac_steps) with two quantile critics over [s | a]:
// tqc_target_kernel truncates the pooled target atoms, tqc_critic_loss_kernel and tqc_policy_loss_kernel are the heads.
// IQL (config algo = 9, create_iql) is a step program of its own (enqueue_iql_steps): network 3 is a trained value
// network, iql_value_loss_kernel and iql_policy_loss_kernel are its heads, sac_q_loss_kernel the critics'.
// REDQ (config algo = 10, create_redq) is a step program of its own (enqueue_redq_steps): SAC's policy over N critics
// run as one ensemble (gemm_ens_kernel, one launch per layer for all of them), the target over a drawn subset of M.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "common.cuh"

namespace b200rl {

constexpr int GT = 32;   // output tile (256x256 outputs -> 64 CTAs; the batch is small, parallelism matters more than reuse)
constexpr int GK = 32;   // k tile
constexpr int GTHREADS = 256;

__device__ __forceinline__ float op_act(float z, int kind) {
  if (kind == B200RL_ACT_TANH) return tanhf(z);
  if (kind == B200RL_ACT_RELU) return fmaxf(z, 0.f);
  return z;
}
__device__ __forceinline__ float op_act_prime(float y, int kind) {  // derivative from the activation OUTPUT
  if (kind == B200RL_ACT_TANH) return 1.f - y * y;
  if (kind == B200RL_ACT_RELU) return y > 0.f ? 1.f : 0.f;
  return 1.f;
}

// a' = clamp(a + clamp(sigma * eps, -c, c), -limit, limit)   (td3.py:326-332)
__device__ __forceinline__ float smooth_target_action(float a, float eps, float sigma, float clipv, float limit) {
  float e = sigma * eps;
  e = fminf(fmaxf(e, -clipv), clipv);
  return fminf(fmaxf(a + e, -limit), limit);
}

// MODE 0 (NT): C[M,N] = act(A[M,K] * B[N,K]^T + bias[N])              forward: A = X, B = W [out,in]
// MODE 1 (NN): C[M,N] = (A (.) act'(Y))[M,K] * B[K,N]                  dX = dZ * W,   A = dY, Y = layer output
// MODE 2 (TN): C[M,N] = (A (.) act'(Y))[K,M]^T * B[K,N]                dW = dZ^T * X, A = dY [rows, out];
//              and, when dbias is set, dbias[M] = column sums of (A (.) act'(Y)) -- the bias gradient rides along
// MODE 3 (NN, split B): MODE 1 with rows >= ksplit of B read from A2[row - ksplit] (ld lda2): dX through a layer whose
//              weight is two [out, in] blocks kept apart, the dueling streams' hidden layers [W_value; W_advantage]
// MODE 4 (NT, gated): C[M,N] = (A[M,K] * B[N,K]^T) (.) act'(Y)[M,N]      EDAC's tangent forward: MODE 0's product with
//              no bias and no activation, its output gated by the derivative at the same position of Y (ld ldy)
// All matrices row-major with explicit leading dimensions.  Y (same shape / ld as A) may be NULL (no derivative).
struct GemmArgs {
  const float* A; int lda;
  const float* B; int ldb;
  float* C; int ldc;
  const float* bias;
  const float* Y; int ldy; int act;  // MODE 0: output activation; MODE 1/2: activation whose derivative gates A
  int M, N, K;
  float* dbias;                      // MODE 2 only
  // the critics' [s | a] input and the target-policy smoothing, fused into the operand load and the epilogue:
  const float* A2; int lda2; int ksplit;  // A2 != NULL: columns >= ksplit of A (MODE 0) / of B (MODE 2) come from
                                          // A2[:, col - ksplit]: the operand is torch.cat([left, A2], -1), never built
  const float* eps; float sigma, clipv, limit;  // eps != NULL: target-policy smoothing on the output (td3.py:326-332)
};

// These GEMMs are tiny (256 x 256 x 256) and sit on a long dependency chain, so latency is what counts: the operands are
// fetched into registers (coalesced along the contiguous dimension of each operand) eight k-tiles at a time and
// multiplied out of shared memory tile by tile.
typedef float GemmTile[GK][GT + 2];

template <int MODE, bool SPLIT_B = false>  // MODE 3 runs as <1, true>: MODE 1 but for where B's rows come from
__device__ __forceinline__ void gemm_tile(const GemmArgs& g, int bx, int by, GemmTile& As, GemmTile& Bs) {
  constexpr bool NT = MODE == 0 || MODE == 4;  // MODE 4 loads its operands as MODE 0 does
  constexpr int KT = 8;  // k-tiles fetched ahead (registers: 8 per k-tile): K = 256 is ONE round of loads
  const int tid = threadIdx.x;
  const int m0 = by * GT, n0 = bx * GT;
  const int tm = (tid / 16) * 2, tn = (tid % 16) * 2;  // 16 x 16 threads, 2 x 2 outputs each
  constexpr int PER = GK * GT / GTHREADS;               // elements of each operand tile per thread (4)
  float rab[KT][PER], rbb[KT][PER];
  // element e of a tile handled by this thread: idx = tid + e * GTHREADS; (hi, lo) = (idx / 32, idx % 32) with `lo`
  // running along the operand's contiguous dimension
  auto fetch = [&](int k0, float (&ra)[PER], float (&rb)[PER]) {
#pragma unroll
    for (int e = 0; e < PER; ++e) {
      const int idx = tid + e * GTHREADS, hi = idx >> 5, lo = idx & 31;
      {  // A
        const int k = MODE == 2 ? hi : lo, m = MODE == 2 ? lo : hi;
        const int gm = m0 + m, gk = k0 + k;
        float a = 0.f;
        if (gm < g.M && gk < g.K) {
          const size_t ia = MODE == 2 ? (size_t)gk * g.lda + gm : (size_t)gm * g.lda + gk;
          if (NT && g.A2 != nullptr && gk >= g.ksplit) a = g.A2[(size_t)gm * g.lda2 + (gk - g.ksplit)];
          else a = g.A[ia];
          if (!NT && g.Y) a *= op_act_prime(g.Y[MODE == 2 ? (size_t)gk * g.ldy + gm : (size_t)gm * g.ldy + gk], g.act);
        }
        ra[e] = a;
      }
      {  // B
        const int k = NT ? lo : hi, n = NT ? hi : lo;
        const int gn = n0 + n, gk = k0 + k;
        float b = 0.f;
        if (gn < g.N && gk < g.K) {
          if constexpr (SPLIT_B) {
            b = gk >= g.ksplit ? g.A2[(size_t)(gk - g.ksplit) * g.lda2 + gn] : g.B[(size_t)gk * g.ldb + gn];
          } else {
            if (MODE == 2 && g.A2 != nullptr && gn >= g.ksplit) b = g.A2[(size_t)gk * g.lda2 + (gn - g.ksplit)];
            else b = NT ? g.B[(size_t)gn * g.ldb + gk] : g.B[(size_t)gk * g.ldb + gn];
          }
        }
        rb[e] = b;
      }
    }
  };
  auto stash = [&](const float (&ra)[PER], const float (&rb)[PER]) {
#pragma unroll
    for (int e = 0; e < PER; ++e) {
      const int idx = tid + e * GTHREADS, hi = idx >> 5, lo = idx & 31;
      if (MODE == 2) As[hi][lo] = ra[e]; else As[lo][hi] = ra[e];
      if (NT) Bs[lo][hi] = rb[e]; else Bs[hi][lo] = rb[e];
    }
  };
  float acc[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
  float colsum[2] = {0.f, 0.f};
  // All loads of up to KT k-tiles are issued back to back (one memory latency for the whole K = 256 product instead of
  // one per k-tile: these GEMMs sit on a dependency chain, their latency is the train step's); the tiles then go through
  // shared memory one after the other, k ascending, so every output's fma chain is the one of a plain k loop.
  for (int kb = 0; kb < g.K; kb += GK * KT) {
#pragma unroll
    for (int t = 0; t < KT; ++t)
      if (kb + t * GK < g.K) fetch(kb + t * GK, rab[t], rbb[t]);
#pragma unroll
    for (int t = 0; t < KT; ++t) {
      if (kb + t * GK < g.K) {  // block-uniform
        stash(rab[t], rbb[t]);
        __syncthreads();
#pragma unroll
        for (int k = 0; k < GK; ++k) {
          const float2 av = *reinterpret_cast<const float2*>(&As[k][tm]);
          const float2 bv = *reinterpret_cast<const float2*>(&Bs[k][tn]);
          const float ar[2] = {av.x, av.y}, br[2] = {bv.x, bv.y};
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            if (MODE == 2) colsum[i] += ar[i];
#pragma unroll
            for (int j = 0; j < 2; ++j) acc[i][j] = fmaf(ar[i], br[j], acc[i][j]);
          }
        }
        __syncthreads();
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int gm = m0 + tm + i, gn = n0 + tn + j;
      if (gm < g.M && gn < g.N) {
        float v = acc[i][j];
        if (MODE == 0) {
          v = op_act(v + (g.bias ? g.bias[gn] : 0.f), g.act);
          if (g.eps != nullptr) v = smooth_target_action(v, g.eps[(size_t)gm * g.N + gn], g.sigma, g.clipv, g.limit);
        } else if (MODE == 4) {
          v *= op_act_prime(g.Y[(size_t)gm * g.ldy + gn], g.act);
        }
        g.C[(size_t)gm * g.ldc + gn] = v;
      }
    }
  if (MODE == 2 && g.dbias != nullptr && bx == 0 && tn == 0) {
#pragma unroll
    for (int i = 0; i < 2; ++i)
      if (m0 + tm + i < g.M) g.dbias[m0 + tm + i] = colsum[i];
  }
}

// Learner groups (b200rl_offpolicy_create_group): everything the engine owns for one learner lives in one arena, and
// the K arenas lie lane_stride bytes apart, so learner z's copy of any engine buffer is ptr + z * lane_stride.  Every
// kernel below has a LANES instantiation that serves all K learners in one launch (learner = blockIdx.z) with the
// arithmetic of the solo kernel; a K = 1 engine launches the LANES = false instantiation, which is the solo kernel.
template <typename T>
__device__ __forceinline__ T* lane_ptr(T* p, size_t off) {  // NULL stays NULL (optional operands)
  return p == nullptr ? p : reinterpret_cast<T*>(reinterpret_cast<uintptr_t>(p) + off);
}

template <int MODE, bool LANES>
__global__ void __launch_bounds__(GTHREADS) gemm_kernel(const GemmArgs g, size_t lane_stride) {
  __shared__ GemmTile As, Bs;
  if (LANES) {
    const size_t off = blockIdx.z * lane_stride;
    GemmArgs a = g;
    a.A = lane_ptr(a.A, off);
    a.B = lane_ptr(a.B, off);
    a.C = lane_ptr(a.C, off);
    a.bias = lane_ptr(a.bias, off);
    a.Y = lane_ptr(a.Y, off);
    a.dbias = lane_ptr(a.dbias, off);
    a.A2 = lane_ptr(a.A2, off);
    a.eps = lane_ptr(a.eps, off);
    gemm_tile<MODE == 3 ? 1 : MODE, MODE == 3>(a, blockIdx.x, blockIdx.y, As, Bs);
  } else {
    gemm_tile<MODE == 3 ? 1 : MODE, MODE == 3>(g, blockIdx.x, blockIdx.y, As, Bs);
  }
}

// ---- device-side draws (opt-in; SURVEY 8f-4): Philox4x32-10, counter-based, so a (seed, call) pair names the whole
// [S, B] index block and the [S, B, A] noise block of one train() call whatever the launch geometry.
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const unsigned long long p0 = (unsigned long long)0xD2511F53u * c.x, p1 = (unsigned long long)0xCD9E8D57u * c.z;
    c = make_uint4((unsigned)(p1 >> 32) ^ c.y ^ k.x, (unsigned)p1, (unsigned)(p0 >> 32) ^ c.w ^ k.y, (unsigned)p0);
    k.x += 0x9E3779B9u;
    k.y += 0xBB67AE85u;
  }
  return c;
}

// Box-Muller of one Philox block: four N(0, 1) values (draw_minibatches_kernel's noise, noisy_draw's weight noise)
__device__ __forceinline__ void box_muller4(uint4 r, float (&z)[4]) {
  const float u1 = ((float)r.x + 1.0f) * 2.3283064365386963e-10f, u2 = (float)r.y * 2.3283064365386963e-10f;
  const float u3 = ((float)r.z + 1.0f) * 2.3283064365386963e-10f, u4 = (float)r.w * 2.3283064365386963e-10f;
  const float m1 = sqrtf(-2.f * logf(u1)), m2 = sqrtf(-2.f * logf(u3));
  float s1, c1, s2, c2;
  sincospif(2.f * u2, &s1, &c1);
  sincospif(2.f * u4, &s2, &c2);
  z[0] = m1 * c1, z[1] = m1 * s1, z[2] = m2 * c2, z[3] = m2 * s2;
}

// (seed, call, ring) of every learner of a launch: one entry for the solo kernel, one per learner for LANES
template <bool LANES>
struct DrawKeys {
  static constexpr int N = LANES ? B200RL_MAX_LEARNERS : 1;
  unsigned long long seed[N], call[N];
  long long start[N], size[N], capacity[N];
};

// idx[j] = physical row of a uniform draw over the `size` live rows of the ring (logical row u sits at
// (start + u) % capacity);  eps[j] = N(0, 1) by Box-Muller.  One thread = one Philox block = 4 values of each.
// A learner's draws depend on its (seed, call) only: in a group they equal those of a solo engine with that key.
template <bool LANES>
__global__ void draw_minibatches_kernel(long long* idx, long long n_idx, float* eps, long long n_eps,
                                        const DrawKeys<LANES> keys, size_t lane_stride) {
  const int z = LANES ? blockIdx.z : 0;
  if (LANES) {
    idx = lane_ptr(idx, blockIdx.z * lane_stride);
    eps = lane_ptr(eps, blockIdx.z * lane_stride);
  }
  const unsigned long long seed = keys.seed[z], call = keys.call[z];
  const long long start = keys.start[z], size = keys.size[z], capacity = keys.capacity[z];
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const uint2 key = make_uint2((unsigned)seed, (unsigned)(seed >> 32));
  if (4 * t < n_idx) {
    const uint4 r = philox4x32_10(make_uint4((unsigned)t, (unsigned)(t >> 32), (unsigned)call, 0x1D5u), key);
    const unsigned v[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (4 * t + j < n_idx) {
        const long long u = (long long)(((unsigned long long)v[j] * (unsigned long long)size) >> 32);  // [0, size)
        idx[4 * t + j] = (start + u) % capacity;
      }
  }
  if (eps != nullptr && 4 * t < n_eps) {
    const uint4 r = philox4x32_10(make_uint4((unsigned)t, (unsigned)(t >> 32), (unsigned)call, 0xE95u), key);
    float z[4];
    box_muller4(r, z);
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (4 * t + j < n_eps) eps[4 * t + j] = z[j];
  }
}

// one replay column of every learner of a launch (each learner has its own replay buffer)
template <bool LANES>
struct LaneSrc {
  const float* p[LANES ? B200RL_MAX_LEARNERS : 1];
};

// staged[i, :] = table[idx[i], :]  (replay-buffer gather; one launch per column)
template <bool LANES>
__global__ void gather_rows_kernel(const LaneSrc<LANES> src, const long long* idx, int width, long long n_out, float* out,
                                   size_t lane_stride) {
  const float* table = src.p[LANES ? blockIdx.z : 0];
  if (LANES) {
    idx = lane_ptr(idx, blockIdx.z * lane_stride);
    out = lane_ptr(out, blockIdx.z * lane_stride);
  }
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_out * width) return;
  const long long r = i / width;
  out[i] = table[idx[r] * width + (i - r * width)];
}

// ---- n-step returns (DQN / C51; b200rl_offpolicy_set_nstep) ----
constexpr int NSTEP_MAX = 32;

// One window from start row p (b200rl.h, "n-step returns"): R = rew[p], g = gamma; for k = 1 .. n - 1 stop at a row that
// is done or ends an episode, else step to the physical successor and take R += g rew, g *= gamma.  Every product and
// sum is rounded on its own (no contraction), so a float32 host walk gives the same bits.  Returns the last row.
__device__ __forceinline__ long long nstep_walk(const float* rew, const float* done, const float* ends, long long rows,
                                                long long p, int n, float gamma, float& R, float& g) {
  R = rew[p];
  g = gamma;
  for (int k = 1; k < n; ++k) {
    if (done[p] != 0.f || ends[p] != 0.f) break;
    p = p + 1 == rows ? 0 : p + 1;  // the window may cross the wrap
    R = __fadd_rn(R, __fmul_rn(g, rew[p]));
    g = __fmul_rn(g, gamma);
  }
  return p;
}

// out[r, :] = table[rows[r], :] for the CTA's nr rows, consecutive threads on consecutive floats
__device__ __forceinline__ void copy_rows(const float* table, const long long* rows, int width, int nr, float* out) {
  for (int i = threadIdx.x; i < nr * width; i += blockDim.x) {
    const int r = i / width;
    out[i] = table[rows[r] * width + (i - r * width)];
  }
}

// the replay columns, episode-end column (n-step calls), sum tree (prioritized calls) and row count of every learner
// of a launch
template <bool LANES>
struct ReplayLanes {
  static constexpr int N = LANES ? B200RL_MAX_LEARNERS : 1;
  LaneSrc<LANES> obs, act, rew, next_obs, done, ends;
  float* tree[N];
  long long rows[N];
};

// The n-step gather of train_gather[_rng] (replaces the five gather_rows_kernel launches): thread i walks the window of
// start row idx[i] and stages rew := R, done := done[last], disc := g and last; then the CTA copies obs and act from the
// start rows and next_obs from the last rows.
template <bool LANES>
__global__ void __launch_bounds__(GTHREADS) nstep_gather_kernel(const ReplayLanes<LANES> src, const long long* idx,
                                                               long long n_out, int O, int A, int n, float gamma,
                                                               float* obs, float* act, float* rew, float* nobs,
                                                               float* done, float* disc, long long* last,
                                                               size_t lane_stride) {
  const int z = LANES ? blockIdx.z : 0;
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    idx = lane_ptr(idx, o), obs = lane_ptr(obs, o), act = lane_ptr(act, o), rew = lane_ptr(rew, o);
    nobs = lane_ptr(nobs, o), done = lane_ptr(done, o), disc = lane_ptr(disc, o), last = lane_ptr(last, o);
  }
  const long long r0 = (long long)blockIdx.x * blockDim.x, i = r0 + threadIdx.x;
  if (i < n_out) {
    float R, g;
    const long long p = nstep_walk(src.rew.p[z], src.done.p[z], src.ends.p[z], src.rows[z], idx[i], n, gamma, R, g);
    rew[i] = R, disc[i] = g, done[i] = src.done.p[z][p], last[i] = p;
  }
  __syncthreads();  // the CTA's last rows are visible to all its threads
  const int nr = (int)min((long long)blockDim.x, n_out - r0);
  copy_rows(src.obs.p[z], idx + r0, O, nr, obs + r0 * O);
  copy_rows(src.act.p[z], idx + r0, A, nr, act + r0 * A);
  copy_rows(src.next_obs.p[z], last + r0, O, nr, nobs + r0 * O);
}

// y = r + gamma * (1 - d) * min(q1t, q2t)   (td3.py:337-339; ddpg.py:280: single target Q)
__device__ __forceinline__ float td_target(float rew, float done, float q1t, const float* q2t, int i, float gamma) {
  const float q = q2t ? fminf(q1t, q2t[i]) : q1t;
  return rew + gamma * (1.f - done) * q;
}

// One CTA: the critic's loss with its TD target computed on the fly: y as above, loss = mean((q - y)^2),
// dq = 2 (q - y) / B (F.mse_loss + backward), q_copy = q (the logged Q-values);  rew == NULL: the policy loss
// -mean(q), dq = -1/B
template <bool LANES>
__global__ void __launch_bounds__(GTHREADS) q_loss_kernel(const float* q, const float* rew, const float* done,
                                                         const float* q1t, const float* q2t, float gamma, int n,
                                                         float* dq, float* loss_out, float* q_copy, size_t lane_stride) {
  __shared__ double red[32];
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    q = lane_ptr(q, o), rew = lane_ptr(rew, o), done = lane_ptr(done, o), q1t = lane_ptr(q1t, o);
    q2t = lane_ptr(q2t, o), dq = lane_ptr(dq, o), loss_out = lane_ptr(loss_out, o), q_copy = lane_ptr(q_copy, o);
  }
  double acc = 0.0;
  const float inv = 1.0f / (float)n;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float qi = q[i];
    if (q_copy) q_copy[i] = qi;
    if (rew) {
      const float d = qi - td_target(rew[i], done[i], q1t[i], q2t, i, gamma);
      acc += (double)d * (double)d;
      dq[i] = (2.f * d) * inv;
    } else {
      acc -= (double)qi;
      dq[i] = -inv;
    }
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[w];
    *loss_out = (float)(t / (double)n);
  }
}

// target <- rho * target + (1 - rho) * param   (utils.py:47-57: f32 tensors tensor(rho), tensor(1 - rho)); the LANES
// instantiation spells out the product the solo kernel fuses (left to the compiler, it fuses the other one)
struct PolyakArgs {
  float* target[3];
  const float* param[3];
  int n[3];
  int n_nets;
};
template <bool LANES>
__global__ void polyak_kernel(const PolyakArgs a, float rho, float one_minus_rho, size_t lane_stride) {  // every network
  const int i = blockIdx.x * blockDim.x + threadIdx.x;                                                   // in one launch
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    for (int k = 0; k < a.n_nets; ++k) {
      float* t = lane_ptr(a.target[k], o);
      const float* p = lane_ptr(a.param[k], o);
      if (i < a.n[k]) t[i] = __fmaf_rn(t[i], rho, __fmul_rn(p[i], one_minus_rho));
    }
  } else {
    for (int k = 0; k < a.n_nets; ++k)
      if (i < a.n[k]) a.target[k][i] = rho * a.target[k][i] + one_minus_rho * a.param[k][i];
  }
}

// *loss_out = (sum of every thread's `acc`) / n, summed as q_loss_kernel sums: a shuffle tree per warp, then the warp
// totals in warp order
__device__ __forceinline__ void block_mean(double acc, int n, float* loss_out, double* red) {
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[w];
    *loss_out = (float)(t / (double)n);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// SAC (algo = 1; Spinning Up sac/core.py SquashedGaussianMLPActor, sac/sac.py compute_loss_q / compute_loss_pi).  The
// policy network's output is [mu | log_std] [B, 2A]; the kernels below are the head and the soft losses around it.
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float softplus_f(float x) { return x > 20.f ? x : log1pf(expf(x)); }  // F.softplus

// One row of the squashed-Gaussian head (out = [mu | log_std] [2A], eps [A]): u = mu + exp(clamp(log_std)) * eps,
// act = limit * tanh(u); returns logp = sum_j Normal(mu, sigma).log_prob(u)_j - sum_j 2 (log 2 - u_j - softplus(-2 u_j))
__device__ __forceinline__ float sac_squash(const float* out, const float* eps, int A, float lmin, float lmax,
                                            float limit, float* act) {
  float lp = 0.f, corr = 0.f;
  for (int j = 0; j < A; ++j) {
    const float mu = out[j];
    const float ls = fminf(fmaxf(out[A + j], lmin), lmax);
    const float sigma = expf(ls);
    const float u = __fadd_rn(mu, __fmul_rn(sigma, eps[j]));  // rsample: loc + eps * scale
    const float d = u - mu;
    lp += -(d * d) / (2.f * (sigma * sigma)) - ls - 0.918938533204672742f;  // - log sqrt(2 pi)
    corr += 2.f * (0.693147180559945309f - u - softplus_f(-2.f * u));
    act[j] = limit * tanhf(u);
  }
  return lp - corr;
}

// One thread per row: sac_squash of row r
template <bool LANES>
__global__ void sac_squash_kernel(const float* out, const float* eps, int B, int A, float lmin, float lmax, float limit,
                                  float* act, float* logp, size_t lane_stride) {
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    out = lane_ptr(out, o), eps = lane_ptr(eps, o), act = lane_ptr(act, o), logp = lane_ptr(logp, o);
  }
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= B) return;
  logp[r] = sac_squash(out + (size_t)r * 2 * A, eps + (size_t)r * A, A, lmin, lmax, limit, act + (size_t)r * A);
}

// One CTA per critic: y = r + gamma (1 - d) (min(Q1targ, Q2targ)(s', a') - alpha log pi(a' | s')), loss = mean((q - y)^2),
// dq = 2 (q - y) / B, q_copy = q (the logged Q-values)
template <bool LANES>
__global__ void __launch_bounds__(GTHREADS) sac_q_loss_kernel(const float* q, const float* rew, const float* done,
                                                             const float* q1t, const float* q2t, const float* logp_next,
                                                             const float* alpha, float gamma, int n, float* dq,
                                                             float* loss_out, float* q_copy, size_t lane_stride) {
  __shared__ double red[32];
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    q = lane_ptr(q, o), rew = lane_ptr(rew, o), done = lane_ptr(done, o), q1t = lane_ptr(q1t, o), q2t = lane_ptr(q2t, o);
    logp_next = lane_ptr(logp_next, o), alpha = lane_ptr(alpha, o), dq = lane_ptr(dq, o);
    loss_out = lane_ptr(loss_out, o), q_copy = lane_ptr(q_copy, o);
  }
  const float a = *alpha;
  const float inv = 1.0f / (float)n;
  double acc = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float qi = q[i];
    q_copy[i] = qi;
    const float y = rew[i] + gamma * (1.f - done[i]) * (fminf(q1t[i], q2t[i]) - a * logp_next[i]);
    const float d = qi - y;
    acc += (double)d * (double)d;
    dq[i] = (2.f * d) * inv;
  }
  block_mean(acc, n, loss_out, red);
}

// One CTA: loss = mean(alpha log pi - min(q1, q2)) at a = pi(s), the per-row gradients w.r.t. q1 and q2 (torch.min's
// rule: equal values share the gradient half and half), and mean(log pi)
template <bool LANES>
__global__ void __launch_bounds__(GTHREADS) sac_policy_loss_kernel(const float* q1, const float* q2, const float* logp,
                                                                  const float* alpha, int n, float* dq1, float* dq2,
                                                                  float* loss_out, float* logp_mean_out,
                                                                  size_t lane_stride) {
  __shared__ double red[32], red_lp[32];
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    q1 = lane_ptr(q1, o), q2 = lane_ptr(q2, o), logp = lane_ptr(logp, o), alpha = lane_ptr(alpha, o);
    dq1 = lane_ptr(dq1, o), dq2 = lane_ptr(dq2, o), loss_out = lane_ptr(loss_out, o);
    logp_mean_out = lane_ptr(logp_mean_out, o);
  }
  const float a = *alpha;
  const float inv = 1.0f / (float)n;
  double acc = 0.0, acc_lp = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float x1 = q1[i], x2 = q2[i], lp = logp[i];
    acc += (double)(a * lp - fminf(x1, x2));
    acc_lp += (double)lp;
    const float w1 = x1 < x2 ? 1.f : (x1 == x2 ? 0.5f : 0.f);
    dq1[i] = -(w1 * inv);
    dq2[i] = -((1.f - w1) * inv);
  }
  block_mean(acc, n, loss_out, red);
  block_mean(acc_lp, n, logp_mean_out, red_lp);
}

// One thread per (row, j): the gradient of the policy loss w.r.t. the network output [mu | log_std], from
// dA = dQ1/da + dQ2/da (the action columns of the critics' input gradients, row stride ldx) and the alpha log pi term;
// u and sigma are recomputed from the output and eps exactly as sac_squash_kernel computed them.  With t = tanh(u) and
// c = alpha / B:  g_u = dA limit (1 - t^2) + 2 c t,  d mu = g_u,  d log_std = g_u sigma eps - c inside the clamp, else 0
// (the Gaussian term's u - mu = sigma eps cancels from d mu and leaves -1 in d log_std).
template <bool LANES>
__global__ void sac_squash_backward_kernel(const float* out, const float* eps, const float* dx1, const float* dx2, int ldx,
                                           int B, int A, float lmin, float lmax, float limit, const float* alpha,
                                           float* dout, size_t lane_stride) {
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    out = lane_ptr(out, o), eps = lane_ptr(eps, o), dx1 = lane_ptr(dx1, o), dx2 = lane_ptr(dx2, o);
    alpha = lane_ptr(alpha, o), dout = lane_ptr(dout, o);
  }
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * A) return;
  const int r = i / A, j = i - r * A;
  const float c = *alpha / (float)B;
  const float mu = out[(size_t)r * 2 * A + j], raw = out[(size_t)r * 2 * A + A + j];
  const float sigma = expf(fminf(fmaxf(raw, lmin), lmax));
  const float e = eps[(size_t)r * A + j];
  const float u = __fadd_rn(mu, __fmul_rn(sigma, e));
  const float t = tanhf(u);
  const float dA = dx1[(size_t)r * ldx + j] + dx2[(size_t)r * ldx + j];
  const float gu = dA * limit * (1.f - t * t) + 2.f * c * t;
  dout[(size_t)r * 2 * A + j] = gu;
  dout[(size_t)r * 2 * A + A + j] = (raw >= lmin && raw <= lmax) ? gu * sigma * e - c : 0.f;
}

// alpha[0..n) = the fixed alpha (learn == 0), or alpha[0] = exp(log_alpha) (learn == 1: the alpha steps fill the rest)
template <bool LANES>
__global__ void sac_alpha_init_kernel(float* alpha, int n, const float* log_alpha, int learn, float fixed,
                                      size_t lane_stride) {
  if (LANES) alpha = lane_ptr(alpha, blockIdx.z * lane_stride), log_alpha = lane_ptr(log_alpha, blockIdx.z * lane_stride);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (learn) {
    if (i == 0) alpha[0] = expf(*log_alpha);
  } else if (i < n) {
    alpha[i] = fixed;
  }
}

// One CTA: the temperature step.  grad = -mean(log pi + target_entropy) (a fixed-order reduction), then torch.optim.Adam
// on the scalar log_alpha (state = {log_alpha, exp_avg, exp_avg_sq}) with the scalars of table[idx]; alpha_next =
// exp(log_alpha), the alpha of the next step
template <bool LANES>
__global__ void __launch_bounds__(GTHREADS) sac_alpha_step_kernel(const float* logp, int n, float target_entropy,
                                                                 float* state, const float2* table, int idx,
                                                                 float one_minus_b1, float b2, float one_minus_b2,
                                                                 float eps, float* alpha_next, size_t lane_stride) {
  __shared__ double red[32];
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    logp = lane_ptr(logp, o), state = lane_ptr(state, o), table = lane_ptr(table, o);
    alpha_next = lane_ptr(alpha_next, o);
  }
  double acc = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) acc += (double)(logp[i] + target_entropy);
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double tot = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += red[w];
    const float g = -(float)(tot / (double)n);
    const float2 t = table[idx];
    float p = state[0], m = state[1], v = state[2];
    m = m + one_minus_b1 * (g - m);  // the arithmetic of adam_step_kernel (adam.cu); LANES: the solo kernel's rounding
    if (LANES) v = __fmaf_rn(__fmul_rn(g, g), one_minus_b2, __fmul_rn(v, b2));
    else v = v * b2 + one_minus_b2 * (g * g);
    const float denom = sqrtf(v) / t.y + eps;
    p = p - t.x * (m / denom);
    state[0] = p;
    state[1] = m;
    state[2] = v;
    *alpha_next = expf(p);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// IQL (algo = 9; Kostrikov, Nair & Levine 2021): the expectile value head and the advantage-weighted policy head.  The
// critics' head is sac_q_loss_kernel with V'(s') as both target inputs and a zero temperature and log density.
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float torch_min(float a, float b) { return isnan(a) || a < b ? a : b; }  // NaN propagates

// One CTA: q^ = min(q1t, q2t), u = q^ - v, w = tau (u > 0) or 1 - tau; loss = mean(w u^2), dv = -2 w u / B,
// mean_out = mean(v) (the value network at the start of the step)
template <bool LANES>
__global__ void __launch_bounds__(GTHREADS) iql_value_loss_kernel(const float* q1t, const float* q2t, const float* v,
                                                                 float tau, float one_minus_tau, int n, float* dv,
                                                                 float* loss_out, float* mean_out, size_t lane_stride) {
  __shared__ double red[32], red_v[32];
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    q1t = lane_ptr(q1t, o), q2t = lane_ptr(q2t, o), v = lane_ptr(v, o), dv = lane_ptr(dv, o);
    loss_out = lane_ptr(loss_out, o), mean_out = lane_ptr(mean_out, o);
  }
  const float inv = 1.0f / (float)n;
  double acc = 0.0, acc_v = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float vi = v[i];
    const float u = torch_min(q1t[i], q2t[i]) - vi;
    const float w = u > 0.f ? tau : one_minus_tau;
    acc += (double)(w * (u * u));
    acc_v += (double)vi;
    dv[i] = -((2.f * w * u) * inv);
  }
  block_mean(acc, n, loss_out, red);
  block_mean(acc_v, n, mean_out, red_v);
}

// One CTA, one thread per row i: the AWR head on the policy output out = [m | l] [B, 2A] at the dataset action act:
// e_i = min(exp(beta (min(q1t, q2t) - v)), W) (NaN stays NaN), log pi_i = sum_j Normal(L tanh m_j, exp(clamp l_j))
// .log_prob(a_j); loss = -mean(e log pi), weight_mean = mean(e), dout = d loss / d [m | l] (b200rl.h, "IQL")
template <bool LANES>
__global__ void __launch_bounds__(GTHREADS) iql_policy_loss_kernel(const float* out, const float* act, const float* q1t,
                                                                  const float* q2t, const float* v, int n, int A,
                                                                  float beta, float max_w, float lmin, float lmax,
                                                                  float limit, float* dout, float* loss_out,
                                                                  float* weight_mean_out, size_t lane_stride) {
  __shared__ double red[32], red_w[32];
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    out = lane_ptr(out, o), act = lane_ptr(act, o), q1t = lane_ptr(q1t, o), q2t = lane_ptr(q2t, o);
    v = lane_ptr(v, o), dout = lane_ptr(dout, o);
  }
  const float inv = 1.0f / (float)n;
  double acc = 0.0, acc_w = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float x = expf(beta * (torch_min(q1t[i], q2t[i]) - v[i]));
    const float e = x > max_w ? max_w : x;
    const float c = e * inv;
    const float* row = out + (size_t)i * 2 * A;
    float* drow = dout + (size_t)i * 2 * A;
    float lp = 0.f;
    for (int j = 0; j < A; ++j) {
      const float t = tanhf(row[j]), raw = row[A + j];
      const float ls = fminf(fmaxf(raw, lmin), lmax);
      const float sigma = expf(ls), var = sigma * sigma;
      const float d = act[(size_t)i * A + j] - limit * t;
      lp += -(d * d) / (2.f * var) - ls - 0.918938533204672742f;  // - log sqrt(2 pi)
      drow[j] = -(c * (d / var)) * (limit * (1.f - t * t));
      drow[A + j] = (raw >= lmin && raw <= lmax) ? -(c * ((d * d) / var - 1.f)) : 0.f;
    }
    acc -= (double)(e * lp);
    acc_w += (double)e;
  }
  if (LANES) {  // offset after the row loop: with both outputs live across it ptxas spills
    const size_t o = blockIdx.z * lane_stride;
    loss_out = lane_ptr(loss_out, o), weight_mean_out = lane_ptr(weight_mean_out, o);
  }
  block_mean(acc, n, loss_out, red);
  block_mean(acc_w, n, weight_mean_out, red_w);
}

// ---------------------------------------------------------------------------------------------------------------
// TQC (algo = 7; Kuznetsov, Shvechikov, Grishin & Vetrov 2020): SAC's step program with two quantile critics over
// [s | a], each mapping it to M quantile locations at tau_m = (2m + 1) / (2M).  The kernels below are its three heads;
// everything else (squash head and its backward pass, temperature, polyak) is SAC's.
// ---------------------------------------------------------------------------------------------------------------
constexpr int TQC_MAX_QUANTILES = 256;  // M per critic; the pooled target holds up to 2M atoms

// x precedes y in torch.sort's ascending order: NaN sorts last
__device__ __forceinline__ bool tqc_before(float x, float y) { return !isnan(x) && (isnan(y) || x < y); }

// One CTA per row i, one thread per pooled atom (blockDim = 2M rounded up to whole warps).  The 2M atoms
// z = [Q1targ(s', a')_0..M-1 | Q2targ(s', a')_0..M-1] are ranked in shared memory: atom k's rank is the number of atoms
// that precede it, ties (and NaNs) broken by pooled index, so the ranks are a permutation and the kept sequence is
// torch.sort's whatever the ties.  The atoms of rank < kN are kept:
//   y[i, rank] = r + gamma (1 - d) (z_k - alpha log pi(a' | s'))   (sac_q_loss_kernel's order of operations)
template <bool LANES>
__global__ void __launch_bounds__(2 * TQC_MAX_QUANTILES) tqc_target_kernel(
    const float* q1t, const float* q2t, const float* rew, const float* done, const float* logp_next,
    const float* alpha, float gamma, int M, int kN, float* y, size_t lane_stride) {
  __shared__ float sz[2 * TQC_MAX_QUANTILES];
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    q1t = lane_ptr(q1t, o), q2t = lane_ptr(q2t, o), rew = lane_ptr(rew, o), done = lane_ptr(done, o);
    logp_next = lane_ptr(logp_next, o), alpha = lane_ptr(alpha, o), y = lane_ptr(y, o);
  }
  const int i = blockIdx.x, k = threadIdx.x, n = 2 * M;
  if (k < n) sz[k] = k < M ? q1t[(size_t)i * M + k] : q2t[(size_t)i * M + k - M];
  __syncthreads();
  if (k >= n) return;
  const float x = sz[k];
  int rank = 0;
  for (int j = 0; j < n; ++j) {
    const float v = sz[j];
    rank += tqc_before(v, x) || (j < k && !tqc_before(x, v));  // v precedes x, or ties with it at a lower index
  }
  if (rank < kN) {
    const float a = *alpha;
    y[(size_t)i * kN + rank] = rew[i] + gamma * (1.f - done[i]) * (x - a * logp_next[i]);
  }
}

// One CTA per row i, thread m owning critic quantile m (blockDim = M rounded up to whole warps): with
// u_mj = y_ij - theta_m(s, a) over the kN kept target atoms j (ascending) and qr_loss_kernel's weights and Huber terms,
//   L = (1 / (kN M)) sum_m sum_j k_mj h(u_mj)  (j, then m, in index order),
//   dOut[i, m] = -(sum_j k_mj clamp(u_mj, -1, 1)) / (kN M) * (1 / B),  q_copy[i] = (sum_m theta_m) / M.
// The last CTA of a learner to finish (sync counts them) writes *loss_out = mean L, summed in double as
// qr_loss_kernel sums, and leaves the counter at 0.  No atomics touch a float.
template <bool LANES>
__global__ void __launch_bounds__(TQC_MAX_QUANTILES) tqc_critic_loss_kernel(
    const float* q, const float* y, int B, int M, int kN, float* dout, float* row_loss, float* q_copy, int* sync,
    float* loss_out, size_t lane_stride) {
  __shared__ float sy[2 * TQC_MAX_QUANTILES], sl[TQC_MAX_QUANTILES], sth[TQC_MAX_QUANTILES];
  __shared__ double red[32];
  __shared__ bool last;
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    q = lane_ptr(q, o), y = lane_ptr(y, o), dout = lane_ptr(dout, o), row_loss = lane_ptr(row_loss, o);
    q_copy = lane_ptr(q_copy, o), sync = lane_ptr(sync, o), loss_out = lane_ptr(loss_out, o);
  }
  const int t = threadIdx.x, i = blockIdx.x;
  for (int j = t; j < kN; j += blockDim.x) sy[j] = y[(size_t)i * kN + j];
  const float th = t < M ? q[(size_t)i * M + t] : 0.f;
  if (t < M) sth[t] = th;
  __syncthreads();
  const float norm = (float)(kN * M);
  if (t < M) {
    const float tau = (float)(2 * t + 1) / (float)(2 * M);
    float lsum = 0.f, gsum = 0.f;
    for (int j = 0; j < kN; ++j) {
      const float u = sy[j] - th;
      const float k = fabsf(tau - (u < 0.f ? 1.f : 0.f));
      const float au = fabsf(u);
      const float hu = au < 1.f ? 0.5f * u * u : au - 0.5f;
      const float c = u > 1.f ? 1.f : (u < -1.f ? -1.f : u);  // NaN passes through, as torch's clamp lets it
      lsum += k * hu;
      gsum += k * c;
    }
    sl[t] = lsum;
    dout[(size_t)i * M + t] = (-gsum / norm) * (1.0f / (float)B);
  }
  __syncthreads();
  if (t == 0) {
    float L = 0.f, qv = 0.f;
    for (int m = 0; m < M; ++m) L += sl[m], qv += sth[m];
    row_loss[i] = L / norm;
    q_copy[i] = qv / (float)M;
  }
  // the last CTA of this learner reads every row's loss
  __threadfence();
  __syncthreads();
  if (t == 0) last = atomicAdd(sync, 1) == (int)gridDim.x - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  double acc = 0.0;
  for (int r = t; r < B; r += blockDim.x) acc += (double)__ldcg(row_loss + r);
  block_mean(acc, B, loss_out, red);
  if (t == 0) sync[0] = 0;
}

// One CTA: the policy step's head at a = pi(s) on the critics just updated (q1, q2 [B, M]).  Per row the loss is
// alpha log pi - (sum_m q1_m + sum_m q2_m) / (2M) (index order, Q1's quantiles first); *loss_out = its mean,
// *logp_mean_out = mean log pi (each summed as block_mean sums), and every entry of dq1 and dq2 is -1 / (2 M B).
template <bool LANES>
__global__ void __launch_bounds__(GTHREADS) tqc_policy_loss_kernel(const float* q1, const float* q2, const float* logp,
                                                                  const float* alpha, int B, int M, float* dq1,
                                                                  float* dq2, float* loss_out, float* logp_mean_out,
                                                                  size_t lane_stride) {
  __shared__ double red[32], red_lp[32];
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    q1 = lane_ptr(q1, o), q2 = lane_ptr(q2, o), logp = lane_ptr(logp, o), alpha = lane_ptr(alpha, o);
    dq1 = lane_ptr(dq1, o), dq2 = lane_ptr(dq2, o), loss_out = lane_ptr(loss_out, o);
    logp_mean_out = lane_ptr(logp_mean_out, o);
  }
  const float a = *alpha;
  const float g = -1.0f / (float)(2 * M * B);
  for (int e = threadIdx.x; e < B * M; e += blockDim.x) dq1[e] = g, dq2[e] = g;
  double acc = 0.0, acc_lp = 0.0;
  for (int i = threadIdx.x; i < B; i += blockDim.x) {
    const float *x1 = q1 + (size_t)i * M, *x2 = q2 + (size_t)i * M;
    float s = 0.f;
    for (int m = 0; m < M; ++m) s += x1[m];
    for (int m = 0; m < M; ++m) s += x2[m];
    const float lp = logp[i];
    acc += (double)(a * lp - s / (float)(2 * M));
    acc_lp += (double)lp;
  }
  block_mean(acc, B, loss_out, red);
  block_mean(acc_lp, B, logp_mean_out, red_lp);
}

// ---------------------------------------------------------------------------------------------------------------
// CQL (algo = 8; Kumar, Zhou, Tucker & Levine 2020, CQL(H)): SAC's step program whose critics also run on 3N sampled
// actions per minibatch row.  The critics' forward and backward passes run on (1 + 3N) B stacked rows: rows 0..B-1 are
// the data rows [s_i | a_i], row B + i 3N + j sample j of row i.  cql_stage_kernel builds that operand, SAC's soft MSE
// head serves the data rows, cql_penalty_kernel adds the log-sum-exp penalty, cql_alpha_prime_kernel is the optional
// Lagrange step.
// ---------------------------------------------------------------------------------------------------------------
constexpr int CQL_MAX_ACTIONS = 64;  // N; a row's penalty runs over 3N values
constexpr int CQL_WARPS = 8;         // rows per penalty CTA
constexpr float CQL_MAX_ALPHA_PRIME = 1e6f;

// Philox tag of CQL's device draws: distinct from the index (0x1D5), noise (0xE95), IQN (0x9E5) and noisy (0xA00 | r)
// blocks, so SAC's draws for the same (seed, call) are unchanged
constexpr unsigned CQL_DRAW_TAG = 0xC91u;

// draws [S][3][B][N][A] per learner: block 0 uniform x in [0, 1) (24-bit), blocks 1 and 2 N(0, 1) by Box-Muller.  One
// thread = one Philox block = 4 consecutive values; each value takes the form of the block it falls in.
template <bool LANES>
__global__ void cql_draw_kernel(float* draws, long long n, long long block, const DrawKeys<LANES> keys,
                                size_t lane_stride) {
  const int zl = LANES ? blockIdx.z : 0;
  if (LANES) draws = lane_ptr(draws, blockIdx.z * lane_stride);
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (4 * t >= n) return;
  const unsigned long long seed = keys.seed[zl], call = keys.call[zl];
  const uint4 r = philox4x32_10(make_uint4((unsigned)t, (unsigned)(t >> 32), (unsigned)call, CQL_DRAW_TAG),
                                make_uint2((unsigned)seed, (unsigned)(seed >> 32)));
  float z[4];
  box_muller4(r, z);
  const unsigned v[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const long long e = 4 * t + j;
    if (e < n) draws[e] = (e / block) % 3 == 0 ? (float)(v[j] >> 8) * 5.9604644775390625e-8f : z[j];
  }
}

// One thread per stacked row r of the critics' operand x [(1 + 3N) B, O + A]: r < B copies [s_r | a_r]; r = B + i 3N + j
// writes [s_i | action] and logp[i 3N + j], with the action u = limit (2 x - 1) and logp = lu for j < N, a squashed
// sample of pi(.|s'_i) for N <= j < 2N and of pi(.|s_i) for 2N <= j < 3N (out_next / out_cur: the policy outputs at
// s' / s; draws [3][B][N][A] the step's x, eps at s and eps at s', in that order).  The squash is sac_squash's.
template <bool LANES>
__global__ void cql_stage_kernel(const float* obs, const float* act, const float* out_next, const float* out_cur,
                                 const float* draws, int B, int N, int O, int A, float lmin, float lmax, float limit,
                                 float lu, float* x, float* logp, size_t lane_stride) {
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    obs = lane_ptr(obs, o), act = lane_ptr(act, o), out_next = lane_ptr(out_next, o), out_cur = lane_ptr(out_cur, o);
    draws = lane_ptr(draws, o), x = lane_ptr(x, o), logp = lane_ptr(logp, o);
  }
  const int n3 = 3 * N;
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= (long long)B * (1 + n3)) return;
  float* xr = x + r * (O + A);
  if (r < B) {
    for (int c = 0; c < O; ++c) xr[c] = obs[r * O + c];
    for (int c = 0; c < A; ++c) xr[O + c] = act[r * A + c];
    return;
  }
  const int k = (int)(r - B), i = k / n3, j = k - i * n3, blk = j / N, jj = j - blk * N;
  for (int c = 0; c < O; ++c) xr[c] = obs[(size_t)i * O + c];
  const float* d = draws + (((size_t)(blk == 0 ? 0 : 3 - blk) * B + i) * N + jj) * A;  // draws: x, eps at s, eps at s'
  if (blk == 0) {
    for (int c = 0; c < A; ++c) xr[O + c] = limit * (2.f * d[c] - 1.f);
    logp[k] = lu;
  } else {
    logp[k] = sac_squash(blk == 1 ? out_next + (size_t)i * 2 * A : out_cur + (size_t)i * 2 * A, d, A, lmin, lmax,
                         limit, xr + O);
  }
}

// One warp per row i over its 3N sampled values q[B + i 3N + j] (CQL_WARPS rows per CTA): z_j = (q_j - logp_j) / T,
// P_i = T (m + log sum_j exp(z_j - m)) with m = max_j z_j and the sum in index order; with w = weight (times
// alpha'[0], clamped, when alpha_prime != NULL)
//   dq[B + i 3N + j] = w softmax_j(z) / B,  dq[i] -= w / B  (behind SAC's soft MSE head, which wrote 2 (q - y) / B).
// The last CTA of a learner (sync counts them) writes gap = mean_i P_i - mean_i q_i (each sum in double, fixed order),
// adds w gap (- alpha' tau) to *loss_out and leaves the counter at 0.  No atomics touch a float.
template <bool LANES>
__global__ void __launch_bounds__(CQL_WARPS * 32) cql_penalty_kernel(
    const float* q, const float* logp, int B, int N, float temperature, float weight, const float* alpha_prime,
    float tau, float* dq, float* row_p, int* sync, float* loss_out, float* gap_out, size_t lane_stride) {
  __shared__ float sz[CQL_WARPS][3 * CQL_MAX_ACTIONS];
  __shared__ double red[32], red_q[32];
  __shared__ bool last;
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    q = lane_ptr(q, o), logp = lane_ptr(logp, o), alpha_prime = lane_ptr(alpha_prime, o), dq = lane_ptr(dq, o);
    row_p = lane_ptr(row_p, o), sync = lane_ptr(sync, o), loss_out = lane_ptr(loss_out, o);
    gap_out = lane_ptr(gap_out, o);
  }
  const int n3 = 3 * N, w_ = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = blockIdx.x * CQL_WARPS + w_;
  const float ap = alpha_prime != nullptr ? fminf(*alpha_prime, CQL_MAX_ALPHA_PRIME) : 1.f;
  const float w = alpha_prime != nullptr ? ap * weight : weight;
  const float invB = 1.0f / (float)B;
  if (i < B) {
    const float* qi = q + B + (size_t)i * n3;
    const float* li = logp + (size_t)i * n3;
    for (int j = lane; j < n3; j += 32) sz[w_][j] = (qi[j] - li[j]) / temperature;
    __syncwarp();
    float m = sz[w_][0], s = 0.f;
    for (int j = 1; j < n3; ++j) m = fmaxf(m, sz[w_][j]);
    for (int j = 0; j < n3; ++j) s += expf(sz[w_][j] - m);
    float* di = dq + B + (size_t)i * n3;
    for (int j = lane; j < n3; j += 32) di[j] = w * (expf(sz[w_][j] - m) / s) * invB;
    if (lane == 0) {
      row_p[i] = temperature * (m + logf(s));
      dq[i] = dq[i] - w * invB;
    }
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(sync, 1) == (int)gridDim.x - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  double acc = 0.0, acc_q = 0.0;
  for (int r = threadIdx.x; r < B; r += blockDim.x) acc += (double)__ldcg(row_p + r), acc_q += (double)q[r];
  acc = warp_sum(acc), acc_q = warp_sum(acc_q);
  if (lane == 0) red[w_] = acc, red_q[w_] = acc_q;
  __syncthreads();
  if (threadIdx.x == 0) {
    double tp = 0.0, tq = 0.0;
    for (int k = 0; k < CQL_WARPS; ++k) tp += red[k], tq += red_q[k];
    const float gap = (float)(tp / (double)B) - (float)(tq / (double)B);
    *gap_out = gap;
    float l = *loss_out + w * gap;
    if (alpha_prime != nullptr) l -= ap * tau;
    *loss_out = l;
    sync[0] = 0;
  }
}

// One thread: the Lagrange step on log alpha' (state = {log alpha', exp_avg, exp_avg_sq}).  Its loss
// -1/2 sum_k alpha' (weight gap_k - tau), alpha' = clamp(exp(log alpha'), 0, 1e6), has the gradient
// g = -1/2 ((weight gap_1 - tau) + (weight gap_2 - tau)) exp(log alpha') (0 where the clamp is active); one
// torch.optim.Adam step with the scalars of table[idx] (sac_alpha_step_kernel's arithmetic); alpha_next = the clamped
// alpha' of the next step.
template <bool LANES>
__global__ void cql_alpha_prime_kernel(const float* gap1, const float* gap2, float weight, float tau, float* state,
                                       const float2* table, int idx, float one_minus_b1, float b2, float one_minus_b2,
                                       float eps, float* alpha_next, size_t lane_stride) {
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    gap1 = lane_ptr(gap1, o), gap2 = lane_ptr(gap2, o), state = lane_ptr(state, o), table = lane_ptr(table, o);
    alpha_next = lane_ptr(alpha_next, o);
  }
  // every operation rounded explicitly, so that both instantiations compute the same bits
  float p = state[0], m = state[1], v = state[2];
  const float e = expf(p);
  const float s = __fadd_rn(__fsub_rn(__fmul_rn(weight, *gap1), tau), __fsub_rn(__fmul_rn(weight, *gap2), tau));
  const float g = e <= CQL_MAX_ALPHA_PRIME ? __fmul_rn(__fmul_rn(-0.5f, s), e) : 0.f;
  const float2 t = table[idx];
  m = __fadd_rn(m, __fmul_rn(one_minus_b1, __fsub_rn(g, m)));
  v = __fmaf_rn(__fmul_rn(g, g), one_minus_b2, __fmul_rn(v, b2));
  const float denom = __fadd_rn(__fdiv_rn(sqrtf(v), t.y), eps);
  p = __fsub_rn(p, __fmul_rn(t.x, __fdiv_rn(m, denom)));
  state[0] = p;
  state[1] = m;
  state[2] = v;
  *alpha_next = fminf(expf(p), CQL_MAX_ALPHA_PRIME);
}

// ---------------------------------------------------------------------------------------------------------------
// REDQ (algo = 10; Chen, Wang, Zhou & Ross 2021): SAC's squashed-Gaussian policy over an ensemble of N critics.  The N
// critics of a learner lie in one block of the arena (parameters, gradients, Adam moments, activations), each member at
// a fixed byte stride from the first, so one launch per layer serves the whole ensemble: gemm_ens_kernel runs member
// blockIdx.z % nm through gemm_tile, the tile function of every other network, so each critic's arithmetic is a solo
// critic's.  The target pass reads its M members from the step's subset table.
// ---------------------------------------------------------------------------------------------------------------
constexpr int REDQ_MAX_CRITICS = 32;  // N; the ensemble axis of a launch is K N <= 512 CTAs deep in z
constexpr unsigned REDQ_DRAW_TAG = 0x7EDu;  // Philox tag of the subset draws: SAC's index / noise draws stay unchanged

// byte strides between consecutive members of the GemmArgs operands (0: an operand every member shares): the bias moves
// with B (both in the parameter block), dbias with C (both in the gradient block), and A2 -- the action columns of the
// first layer's input -- is shared by every member.  32 bits keep the kernel within its registers.
struct EnsStrides {
  unsigned a, b, c, y;
};

// z = learner nm + slot; the slot's member is sub[slot] (a subset table, per learner) or the slot itself.  The weights
// and bias (B and bias in MODE 0 / 1) move with the member, every other operand with the slot; MODE 2 runs without a
// table, where member and slot agree.
template <int MODE, bool LANES>
__global__ void __launch_bounds__(GTHREADS, 1) gemm_ens_kernel(const GemmArgs g, const EnsStrides es, const int* sub,
                                                            int nm, size_t lane_stride) {
  __shared__ GemmTile As, Bs;
  const int lane = LANES ? (int)blockIdx.z / nm : 0, slot = (int)blockIdx.z - lane * nm;
  const size_t off = LANES ? (size_t)lane * lane_stride : 0;
  const int mem = sub != nullptr ? lane_ptr(sub, off)[slot] : slot;
  GemmArgs a = g;
  const size_t sl = (size_t)slot, ob = off + (size_t)(MODE == 2 ? slot : mem) * es.b, oc = off + sl * es.c;
  a.A = lane_ptr(a.A, off + sl * es.a);
  a.B = lane_ptr(a.B, ob);
  a.C = lane_ptr(a.C, oc);
  a.bias = lane_ptr(a.bias, ob);
  a.Y = lane_ptr(a.Y, off + sl * es.y);
  a.dbias = lane_ptr(a.dbias, oc);
  a.A2 = lane_ptr(a.A2, off);
  gemm_tile<MODE>(a, blockIdx.x, blockIdx.y, As, Bs);
}

// One Adam step for every critic of the ensemble (blockIdx.y = critic k) with the scalars of table[idx]: the arithmetic
// of adam_step_kernel (adam.cu) on critic k's parameters and gradient (k pg bytes after critic 0's) and its moments
// (k mv bytes after), the exp_avg_sq product rounded as that kernel's solo instantiation rounds it.  grad2 != NULL (EDAC's
// diversity gradient, laid out as grad): the step is on grad[i] + grad2[i], added in that order.
template <bool LANES>
__global__ void __launch_bounds__(256) redq_adam_kernel(float* params, const float* grad, const float* grad2, float* m,
                                                        float* v, long long n, size_t pg, size_t mv,
                                                        const float2* table, int idx, float one_minus_b1, float b2,
                                                        float one_minus_b2, float eps, size_t lane_stride) {
  const size_t o = LANES ? blockIdx.z * lane_stride : 0, k = blockIdx.y;
  params = lane_ptr(params, o + k * pg), grad = lane_ptr(grad, o + k * pg), grad2 = lane_ptr(grad2, o + k * pg);
  m = lane_ptr(m, o + k * mv), v = lane_ptr(v, o + k * mv), table = lane_ptr(table, o);
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float2 t = table[idx];
  const float g = grad2 != nullptr ? grad[i] + grad2[i] : grad[i];
  float mi = m[i], vi = v[i];
  mi = mi + one_minus_b1 * (g - mi);
  vi = __fmaf_rn(vi, b2, __fmul_rn(__fmul_rn(g, g), one_minus_b2));
  const float denom = sqrtf(vi) / t.y + eps;
  m[i] = mi;
  v[i] = vi;
  params[i] = params[i] - t.x * (mi / denom);
}

// One thread per step: sub[st][0..M) = the first M entries of a partial Fisher-Yates shuffle of 0..N-1, entry j
// swapping position j with j + floor(u (N - j) / 2^32), u the (j % 4)-th word of Philox block (j / 4, st, call, tag)
template <bool LANES>
__global__ void redq_draw_kernel(int* sub, int S, int N, int M, const DrawKeys<LANES> keys, size_t lane_stride) {
  const int zl = LANES ? blockIdx.z : 0;
  if (LANES) sub = lane_ptr(sub, blockIdx.z * lane_stride);
  const int st = blockIdx.x * blockDim.x + threadIdx.x;
  if (st >= S) return;
  const unsigned long long seed = keys.seed[zl], call = keys.call[zl];
  const uint2 key = make_uint2((unsigned)seed, (unsigned)(seed >> 32));
  int perm[REDQ_MAX_CRITICS];
  for (int j = 0; j < N; ++j) perm[j] = j;
  uint4 r = make_uint4(0u, 0u, 0u, 0u);
  for (int j = 0; j < M; ++j) {
    if ((j & 3) == 0) r = philox4x32_10(make_uint4((unsigned)(j >> 2), (unsigned)st, (unsigned)call, REDQ_DRAW_TAG), key);
    const unsigned u = (j & 3) == 0 ? r.x : (j & 3) == 1 ? r.y : (j & 3) == 2 ? r.z : r.w;
    const int k = j + (int)(((unsigned long long)u * (unsigned long long)(N - j)) >> 32);
    const int t = perm[j];
    perm[j] = perm[k], perm[k] = t;
    sub[st * M + j] = perm[j];
  }
}

// One thread per row i: qmin[i] = fminf over the M gathered target critics qt[j qt_stride + i] in slot order (fminf: a
// NaN loses to a number, as in SAC's target); thread 0 also carries the step's temperature to the next step,
// alpha[1] = alpha[0] (a policy step's temperature step overwrites it later in the step)
template <bool LANES>
__global__ void redq_target_kernel(const float* qt, int qt_stride, int M, int B, float* qmin, float* alpha,
                                   size_t lane_stride) {
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    qt = lane_ptr(qt, o), qmin = lane_ptr(qmin, o), alpha = lane_ptr(alpha, o);
  }
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) alpha[1] = alpha[0];
  if (i >= B) return;
  float m = qt[i];
  for (int j = 1; j < M; ++j) m = fminf(m, qt[(size_t)j * qt_stride + i]);
  qmin[i] = m;
}

// One CTA per critic k = blockIdx.x: sac_q_loss_kernel's head with min(Q1targ, Q2targ) replaced by qmin:
// y = r + gamma (1 - d) (qmin - alpha log pi'), loss_k = mean((q_k - y)^2), dq_k = 2 (q_k - y) / B, the logged values
// q_copy_k = q_k.  Member k's q, dq, loss and q_copy are q_stride, B, loss_stride and copy_stride floats apart.
template <bool LANES>
__global__ void __launch_bounds__(GTHREADS) redq_q_loss_kernel(const float* q, int q_stride, const float* rew,
                                                              const float* done, const float* qmin,
                                                              const float* logp_next, const float* alpha, float gamma,
                                                              int n, float* dq, float* loss_out, int loss_stride,
                                                              float* q_copy, int copy_stride, size_t lane_stride) {
  __shared__ double red[32];
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    q = lane_ptr(q, o), rew = lane_ptr(rew, o), done = lane_ptr(done, o), qmin = lane_ptr(qmin, o);
    logp_next = lane_ptr(logp_next, o), alpha = lane_ptr(alpha, o), dq = lane_ptr(dq, o);
    loss_out = lane_ptr(loss_out, o), q_copy = lane_ptr(q_copy, o);
  }
  const int k = blockIdx.x;
  q += (size_t)k * q_stride, dq += (size_t)k * n, loss_out += (size_t)k * loss_stride;
  q_copy += (size_t)k * copy_stride;
  const float a = *alpha;
  const float inv = 1.0f / (float)n;
  double acc = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float qi = q[i];
    q_copy[i] = qi;
    const float y = rew[i] + gamma * (1.f - done[i]) * (qmin[i] - a * logp_next[i]);
    const float d = qi - y;
    acc += (double)d * (double)d;
    dq[i] = (2.f * d) * inv;
  }
  block_mean(acc, n, loss_out, red);
}

// One CTA: the policy step's head at a = pi(s) on the N critics just updated (member k's output at q + k q_stride).
// Per row the loss is alpha log pi - (sum_k q_k) / N (k in index order); *loss_out = its mean, *logp_mean_out = mean
// log pi (each summed as block_mean sums), and every dq_k[i] (member k's at dq + k B) is -1 / (N B).
template <bool LANES>
__global__ void __launch_bounds__(GTHREADS) redq_policy_loss_kernel(const float* q, int q_stride, int N,
                                                                   const float* logp, const float* alpha, int B,
                                                                   float* dq, float* loss_out, float* logp_mean_out,
                                                                   size_t lane_stride) {
  __shared__ double red[32], red_lp[32];
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    q = lane_ptr(q, o), logp = lane_ptr(logp, o), alpha = lane_ptr(alpha, o), dq = lane_ptr(dq, o);
    loss_out = lane_ptr(loss_out, o), logp_mean_out = lane_ptr(logp_mean_out, o);
  }
  const float a = *alpha;
  const float g = -1.0f / (float)(N * B);
  for (int e = threadIdx.x; e < N * B; e += blockDim.x) dq[e] = g;
  double acc = 0.0, acc_lp = 0.0;
  for (int i = threadIdx.x; i < B; i += blockDim.x) {
    float s = 0.f;
    for (int k = 0; k < N; ++k) s += q[(size_t)k * q_stride + i];
    const float lp = logp[i];
    acc += (double)(a * lp - s / (float)N);
    acc_lp += (double)lp;
  }
  block_mean(acc, B, loss_out, red);
  block_mean(acc_lp, B, logp_mean_out, red_lp);
}

// sac_squash_backward_kernel with dA = the sum of the N critics' action-column input gradients in index order (member
// k's input gradient at dx + k dx_stride, row stride ldx); the rest of the arithmetic is that kernel's
template <bool LANES>
__global__ void redq_squash_backward_kernel(const float* out, const float* eps, const float* dx, int dx_stride, int N,
                                            int ldx, int B, int A, float lmin, float lmax, float limit,
                                            const float* alpha, float* dout, size_t lane_stride) {
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    out = lane_ptr(out, o), eps = lane_ptr(eps, o), dx = lane_ptr(dx, o), alpha = lane_ptr(alpha, o);
    dout = lane_ptr(dout, o);
  }
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * A) return;
  const int r = i / A, j = i - r * A;
  const float c = *alpha / (float)B;
  const float mu = out[(size_t)r * 2 * A + j], raw = out[(size_t)r * 2 * A + A + j];
  const float sigma = expf(fminf(fmaxf(raw, lmin), lmax));
  const float e = eps[(size_t)r * A + j];
  const float u = __fadd_rn(mu, __fmul_rn(sigma, e));
  const float t = tanhf(u);
  float dA = dx[(size_t)r * ldx + j];
  for (int k = 1; k < N; ++k) dA = dA + dx[(size_t)k * dx_stride + (size_t)r * ldx + j];
  const float gu = dA * limit * (1.f - t * t) + 2.f * c * t;
  dout[(size_t)r * 2 * A + j] = gu;
  dout[(size_t)r * 2 * A + A + j] = (raw >= lmin && raw <= lmax) ? gu * sigma * e - c : 0.f;
}

// ---------------------------------------------------------------------------------------------------------------
// EDAC / SAC-N (algo = 11; An, Moon, Kim & Song 2021): REDQ's ensemble with M = N, a policy step every step on the min
// over all N critics, and (eta > 0) a penalty eta D that pushes the critics' action gradients g_k = dQ_k / da apart.  D's
// parameter gradient is taken without autograd: with ReLU hidden layers the masks are fixed, and for u_k = d(eta D) /
// d g_k held fixed it is the gradient of the directional derivative g_k . u_k, which the existing GEMM modes give:
//   ones-backward (MODE 1 from dOut = 1; the first layer on its action columns only) -> g_k
//   edac_diversity_kernel                                                             -> u_k, D
//   tangent forward (MODE 4: h'_1 = act'(h_1) (.) u W_1a^T, h'_l = act'(h_l) (.) h'_{l-1} W_l^T)
//   weight gradients (MODE 2 without dbias: dW_1[:, act] = sum_b d_1 u^T, dW_l = sum_b d_l h'_{l-1}^T)
// with d_l the ones-backward's gated input gradients.  The bias and obs-column gradients of D are exactly 0.
// ---------------------------------------------------------------------------------------------------------------
constexpr int EDAC_THREADS = 1024;  // one CTA per learner, one warp per row at a time, lane k = critic k
constexpr double EDAC_NORM_EPS = 1e-10;

// The diversity head of one learner.  g: member k's action gradients [B][A] at g + k B A (u likewise).  Per row b, with
// n_k = |g_k|, gh_k = g_k / (n_k + 1e-10) and S = sum_k gh_k: v_k = c (S - gh_k), c = 2 eta / (B (N - 1)), and
// u_k = v_k / (n_k + 1e-10) - g_k (g_k . v_k) / (n_k (n_k + 1e-10)^2) (the second term 0 at n_k = 0, as torch's norm
// backward).  *div_out = D = sum_b sum_{i != j} gh_i . gh_j / (B (N - 1)).  Arithmetic in double; the sums over the
// critics are warp shuffle trees (every lane gets the same bits), the rows' sums block_mean's fixed order.
template <bool LANES>
__global__ void __launch_bounds__(EDAC_THREADS) edac_diversity_kernel(const float* g, int N, int B, int A, double c,
                                                                      float* u, float* div_out, size_t lane_stride) {
  __shared__ double red[32];
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    g = lane_ptr(g, o), u = lane_ptr(u, o), div_out = lane_ptr(div_out, o);
  }
  const int lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  const bool on = lane < N;
  const size_t mo = (size_t)(on ? lane : 0) * B * A;
  double acc = 0.0;
  for (int b = threadIdx.x >> 5; b < B; b += nw) {  // warp-uniform
    const float* gr = g + mo + (size_t)b * A;
    double nn = 0.0;
    for (int j = 0; on && j < A; ++j) nn += (double)gr[j] * (double)gr[j];
    const double n = sqrt(nn), inv = 1.0 / (n + EDAC_NORM_EPS);
    double dot = 0.0, drow = 0.0;
    for (int j = 0; j < A; ++j) {
      const double gj = on ? (double)gr[j] : 0.0, gh = gj * inv, s = warp_sum(gh);
      dot += gj * (c * (s - gh));
      drow += gh * (s - gh);
    }
    const double corr = n > 0.0 ? dot / (n * (n + EDAC_NORM_EPS) * (n + EDAC_NORM_EPS)) : 0.0;
    for (int j = 0; j < A; ++j) {
      const double gj = on ? (double)gr[j] : 0.0, gh = gj * inv, s = warp_sum(gh);
      if (on) u[mo + (size_t)b * A + j] = (float)(c * (s - gh) * inv - gj * corr);
    }
    drow = warp_sum(drow);
    if (lane == 0) acc += drow;
  }
  block_mean(acc, B * (N - 1), div_out, red);
}

// One CTA: the policy step's head at a = pi(s) on the N critics just updated (member k's output at q + k q_stride).  Per
// row the loss is alpha log pi - min_k q_k (the first critic that attains the min, in index order; a NaN loses to a
// number, as fminf); *loss_out = its mean, *logp_mean_out = mean log pi (summed as redq_policy_loss_kernel sums them);
// dq_k[i] (member k's at dq + k B) is -1 / B on row i's argmin critic and 0 on the others.
template <bool LANES>
__global__ void __launch_bounds__(GTHREADS) edac_policy_loss_kernel(const float* q, int q_stride, int N,
                                                                   const float* logp, const float* alpha, int B,
                                                                   float* dq, float* loss_out, float* logp_mean_out,
                                                                   size_t lane_stride) {
  __shared__ double red[32], red_lp[32];
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    q = lane_ptr(q, o), logp = lane_ptr(logp, o), alpha = lane_ptr(alpha, o), dq = lane_ptr(dq, o);
    loss_out = lane_ptr(loss_out, o), logp_mean_out = lane_ptr(logp_mean_out, o);
  }
  const float a = *alpha;
  const float g = -1.0f / (float)B;
  double acc = 0.0, acc_lp = 0.0;
  for (int i = threadIdx.x; i < B; i += blockDim.x) {
    float m = q[i];
    int km = 0;
    for (int k = 1; k < N; ++k) {
      const float v = q[(size_t)k * q_stride + i];
      if (v < m || (m != m && v == v)) m = v, km = k;
    }
    for (int k = 0; k < N; ++k) dq[(size_t)k * B + i] = k == km ? g : 0.f;
    const float lp = logp[i];
    acc += (double)(a * lp - m);
    acc_lp += (double)lp;
  }
  block_mean(acc, B, loss_out, red);
  block_mean(acc_lp, B, logp_mean_out, red_lp);
}

// ---------------------------------------------------------------------------------------------------------------
// Discrete SAC (algo = 5; Christodoulou 2019).  The policy network maps obs -> [n] logits, both critics and their
// targets obs -> [n] Q-values; the action column holds the action index as float32.  Every expectation over actions
// is exact: no noise, no squash head, and no gradient through the critics into the policy.
// ---------------------------------------------------------------------------------------------------------------
// log_softmax of one row's n logits x: log pi_j = (x_j - m) - ls with m = max_j x_j and ls = log(sum_j exp(x_j - m)),
// the sum in index order (c51_expected's arithmetic); returns ls and sets m.  pi_j = exp(log pi_j), so a vanishing
// probability gives pi log pi = 0, never 0 * -inf.
__device__ __forceinline__ float dsac_log_norm(const float* x, int n, float& m) {
  m = x[0];
  for (int j = 1; j < n; ++j) m = fmaxf(m, x[j]);
  float s = 0.f;
  for (int j = 0; j < n; ++j) s += expf(x[j] - m);
  return logf(s);
}

// One CTA per critic (each critic's launch on its own stream): per row i with action a = act[i],
//   V(s') = sum_j pi'_j (min(Q1targ, Q2targ)(s')_j - alpha log pi'_j) from the policy's logits at s' (index order),
//   y = r + gamma (1 - d) V(s'), loss = mean((Q(s)[a] - y)^2),
//   dOut[i, :] = 0 except dOut[i, a] = 2 (Q(s)[a] - y) / B, q_copy[i] = Q(s)[a] (the logged Q-value).
// A row whose action is not an integer in [0, n) is never used as an index: it adds nothing to the loss or dOut, logs
// NaN, and is counted in *bad_out (when bad_out != NULL; both critics see the same actions, so one of them counts).
// The loss is summed as q_loss_kernel sums it, in a fixed order with no float atomics.
template <bool LANES>
__global__ void __launch_bounds__(GTHREADS) dsac_q_loss_kernel(const float* q, const float* logits_next,
                                                              const float* q1t, const float* q2t, const float* act,
                                                              const float* rew, const float* done, const float* alpha,
                                                              float gamma, int B, int n, float* dout, float* loss_out,
                                                              float* q_copy, int* bad_out, size_t lane_stride) {
  __shared__ double red[32];
  __shared__ int bad_rows;
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    q = lane_ptr(q, o), logits_next = lane_ptr(logits_next, o), q1t = lane_ptr(q1t, o), q2t = lane_ptr(q2t, o);
    act = lane_ptr(act, o), rew = lane_ptr(rew, o), done = lane_ptr(done, o), alpha = lane_ptr(alpha, o);
    dout = lane_ptr(dout, o), loss_out = lane_ptr(loss_out, o), q_copy = lane_ptr(q_copy, o);
    bad_out = lane_ptr(bad_out, o);
  }
  if (threadIdx.x == 0) bad_rows = 0;
  __syncthreads();
  const float al = *alpha;
  const float inv = 1.0f / (float)B;
  double acc = 0.0;
  int bad = 0;
  for (int i = threadIdx.x; i < B; i += blockDim.x) {
    const float af = act[i];
    const bool valid = af >= 0.f && af < (float)n && af == floorf(af);  // false for NaN
    const int a = valid ? (int)af : -1;
    float g = 0.f;
    if (valid) {
      const float *x = logits_next + (size_t)i * n, *t1 = q1t + (size_t)i * n, *t2 = q2t + (size_t)i * n;
      float m;
      const float ls = dsac_log_norm(x, n, m);
      float v = 0.f;
      for (int j = 0; j < n; ++j) {
        const float lp = (x[j] - m) - ls;
        v += expf(lp) * (fminf(t1[j], t2[j]) - al * lp);
      }
      const float qi = q[(size_t)i * n + a];
      const float d = qi - (rew[i] + gamma * (1.f - done[i]) * v);
      acc += (double)d * (double)d;
      g = (2.f * d) * inv;
      q_copy[i] = qi;
    } else {
      q_copy[i] = __int_as_float(0x7fc00000);
      ++bad;
    }
    for (int j = 0; j < n; ++j) dout[(size_t)i * n + j] = j == a ? g : 0.f;
  }
  if (bad) atomicAdd(&bad_rows, bad);
  block_mean(acc, B, loss_out, red);  // its __syncthreads orders every thread's atomicAdd before thread 0 reads
  if (threadIdx.x == 0 && bad_out != nullptr) *bad_out = bad_rows;
}

// One CTA: the policy step's head.  Per row i, with pi from the logits x of the policy at s, m_j = min(Q1, Q2)(s)_j of
// the critics just updated and c_j = alpha log pi_j - m_j:
//   L_i = sum_j pi_j c_j, E_i = sum_j pi_j log pi_j (index order),
//   dOut[i, k] = pi_k (c_k - L_i) / B (the alpha term of d log pi cancels: sum_j pi_j = 1), ent[i] = E_i;
// *loss_out = mean L_i and *ent_mean_out = mean E_i, each summed as block_mean sums.  ent is what
// sac_alpha_step_kernel reads in place of log pi.
template <bool LANES>
__global__ void __launch_bounds__(GTHREADS) dsac_policy_loss_kernel(const float* logits, const float* q1,
                                                                   const float* q2, const float* alpha, int B, int n,
                                                                   float* dout, float* ent, float* loss_out,
                                                                   float* ent_mean_out, size_t lane_stride) {
  __shared__ double red[32], red_e[32];
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    logits = lane_ptr(logits, o), q1 = lane_ptr(q1, o), q2 = lane_ptr(q2, o), alpha = lane_ptr(alpha, o);
    dout = lane_ptr(dout, o), ent = lane_ptr(ent, o), loss_out = lane_ptr(loss_out, o);
    ent_mean_out = lane_ptr(ent_mean_out, o);
  }
  const float al = *alpha;
  const float inv = 1.0f / (float)B;
  double acc = 0.0, acc_e = 0.0;
  for (int i = threadIdx.x; i < B; i += blockDim.x) {
    const float *x = logits + (size_t)i * n, *a1 = q1 + (size_t)i * n, *a2 = q2 + (size_t)i * n;
    float m;
    const float ls = dsac_log_norm(x, n, m);
    float L = 0.f, E = 0.f;
    for (int j = 0; j < n; ++j) {
      const float lp = (x[j] - m) - ls, p = expf(lp);
      L += p * (al * lp - fminf(a1[j], a2[j]));
      E += p * lp;
    }
    for (int j = 0; j < n; ++j) {
      const float lp = (x[j] - m) - ls;
      dout[(size_t)i * n + j] = (expf(lp) * ((al * lp - fminf(a1[j], a2[j])) - L)) * inv;
    }
    ent[i] = E;
    acc += (double)L;
    acc_e += (double)E;
  }
  block_mean(acc, B, loss_out, red);
  block_mean(acc_e, B, ent_mean_out, red_e);
}

// ---------------------------------------------------------------------------------------------------------------
// DQN (algo = 2; Mnih et al. 2015, Double DQN: van Hasselt et al. 2016).  The Q network maps obs -> [n] values; the
// action column holds the action index as float32.
// ---------------------------------------------------------------------------------------------------------------
// index of the largest of q[0..n) as torch.argmax takes it: a NaN wins (the first NaN), ties go to the first index
__device__ __forceinline__ int argmax_row(const float* q, int n) {
  int best = 0;
  float bv = q[0];
  for (int j = 1; j < n && !isnan(bv); ++j) {
    const float v = q[j];
    if (isnan(v) || v > bv) bv = v, best = j;
  }
  return best;
}

// One CTA: per row i with action a = act[i]
//   v = Q_targ(s')[i, argmax_j Q(s')[i, j]] (Double DQN: qn != NULL) or max_j Q_targ(s')[i, j],
//   y = r + gamma (1 - d) v (td_target's order), delta = Q(s)[i, a] - y,
//   loss = mean(0.5 delta^2 if |delta| < 1 else |delta| - 0.5)  (F.smooth_l1_loss, beta = 1),
//   dOut[i, :] = 0 except dOut[i, a] = clamp(delta, -1, 1) / B, q_copy[i] = Q(s)[i, a] (the logged Q-value).
// A row whose action is not an integer in [0, n) is never used as an index: it adds nothing to the loss or dOut, logs
// NaN, and is counted in *bad_out (0 when every action is valid).
// WEIGHTED (prioritized replay): row i's loss and gradient are scaled by w[i] -- loss = (1/B) sum_i w_i huber(delta_i),
// dOut[i, a] = w_i clamp(delta_i, -1, 1) / B -- and absd[i] = |delta_i| (-1 for a row with an invalid action).  With
// every w_i = 1 both are bit for bit those of the unweighted head: the products by 1 are exact.
// NSTEP (n-step returns): row i's discount is disc[i] (gamma^k of its window) in place of gamma.
// Each flag's operands are read only by the instantiations that set it.
template <bool LANES, bool WEIGHTED, bool NSTEP>
__global__ void __launch_bounds__(GTHREADS) dqn_loss_kernel(const float* q, const float* qt_next, const float* qn,
                                                           const float* act, const float* rew, const float* done,
                                                           const float* disc, float gamma, int B, int n, float* dout,
                                                           float* loss_out, float* q_copy, int* bad_out, const float* w,
                                                           float* absd, size_t lane_stride) {
  __shared__ double red[32];
  __shared__ int bad_rows;
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    q = lane_ptr(q, o), qt_next = lane_ptr(qt_next, o), qn = lane_ptr(qn, o), act = lane_ptr(act, o);
    rew = lane_ptr(rew, o), done = lane_ptr(done, o), dout = lane_ptr(dout, o), loss_out = lane_ptr(loss_out, o);
    q_copy = lane_ptr(q_copy, o), bad_out = lane_ptr(bad_out, o);
    if (WEIGHTED) w = lane_ptr(w, o), absd = lane_ptr(absd, o);
    if (NSTEP) disc = lane_ptr(disc, o);
  }
  if (threadIdx.x == 0) bad_rows = 0;
  __syncthreads();
  const float inv = 1.0f / (float)B;
  double acc = 0.0;
  int bad = 0;
  for (int i = threadIdx.x; i < B; i += blockDim.x) {
    const float af = act[i];
    const bool valid = af >= 0.f && af < (float)n && af == floorf(af);  // false for NaN
    const int a = valid ? (int)af : -1;
    float g = 0.f;
    if (valid) {
      const float* tn = qt_next + (size_t)i * n;
      const float v = qn != nullptr ? tn[argmax_row(qn + (size_t)i * n, n)] : tn[argmax_row(tn, n)];
      const float qi = q[(size_t)i * n + a];
      const float d = qi - td_target(rew[i], done[i], v, nullptr, i, NSTEP ? disc[i] : gamma);
      const float ad = fabsf(d);
      const double hub = ad < 1.f ? 0.5 * (double)d * (double)d : (double)ad - 0.5;
      const float c = d > 1.f ? 1.f : (d < -1.f ? -1.f : d);  // NaN passes through, as torch's clamp lets it
      if (WEIGHTED) {
        const float wi = w[i];
        acc += (double)wi * hub;
        g = (wi * c) * inv;
        absd[i] = ad;
      } else {
        acc += hub;
        g = c * inv;
      }
      q_copy[i] = qi;
    } else {
      q_copy[i] = __int_as_float(0x7fc00000);
      if (WEIGHTED) absd[i] = -1.f;
      ++bad;
    }
    for (int j = 0; j < n; ++j) dout[(size_t)i * n + j] = j == a ? g : 0.f;
  }
  if (bad) atomicAdd(&bad_rows, bad);
  block_mean(acc, B, loss_out, red);  // its __syncthreads orders every thread's atomicAdd before thread 0 reads
  if (threadIdx.x == 0) *bad_out = bad_rows;
}

// target <- param on the steps the copy table marks (flags[idx].x != 0): the graph launches the copy every step and
// the host decides per learner, from its Q optimizer's step count, which steps it takes effect on
template <bool LANES>
__global__ void dqn_target_copy_kernel(float* target, const float* param, int n, const float2* flags, int idx,
                                       size_t lane_stride) {
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    target = lane_ptr(target, o), param = lane_ptr(param, o), flags = lane_ptr(flags, o);
  }
  if (flags[idx].x == 0.f) return;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) target[i] = param[i];
}

// ---------------------------------------------------------------------------------------------------------------
// Dueling Q networks (config dueling_k = K; Wang et al. 2016, eq. 9, per output column): the value stream's V [B, K] and
// the advantage stream's A [B, n K] sit side by side in va [B, K + n K] (row b = [V_b | A_b], action a owning A's
// columns a K .. a K + K - 1).  One thread per (row, column i < K); both sums run over the actions in index order.
//   forward   mean_i = (sum_a A[a, i]) / n,  Q[a, i] = V[i] + (A[a, i] - mean_i)          -> q [B, n K]
//   backward  s_i = sum_a dQ[a, i],  dV[i] = s_i,  dA[a, i] = dQ[a, i] - s_i / n            -> dva [B, K + n K]
template <bool LANES>
__global__ void __launch_bounds__(GTHREADS) dueling_forward_kernel(const float* va, int B, int n, int k, float* q,
                                                                  size_t lane_stride) {
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    va = lane_ptr(va, o), q = lane_ptr(q, o);
  }
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= B * k) return;
  const int b = t / k, i = t - b * k;
  const float* v = va + (size_t)b * (k + n * k);
  const float* a = v + k + i;
  float s = 0.f;
  for (int j = 0; j < n; ++j) s += a[(size_t)j * k];
  const float mean = s / (float)n, vi = v[i];
  float* out = q + (size_t)b * n * k + i;
  for (int j = 0; j < n; ++j) out[(size_t)j * k] = vi + (a[(size_t)j * k] - mean);
}

template <bool LANES>
__global__ void __launch_bounds__(GTHREADS) dueling_backward_kernel(const float* dq, int B, int n, int k, float* dva,
                                                                   size_t lane_stride) {
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    dq = lane_ptr(dq, o), dva = lane_ptr(dva, o);
  }
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= B * k) return;
  const int b = t / k, i = t - b * k;
  const float* g = dq + (size_t)b * n * k + i;
  float s = 0.f;
  for (int j = 0; j < n; ++j) s += g[(size_t)j * k];
  const float mean = s / (float)n;
  float* dv = dva + (size_t)b * (k + n * k);
  dv[i] = s;
  float* da = dv + k + i;
  for (int j = 0; j < n; ++j) da[(size_t)j * k] = g[(size_t)j * k] - mean;
}

// ---------------------------------------------------------------------------------------------------------------
// Noisy networks (config noisy_layers; Fortunato et al. 2018, factorized Gaussian noise).  A noisy layer's
// parameters are W_mu, W_sigma [out, in], b_mu, b_sigma [out] in the noisy vector; per draw eps_in [in], eps_out [out]
// ~ N(0, 1), f(x) = copysign(sqrt(|x|), x), e_ij = f(eps_out_i) f(eps_in_j), and the composed layer the GEMMs read is
// W = W_mu + W_sigma e, b = b_mu + b_sigma f(eps_out), every product and sum rounded on its own.  A plain layer of the
// network is copied.  The work is cut into tiles of up to NOISY_TR rows x NOISY_TC columns of one layer's W (the tiles
// of the first column also take the rows' biases): one CTA each, in layer order.
constexpr int NOISY_MAX_LAYERS = 5;  // a dueling network's five Linear layers
constexpr int NOISY_TR = 32, NOISY_TC = 256;

struct NoisyLayout {
  int n;          // Linear layers in flat order
  unsigned mask;  // bit l: layer l is noisy
  int in[NOISY_MAX_LAYERS], out[NOISY_MAX_LAYERS];
  int cw[NOISY_MAX_LAYERS], cb[NOISY_MAX_LAYERS];  // W and b in the composed (plain-layout) vector
  int fw[NOISY_MAX_LAYERS], fb[NOISY_MAX_LAYERS];  // W (W_mu, then W_sigma) and b (b_mu, then b_sigma) in the noisy vector
  int eo[NOISY_MAX_LAYERS];                        // eps_in of a noisy layer in the draw vector; eps_out follows it
  int E;                                           // draws per network: the sum of in + out over the noisy layers
  int tiles[NOISY_MAX_LAYERS + 1];                 // first tile of each layer; tiles[n] = all tiles
};

__device__ __forceinline__ float noisy_f(float x) { return copysignf(sqrtf(fabsf(x)), x); }

// draw k of network r (0 online, 1 target) at step st: element k % 4 of the Box-Muller block k / 4, Philox counter
// (k / 4, st, call, 0xA00 | r) under key seed
__device__ __forceinline__ float noisy_draw(int k, int st, int r, unsigned long long seed, unsigned long long call) {
  const uint4 c = philox4x32_10(make_uint4((unsigned)(k >> 2), (unsigned)st, (unsigned)call, 0xA00u | (unsigned)r),
                                make_uint2((unsigned)seed, (unsigned)(seed >> 32)));
  float z[4];
  box_muller4(c, z);
  const int j = k & 3;  // selected, not indexed: z stays in registers
  return j == 0 ? z[0] : j == 1 ? z[1] : j == 2 ? z[2] : z[3];
}

// The tile of CTA `bid`: its layer l, first row r0 and column c0, rows nr and columns nc
__device__ __forceinline__ int noisy_tile(const NoisyLayout& lay, int bid, int& r0, int& c0, int& nr, int& nc) {
  int l = 0;
  while (bid >= lay.tiles[l + 1]) ++l;
  const int ct = (lay.in[l] + NOISY_TC - 1) / NOISY_TC, t = bid - lay.tiles[l];
  r0 = (t / ct) * NOISY_TR, c0 = (t % ct) * NOISY_TC;
  nr = min(NOISY_TR, lay.out[l] - r0), nc = min(NOISY_TC, lay.in[l] - c0);
  return l;
}

// One launch per step for both networks (blockIdx.y = r: 0 composes the online network from flat_q into comp_q, 1 the
// target from flat_t into comp_t), each from its own draw.  The tile's f(eps_in) and f(eps_out) are drawn into shared
// memory; the CTAs past the tiles write the network's E raw draws, one Box-Muller block per thread, to draws[r * E ..]
// (the step's slice of the call's [S, 2, E] record, which noisy_expand_kernel and b200rl_offpolicy_get_noisy_draws
// read).  keys = the learner's (seed, call).
template <bool LANES>
__global__ void __launch_bounds__(GTHREADS) noisy_compose_kernel(const NoisyLayout lay, const float* flat_q,
                                                                const float* flat_t, float* comp_q, float* comp_t,
                                                                const unsigned long long* keys, int st, float* draws,
                                                                size_t lane_stride) {
  __shared__ float fi[NOISY_TC], fo[NOISY_TR];
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    flat_q = lane_ptr(flat_q, o), flat_t = lane_ptr(flat_t, o), comp_q = lane_ptr(comp_q, o);
    comp_t = lane_ptr(comp_t, o), keys = lane_ptr(keys, o), draws = lane_ptr(draws, o);
  }
  const int r = blockIdx.y;
  const float* flat = r ? flat_t : flat_q;
  float* comp = r ? comp_t : comp_q;
  const unsigned long long seed = keys[0], call = keys[1];
  if ((int)blockIdx.x >= lay.tiles[lay.n]) {
    const int t = ((int)blockIdx.x - lay.tiles[lay.n]) * blockDim.x + threadIdx.x;
    if (4 * t >= lay.E) return;
    const uint4 c = philox4x32_10(make_uint4((unsigned)t, (unsigned)st, (unsigned)call, 0xA00u | (unsigned)r),
                                  make_uint2((unsigned)seed, (unsigned)(seed >> 32)));
    float z[4];
    box_muller4(c, z);
    float* d = draws + ((size_t)st * 2 + r) * lay.E + 4 * t;
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (4 * t + j < lay.E) d[j] = z[j];
    return;
  }
  int r0, c0, nr, nc;
  const int l = noisy_tile(lay, blockIdx.x, r0, c0, nr, nc);
  const int in = lay.in[l], out = lay.out[l];
  const float* W = flat + lay.fw[l];
  const float* b = flat + lay.fb[l];
  float* cW = comp + lay.cw[l];
  float* cb = comp + lay.cb[l];
  if (!((lay.mask >> l) & 1u)) {  // a plain layer: copied
    for (int i = threadIdx.x; i < nr * nc; i += blockDim.x) {
      const size_t at = (size_t)(r0 + i / nc) * in + c0 + i % nc;
      cW[at] = W[at];
    }
    if (c0 == 0)
      for (int i = threadIdx.x; i < nr; i += blockDim.x) cb[r0 + i] = b[r0 + i];
    return;
  }
  for (int j = threadIdx.x; j < nc; j += blockDim.x) fi[j] = noisy_f(noisy_draw(lay.eo[l] + c0 + j, st, r, seed, call));
  for (int i = threadIdx.x; i < nr; i += blockDim.x)
    fo[i] = noisy_f(noisy_draw(lay.eo[l] + in + r0 + i, st, r, seed, call));
  __syncthreads();
  const float* Ws = W + (size_t)out * in;
  for (int i = threadIdx.x; i < nr * nc; i += blockDim.x) {
    const int ri = i / nc, cj = i - ri * nc;
    const size_t at = (size_t)(r0 + ri) * in + c0 + cj;
    cW[at] = __fadd_rn(W[at], __fmul_rn(Ws[at], __fmul_rn(fo[ri], fi[cj])));
  }
  if (c0 == 0)
    for (int i = threadIdx.x; i < nr; i += blockDim.x) cb[r0 + i] = __fadd_rn(b[r0 + i], __fmul_rn(b[out + r0 + i], fo[i]));
}

// After the backward pass: the composed layer's gradient (dW, db in grad, plain layout) -> the noisy vector's
// (ngrad): dW_mu = dW, dW_sigma = dW e, db_mu = db, db_sigma = db f(eps_out), with e recomputed from the online
// network's raw draws of step st as noisy_compose_kernel rounded it; a plain layer's gradient is copied.
template <bool LANES>
__global__ void __launch_bounds__(GTHREADS) noisy_expand_kernel(const NoisyLayout lay, const float* grad,
                                                               const float* draws, int st, float* ngrad,
                                                               size_t lane_stride) {
  __shared__ float fi[NOISY_TC], fo[NOISY_TR];
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    grad = lane_ptr(grad, o), draws = lane_ptr(draws, o), ngrad = lane_ptr(ngrad, o);
  }
  int r0, c0, nr, nc;
  const int l = noisy_tile(lay, blockIdx.x, r0, c0, nr, nc);
  const int in = lay.in[l], out = lay.out[l];
  const float* dW = grad + lay.cw[l];
  const float* db = grad + lay.cb[l];
  float* gW = ngrad + lay.fw[l];
  float* gb = ngrad + lay.fb[l];
  if (!((lay.mask >> l) & 1u)) {
    for (int i = threadIdx.x; i < nr * nc; i += blockDim.x) {
      const size_t at = (size_t)(r0 + i / nc) * in + c0 + i % nc;
      gW[at] = dW[at];
    }
    if (c0 == 0)
      for (int i = threadIdx.x; i < nr; i += blockDim.x) gb[r0 + i] = db[r0 + i];
    return;
  }
  const float* d = draws + (size_t)st * 2 * lay.E + lay.eo[l];
  for (int j = threadIdx.x; j < nc; j += blockDim.x) fi[j] = noisy_f(d[c0 + j]);
  for (int i = threadIdx.x; i < nr; i += blockDim.x) fo[i] = noisy_f(d[in + r0 + i]);
  __syncthreads();
  float* gWs = gW + (size_t)out * in;
  for (int i = threadIdx.x; i < nr * nc; i += blockDim.x) {
    const int ri = i / nc, cj = i - ri * nc;
    const size_t at = (size_t)(r0 + ri) * in + c0 + cj;
    const float g = dW[at];
    gW[at] = g;
    gWs[at] = __fmul_rn(g, __fmul_rn(fo[ri], fi[cj]));
  }
  if (c0 == 0)
    for (int i = threadIdx.x; i < nr; i += blockDim.x) {
      const float g = db[r0 + i];
      gb[r0 + i] = g;
      gb[out + r0 + i] = __fmul_rn(g, fo[i]);
    }
}

// ---------------------------------------------------------------------------------------------------------------
// C51 (algo = 3; Bellemare, Dabney & Munos 2017): DQN's step program with a categorical head.  The Q network maps obs
// -> [n * N] logits, action a owning columns a*N .. a*N + N - 1; p(s, a) = softmax over them, Q(s, a) = sum_i z_i p_i.
// ---------------------------------------------------------------------------------------------------------------
constexpr int C51_MAX_ATOMS = 256, C51_WARPS = 8;
constexpr int C51_SMEM_FLOATS = 48 * 1024 / 4;  // the dynamic shared memory of one CTA without an opt-in

// warps per CTA of the head at n actions x N atoms: each warp holds 3N + n floats, the CTA the support (N floats)
__host__ __device__ __forceinline__ int c51_warps(int n, int N) {
  const int w = (C51_SMEM_FLOATS - N) / (3 * N + n);
  return w < C51_WARPS ? w : C51_WARPS;
}

// sum_j z_j p_j of one action's N logits x, p = exp(x - max - log(sum exp(x - max))); every sum in index order
__device__ __forceinline__ float c51_expected(const float* x, const float* z, int N) {
  float m = x[0];
  for (int j = 1; j < N; ++j) m = fmaxf(m, x[j]);
  float s = 0.f;
  for (int j = 0; j < N; ++j) s += expf(x[j] - m);
  const float ls = logf(s);
  float e = 0.f;
  for (int j = 0; j < N; ++j) e += z[j] * expf((x[j] - m) - ls);
  return e;
}

// The warp's log_softmax of one action's N logits x (lane l: atoms l, l + 32, ...): logp[k] for atom lane + 32k, and
// p = exp(logp) in sp[0..N).  The same arithmetic as c51_expected: the max is exact in any order, the sum runs in index
// order (every lane adds up sp itself).
__device__ __forceinline__ void c51_warp_log_softmax(const float* x, int N, float* sp, float (&logp)[C51_MAX_ATOMS / 32]) {
  const int lane = threadIdx.x & 31;
  float m = -INFINITY;
#pragma unroll
  for (int k = 0; k < C51_MAX_ATOMS / 32; ++k)
    if (lane + 32 * k < N) m = fmaxf(m, x[lane + 32 * k]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
#pragma unroll
  for (int k = 0; k < C51_MAX_ATOMS / 32; ++k)
    if (lane + 32 * k < N) {
      logp[k] = x[lane + 32 * k] - m;
      sp[lane + 32 * k] = expf(logp[k]);
    }
  __syncwarp();
  float s = 0.f;
  for (int j = 0; j < N; ++j) s += sp[j];
  const float ls = logf(s);
  __syncwarp();
#pragma unroll
  for (int k = 0; k < C51_MAX_ATOMS / 32; ++k)
    if (lane + 32 * k < N) {
      logp[k] -= ls;
      sp[lane + 32 * k] = expf(logp[k]);
    }
  __syncwarp();
}

// One warp per row i with action a = act[i] (a grid of ceil(B / warps) CTAs per learner):
//   a* = argmax_j Q(s')_j over the expected values of qn (Double DQN: qn != NULL) or of qt_next (argmax_row's rule),
//   Tz_j = clamp(r + gamma (1 - d) z_j, v_min, v_max), b_j = (Tz_j - v_min) / dz,
//   m_i = sum_j max(0, 1 - |b_j - i|) p_j(s', a*) from Q_targ(s'), L_i = -sum_i m_i log p_i(s, a),
//   dOut[i, a*N + k] = (p_k(s, a) sum m - m_k) * (1 / B) and 0 elsewhere, q_copy[i] = Q(s, a) (the logged Q-value).
// A row whose action is not an integer in [0, n) is never used as an index: its dOut row is 0, its loss 0, q_copy NaN,
// and it is counted.  The last CTA of a learner to finish (sync[0] counts them) writes *loss_out = mean L, summed in
// double as block_mean sums, and *bad_out = the invalid rows (sync[1]), and leaves both counters at 0 for the next
// launch.  No atomics touch a float: the head is deterministic.
// act == NULL (D4PG's critic over [s | a], n = 1): every row's action is index 0 and a* = 0; no row is invalid.
// WEIGHTED (prioritized replay, D4PG engines): row i's loss and gradient are scaled by w[i], and absd[i] = KL_i =
// L_i + sum_j m_j log m_j (0 log 0 = 0, summed in index order; a rounding-level negative KL is raised to 0, a NaN
// passes), the base of its priority (-1 for a row with an invalid action).  With every w_i = 1 loss and gradient are
// bit for bit those of the unweighted head: the products by 1 are exact.
// NSTEP (n-step returns): row i's discount is disc[i] (gamma^k of its window) in place of gamma (unread otherwise).
// Each flag's operands are read only by the instantiations that set it.
template <bool LANES, bool WEIGHTED, bool NSTEP>
__global__ void __launch_bounds__(C51_WARPS * 32) c51_loss_kernel(
    const float* q, const float* qt_next, const float* qn, const float* act, const float* rew, const float* done,
    const float* disc, const float* support, float gamma, float v_min, float v_max, float dz, int B, int n, int N,
    float* dout, float* row_loss, float* q_copy, int* sync, float* loss_out, int* bad_out, const float* w, float* absd,
    size_t lane_stride) {
  extern __shared__ float c51_smem[];
  __shared__ double red[32];
  __shared__ bool last;
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    q = lane_ptr(q, o), qt_next = lane_ptr(qt_next, o), qn = lane_ptr(qn, o), act = lane_ptr(act, o);
    rew = lane_ptr(rew, o), done = lane_ptr(done, o), support = lane_ptr(support, o), dout = lane_ptr(dout, o);
    row_loss = lane_ptr(row_loss, o), q_copy = lane_ptr(q_copy, o), sync = lane_ptr(sync, o);
    loss_out = lane_ptr(loss_out, o), bad_out = lane_ptr(bad_out, o);
    if (WEIGHTED) w = lane_ptr(w, o), absd = lane_ptr(absd, o);
    if (NSTEP) disc = lane_ptr(disc, o);
  }
  const int nN = n * N, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float* z = c51_smem;
  for (int j = threadIdx.x; j < N; j += blockDim.x) z[j] = support[j];
  __syncthreads();
  float* sp = c51_smem + N + warp * (3 * N + n);  // p(s', a*), then p(s, a)
  float* sb = sp + N;                             // b_j, then m_i
  float* sx = sb + N;                             // log p(s, a)
  float* sq = sx + N;                             // expected values of Q(s') (argmax net)
  const int i = blockIdx.x * (blockDim.x >> 5) + warp;
  if (i < B) {
    const float af = act != nullptr ? act[i] : 0.f;
    const bool valid = af >= 0.f && af < (float)n && af == floorf(af);  // false for NaN
    const int a = valid ? (int)af : -1;
    float* drow = dout + (size_t)i * nN;
    for (int c = lane; c < nN; c += 32)
      if (c / N != a) drow[c] = 0.f;
    if (!valid) {
      if (lane == 0) {
        q_copy[i] = __int_as_float(0x7fc00000);
        row_loss[i] = 0.f;
        if (WEIGHTED) absd[i] = -1.f;
        atomicAdd(sync + 1, 1);
      }
    } else {
      int a_star = 0;  // D4PG (act == NULL): the one action
      if (act != nullptr) {
        // a*: the expected values of the argmax net, one lane per action, then argmax_row over them
        const float* an = (qn != nullptr ? qn : qt_next) + (size_t)i * nN;
        for (int j = lane; j < n; j += 32) sq[j] = c51_expected(an + (size_t)j * N, z, N);
        __syncwarp();
        a_star = argmax_row(sq, n);
      }
      float logp[C51_MAX_ATOMS / 32];
      c51_warp_log_softmax(qt_next + (size_t)i * nN + (size_t)a_star * N, N, sp, logp);
      const float g1d = (NSTEP ? disc[i] : gamma) * (1.f - done[i]), r = rew[i];
#pragma unroll
      for (int k = 0; k < C51_MAX_ATOMS / 32; ++k)
        if (lane + 32 * k < N) {
          float tz = r + g1d * z[lane + 32 * k];
          tz = tz < v_min ? v_min : (tz > v_max ? v_max : tz);  // NaN passes through, as torch's clamp lets it
          sb[lane + 32 * k] = (tz - v_min) / dz;
        }
      __syncwarp();
      float m[C51_MAX_ATOMS / 32];
#pragma unroll
      for (int k = 0; k < C51_MAX_ATOMS / 32; ++k)
        if (lane + 32 * k < N) {
          const float at = (float)(lane + 32 * k);
          float acc = 0.f;
          for (int j = 0; j < N; ++j) {
            float w = 1.f - fabsf(sb[j] - at);
            w = w < 0.f ? 0.f : w;
            acc += w * sp[j];
          }
          m[k] = acc;
        }
      __syncwarp();  // every lane is done with sp and sb
      c51_warp_log_softmax(q + (size_t)i * nN + (size_t)a * N, N, sp, logp);
#pragma unroll
      for (int k = 0; k < C51_MAX_ATOMS / 32; ++k)
        if (lane + 32 * k < N) sb[lane + 32 * k] = m[k], sx[lane + 32 * k] = logp[k];
      __syncwarp();
      float qv = 0.f, ce = 0.f, msum = 0.f, ment = 0.f;
      for (int j = 0; j < N; ++j) {
        qv += z[j] * sp[j];
        ce += sb[j] * sx[j];
        msum += sb[j];
        if (WEIGHTED) ment += sb[j] > 0.f ? sb[j] * logf(sb[j]) : 0.f;
      }
      const float inv = 1.0f / (float)B;  // dqn_loss_kernel's scaling
      const float wi = WEIGHTED ? w[i] : 1.f;
#pragma unroll
      for (int k = 0; k < C51_MAX_ATOMS / 32; ++k)
        if (lane + 32 * k < N) {
          const float g = sp[lane + 32 * k] * msum - m[k];
          drow[(size_t)a * N + lane + 32 * k] = (WEIGHTED ? wi * g : g) * inv;
        }
      if (lane == 0) {
        q_copy[i] = qv;
        row_loss[i] = WEIGHTED ? wi * -ce : -ce;
        if (WEIGHTED) {
          const float kl = -ce + ment;
          absd[i] = kl < 0.f ? 0.f : kl;  // NaN passes
        }
      }
    }
  }
  // the last CTA of this learner reads every row's loss
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(sync, 1) == (int)gridDim.x - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  double acc = 0.0;
  for (int r = threadIdx.x; r < B; r += blockDim.x) acc += (double)__ldcg(row_loss + r);
  block_mean(acc, B, loss_out, red);
  if (threadIdx.x == 0) {
    *bad_out = atomicExch(sync + 1, 0);
    sync[0] = 0;
  }
}

// D4PG's policy head (algo = 6): one warp per row i of the critic's N logits x at [s | mu(s)] (the grid and shared
// memory of c51_loss_kernel at n = 1): p = c51_warp_log_softmax's, Q = sum_j z_j p_j in index order,
//   dOut[i, k] = -(p_k (z_k - Q)) * (1 / B)   (the gradient of -(1/B) sum_i Q_i w.r.t. the logits), row_loss[i] = -Q.
// The last CTA of a learner to finish (sync[0] counts them) writes *loss_out = -mean Q, summed in double as
// c51_loss_kernel sums, and leaves the counter at 0.  No atomics touch a float.
template <bool LANES>
__global__ void __launch_bounds__(C51_WARPS * 32) d4pg_policy_loss_kernel(const float* q, const float* support, int B,
                                                                          int N, float* dout, float* row_loss, int* sync,
                                                                          float* loss_out, size_t lane_stride) {
  extern __shared__ float d4pg_smem[];
  __shared__ double red[32];
  __shared__ bool last;
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    q = lane_ptr(q, o), support = lane_ptr(support, o), dout = lane_ptr(dout, o), row_loss = lane_ptr(row_loss, o);
    sync = lane_ptr(sync, o), loss_out = lane_ptr(loss_out, o);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float* z = d4pg_smem;
  for (int j = threadIdx.x; j < N; j += blockDim.x) z[j] = support[j];
  __syncthreads();
  float* sp = d4pg_smem + N + warp * N;  // p(s, mu(s))
  const int i = blockIdx.x * (blockDim.x >> 5) + warp;
  if (i < B) {
    float logp[C51_MAX_ATOMS / 32];
    c51_warp_log_softmax(q + (size_t)i * N, N, sp, logp);
    float qv = 0.f;
    for (int j = 0; j < N; ++j) qv += z[j] * sp[j];
    const float inv = 1.0f / (float)B;
    float* drow = dout + (size_t)i * N;
#pragma unroll
    for (int k = 0; k < C51_MAX_ATOMS / 32; ++k)
      if (lane + 32 * k < N) drow[lane + 32 * k] = -(sp[lane + 32 * k] * (z[lane + 32 * k] - qv)) * inv;
    if (lane == 0) row_loss[i] = -qv;
  }
  // the last CTA of this learner reads every row's loss
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(sync, 1) == (int)gridDim.x - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  double acc = 0.0;
  for (int r = threadIdx.x; r < B; r += blockDim.x) acc += (double)__ldcg(row_loss + r);
  block_mean(acc, B, loss_out, red);
  if (threadIdx.x == 0) sync[0] = 0;
}

// ---------------------------------------------------------------------------------------------------------------
// QR-DQN (b200rl_offpolicy_set_qr; Dabney, Rowland, Bellemare & Munos 2018): a head of the DQN engine.  The Q network
// maps obs -> [n * N] quantile locations, action a owning columns a*N .. a*N + N - 1; Q(s, a) = their mean.
// ---------------------------------------------------------------------------------------------------------------
constexpr int QR_MAX_QUANTILES = 256;

// shared-memory floats of one row at n actions x N quantiles: T and the quantile losses, theta(s, a), the argmax
// net's means and its row
__host__ __device__ __forceinline__ int qr_smem_floats(int n, int N) { return 2 * N + n + n * N; }

// sum_k x[k] / N over one action's N quantiles (in shared memory), added in index order
__device__ __forceinline__ float qr_mean(const float* x, int N) {
  float s = 0.f;
#pragma unroll 8
  for (int k = 0; k < N; ++k) s += x[k];
  return s / (float)N;
}

// One CTA per row i with action a = act[i] (grid = B rows per learner), thread t owning quantile t (blockDim = N
// rounded up to whole warps): every row spreads its N^2 pairs over N threads, and each thread's sum over the target
// quantiles j runs in index order.  The sums in index order (the means, the row loss) read rows the CTA first copies to
// shared memory with coalesced loads.
//   a* = argmax_j Q(s')_j over the means of qn (Double DQN: qn != NULL) or of qt_next (argmax_row's rule),
//   T_j = r + gamma (1 - d) theta_j(s', a*) from Q_targ (C51's Tz order), u_tj = T_j - theta_t(s, a),
//   tau_t = (2t + 1) / (2N), k_tj = |tau_t - 1{u_tj < 0}|, h(u) = 0.5 u^2 if |u| < 1 else |u| - 0.5,
//   L = (1/N) sum_t sum_j k_tj h(u_tj)  (j, then t, in index order),
//   dOut[i, a*N + t] = -(sum_j k_tj clamp(u_tj, -1, 1)) / N * (1 / B) and 0 elsewhere, q_copy[i] = Q(s, a).
// A row whose action is not an integer in [0, n) is never used as an index: its dOut row is 0, its loss 0, q_copy NaN,
// and it is counted.  The last CTA of a learner to finish sums the row losses and reads and resets the counters as
// c51_loss_kernel does; no atomics touch a float.
// WEIGHTED (prioritized replay): row i's loss and gradient are scaled by w[i], and absd[i] = its unweighted L (-1 for
// a row with an invalid action), the base of its priority.  With every w_i = 1 both are bit for bit those of the
// unweighted head.  NSTEP: row i's discount is disc[i] in place of gamma.  Each flag's operands are read only by the
// instantiations that set it.
template <bool LANES, bool WEIGHTED, bool NSTEP>
__global__ void __launch_bounds__(QR_MAX_QUANTILES) qr_loss_kernel(
    const float* q, const float* qt_next, const float* qn, const float* act, const float* rew, const float* done,
    const float* disc, float gamma, int B, int n, int N, float* dout, float* row_loss, float* q_copy, int* sync,
    float* loss_out, int* bad_out, const float* w, float* absd, size_t lane_stride) {
  extern __shared__ float qr_smem[];
  __shared__ double red[32];
  __shared__ bool last;
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    q = lane_ptr(q, o), qt_next = lane_ptr(qt_next, o), qn = lane_ptr(qn, o), act = lane_ptr(act, o);
    rew = lane_ptr(rew, o), done = lane_ptr(done, o), dout = lane_ptr(dout, o), row_loss = lane_ptr(row_loss, o);
    q_copy = lane_ptr(q_copy, o), sync = lane_ptr(sync, o), loss_out = lane_ptr(loss_out, o);
    bad_out = lane_ptr(bad_out, o);
    if (WEIGHTED) w = lane_ptr(w, o), absd = lane_ptr(absd, o);
    if (NSTEP) disc = lane_ptr(disc, o);
  }
  const int nN = n * N, t = threadIdx.x, i = blockIdx.x;
  float* st = qr_smem;        // T_j, then each quantile's loss sum
  float* sth = st + N;        // theta(s, a)
  float* sq = sth + N;        // the means of the argmax net
  float* sa = sq + n;         // the argmax net's row
  const float af = act[i];
  const bool valid = af >= 0.f && af < (float)n && af == floorf(af);  // false for NaN
  const int a = valid ? (int)af : -1;
  float* drow = dout + (size_t)i * nN;
  for (int c = t; c < nN; c += blockDim.x)
    if (c / N != a) drow[c] = 0.f;
  if (!valid) {
    if (t == 0) {
      q_copy[i] = __int_as_float(0x7fc00000);
      row_loss[i] = 0.f;
      if (WEIGHTED) absd[i] = -1.f;
      atomicAdd(sync + 1, 1);
    }
  } else {
    const float* an = (qn != nullptr ? qn : qt_next) + (size_t)i * nN;
    for (int c = t; c < nN; c += blockDim.x) sa[c] = an[c];
    const float th = t < N ? q[(size_t)i * nN + (size_t)a * N + t] : 0.f;
    if (t < N) sth[t] = th;
    __syncthreads();
    for (int j = t; j < n; j += blockDim.x) sq[j] = qr_mean(sa + (size_t)j * N, N);
    __syncthreads();
    const int a_star = argmax_row(sq, n);
    const float g1d = (NSTEP ? disc[i] : gamma) * (1.f - done[i]), r = rew[i];
    const float* tq = qn != nullptr ? qt_next + (size_t)i * nN : sa;  // without Double DQN the argmax net is Q_targ
    if (t < N) st[t] = r + g1d * tq[(size_t)a_star * N + t];
    __syncthreads();
    float lsum = 0.f, gsum = 0.f;
    if (t < N) {
      const float tau = (float)(2 * t + 1) / (float)(2 * N);
      for (int j = 0; j < N; ++j) {
        const float u = st[j] - th;
        const float k = fabsf(tau - (u < 0.f ? 1.f : 0.f));
        const float au = fabsf(u);
        const float hu = au < 1.f ? 0.5f * u * u : au - 0.5f;
        const float c = u > 1.f ? 1.f : (u < -1.f ? -1.f : u);  // NaN passes through, as torch's clamp lets it
        lsum += k * hu;
        gsum += k * c;
      }
    }
    __syncthreads();  // every thread is done with T
    const float inv = 1.0f / (float)B;  // dqn_loss_kernel's scaling
    if (t < N) {
      st[t] = lsum;
      const float g = -gsum / (float)N;
      drow[(size_t)a * N + t] = (WEIGHTED ? w[i] * g : g) * inv;
    }
    __syncthreads();
    if (t == 0) {
      float L = 0.f, qv = 0.f;
#pragma unroll 8
      for (int k = 0; k < N; ++k) L += st[k], qv += sth[k];
      L /= (float)N;
      q_copy[i] = qv / (float)N;
      row_loss[i] = WEIGHTED ? w[i] * L : L;
      if (WEIGHTED) absd[i] = L;
    }
  }
  // the last CTA of this learner reads every row's loss
  __threadfence();
  __syncthreads();
  if (t == 0) last = atomicAdd(sync, 1) == (int)gridDim.x - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  double acc = 0.0;
  for (int r = t; r < B; r += blockDim.x) acc += (double)__ldcg(row_loss + r);
  block_mean(acc, B, loss_out, red);
  if (t == 0) {
    *bad_out = atomicExch(sync + 1, 0);
    sync[0] = 0;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// IQN (algo = 4; Dabney, Ostrovski, Silver & Munos 2018): DQN's step program over an implicit quantile network.  Every
// minibatch row fans out into one network row per sampled fraction tau: Z(s, tau) = head(psi(s) * phi(cos(pi i tau))),
// psi and the head plain GEMM layers, phi a GEMM layer over the fraction's cosine features (b200rl.h, "IQN").
// ---------------------------------------------------------------------------------------------------------------
constexpr int IQN_MAX = 256;  // the largest n_cos, N, N' and K

// The activations of one IQN forward pass on B rows with M fractions each (R = B M network rows)
struct IqnPass {
  float* psi;  // [B, d]
  float* phi;  // [R, d]
  float* z;    // [R, d]  psi(s) * phi(tau)
  float* hid;  // [R, h]
  float* out;  // [R, n]  Z(s, tau)
};

// Draw t of step st (t = b (N + N' + K) + j for row b's j-th fraction): lane t % 4 of Philox4x32-10(counter
// (t / 4, st, call, 0xB00), key seed) = r, and tau = (2 (r >> 9) + 1) 2^-24, an odd multiple of 2^-24 in (0, 1)
__device__ __forceinline__ float iqn_tau(long long t, int st, unsigned long long seed, unsigned long long call) {
  const uint4 c = philox4x32_10(make_uint4((unsigned)(t >> 2), (unsigned)st, (unsigned)call, 0xB00u),
                                make_uint2((unsigned)seed, (unsigned)(seed >> 32)));
  const int j = (int)(t & 3);  // selected, not indexed: c stays in registers
  const unsigned r = j == 0 ? c.x : j == 1 ? c.y : j == 2 ? c.z : c.w;
  return (float)(2u * (r >> 9) + 1u) * 5.9604644775390625e-8f;
}

// One thread per (draw t, feature i) of step st over the B rows' Mt = N + N' + K draws: tau goes to the call's record
// (taus = the step's [B, Mt] slice; written by the i = 0 threads), x_i = cospi(float32(i tau)) to the rows of the
// forward passes that read it: an online draw (j < N) to cos_q row b N + j; a target or argmax draw to cos_t row
// b (N' + K) + j - N; an argmax draw (j >= N + N') also to cos_n row b K + j - N - N' (Double DQN's Q(s')).
template <bool LANES>
__global__ void iqn_draw_kernel(int B, int N, int Nt, int K, int n_cos, const unsigned long long* keys, int st,
                                float* taus, float* cos_q, float* cos_t, float* cos_n, size_t lane_stride) {
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    keys = lane_ptr(keys, o), taus = lane_ptr(taus, o), cos_q = lane_ptr(cos_q, o), cos_t = lane_ptr(cos_t, o);
    cos_n = lane_ptr(cos_n, o);
  }
  const int Mt = N + Nt + K;
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)B * Mt * n_cos) return;
  const long long t = e / n_cos;
  const int i = (int)(e - t * n_cos);
  const float tau = iqn_tau(t, st, keys[0], keys[1]);
  if (i == 0) taus[t] = tau;
  const float x = cospif(__fmul_rn((float)i, tau));
  const long long b = t / Mt;
  const int j = (int)(t - b * Mt);
  if (j < N) {
    cos_q[(b * N + j) * n_cos + i] = x;
  } else {
    cos_t[(b * (Nt + K) + j - N) * n_cos + i] = x;
    if (j >= N + Nt) cos_n[(b * K + j - N - Nt) * n_cos + i] = x;
  }
}

// z[r, c] = psi[r / M, c] * phi[r, c] over the R = B M rows of width d: one float32 product per element
template <bool LANES>
__global__ void iqn_mul_kernel(const float* psi, const float* phi, long long R, int M, int d, float* z,
                               size_t lane_stride) {
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    psi = lane_ptr(psi, o), phi = lane_ptr(phi, o), z = lane_ptr(z, o);
  }
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= R * d) return;
  const long long r = e / d;
  const int c = (int)(e - r * d);
  z[e] = __fmul_rn(psi[(r / M) * d + c], phi[e]);
}

// The product's backward pass, one thread per (row b, column c) over its N online rows:
//   dphi[b N + i, c] = dz[b N + i, c] psi[b, c],  dpsi[b, c] = sum_i dz[b N + i, c] phi[b N + i, c]
// the sum over i in index order, every product rounded before it is added.
template <bool LANES>
__global__ void iqn_mul_backward_kernel(const float* dz, const float* psi, const float* phi, int B, int N, int d,
                                        float* dphi, float* dpsi, size_t lane_stride) {
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    dz = lane_ptr(dz, o), psi = lane_ptr(psi, o), phi = lane_ptr(phi, o), dphi = lane_ptr(dphi, o);
    dpsi = lane_ptr(dpsi, o);
  }
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= B * d) return;
  const int b = e / d, c = e - b * d;
  const float p = psi[e];
  float s = 0.f;
  for (int i = 0; i < N; ++i) {
    const size_t at = ((size_t)b * N + i) * d + c;
    const float g = dz[at];
    dphi[at] = __fmul_rn(g, p);
    s = __fadd_rn(s, __fmul_rn(g, phi[at]));
  }
  dpsi[e] = s;
}

// shared-memory floats of one row's head: T_j and then the samples' loss sums, theta(s, tau_i, a), the argmax means
__host__ __device__ __forceinline__ int iqn_smem_floats(int n, int N, int Nt) { return (N > Nt ? N : Nt) + N + n; }

// One CTA per row i with action a = act[i] (grid = B rows per learner), thread t owning online sample t (blockDim = N
// rounded up to whole warps; every sum below runs in index order, no float atomics).  q = Z(s) [B N, n], qt_next =
// Q_targ(s') [B (N' + K), n] (per row its N' target samples, then its K argmax samples), qn = Double DQN's Q(s')
// [B K, n] or NULL, taus = the step's fractions [B, N + N' + K] (the online ones first).
//   a* = argmax_a (sum_k Z(s', tau~_k, a)) / K over the argmax samples of qn, or of qt_next without Double DQN,
//   T_j = r + gamma (1 - d) Z_targ(s', tau'_j, a*), u_tj = T_j - theta_t with theta_t = Z(s, tau_t, a),
//   k_tj = |tau_t - 1{u_tj < 0}|, h(u) = 0.5 u^2 if |u| < 1 else |u| - 0.5,
//   L = (1/N') sum_t sum_j k_tj h(u_tj)  (j, then t),
//   dOut[i N + t, a] = -(sum_j k_tj clamp(u_tj, -1, 1)) / N' * (1 / B) and 0 in every other column of the row's N
//   online rows, q_copy[i] = (sum_t theta_t) / N.
// Invalid actions, the row losses, the counters, WEIGHTED and NSTEP as in qr_loss_kernel.
template <bool LANES, bool WEIGHTED, bool NSTEP>
__global__ void __launch_bounds__(IQN_MAX) iqn_loss_kernel(
    const float* q, const float* qt_next, const float* qn, const float* taus, const float* act, const float* rew,
    const float* done, const float* disc, float gamma, int B, int n, int N, int Nt, int K, float* dout,
    float* row_loss, float* q_copy, int* sync, float* loss_out, int* bad_out, const float* w, float* absd,
    size_t lane_stride) {
  extern __shared__ float iqn_smem[];
  __shared__ double red[32];
  __shared__ bool last;
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    q = lane_ptr(q, o), qt_next = lane_ptr(qt_next, o), qn = lane_ptr(qn, o), taus = lane_ptr(taus, o);
    act = lane_ptr(act, o), rew = lane_ptr(rew, o), done = lane_ptr(done, o), dout = lane_ptr(dout, o);
    row_loss = lane_ptr(row_loss, o), q_copy = lane_ptr(q_copy, o), sync = lane_ptr(sync, o);
    loss_out = lane_ptr(loss_out, o), bad_out = lane_ptr(bad_out, o);
    if (WEIGHTED) w = lane_ptr(w, o), absd = lane_ptr(absd, o);
    if (NSTEP) disc = lane_ptr(disc, o);
  }
  const int t = threadIdx.x, i = blockIdx.x;
  float* st = iqn_smem;                // T_j, then each online sample's loss sum
  float* sth = st + (N > Nt ? N : Nt);  // theta(s, tau_t, a)
  float* sq = sth + N;                 // the argmax samples' means per action
  const float af = act[i];
  const bool valid = af >= 0.f && af < (float)n && af == floorf(af);  // false for NaN
  const int a = valid ? (int)af : -1;
  float* drow = dout + (size_t)i * N * n;
  for (int c = t; c < N * n; c += blockDim.x)
    if (c % n != a) drow[c] = 0.f;
  if (!valid) {
    if (t == 0) {
      q_copy[i] = __int_as_float(0x7fc00000);
      row_loss[i] = 0.f;
      if (WEIGHTED) absd[i] = -1.f;
      atomicAdd(sync + 1, 1);
    }
  } else {
    const float th = t < N ? q[((size_t)i * N + t) * n + a] : 0.f;
    if (t < N) sth[t] = th;
    const float* an = qn != nullptr ? qn + (size_t)i * K * n : qt_next + ((size_t)i * (Nt + K) + Nt) * n;
    for (int c = t; c < n; c += blockDim.x) {
      float s = 0.f;
      for (int k = 0; k < K; ++k) s += an[(size_t)k * n + c];
      sq[c] = s / (float)K;
    }
    __syncthreads();
    const int a_star = argmax_row(sq, n);
    const float g1d = (NSTEP ? disc[i] : gamma) * (1.f - done[i]), r = rew[i];
    const float* tq = qt_next + (size_t)i * (Nt + K) * n + a_star;
    for (int j = t; j < Nt; j += blockDim.x) st[j] = r + g1d * tq[(size_t)j * n];
    __syncthreads();
    float lsum = 0.f, gsum = 0.f;
    if (t < N) {
      const float tau = taus[(size_t)i * (N + Nt + K) + t];
      for (int j = 0; j < Nt; ++j) {
        const float u = st[j] - th;
        const float k = fabsf(tau - (u < 0.f ? 1.f : 0.f));
        const float au = fabsf(u);
        const float hu = au < 1.f ? 0.5f * u * u : au - 0.5f;
        const float c = u > 1.f ? 1.f : (u < -1.f ? -1.f : u);  // NaN passes through, as torch's clamp lets it
        lsum += k * hu;
        gsum += k * c;
      }
    }
    __syncthreads();  // every thread is done with T
    const float inv = 1.0f / (float)B;  // dqn_loss_kernel's scaling
    const float wi = WEIGHTED ? w[i] : 1.f;
    if (t < N) {
      st[t] = lsum;
      const float g = -gsum / (float)Nt;
      drow[(size_t)t * n + a] = (WEIGHTED ? wi * g : g) * inv;
    }
    __syncthreads();
    if (t == 0) {
      float L = 0.f, qv = 0.f;
      for (int k = 0; k < N; ++k) L += st[k], qv += sth[k];
      L /= (float)Nt;
      q_copy[i] = qv / (float)N;
      row_loss[i] = WEIGHTED ? wi * L : L;
      if (WEIGHTED) absd[i] = L;
    }
  }
  // the last CTA of this learner reads every row's loss
  __threadfence();
  __syncthreads();
  if (t == 0) last = atomicAdd(sync, 1) == (int)gridDim.x - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  double acc = 0.0;
  for (int r = t; r < B; r += blockDim.x) acc += (double)__ldcg(row_loss + r);
  block_mean(acc, B, loss_out, red);
  if (t == 0) {
    *bad_out = atomicExch(sync + 1, 0);
    sync[0] = 0;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Prioritized experience replay (Schaul et al. 2016, proportional variant).  A sum tree over the physical rows of a
// replay buffer with 32 children per node, all levels in one float array (b200rl.h, b200rl_per_tree_floats): level 0
// holds the leaves, level k + 1 the sums of 32 consecutive nodes of level k, every level padded with zeros to a multiple
// of 32 floats so that a node's children are one aligned 128-byte line.  The last level is [root, running max, 0...].
// An interior node is always recomputed from its children by per_node_sum (never updated by adding a difference), so
// the tree carries no drift and any two ways of reaching the same leaves give the same bits.  Nothing here depends on
// DQN: the draw and the tree update take a row count, the tree and the replay columns.
// ---------------------------------------------------------------------------------------------------------------
constexpr int PER_FAN = 32, PER_MAX_LEVELS = 8;

// offsets of levels 0..top of a tree over n leaves; returns top (the root's level, >= 1)
__host__ __device__ __forceinline__ int per_levels(long long n, long long* off) {
  off[0] = 0;
  long long c = n;
  int k = 0;
  do {
    off[k + 1] = off[k] + ((c + PER_FAN - 1) / PER_FAN) * PER_FAN;
    c = (c + PER_FAN - 1) / PER_FAN;
    ++k;
  } while (c > 1);
  return k;
}

// the sum of the 32 children at ch[0..32), added in index order: the one rule every interior node is computed by
__device__ __forceinline__ float per_node_sum(const float* ch) {
  float s = 0.f;
#pragma unroll
  for (int v = 0; v < PER_FAN / 4; ++v) {
    const float4 x = reinterpret_cast<const float4*>(ch)[v];
    s += x.x;
    s += x.y;
    s += x.z;
    s += x.w;
  }
  return s;
}

// level `parent` nodes [lo, hi) recomputed from level parent - 1 (tree building; one thread per node)
__global__ void per_tree_level_kernel(float* tree, long long child_off, long long parent_off, long long lo,
                                      long long hi) {
  const long long i = lo + (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < hi) tree[parent_off + i] = per_node_sum(tree + child_off + i * PER_FAN);
}

// leaves [lo, lo + count) <- the running max (read on the device: it is whatever the last train call left)
__global__ void per_tree_fill_kernel(float* tree, long long lo, long long count, long long max_at) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < count) tree[lo + i] = tree[max_at];
}

// One CTA per learner, one thread per row (looping for B > blockDim): the stratified proportional draw of step st and
// the importance weights.
//   u_j = (j + U_j) * (M / B), M = the root, U_j = the top 24 bits of Philox4x32-10(counter (j, st, call, 0x9E5),
//   key seed) times 2^-24; descend from the root: at each node take the first child with a nonzero value whose
//   inclusive prefix (summed in per_node_sum's order, so the last prefix is the parent itself) exceeds u, else the last
//   nonzero child, and subtract the exclusive prefix;  w_j = (min_k p[idx_k] / p[idx_j])^beta.
// seed and call are the two 64-bit words at keys[0..2), beta the .y of betas[st]: they change between calls and are read
// from device memory, so a captured graph stays valid.  Ends with a __syncthreads after idx and w are written.
__device__ __forceinline__ void per_draw_rows(const float* tree, long long rows, const float2* betas,
                                              const unsigned long long* keys, int st, int B, long long* idx, float* w) {
  __shared__ float red[32];
  long long off[PER_MAX_LEVELS + 1];
  const int top = per_levels(rows, off);
  const float M = tree[off[top]];
  const unsigned long long seed = keys[0], call = keys[1];
  const uint2 key = make_uint2((unsigned)seed, (unsigned)(seed >> 32));
  const float beta = betas[st].y, step = M / (float)B;
  float pmin = INFINITY;
  for (int j = threadIdx.x; j < B; j += blockDim.x) {
    const uint4 r = philox4x32_10(make_uint4((unsigned)j, (unsigned)st, (unsigned)call, 0x9E5u), key);
    float u = ((float)j + (float)(r.x >> 8) * 5.9604644775390625e-8f) * step;
    long long node = 0;
    for (int k = top; k >= 1; --k) {
      const float* ch = tree + off[k - 1] + node * PER_FAN;
      float c[PER_FAN];
#pragma unroll
      for (int v = 0; v < PER_FAN / 4; ++v) {
        const float4 x = reinterpret_cast<const float4*>(ch)[v];
        c[4 * v] = x.x, c[4 * v + 1] = x.y, c[4 * v + 2] = x.z, c[4 * v + 3] = x.w;
      }
      int pick = -1, last = 0;
      float s = 0.f, before = 0.f, before_last = 0.f;
#pragma unroll
      for (int i = 0; i < PER_FAN; ++i) {
        const float prev = s;
        s += c[i];
        if (c[i] > 0.f) {
          last = i, before_last = prev;
          if (pick < 0 && u < s) pick = i, before = prev;
        }
      }
      if (pick < 0) pick = last, before = before_last;  // rounding put u at or past the last boundary
      u = fmaxf(u - before, 0.f);
      node = node * PER_FAN + pick;
    }
    const float p = tree[node];
    idx[j] = node;
    w[j] = p;
    pmin = fminf(pmin, p);
  }
  // min over the minibatch (exact in any order)
  for (int o = 16; o > 0; o >>= 1) pmin = fminf(pmin, __shfl_xor_sync(0xffffffffu, pmin, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = pmin;
  __syncthreads();
  pmin = red[0];
  for (int i = 1; i < (int)(blockDim.x >> 5); ++i) pmin = fminf(pmin, red[i]);
  for (int j = threadIdx.x; j < B; j += blockDim.x) w[j] = powf(pmin / w[j], beta);
}

// The draw of a prioritized step, then the minibatch staged from the drawn rows (idx was written above by this CTA:
// visible after the __syncthreads).  Without NSTEP the five columns are gathered.  With NSTEP (n-step returns) row j's
// window from idx[j] (nstep_walk over the learner's episode-end column) stages rew := R, done := done[last], disc := g
// and last; obs and act come from the drawn rows, next_obs from the last rows.  n, gamma, disc and last are read by the
// NSTEP instantiations only.
template <bool LANES, bool NSTEP>
__global__ void __launch_bounds__(GTHREADS) per_draw_kernel(const ReplayLanes<LANES> pl, const float2* betas,
                                                           const unsigned long long* keys, int st, int B, int O, int A,
                                                           int n, float gamma, long long* idx, float* w, float* obs,
                                                           float* act, float* rew, float* nobs, float* done,
                                                           float* disc, long long* last, size_t lane_stride) {
  const int z = LANES ? blockIdx.z : 0;
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    betas = lane_ptr(betas, o), keys = lane_ptr(keys, o), idx = lane_ptr(idx, o), w = lane_ptr(w, o);
    obs = lane_ptr(obs, o), act = lane_ptr(act, o), rew = lane_ptr(rew, o), nobs = lane_ptr(nobs, o);
    done = lane_ptr(done, o);
    if (NSTEP) disc = lane_ptr(disc, o), last = lane_ptr(last, o);
  }
  per_draw_rows(pl.tree[z], pl.rows[z], betas, keys, st, B, idx, w);
  if (NSTEP) {
    for (int j = threadIdx.x; j < B; j += blockDim.x) {
      float R, g;
      const long long p = nstep_walk(pl.rew.p[z], pl.done.p[z], pl.ends.p[z], pl.rows[z], idx[j], n, gamma, R, g);
      rew[j] = R, disc[j] = g, done[j] = pl.done.p[z][p], last[j] = p;
    }
    __syncthreads();  // every row's last row is visible to the CTA
    copy_rows(pl.obs.p[z], idx, O, B, obs);
    copy_rows(pl.act.p[z], idx, A, B, act);
    copy_rows(pl.next_obs.p[z], last, O, B, nobs);
  } else {
    const float* src[5] = {pl.obs.p[z], pl.act.p[z], pl.rew.p[z], pl.next_obs.p[z], pl.done.p[z]};
    float* dst[5] = {obs, act, rew, nobs, done};
    const int width[5] = {O, A, 1, O, 1};
#pragma unroll
    for (int c = 0; c < 5; ++c) {
      const int wd = width[c];
      for (int i = threadIdx.x; i < B * wd; i += blockDim.x) {
        const int r = i / wd;
        dst[c][i] = src[c][idx[r] * wd + (i - r * wd)];
      }
    }
  }
}

// One CTA per learner: the priority update of one step.  Row j (in row order; a later row on the same leaf wins) sets
// leaf idx[j] to (absd[j] + eps)^alpha and raises the running max to it; a row with absd = -1 (invalid action) is
// skipped, and a non-finite |delta| or priority leaves its leaf unchanged and is counted in *bad_out.  Then every
// ancestor of a drawn leaf is recomputed, level by level.  newp [B] = the new priority of each row (NaN when skipped).
template <bool LANES>
__global__ void __launch_bounds__(GTHREADS) per_update_kernel(const ReplayLanes<LANES> pl, const long long* idx,
                                                             const float* absd, int B, float alpha, float eps,
                                                             float* newp, int* bad_out, size_t lane_stride) {
  __shared__ long long leaf_s[GTHREADS];
  __shared__ float red[32];
  __shared__ int bad_rows;
  const int z = LANES ? blockIdx.z : 0;
  if (LANES) {
    const size_t o = blockIdx.z * lane_stride;
    idx = lane_ptr(idx, o), absd = lane_ptr(absd, o), newp = lane_ptr(newp, o), bad_out = lane_ptr(bad_out, o);
  }
  float* tree = pl.tree[z];
  long long off[PER_MAX_LEVELS + 1];
  const int top = per_levels(pl.rows[z], off);
  if (threadIdx.x == 0) bad_rows = 0;
  float mx = 0.f;
  int bad = 0;
  for (int base = 0; base < B; base += blockDim.x) {  // rows in chunks of blockDim, in order
    const int j = base + threadIdx.x;
    long long leaf = -1;
    float p = 0.f;
    if (j < B) {
      const float ad = absd[j];
      p = __int_as_float(0x7fc00000);
      if (ad != -1.f) {
        p = powf(ad + eps, alpha);
        if (isfinite(ad) && isfinite(p)) leaf = idx[j], mx = fmaxf(mx, p);
        else ++bad;
      }
      newp[j] = p;
    }
    leaf_s[threadIdx.x] = leaf;
    __syncthreads();
    if (leaf >= 0) {
      bool last = true;
      const int n = min((int)blockDim.x, B - base);
      for (int k = threadIdx.x + 1; k < n && last; ++k) last = leaf_s[k] != leaf;
      if (last) tree[leaf] = p;
    }
    __syncthreads();
  }
  if (bad) atomicAdd(&bad_rows, bad);
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  for (int k = 1; k <= top; ++k) {  // the leaves' writes (and each level's) are visible to the CTA after the barrier
    __syncthreads();
    for (int j = threadIdx.x; j < B; j += blockDim.x) {
      const long long node = idx[j] >> (5 * k);
      tree[off[k] + node] = per_node_sum(tree + off[k - 1] + node * PER_FAN);
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) mx = fmaxf(mx, red[i]);
    float& m = tree[off[top] + 1];
    m = fmaxf(m, mx);
    *bad_out = bad_rows;
  }
}

}  // namespace b200rl

using namespace b200rl;

// ---------------------------------------------------------------------------------------------------------------
struct NetBuf {
  b200rl_mlp_desc d;
  int64_t P = 0;
  float* params = nullptr;
  float *m = nullptr, *v = nullptr;  // Adam state (trainable nets only)
  float* grad = nullptr;
  bool present = false;
  int64_t step[B200RL_MAX_LEARNERS] = {};  // Adam step count of each learner
  int w_off[B200RL_MAX_LAYERS], b_off[B200RL_MAX_LAYERS];
  // dueling Q network (config dueling_k = K > 0; d = [obs, h1, h2, n K]): its five Linear layers' offsets, in the
  // order trunk, value hidden, value out, advantage hidden, advantage out
  int duel_k = 0;
  int dw_off[5] = {}, db_off[5] = {};  // an IQN network (config algo = 4) keeps its four layers' offsets here too: psi,
                                       // phi, head hidden, head out
  // the vector set_params / get_params, the state blob, Adam and the target copy work on, P_flat floats: params /
  // grad themselves, except for networks 1 and 4 of an engine with noisy layers, where params / grad hold the composed
  // network the GEMMs read and flat / flat_grad the noisy vector (noisy_compose_kernel, noisy_expand_kernel)
  float *flat = nullptr, *flat_grad = nullptr;
  int64_t P_flat = 0;
};

// What a captured step program holds in its nodes besides the engine's own buffers: a graph is replayed only for a call
// with the same key.  Zero-initialised as a whole (compared with memcmp).  A prioritized call's nodes also hold alpha /
// eps and the trees' and columns' addresses and row counts (and with n > 1 the episode-end columns its draw walks);
// `per` and `replay` stay zero for every other call.
struct GraphKey {
  int S, B, nstep;
  b200rl_offpolicy_hparams hp;
  b200rl_sac_hparams sac;
  b200rl_dqn_hparams dqn;
  b200rl_c51_hparams c51;
  b200rl_qr_hparams qr;
  b200rl_per_hparams per;
  ReplayLanes<true> replay;
  b200rl_cql_hparams cql;
  b200rl_iql_hparams iql;  // v_lr zeroed: V's learning rate is read per call, like q1_lr / q2_lr
};

struct b200rl_offpolicy {
  b200rl_offpolicy_config cfg;
  // learners of the group (1 = a solo engine) and the byte distance between their arenas: every pointer below is
  // learner 0's copy, learner z's is at + z * lane_stride (see lane_ptr)
  int K = 1;
  size_t lane_stride = 0;
  std::vector<std::pair<void**, size_t>> pieces;  // (pointer to set, offset in the arena) of every engine buffer
  size_t arena_bytes = 0;
  NetBuf net[2 * REDQ_MAX_CRITICS + 1];  // 0 pi, 1 Q1, 2 Q2, 3 pi_targ, 4 Q1_targ, 5 Q2_targ (REDQ: 0 pi, 1..N the
                                         // critics, N+1..2N their targets)
  int O = 0, A = 0, maxw = 0;
  // staged minibatches [S,B,*]
  float *obs = nullptr, *act = nullptr, *rew = nullptr, *nobs = nullptr, *done = nullptr, *eps = nullptr;
  // per-step workspace
  float* acts[5][B200RL_MAX_LAYERS + 1];  // activation stacks [B, width]: 0 scratch/target (Q1 side), 1 Q1, 2 policy,
                                          // 3 target Q2, 4 Q2 (the twin critic runs on a second stream)
  float* acts_tq[B200RL_MAX_LAYERS + 1];  // Q1's target critic gets a stack of its own: in stack 0, a critic deeper than
                                          // the policy would overwrite the target action, which the twin target
                                          // critic on s2 may still be reading
  float *x_cat = nullptr, *x_cat2 = nullptr, *qt1 = nullptr, *qt2 = nullptr, *dq = nullptr;
  float *dbuf0 = nullptr, *dbuf1 = nullptr;  // gradient ping-pong [B, maxw]
  float *dbuf2 = nullptr, *dbuf3 = nullptr, *dq2 = nullptr;  // the same for the twin critic's branch
  cudaStream_t s2 = nullptr;                // side stream of the twin critic (forked / joined with events)
  cudaStream_t s3 = nullptr, s4 = nullptr;  // the critics' forward passes on [s | a] beside the target path; the
                                            // weight-gradient products beside the dX chains
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr, ev_side = nullptr;
  // outputs
  float *out_q1 = nullptr, *out_q2 = nullptr, *out_l1 = nullptr, *out_l2 = nullptr, *out_lp = nullptr;
  // CUDA graph of the S-step loop: node arguments are fixed per (S, B, hyper-parameters); what changes between calls
  // (minibatch contents, Adam bias-correction scalars) lives in device buffers refreshed before each launch
  long long* idx = nullptr;      // [max_steps * max_minibatch] replay rows of train_gather
  float2* adam_tab = nullptr;    // [3][max_steps] {lr / (1 - beta1^t), sqrt(1 - beta2^t)} for policy, Q1, Q2
  float2* h_adam_tab = nullptr;  // pinned mirror, [K][table]
  cudaStream_t gs = nullptr;     // internal stream (the caller's may be the legacy default stream: not capturable)
  cudaEvent_t ev = nullptr;
  cudaGraphExec_t graph = nullptr;
  GraphKey graph_key;  // the call the graph was captured for
  int graph_npol = 0, graph_launches = 0;
  int last_npol = 0;   // the policy steps of the last train call that ran steps (get_policy_losses)
  float* state = nullptr;  // parameters + Adam state of every network, blob order (see b200rl_offpolicy_create)
  int64_t state_n = 0;
  // SAC (cfg.algo == 1): network 3 is absent; h->eps holds [S, 2, B, A] (the draw for s', then the one for s)
  bool sac = false, sac_set = false;
  b200rl_sac_hparams sac_hp{};
  float *sac_act_next = nullptr, *sac_logp_next = nullptr;  // [B, A] / [B]: a' and log pi(a' | s')
  float *sac_act = nullptr, *sac_logp = nullptr;            // the same at s (the policy step)
  float* sac_dout = nullptr;                                // [B, 2A] gradient w.r.t. the policy output
  float* sac_alpha = nullptr;                               // [max_steps + 1] alpha of step st at [st]
  float* sac_state = nullptr;                               // {log_alpha, exp_avg, exp_avg_sq}
  float* out_logp = nullptr;                                // [max_steps] mean log pi of each policy step
  int64_t alpha_step[B200RL_MAX_LEARNERS] = {};
  // discrete SAC (cfg.algo == 5): SAC's networks, temperature and outputs (every SAC buffer above except the act /
  // log pi ones), DQN's index action column (A = 1) and invalid-action count (dqn_bad); h->sac stays false.  dq / dq2
  // are [B, n], sac_dout the policy's [B, n] logit gradient and sac_logp each row's E_i = sum_j pi_j log pi_j
  bool dsac = false;
  // DQN (cfg.algo == 2): networks 1 (Q) and 4 (target Q) only; the action column is 1 wide (the index as float32);
  // adam_tab row 3 holds the target-copy flags of the call's steps
  bool dqn = false, dqn_set = false;
  b200rl_dqn_hparams dqn_hp{};
  float* dqn_dout = nullptr;  // [B, n] gradient w.r.t. the Q output
  int* dqn_bad = nullptr;     // [max_steps] rows of each step whose action was not a valid index
  // C51 (cfg.algo == 3): a DQN engine (h->dqn is set) whose loss head is c51_loss_kernel
  bool c51 = false, c51_set = false;
  b200rl_c51_hparams c51_hp{};
  float* c51_support = nullptr;   // [C51_MAX_ATOMS] z_0 .. z_{N-1}
  float* c51_row_loss = nullptr;  // [B] each row's cross-entropy (QR-DQN: quantile loss) of the current step
  int* c51_sync = nullptr;        // {CTAs done, invalid rows} of the current step; 0 between launches
  // QR-DQN (b200rl_offpolicy_set_qr on a DQN engine): the loss head is qr_loss_kernel, with C51's row losses and counters
  bool qr = false;
  b200rl_qr_hparams qr_hp{};
  // prioritized replay (DQN engines): a prioritized call draws, weighs and gathers inside the step program; adam_tab
  // row 3's .y then holds each step's beta and the table's last two float2 the call's (seed, call) words
  bool per_set = false, per_run = false;
  bool per_last = false;                       // the last call that ran steps was a prioritized one
  b200rl_per_hparams per_hp{};
  float *per_w = nullptr, *per_newp = nullptr;  // [max_steps * B] importance weights / new priorities of each row
  float* per_absd = nullptr;                    // [B] |delta| of the current step
  int* per_bad = nullptr;                       // [max_steps] rows of each step whose new priority was not finite
  // n-step returns (DQN engines; b200rl_offpolicy_set_nstep): an n-step call stages R in rew, done[last] in done, and
  // each row's discount and last row beside them
  int nstep = 1;
  LaneSrc<true> nstep_ends{};         // each learner's episode-end column (n > 1)
  bool nstep_last = false;            // the last call that ran steps was an n-step one
  float* nstep_disc = nullptr;        // [max_steps * B] gamma^k of each row's window
  long long* nstep_rows = nullptr;    // [max_steps * B] the last row of each row's window
  // noisy layers (config noisy_layers != 0; DQN engines): adam_tab's last two float2 hold the (seed, call) words of
  // set_noise_keys, which every train call needs afresh
  bool noisy = false, noisy_keys = false;
  NoisyLayout noisy_lay{};
  float* noisy_draws = nullptr;  // [max_steps][2][E] raw draws of the call's steps (online, target)
  // IQN (cfg.algo == 4): a DQN engine (h->dqn is set) over an implicit quantile network; its draws take their keys from
  // set_noise_keys, in the adam_tab slot a noisy engine's keys take
  bool iqn = false;
  b200rl_iqn_config iqn_cfg{};         // n_cos, N, N', K
  int iqn_last_B = 0;                  // the minibatch of the last call that ran steps (0: none yet)
  float* iqn_taus = nullptr;           // [max_steps][B][N + N' + K] fractions of the call's steps
  float *iqn_cos_q = nullptr, *iqn_cos_t = nullptr, *iqn_cos_n = nullptr;  // the step's cosine features (iqn_draw_kernel)
  IqnPass iqn_pass[3] = {};            // Q(s) with N, Q_targ(s') with N' + K, Q(s') with K fractions per row
  float *iqn_dhid = nullptr, *iqn_dz = nullptr, *iqn_dphi = nullptr, *iqn_dpsi = nullptr;  // the backward pass's
  // D4PG (cfg.algo == 6): DDPG's networks with an N-wide critic; C51's support, row losses and counters, DQN's
  // prioritized and n-step buffers; dq and qt1 are [B, N]
  bool d4pg = false;
  b200rl_d4pg_config d4pg_cfg{};
  // TQC (cfg.algo == 7): a SAC engine (h->sac is set: every SAC buffer, the temperature and the outputs) whose critics
  // map [s | a] -> M quantiles; qt1, qt2, dq and dq2 are [B, M]
  bool tqc = false;
  b200rl_tqc_config tqc_cfg{};
  float* tqc_y = nullptr;         // [B, kN] the step's truncated target atoms, ascending
  float* tqc_row_loss = nullptr;  // [2][B] each critic's row losses
  int* tqc_sync = nullptr;        // [2] each critic head's CTAs done; 0 between launches
  // CQL (cfg.algo == 8): a SAC engine (h->sac is set) whose critics run on R = (1 + 3N) B stacked rows in the critic
  // step; dq, dq2 and dbuf0..3 are R rows deep.  adam_tab row 4 holds the Lagrange step's Adam scalars.
  bool cql = false, cql_set = false;
  b200rl_cql_config cql_cfg{};
  b200rl_cql_hparams cql_hp{};
  int cql_staged_S = -1, cql_staged_B = -1;      // the (S, B) of host draws staged for the next train call
  float* cql_draws = nullptr;                    // [max_steps][3][B][N][A] the call's draws (uniform x, eps at s', at s)
  float* cql_x = nullptr;                        // [R, O + A] the stacked critic operand
  float* cql_logp = nullptr;                     // [B, 3N] each sample's log density
  float* cql_acts[2][B200RL_MAX_LAYERS + 1];     // the critics' activation stacks [R, width]
  float* cql_row_p = nullptr;                    // [2][B] each critic's P_i
  int* cql_sync = nullptr;                       // [2] each penalty head's CTAs done; 0 between launches
  float* cql_gap = nullptr;                      // [2][max_steps] gap_k of each step
  float* cql_ap = nullptr;                       // [max_steps + 1] alpha' of step st at [st]
  float* cql_ap_state = nullptr;                 // {log alpha', exp_avg, exp_avg_sq}
  float* cql_zero = nullptr;                     // one 0.f: the temperature of a backup without the entropy term
  int64_t ap_step[B200RL_MAX_LEARNERS] = {};
  // IQL (cfg.algo == 9): network 3 is the value network V, trained by optimizer 3 (adam_tab row 3); networks 0, 1, 2,
  // 4, 5 are SAC's.  The critics' backward passes run beside the policy's, so Q1's takes a third gradient ping-pong.
  bool iql = false, iql_set = false;
  b200rl_iql_hparams iql_hp{};
  float *dbuf4 = nullptr, *dbuf5 = nullptr;   // [B, maxw] Q1's gradient ping-pong
  float* iql_dv = nullptr;                     // [B] d L_V / d V(s)
  float* iql_dout = nullptr;                   // [B, 2A] d L_pi / d [m | l]
  float* iql_zero = nullptr;                   // [B] zeros: the critics' head's temperature and log density
  float *out_vl = nullptr, *out_vm = nullptr, *out_wm = nullptr;  // [max_steps] value loss, value mean, weight mean
  // REDQ (cfg.algo == 10): a SAC engine (h->sac is set: the policy, its buffers, the temperature and the outputs) whose
  // N critics are networks 1..N, run as one ensemble.  Member k of every ensemble buffer below sits k member strides
  // after member 0; out_q1 / out_l1 hold every critic's values [N][S][B] and losses [N][S] of the call.
  bool redq = false;
  b200rl_redq_config redq_cfg{};
  int redq_staged_S = -1;                        // the S of host subsets staged for the next train call
  int* redq_sub = nullptr;                       // [max_steps][M] the call's subsets
  float* redq_acts[B200RL_MAX_LAYERS + 1];       // the critics' activation stacks, [N][B][maxw] per layer
  float* redq_tacts[B200RL_MAX_LAYERS + 1];      // the drawn target critics' stacks, [M][B][maxw] per layer
  float *redq_d0 = nullptr, *redq_d1 = nullptr;  // [N][B][maxw] gradient ping-pong
  float* redq_dq = nullptr;                      // [N][B] d loss / d Q_k
  float* redq_dx = nullptr;                      // [N][B][O + A] the critics' input gradients (policy step)
  float* redq_qmin = nullptr;                    // [B] min over the drawn target critics
  int redq_last_S = 0, redq_last_B = 0;          // the (S, B) of the last call that ran steps (redq_outputs)
  // EDAC / SAC-N (cfg.algo == 11): a REDQ engine (h->redq is set, M = N) with its own step program.  With eta > 0 the
  // diversity pass keeps every hidden layer's ones-backward gradient and tangent in buffers of their own (the TD
  // backward's redq_d0 / redq_d1 run at the same time), and its weight gradient in a second gradient block laid out as
  // the critics' (zeroed at create; its obs columns and biases are never written)
  bool edac = false;
  double edac_eta = 0.0;
  float* edac_ones = nullptr;                   // [max_minibatch] ones: the ones-backward's dOut
  float* edac_e[B200RL_MAX_LAYERS + 1];         // [N][B][maxw] layer l's ungated input gradient of sum Q_k, l >= 1
  float* edac_t[B200RL_MAX_LAYERS + 1];         // [N][B][maxw] layer l's tangent h'_l, l >= 1
  float *edac_g = nullptr, *edac_u = nullptr;   // [N][B][A] the action gradients and d(eta D) / d g
  float* edac_grad = nullptr;                   // [N][state_pad(P)] the diversity term's parameter gradient
  float* edac_div = nullptr;                    // [max_steps] D per step
  // the replay columns, episode-end columns, trees and row counts of this call (train_gather[_rng], train_prioritized)
  ReplayLanes<true> replay{};
  std::vector<void*> allocs;
};

namespace {

inline int64_t state_pad(int64_t n) { return (n + 63) & ~(int64_t)63; }

// the optimizers of the state blob and of steps[]: policy, Q1, Q2 (and V on an IQL engine; policy and N critics on a
// REDQ engine)
inline int n_opt(const b200rl_offpolicy* h) { return h->iql ? 4 : h->redq ? 1 + h->redq_cfg.n_critics : 3; }
// the network slots of the engine: 6, or 1 + 2N on a REDQ engine
inline int n_nets(const b200rl_offpolicy* h) { return h->redq ? 1 + 2 * h->redq_cfg.n_critics : 6; }

// float2 entries of one learner's adam_tab: the Adam scalar rows (+ SAC's temperature row, DQN's copy flags or D4PG's
// betas), then DQN's or D4PG's prioritized (seed, call) at 4 max_steps and a noisy or IQN engine's draw keys (seed,
// call) after it
inline size_t adam_tab_len(const b200rl_offpolicy* h) {
  const bool per = h->dqn || h->d4pg;  // engines that take prioritized replay: row 3's .y holds the betas
  return (h->cql ? 5 : h->sac || h->dsac || h->iql || per ? 4 : 3) * (size_t)h->cfg.max_steps + (per ? 2 : 0) +
         (h->noisy || h->iqn ? 2 : 0);
}

// A piece of the learner arena: recorded here (256-byte aligned), placed by arena_commit
template <typename T>
int oalloc(b200rl_offpolicy* h, T** p, size_t count) {
  h->pieces.emplace_back(reinterpret_cast<void**>(p), h->arena_bytes);
  h->arena_bytes += ((count ? count : 1) * sizeof(T) + 255) & ~(size_t)255;
  return 0;
}

// ONE zeroed allocation of K arenas at a fixed stride (a multiple of 256 bytes); every recorded buffer points into
// learner 0's arena
int arena_commit(b200rl_offpolicy* h) {
  h->lane_stride = h->arena_bytes;
  void* q = nullptr;
  B200RL_CUDA(cudaMalloc(&q, (size_t)h->K * h->lane_stride));
  h->allocs.push_back(q);
  B200RL_CUDA(cudaMemset(q, 0, (size_t)h->K * h->lane_stride));
  for (const auto& pc : h->pieces) *pc.first = static_cast<char*>(q) + pc.second;
  h->pieces.clear();
  return 0;
}

inline dim3 lane_grid(dim3 g, int K) {
  g.z = (unsigned)K;
  return g;
}

// The LANES = false slice of a per-learner table: learner 0's entry, a solo engine's only one.  Every other kernel
// argument is the same for both instantiations.
template <typename T>
const T& solo(const T& arg) { return arg; }
LaneSrc<false> solo(const LaneSrc<true>& t) { return {{t.p[0]}}; }
DrawKeys<false> solo(const DrawKeys<true>& k) {
  return {{k.seed[0]}, {k.call[0]}, {k.start[0]}, {k.size[0]}, {k.capacity[0]}};
}
ReplayLanes<false> solo(const ReplayLanes<true>& r) {
  return {solo(r.obs), solo(r.act), solo(r.rew), solo(r.next_obs), solo(r.done), solo(r.ends),
          {r.tree[0]}, {r.rows[0]}};
}

// One launch for every learner: a solo engine runs the solo kernel kern<false> on `grid` with each table argument cut
// to its solo slice, a group kern<true> over blockIdx.z = learner.  `args` are the kernel's arguments up to its lane
// stride, tables in their LANES = true form.
template <typename... Solo, typename... Lanes, typename... Args>
int launch(const b200rl_offpolicy* h, void (*solo_kern)(Solo...), void (*lanes_kern)(Lanes...), dim3 grid, dim3 block,
           size_t smem, cudaStream_t s, const Args&... args) {
  if (h->K == 1) solo_kern<<<grid, block, smem, s>>>(solo(args)..., (size_t)0);
  else lanes_kern<<<lane_grid(grid, h->K), block, smem, s>>>(args..., h->lane_stride);
  B200RL_CUDA(cudaGetLastError());
  count_launch(1);
  return 0;
}

// work queued on `to` from here on waits for everything queued on `from` so far (a graph edge under capture)
int edge(const b200rl_offpolicy* h, cudaStream_t from, cudaStream_t to) {
  B200RL_CUDA(cudaEventRecord(h->ev_fork, from));
  B200RL_CUDA(cudaStreamWaitEvent(to, h->ev_fork, 0));
  return 0;
}

template <int MODE>
int gemm(const b200rl_offpolicy* h, const GemmArgs& g, cudaStream_t s) {
  const dim3 grid((g.N + GT - 1) / GT, (g.M + GT - 1) / GT);
  return launch(h, gemm_kernel<MODE, false>, gemm_kernel<MODE, true>, grid, GTHREADS, 0, s, g);
}

// forward through one network: acts[0] = input [rows, n0] (ld = n0); acts[l+1] = layer outputs.
// in_b != NULL: the input is torch.cat([acts[0] (ksplit columns), in_b (ld_b)], -1), read in place by the first layer
// (q_function.py:30); eps != NULL: target-policy smoothing on the output (td3.py:326-332)
int net_forward(const b200rl_offpolicy* h, const NetBuf& nb, float* const* acts, int rows, cudaStream_t s,
                const float* in_b = nullptr, int ld_b = 0, int ksplit = 0, const float* eps = nullptr,
                const b200rl_offpolicy_hparams* hp = nullptr) {
  const int L = nb.d.n_layers;
  for (int l = 0; l < L; ++l) {
    GemmArgs g{};
    g.A = acts[l]; g.lda = nb.d.sizes[l];
    if (l == 0 && in_b != nullptr) {
      g.lda = ksplit;
      g.A2 = in_b; g.lda2 = ld_b; g.ksplit = ksplit;
    }
    if (l == L - 1 && eps != nullptr) {
      g.eps = eps;
      g.sigma = (float)hp->target_noise_scale;
      g.clipv = (float)hp->target_noise_clip;
      g.limit = (float)hp->action_limit;
    }
    g.B = nb.params + nb.w_off[l]; g.ldb = nb.d.sizes[l];
    g.C = acts[l + 1]; g.ldc = nb.d.sizes[l + 1];
    g.bias = nb.params + nb.b_off[l];
    g.act = (l == L - 1) ? nb.d.out_act : nb.d.hidden_act;
    g.M = rows; g.N = nb.d.sizes[l + 1]; g.K = nb.d.sizes[l];
    if (gemm<0>(h, g, s)) return 1;
  }
  return 0;
}

// backward: dOut = gradient w.r.t. the network OUTPUT (after the output activation) [rows, nL] with ld ld_dout.
// want_param_grads: write nb.grad (flat).  dx_out (optional): gradient w.r.t. the input [rows, n0].
// s_dw != NULL (and at most 3 layers: the two ping-pong buffers then never see a writer while a reader is pending): the
// weight-gradient products go to that stream, behind the gradient they read, and the dX chain -- the critical path --
// stays on `s`; both are joined before returning.
int net_backward(b200rl_offpolicy* h, const NetBuf& nb, float* const* acts, const float* dOut, int ld_dout, int rows,
                 bool want_param_grads, float* dx_out, cudaStream_t s, int branch = 0,
                 const float* in_b = nullptr, int ld_b = 0, int ksplit = 0, cudaStream_t s_dw = nullptr) {
  const int L = nb.d.n_layers;
  const bool side = s_dw != nullptr && want_param_grads && L <= 3;
  const float* dY = dOut;
  int ldd = ld_dout;
  // the gradient ping-pong of the branch: 0 dbuf0/1, 1 (the twin critic) dbuf2/3, 2 (IQL's Q1) dbuf4/5
  float* pp[2] = {branch == 0 ? h->dbuf0 : branch == 1 ? h->dbuf2 : h->dbuf4,
                  branch == 0 ? h->dbuf1 : branch == 1 ? h->dbuf3 : h->dbuf5};
  for (int l = L - 1; l >= 0; --l) {
    const int nout = nb.d.sizes[l + 1], nin = nb.d.sizes[l];
    const int act = (l == L - 1) ? nb.d.out_act : nb.d.hidden_act;
    const float* Y = acts[l + 1];
    if (want_param_grads) {
      GemmArgs g{};  // dW[nout, nin] = (dY . act'(Y))^T [nout, rows] * X[rows, nin]
      g.A = dY; g.lda = ldd; g.Y = Y; g.ldy = nout; g.act = act;
      g.B = acts[l]; g.ldb = nin;
      if (l == 0 && in_b != nullptr) {  // the layer's input is [acts[0] | in_b], never materialised
        g.ldb = ksplit;
        g.A2 = in_b; g.lda2 = ld_b; g.ksplit = ksplit;
      }
      g.C = nb.grad + nb.w_off[l]; g.ldc = nin;
      g.M = nout; g.N = nin; g.K = rows;
      g.dbias = nb.grad + nb.b_off[l];  // db = column sums of dZ, accumulated by the same kernel
      if (side) {  // dY of this layer is complete on `s` at this point
        B200RL_CUDA(cudaEventRecord(h->ev_side, s));
        B200RL_CUDA(cudaStreamWaitEvent(s_dw, h->ev_side, 0));
      }
      if (gemm<2>(h, g, side ? s_dw : s)) return 1;
    }
    if (l > 0 || dx_out) {
      float* dst = (l == 0) ? dx_out : pp[l & 1];
      GemmArgs g{};  // dX[rows, nin] = (dY . act'(Y))[rows, nout] * W[nout, nin]
      g.A = dY; g.lda = ldd; g.Y = Y; g.ldy = nout; g.act = act;
      g.B = nb.params + nb.w_off[l]; g.ldb = nin;
      g.C = dst; g.ldc = nin;
      g.M = rows; g.N = nin; g.K = nout;
      if (gemm<1>(h, g, s)) return 1;
      dY = dst;
      ldd = nin;
    }
  }
  if (side) {
    B200RL_CUDA(cudaEventRecord(h->ev_side, s_dw));
    B200RL_CUDA(cudaStreamWaitEvent(s, h->ev_side, 0));
  }
  return 0;
}

// A dueling Q network (nb.duel_k = K; nb.d = [O, h1, h2, n K]) on acts[0] = input [rows, O]: acts[1] = trunk [rows, h1],
// acts[2] = [value hidden | advantage hidden] [rows, 2 h2], acts[4] = [V | A] [rows, K + n K], and acts[3] = Q [rows, n K]
// (dueling_forward_kernel), the slot a plain network's output takes, where the loss heads read it.
int dueling_forward(const b200rl_offpolicy* h, const NetBuf& nb, float* const* acts, int rows, cudaStream_t s) {
  const int O = nb.d.sizes[0], h1 = nb.d.sizes[1], h2 = nb.d.sizes[2], nK = nb.d.sizes[3], K = nb.duel_k;
  auto layer = [&](int l, const float* x, int ldx, int nin, float* y, int ldy, int nout, int act) {
    GemmArgs g{};
    g.A = x; g.lda = ldx;
    g.B = nb.params + nb.dw_off[l]; g.ldb = nin;
    g.C = y; g.ldc = ldy;
    g.bias = nb.params + nb.db_off[l];
    g.act = act;
    g.M = rows; g.N = nout; g.K = nin;
    return gemm<0>(h, g, s);
  };
  const int hid = nb.d.hidden_act, out = nb.d.out_act;
  if (layer(0, acts[0], O, O, acts[1], h1, h1, hid) || layer(1, acts[1], h1, h1, acts[2], 2 * h2, h2, hid) ||
      layer(3, acts[1], h1, h1, acts[2] + h2, 2 * h2, h2, hid) ||
      layer(2, acts[2], 2 * h2, h2, acts[4], K + nK, K, out) ||
      layer(4, acts[2] + h2, 2 * h2, h2, acts[4] + K, K + nK, nK, out))
    return 1;
  return launch(h, dueling_forward_kernel<false>, dueling_forward_kernel<true>, (unsigned)((rows * K + GTHREADS - 1) / GTHREADS),
                GTHREADS, 0, s, acts[4], rows, nK / K, K, acts[3]);
}

// Its backward pass from dOut = dL/dQ [rows, n K] into nb.grad: dueling_backward_kernel, then each stream's output and
// hidden layer, then the trunk, whose input gradient dZv Wv + dZa Wa is one split-B GEMM (k over [value | advantage]
// in that order).  The dX chain stays on `s`, the weight-gradient products go to s_dw behind the gradient they read;
// dbuf0 / dbuf1 / dbuf2 hold dL/d[V | A], dL/d(stream hidden) and dL/d(trunk), each written once per step.
int dueling_backward(b200rl_offpolicy* h, const NetBuf& nb, float* const* acts, const float* dOut, int rows,
                     cudaStream_t s, cudaStream_t s_dw) {
  const int O = nb.d.sizes[0], h1 = nb.d.sizes[1], h2 = nb.d.sizes[2], nK = nb.d.sizes[3], K = nb.duel_k;
  const int hid = nb.d.hidden_act;
  float *dva = h->dbuf0, *dh2 = h->dbuf1, *dh1 = h->dbuf2;
  auto fork = [&]() {  // what `s` has queued so far is complete before the next products on s_dw
    B200RL_CUDA(cudaEventRecord(h->ev_side, s));
    B200RL_CUDA(cudaStreamWaitEvent(s_dw, h->ev_side, 0));
    return 0;
  };
  // dW[nout, nin] = (dY . act'(Y))^T X and db on s_dw
  auto dw = [&](int l, const float* dY, int ldd, const float* Y, int act, const float* X, int ldx, int nout, int nin) {
    GemmArgs g{};
    g.A = dY; g.lda = ldd; g.Y = Y; g.ldy = ldd; g.act = act;
    g.B = X; g.ldb = ldx;
    g.C = nb.grad + nb.dw_off[l]; g.ldc = nin;
    g.M = nout; g.N = nin; g.K = rows;
    g.dbias = nb.grad + nb.db_off[l];
    return gemm<2>(h, g, s_dw);
  };
  // dX[rows, nin] = dY[rows, nout] W[nout, nin] on s (the output layers are linear: no derivative)
  auto dx = [&](int l, const float* dY, int ldd, float* dst, int ldc, int nout, int nin) {
    GemmArgs g{};
    g.A = dY; g.lda = ldd;
    g.B = nb.params + nb.dw_off[l]; g.ldb = nin;
    g.C = dst; g.ldc = ldc;
    g.M = rows; g.N = nin; g.K = nout;
    return gemm<1>(h, g, s);
  };
  if (launch(h, dueling_backward_kernel<false>, dueling_backward_kernel<true>,
             (unsigned)((rows * K + GTHREADS - 1) / GTHREADS), GTHREADS, 0, s, dOut, rows, nK / K, K, dva))
    return 1;
  if (fork() || dw(2, dva, K + nK, nullptr, B200RL_ACT_IDENTITY, acts[2], 2 * h2, K, h2) ||
      dw(4, dva + K, K + nK, nullptr, B200RL_ACT_IDENTITY, acts[2] + h2, 2 * h2, nK, h2))
    return 1;
  if (dx(2, dva, K + nK, dh2, 2 * h2, K, h2) || dx(4, dva + K, K + nK, dh2 + h2, 2 * h2, nK, h2)) return 1;
  if (fork() || dw(1, dh2, 2 * h2, acts[2], hid, acts[1], h1, h2, h1) ||
      dw(3, dh2 + h2, 2 * h2, acts[2] + h2, hid, acts[1], h1, h2, h1))
    return 1;
  {
    GemmArgs g{};  // dX[rows, h1] = (dH . act'(H))[rows, 2 h2] [Wv; Wa][2 h2, h1]
    g.A = dh2; g.lda = 2 * h2; g.Y = acts[2]; g.ldy = 2 * h2; g.act = hid;
    g.B = nb.params + nb.dw_off[1]; g.ldb = h1;
    g.A2 = nb.params + nb.dw_off[3]; g.lda2 = h1; g.ksplit = h2;
    g.C = dh1; g.ldc = h1;
    g.M = rows; g.N = h1; g.K = 2 * h2;
    if (gemm<3>(h, g, s)) return 1;
  }
  if (fork() || dw(0, dh1, h1, acts[1], hid, acts[0], O, h1, O)) return 1;
  B200RL_CUDA(cudaEventRecord(h->ev_side, s_dw));
  B200RL_CUDA(cudaStreamWaitEvent(s, h->ev_side, 0));
  return 0;
}

// An IQN network (nb.d = [obs, d, h, n]) on x [B, obs] and the cosine features cos [B M, n_cos] of M fractions per
// row: psi, phi, their product and the head's two layers into p, 5 launches.
int iqn_forward(const b200rl_offpolicy* h, const NetBuf& nb, const float* x, const float* cos, int B, int M,
                const IqnPass& p, cudaStream_t s) {
  const int O = nb.d.sizes[0], D = nb.d.sizes[1], H = nb.d.sizes[2], n = nb.d.sizes[3], C = h->iqn_cfg.n_cos;
  const int R = B * M, hid = nb.d.hidden_act;
  auto layer = [&](int l, const float* X, int rows, int nin, float* Y, int nout, int act) {
    GemmArgs g{};
    g.A = X; g.lda = nin;
    g.B = nb.params + nb.dw_off[l]; g.ldb = nin;
    g.C = Y; g.ldc = nout;
    g.bias = nb.params + nb.db_off[l];
    g.act = act;
    g.M = rows; g.N = nout; g.K = nin;
    return gemm<0>(h, g, s);
  };
  if (layer(0, x, B, O, p.psi, D, hid) || layer(1, cos, R, C, p.phi, D, hid)) return 1;
  if (launch(h, iqn_mul_kernel<false>, iqn_mul_kernel<true>, (unsigned)(((long long)R * D + GTHREADS - 1) / GTHREADS),
             GTHREADS, 0, s, p.psi, p.phi, (long long)R, M, D, p.z))
    return 1;
  return layer(2, p.z, R, D, p.hid, H, hid) || layer(3, p.hid, R, H, p.out, n, nb.d.out_act);
}

// Its backward pass from dOut = dL/dZ [B N, n] into nb.grad, 7 launches: the dX chain (dhid, dz, the product's
// backward) on `s`, the four weight-gradient products on s_dw behind the gradient they read.  No input gradient.
int iqn_backward(b200rl_offpolicy* h, const NetBuf& nb, const float* x, const float* cos, int B, const IqnPass& p,
                 const float* dOut, cudaStream_t s, cudaStream_t s_dw) {
  const int O = nb.d.sizes[0], D = nb.d.sizes[1], H = nb.d.sizes[2], n = nb.d.sizes[3], C = h->iqn_cfg.n_cos;
  const int N = h->iqn_cfg.n, R = B * N, hid = nb.d.hidden_act;
  auto fork = [&]() {  // what `s` has queued so far is complete before the next products on s_dw
    B200RL_CUDA(cudaEventRecord(h->ev_side, s));
    B200RL_CUDA(cudaStreamWaitEvent(s_dw, h->ev_side, 0));
    return 0;
  };
  // dW[nout, nin] = (dY . act'(Y))^T X and db on s_dw
  auto dw = [&](int l, const float* dY, const float* Y, int act, const float* X, int rows, int nout, int nin) {
    GemmArgs g{};
    g.A = dY; g.lda = nout; g.Y = Y; g.ldy = nout; g.act = act;
    g.B = X; g.ldb = nin;
    g.C = nb.grad + nb.dw_off[l]; g.ldc = nin;
    g.M = nout; g.N = nin; g.K = rows;
    g.dbias = nb.grad + nb.db_off[l];
    return gemm<2>(h, g, s_dw);
  };
  // dX[R, nin] = (dY . act'(Y))[R, nout] W[nout, nin] on s
  auto dx = [&](int l, const float* dY, const float* Y, int act, float* dst, int nout, int nin) {
    GemmArgs g{};
    g.A = dY; g.lda = nout; g.Y = Y; g.ldy = nout; g.act = act;
    g.B = nb.params + nb.dw_off[l]; g.ldb = nin;
    g.C = dst; g.ldc = nin;
    g.M = R; g.N = nin; g.K = nout;
    return gemm<1>(h, g, s);
  };
  const int idt = B200RL_ACT_IDENTITY;
  if (fork() || dw(3, dOut, nullptr, idt, p.hid, R, n, H) || dx(3, dOut, nullptr, idt, h->iqn_dhid, n, H)) return 1;
  if (fork() || dw(2, h->iqn_dhid, p.hid, hid, p.z, R, H, D) || dx(2, h->iqn_dhid, p.hid, hid, h->iqn_dz, H, D))
    return 1;
  if (launch(h, iqn_mul_backward_kernel<false>, iqn_mul_backward_kernel<true>, (unsigned)((B * D + GTHREADS - 1) / GTHREADS),
             GTHREADS, 0, s, h->iqn_dz, p.psi, p.phi, B, N, D, h->iqn_dphi, h->iqn_dpsi))
    return 1;
  if (fork() || dw(1, h->iqn_dphi, p.phi, hid, cos, R, D, C) || dw(0, h->iqn_dpsi, p.psi, hid, x, B, D, O)) return 1;
  B200RL_CUDA(cudaEventRecord(h->ev_side, s_dw));
  B200RL_CUDA(cudaStreamWaitEvent(s, h->ev_side, 0));
  return 0;
}

int adam_net(const b200rl_offpolicy* h, NetBuf& nb, const float2* table, int idx, double b1, double b2, double eps,
             cudaStream_t s) {
  return adam_step_table(nb.flat, nb.flat_grad, nb.m, nb.v, nb.P_flat, table, idx, b1, b2, eps, s, h->K,
                         h->lane_stride);
}

}  // namespace

// The engine of create_group (ic = dc = tc = NULL), of create_iqn (ic = the IQN counts, config algo 4), of create_d4pg
// (dc = the support, config algo 6), of create_tqc (tc = the quantile counts, config algo 7), of create_cql (cc, algo
// 8) and of create_iql (vc = the value network, config algo 9)
static int create_engine(const b200rl_offpolicy_config* cfg, const b200rl_iqn_config* ic,
                         const b200rl_d4pg_config* dc, int32_t n_learners, b200rl_offpolicy** out,
                         const b200rl_tqc_config* tc = nullptr, const b200rl_cql_config* cc = nullptr,
                         const b200rl_iql_config* vc = nullptr, const b200rl_redq_config* rq = nullptr,
                         const b200rl_edac_config* ec = nullptr) {
  B200RL_REQUIRE(cfg && out, "offpolicy_create: NULL argument");
  B200RL_REQUIRE(n_learners >= 1 && n_learners <= B200RL_MAX_LEARNERS,
                 "offpolicy_create_group: n_learners must be 1..%d, got %d", B200RL_MAX_LEARNERS, n_learners);
  B200RL_REQUIRE(cfg->n_q == 1 || cfg->n_q == 2, "offpolicy_create: n_q must be 1 (DDPG) or 2 (TD3)");
  B200RL_REQUIRE((cfg->algo >= 0 && cfg->algo <= 3) || cfg->algo == 5 || (cfg->algo == 4 && ic != nullptr) ||
                     (cfg->algo == 6 && dc != nullptr) || (cfg->algo == 7 && tc != nullptr) ||
                     (cfg->algo == 8 && cc != nullptr) || (cfg->algo == 9 && vc != nullptr) ||
                     (cfg->algo == 10 && rq != nullptr) || (cfg->algo == 11 && rq != nullptr && ec != nullptr),
                 "offpolicy_create: algo must be 0 (DDPG / TD3), 1 (SAC), 2 (DQN), 3 (C51) or 5 (discrete SAC), got %d "
                 "(algo 4, IQN, is created by b200rl_offpolicy_create_iqn with its counts, algo 6, D4PG, by "
                 "b200rl_offpolicy_create_d4pg with its support, algo 7, TQC, by b200rl_offpolicy_create_tqc, algo 8, "
                 "CQL, by b200rl_offpolicy_create_cql, algo 9, IQL, by b200rl_offpolicy_create_iql, algo 10, REDQ, by "
                 "b200rl_offpolicy_create_redq, algo 11, EDAC, by b200rl_offpolicy_create_edac)", cfg->algo);
  B200RL_REQUIRE(ic == nullptr || cfg->algo == 4, "offpolicy_create_iqn: the config's algo must be 4 (IQN), got %d",
                 cfg->algo);
  B200RL_REQUIRE(dc == nullptr || cfg->algo == 6, "offpolicy_create_d4pg: the config's algo must be 6 (D4PG), got %d",
                 cfg->algo);
  B200RL_REQUIRE(tc == nullptr || cfg->algo == 7, "offpolicy_create_tqc: the config's algo must be 7 (TQC), got %d",
                 cfg->algo);
  B200RL_REQUIRE(cc == nullptr || cfg->algo == 8, "offpolicy_create_cql: the config's algo must be 8 (CQL), got %d",
                 cfg->algo);
  B200RL_REQUIRE(vc == nullptr || cfg->algo == 9, "offpolicy_create_iql: the config's algo must be 9 (IQL), got %d",
                 cfg->algo);
  B200RL_REQUIRE(rq == nullptr || cfg->algo == 10 || ec != nullptr, "offpolicy_create_redq: the config's algo must "
                 "be 10 (REDQ), got %d", cfg->algo);
  // SAC's policy over an ensemble of N critics (EDAC: create_edac passes M = N)
  const bool redq = (cfg->algo == 10 || cfg->algo == 11) && rq != nullptr;
  const int RN = redq ? rq->n_critics : 0;
  if (redq) {
    B200RL_REQUIRE(cfg->n_q == 2, "offpolicy_create_redq: REDQ needs n_q = 2 (its first two critics are the train "
                   "call's q1 / q2), got %d", cfg->n_q);
    B200RL_REQUIRE(cfg->dueling_k == 0 && cfg->noisy_layers == 0, "offpolicy_create_redq: REDQ takes neither "
                   "dueling_k nor noisy_layers: dueling and noisy networks are not implemented for it");
    B200RL_REQUIRE(RN >= 2 && RN <= REDQ_MAX_CRITICS, "offpolicy_create_redq: n_critics must be 2..%d, got %d",
                   REDQ_MAX_CRITICS, RN);
    B200RL_REQUIRE(rq->n_min >= 1 && rq->n_min <= RN, "offpolicy_create_redq: n_min must be 1..n_critics = %d, got %d",
                   RN, rq->n_min);
    const b200rl_mlp_desc &p = cfg->policy, &q = cfg->q;
    const int O_ = p.sizes[0], A_ = q.sizes[0] - O_;
    B200RL_REQUIRE(b200rl_mlp_param_count(&p) > 0 && A_ >= 1 && p.sizes[p.n_layers] == 2 * A_,
                   "offpolicy_create_redq: the policy must map [obs %d] -> [mean | log_std] = 2 x %d values, got %d -> "
                   "%d", O_, A_, O_, p.sizes[p.n_layers]);
    B200RL_REQUIRE(b200rl_mlp_param_count(&q) > 0 && q.sizes[q.n_layers] == 1, "offpolicy_create_redq: the critics "
                   "must map [obs %d + act %d] -> 1, got %d -> %d", O_, A_, q.sizes[0], q.sizes[q.n_layers]);
  }
  const bool iql = cfg->algo == 9 && vc != nullptr;  // policy, twin critics and a trained value network in slot 3
  int64_t Pv = 0;
  if (iql) {
    B200RL_REQUIRE(cfg->n_q == 2, "offpolicy_create_iql: IQL needs n_q = 2 (twin critics), got %d", cfg->n_q);
    B200RL_REQUIRE(cfg->dueling_k == 0 && cfg->noisy_layers == 0, "offpolicy_create_iql: IQL takes neither dueling_k "
                   "nor noisy_layers: dueling and noisy networks are not implemented for it");
    const b200rl_mlp_desc &p = cfg->policy, &q = cfg->q, &v = vc->value;
    Pv = b200rl_mlp_param_count(&v);
    const int O_ = p.sizes[0], A_ = q.sizes[0] - O_;
    B200RL_REQUIRE(b200rl_mlp_param_count(&p) > 0 && A_ >= 1 && p.sizes[p.n_layers] == 2 * A_,
                   "offpolicy_create_iql: the policy must map [obs %d] -> [mean | log_std] = 2 x %d values, got %d -> %d",
                   O_, A_, O_, p.sizes[p.n_layers]);
    B200RL_REQUIRE(b200rl_mlp_param_count(&q) > 0 && q.sizes[q.n_layers] == 1, "offpolicy_create_iql: the critics must "
                   "map [obs %d + act %d] -> 1, got %d -> %d", O_, A_, q.sizes[0], q.sizes[q.n_layers]);
    B200RL_REQUIRE(Pv > 0 && v.sizes[0] == O_ && v.sizes[v.n_layers] == 1, "offpolicy_create_iql: the value network "
                   "must map [obs %d] -> 1, got %d -> %d", O_, v.sizes[0], v.sizes[v.n_layers]);
  }
  const bool cql = cfg->algo == 8 && cc != nullptr;  // a SAC engine whose critic step runs on stacked sampled rows
  const int CN = cql ? cc->n_actions : 0;
  if (cql) {
    B200RL_REQUIRE(cfg->n_q == 2, "offpolicy_create_cql: CQL needs n_q = 2 (twin soft critics), got %d", cfg->n_q);
    B200RL_REQUIRE(cfg->dueling_k == 0 && cfg->noisy_layers == 0, "offpolicy_create_cql: CQL takes neither dueling_k "
                   "nor noisy_layers: dueling and noisy networks are not implemented for it");
    B200RL_REQUIRE(CN >= 1 && CN <= CQL_MAX_ACTIONS, "offpolicy_create_cql: n_actions must be 1..%d, got %d",
                   CQL_MAX_ACTIONS, CN);
    B200RL_REQUIRE(cc->lagrange == 0 || cc->lagrange == 1, "offpolicy_create_cql: lagrange must be 0 or 1, got %d",
                   cc->lagrange);
    B200RL_REQUIRE((long long)cfg->max_minibatch * (1 + 3 * CN) <= 65535LL * GT, "offpolicy_create_cql: max_minibatch "
                   "%d x %d stacked rows per row exceed the %lld network rows of one pass", cfg->max_minibatch,
                   1 + 3 * CN, 65535LL * GT);
  }
  const bool tqc = cfg->algo == 7 && tc != nullptr;  // a SAC engine with quantile critics
  const int TM = tqc ? tc->n_quantiles : 0, TD = tqc ? tc->n_drop_per_net : 0;
  if (tqc) {
    B200RL_REQUIRE(cfg->n_q == 2, "offpolicy_create_tqc: TQC needs n_q = 2 (two quantile critics), got %d", cfg->n_q);
    B200RL_REQUIRE(cfg->dueling_k == 0 && cfg->noisy_layers == 0, "offpolicy_create_tqc: TQC takes neither dueling_k "
                   "nor noisy_layers: dueling and noisy networks are not implemented for it");
    B200RL_REQUIRE(TM >= 1 && TM <= TQC_MAX_QUANTILES, "offpolicy_create_tqc: n_quantiles must be 1..%d, got %d",
                   TQC_MAX_QUANTILES, TM);
    B200RL_REQUIRE(TD >= 0 && TD <= TM - 1, "offpolicy_create_tqc: n_drop_per_net must be 0..n_quantiles - 1 = %d, "
                   "got %d", TM - 1, TD);
  }
  const bool sac = cfg->algo == 1 || tqc || cql || redq, c51 = cfg->algo == 3, iqn = cfg->algo == 4, dsac = cfg->algo == 5;
  const bool d4pg = cfg->algo == 6 && dc != nullptr;
  const int NA = d4pg ? dc->n_atoms : 0;
  if (d4pg) {
    B200RL_REQUIRE(cfg->n_q == 1, "offpolicy_create_d4pg: D4PG needs n_q = 1 (one distributional critic), got %d",
                   cfg->n_q);
    B200RL_REQUIRE(cfg->dueling_k == 0 && cfg->noisy_layers == 0, "offpolicy_create_d4pg: D4PG takes neither "
                   "dueling_k nor noisy_layers: dueling and noisy networks are not implemented for it");
    B200RL_REQUIRE(NA >= 2 && NA <= C51_MAX_ATOMS, "offpolicy_create_d4pg: n_atoms must be 2..%d, got %d",
                   C51_MAX_ATOMS, NA);
    B200RL_REQUIRE(std::isfinite(dc->v_min) && std::isfinite(dc->v_max) && dc->v_min < dc->v_max,
                   "offpolicy_create_d4pg: the support needs finite v_min < v_max, got [%g, %g]", dc->v_min, dc->v_max);
    B200RL_REQUIRE(c51_warps(1, NA) >= 1, "offpolicy_create_d4pg: %d atoms are too many for the head's shared memory",
                   NA);
  }
  const bool dqn = cfg->algo == 2 || c51 || iqn;  // C51 and IQN are DQN engines
  B200RL_REQUIRE(!sac || cfg->n_q == 2, "offpolicy_create: SAC needs n_q = 2 (twin soft critics), got %d", cfg->n_q);
  B200RL_REQUIRE(!dsac || cfg->n_q == 2, "offpolicy_create: discrete SAC (algo = 5) needs n_q = 2 (twin soft critics), "
                 "got %d", cfg->n_q);
  B200RL_REQUIRE(!dsac || (cfg->dueling_k == 0 && cfg->noisy_layers == 0), "offpolicy_create: discrete SAC (algo = 5) "
                 "takes neither dueling_k nor noisy_layers: dueling and noisy networks are not implemented for it");
  B200RL_REQUIRE(!dqn || cfg->n_q == 1, "offpolicy_create: DQN needs n_q = 1 (one Q network), got %d", cfg->n_q);
  B200RL_REQUIRE(cfg->max_minibatch >= 1 && cfg->max_minibatch <= 65536 && cfg->max_steps >= 1,
                 "offpolicy_create: bad capacities");
  if (dqn) {
    const b200rl_mlp_desc zero{};
    B200RL_REQUIRE(memcmp(&cfg->policy, &zero, sizeof(zero)) == 0,
                   "offpolicy_create: DQN has no policy network: the policy description must be zeroed");
  }
  int64_t Pp = dqn ? 0 : b200rl_mlp_param_count(&cfg->policy), Pq = b200rl_mlp_param_count(&cfg->q);
  B200RL_REQUIRE((dqn || Pp > 0) && Pq > 0, "offpolicy_create: invalid MLP description");
  const int DK = cfg->dueling_k;
  B200RL_REQUIRE(DK == 0 || dqn, "offpolicy_create: dueling_k must be 0 unless algo = 2 (DQN / QR-DQN) or 3 (C51), got "
                 "%d", DK);
  if (DK != 0) {
    const b200rl_mlp_desc& d = cfg->q;
    B200RL_REQUIRE(DK >= 1, "offpolicy_create: dueling_k must be >= 1 (or 0: a plain MLP), got %d", DK);
    B200RL_REQUIRE(d.n_layers == 3, "offpolicy_create: a dueling Q network is described as [obs, h_trunk, h_stream, "
                   "n_actions x dueling_k] (3 layers), got %d layers", d.n_layers);
    B200RL_REQUIRE(d.sizes[3] % DK == 0, "offpolicy_create: the dueling Q network's output width %d is not n_actions x "
                   "dueling_k for dueling_k = %d", d.sizes[3], DK);
    B200RL_REQUIRE(d.out_act == B200RL_ACT_IDENTITY, "offpolicy_create: a dueling Q network's stream outputs must be "
                   "linear (out_act identity)");
    // trunk, value hidden, value out, advantage hidden, advantage out
    Pq = (int64_t)d.sizes[1] * (d.sizes[0] + 1) + 2 * (int64_t)d.sizes[2] * (d.sizes[1] + 1) +
         (int64_t)(DK + d.sizes[3]) * (d.sizes[2] + 1);
  }
  const int IC = iqn ? ic->n_cos : 0, IN = iqn ? ic->n : 0, INt = iqn ? ic->n_target : 0, IK = iqn ? ic->k : 0;
  if (iqn) {
    const b200rl_mlp_desc& d = cfg->q;
    B200RL_REQUIRE(DK == 0 && cfg->noisy_layers == 0, "offpolicy_create: IQN takes neither dueling_k nor noisy_layers: "
                   "dueling and noisy IQN networks are not implemented");
    B200RL_REQUIRE(IC >= 1 && IC <= IQN_MAX && IN >= 1 && IN <= IQN_MAX && INt >= 1 && INt <= IQN_MAX && IK >= 1 &&
                   IK <= IQN_MAX, "offpolicy_create: the IQN counts n_cos, n, n_target and k must each be 1..%d, got "
                   "%d, %d, %d, %d", IQN_MAX, IC, IN, INt, IK);
    B200RL_REQUIRE(d.n_layers == 3, "offpolicy_create: an IQN network is described as [obs, d, h, n_actions] (3 "
                   "layers), got %d layers", d.n_layers);
    B200RL_REQUIRE(d.out_act == B200RL_ACT_IDENTITY, "offpolicy_create: an IQN network's output must be linear "
                   "(out_act identity)");
    B200RL_REQUIRE(iqn_smem_floats(d.sizes[3], IN, INt) <= C51_SMEM_FLOATS, "offpolicy_create: %d actions are too "
                   "many for the IQN head's shared memory", d.sizes[3]);
    B200RL_REQUIRE((long long)cfg->max_minibatch * std::max(IN, INt + IK) <= 65535LL * GT, "offpolicy_create: "
                   "max_minibatch %d x %d fractions per row exceed the %lld network rows of one pass",
                   cfg->max_minibatch, std::max(IN, INt + IK), 65535LL * GT);
    // psi, phi, head hidden, head out
    Pq = (int64_t)d.sizes[1] * (d.sizes[0] + 1) + (int64_t)d.sizes[1] * (IC + 1) +
         (int64_t)d.sizes[2] * (d.sizes[1] + 1) + (int64_t)d.sizes[3] * (d.sizes[2] + 1);
  }
  const unsigned NM = (unsigned)cfg->noisy_layers;
  const int n_lin = DK != 0 ? 5 : cfg->q.n_layers;  // the Q network's Linear layers in flat order
  B200RL_REQUIRE(NM == 0 || dqn, "offpolicy_create: noisy_layers must be 0 unless algo = 2 (DQN / QR-DQN) or 3 (C51), "
                 "got 0x%x", NM);
  B200RL_REQUIRE((NM >> n_lin) == 0, "offpolicy_create: noisy_layers 0x%x has bits beyond the Q network's %d Linear "
                 "layers", NM, n_lin);
  const int O = dqn ? cfg->q.sizes[0] : cfg->policy.sizes[0], P_out = cfg->policy.sizes[cfg->policy.n_layers];
  // SAC: the policy outputs [mean | log_std], 2A wide; DQN: the action column holds the index (1 wide)
  const int A = dqn || dsac ? 1 : sac || iql ? cfg->q.sizes[0] - O : P_out;
  B200RL_REQUIRE(!sac || (A >= 1 && P_out == 2 * A),
                 "offpolicy_create: the SAC policy must output [mean | log_std] = 2 x %d values, got %d", A, P_out);
  if (dsac) {  // policy and critics both map obs -> [n]
    const int nq = cfg->q.sizes[cfg->q.n_layers];
    B200RL_REQUIRE(cfg->q.sizes[0] == O && nq == P_out && nq >= 2, "offpolicy_create: discrete SAC (algo = 5) needs a "
                   "policy [obs, ..., n] and critics [obs, ..., n] with n >= 2 actions, got policy %d -> %d and critics "
                   "%d -> %d", O, P_out, cfg->q.sizes[0], nq);
  }
  B200RL_REQUIRE(dqn || dsac || d4pg || tqc || (cfg->q.sizes[0] == O + A && cfg->q.sizes[cfg->q.n_layers] == 1),
                 "offpolicy_create: Q network must map [obs %d + act %d] -> 1", O, A);
  B200RL_REQUIRE(!tqc || (cfg->q.sizes[0] == O + A && cfg->q.sizes[cfg->q.n_layers] == TM),
                 "offpolicy_create_tqc: the critics must map [obs %d + act %d] -> %d quantiles, got %d -> %d", O, A, TM,
                 cfg->q.sizes[0], cfg->q.sizes[cfg->q.n_layers]);
  B200RL_REQUIRE(!d4pg || (cfg->q.sizes[0] == O + A && cfg->q.sizes[cfg->q.n_layers] == NA),
                 "offpolicy_create_d4pg: the critic must map [obs %d + act %d] -> %d atoms' logits, got %d -> %d", O, A,
                 NA, cfg->q.sizes[0], cfg->q.sizes[cfg->q.n_layers]);
  B200RL_REQUIRE(device_sm_count() > 0, "offpolicy_create: no CUDA device");
  b200rl_offpolicy* h = new b200rl_offpolicy();
  h->cfg = *cfg;
  h->K = n_learners;
  h->O = O;
  h->A = A;
  h->sac = sac;
  h->dsac = dsac;
  h->dqn = dqn;
  h->c51 = c51;
  h->iqn = iqn;
  if (iqn) h->iqn_cfg = *ic;
  h->d4pg = d4pg;
  if (d4pg) h->d4pg_cfg = *dc, h->d4pg_cfg.reserved = 0;
  h->tqc = tqc;
  if (tqc) h->tqc_cfg = *tc;
  h->cql = cql;
  if (cql) h->cql_cfg = *cc;
  h->iql = iql;
  h->redq = redq;
  if (redq) h->redq_cfg = *rq;
  h->edac = ec != nullptr;
  if (ec) h->edac_eta = ec->eta;
  h->noisy = NM != 0;
  int rc = 0;
  int maxw = O + A;
  for (int i = 0; i < n_nets(h); ++i) {
    NetBuf& nb = h->net[i];
    const bool pol = redq ? i == 0 : i == 0 || i == 3;
    nb.d = iql && i == 3 ? vc->value : pol ? cfg->policy : cfg->q;
    nb.P = iql && i == 3 ? Pv : pol ? Pp : Pq;
    int off = 0;
    for (int l = 0; l < nb.d.n_layers; ++l) {
      nb.w_off[l] = off;
      off += nb.d.sizes[l + 1] * nb.d.sizes[l];
      nb.b_off[l] = off;
      off += nb.d.sizes[l + 1];
      maxw = nb.d.sizes[l + 1] > maxw ? nb.d.sizes[l + 1] : maxw;
    }
    if (DK != 0 && (i == 1 || i == 4)) {  // the activation stacks also hold [rows, 2 h2] and [rows, K + n K]
      const int O_ = nb.d.sizes[0], h1 = nb.d.sizes[1], h2 = nb.d.sizes[2], nK = nb.d.sizes[3];
      const int ins[5] = {O_, h1, h2, h1, h2}, outs[5] = {h1, h2, DK, h2, nK};
      nb.duel_k = DK;
      off = 0;
      for (int l = 0; l < 5; ++l) {
        nb.dw_off[l] = off;
        off += outs[l] * ins[l];
        nb.db_off[l] = off;
        off += outs[l];
      }
      maxw = std::max(maxw, std::max(2 * h2, DK + nK));
    }
    if (iqn && (i == 1 || i == 4)) {
      const int ins[4] = {nb.d.sizes[0], IC, nb.d.sizes[1], nb.d.sizes[2]};
      const int outs[4] = {nb.d.sizes[1], nb.d.sizes[1], nb.d.sizes[2], nb.d.sizes[3]};
      off = 0;
      for (int l = 0; l < 4; ++l) {
        nb.dw_off[l] = off;
        off += outs[l] * ins[l];
        nb.db_off[l] = off;
        off += outs[l];
      }
    }
    nb.P_flat = nb.P;
    if (NM != 0 && (i == 1 || i == 4)) {  // the noisy vector: [W_mu, W_sigma, b_mu, b_sigma] per noisy layer, [W, b] else
      NoisyLayout& lay = h->noisy_lay;
      const b200rl_mlp_desc& d = nb.d;
      const int ins[5] = {d.sizes[0], d.sizes[1], d.sizes[2], d.sizes[1], d.sizes[2]};
      const int outs[5] = {d.sizes[1], d.sizes[2], DK, d.sizes[2], d.sizes[3]};
      lay = NoisyLayout{};
      lay.n = n_lin, lay.mask = NM;
      int fo = 0;
      for (int l = 0; l < n_lin; ++l) {
        const int in = DK ? ins[l] : d.sizes[l], out = DK ? outs[l] : d.sizes[l + 1], w = (NM >> l) & 1u ? 2 : 1;
        lay.in[l] = in, lay.out[l] = out;
        lay.cw[l] = DK ? nb.dw_off[l] : nb.w_off[l], lay.cb[l] = DK ? nb.db_off[l] : nb.b_off[l];
        lay.fw[l] = fo, fo += w * out * in;
        lay.fb[l] = fo, fo += w * out;
        if (w == 2) lay.eo[l] = lay.E, lay.E += in + out;
        lay.tiles[l + 1] = lay.tiles[l] + ((out + NOISY_TR - 1) / NOISY_TR) * ((in + NOISY_TC - 1) / NOISY_TC);
      }
      nb.P_flat = fo;
    }
    if (cfg->n_q == 1 && (i == 2 || i == 5)) continue;
    if ((sac || dsac) && !redq && i == 3) continue;  // SAC has no target policy
    if (dqn && (i == 0 || i == 3)) continue;  // DQN has no policy
    nb.present = true;
    if (i < n_opt(h)) rc |= oalloc(h, &nb.grad, (size_t)nb.P);  // REDQ: critic k's at k state_pad(P) after critic 1's
    if (nb.P_flat != nb.P) {  // the composed network beside the noisy vector in the slab (and its gradient)
      rc |= oalloc(h, &nb.params, (size_t)nb.P);
      if (i < 3) rc |= oalloc(h, &nb.flat_grad, (size_t)nb.P_flat);
    }
  }
  // parameters and Adam state live in ONE slab in the order of the state blob (b200rl_offpolicy_get_state): the
  // parameters of networks 0..5, then exp_avg / exp_avg_sq of optimizers 0..2 (0..3 for IQL), every segment padded to
  // 64 floats (REDQ: networks 0..2N, optimizers 0..N)
  {
    int64_t n = 0;
    for (int i = 0; i < n_nets(h); ++i)
      if (h->net[i].present) n += state_pad(h->net[i].P_flat);
    for (int i = 0; i < n_opt(h); ++i)
      if (h->net[i].present) n += 2 * state_pad(h->net[i].P_flat);
    h->state_n = n;
    rc |= oalloc(h, &h->state, (size_t)n);
  }
  h->maxw = maxw;
  const size_t B = (size_t)cfg->max_minibatch, S = (size_t)cfg->max_steps;
  const size_t R = B * (size_t)(1 + 3 * CN);  // CQL's stacked critic rows; the gradient buffers are that deep
  const size_t RD = cql ? R : B;
  rc |= oalloc(h, &h->obs, S * B * O);
  rc |= oalloc(h, &h->act, S * B * A);
  rc |= oalloc(h, &h->rew, S * B);
  rc |= oalloc(h, &h->nobs, S * B * O);
  rc |= oalloc(h, &h->done, S * B);
  rc |= oalloc(h, &h->eps, iql ? 0 : (sac ? 2 : 1) * S * B * A);  // IQL draws no noise
  for (int k = 0; k < 5; ++k)
    for (int l = 0; l <= B200RL_MAX_LAYERS; ++l) rc |= oalloc(h, &h->acts[k][l], B * (size_t)maxw);
  for (int l = 0; l <= B200RL_MAX_LAYERS; ++l) rc |= oalloc(h, &h->acts_tq[l], B * (size_t)maxw);
  rc |= oalloc(h, &h->x_cat, B * (size_t)(O + A));
  rc |= oalloc(h, &h->x_cat2, B * (size_t)(O + A));
  // discrete SAC: [B, n] per critic; D4PG: [B, N] (the target critic's logits, the output gradient); TQC: [B, M]
  const size_t n_dq = dsac || d4pg || tqc ? (size_t)cfg->q.sizes[cfg->q.n_layers] : 1;
  rc |= oalloc(h, &h->qt1, B * n_dq);
  rc |= oalloc(h, &h->qt2, B * (tqc ? n_dq : 1));
  rc |= oalloc(h, &h->dq, RD * n_dq);
  rc |= oalloc(h, &h->dbuf0, RD * (size_t)maxw);
  rc |= oalloc(h, &h->dbuf1, RD * (size_t)maxw);
  rc |= oalloc(h, &h->dbuf2, RD * (size_t)maxw);
  rc |= oalloc(h, &h->dbuf3, RD * (size_t)maxw);
  rc |= oalloc(h, &h->dq2, RD * n_dq);
  rc |= oalloc(h, &h->out_q1, S * B * (redq ? RN : 1));
  rc |= oalloc(h, &h->out_q2, S * B);
  rc |= oalloc(h, &h->out_l1, S * (redq ? RN : 1));
  rc |= oalloc(h, &h->out_l2, S);
  rc |= oalloc(h, &h->out_lp, S);
  rc |= oalloc(h, &h->adam_tab, adam_tab_len(h));
  rc |= oalloc(h, &h->idx, S * B);
  if (h->noisy) rc |= oalloc(h, &h->noisy_draws, S * 2 * (size_t)h->noisy_lay.E);
  if (sac) {
    rc |= oalloc(h, &h->sac_act_next, B * (size_t)A);
    rc |= oalloc(h, &h->sac_logp_next, B);
    rc |= oalloc(h, &h->sac_act, B * (size_t)A);
    rc |= oalloc(h, &h->sac_logp, B);
    rc |= oalloc(h, &h->sac_dout, B * (size_t)(2 * A));
    rc |= oalloc(h, &h->sac_alpha, S + 1);
    rc |= oalloc(h, &h->sac_state, 3);
    rc |= oalloc(h, &h->out_logp, S);
  }
  if (tqc) {
    rc |= oalloc(h, &h->tqc_y, B * (size_t)(2 * (TM - TD)));
    rc |= oalloc(h, &h->tqc_row_loss, 2 * B);
    rc |= oalloc(h, &h->tqc_sync, 2);
  }
  if (cql) {
    rc |= oalloc(h, &h->cql_draws, S * 3 * B * CN * A);
    rc |= oalloc(h, &h->cql_x, R * (O + A));
    rc |= oalloc(h, &h->cql_logp, B * 3 * CN);
    for (int k = 0; k < 2; ++k)
      for (int l = 1; l <= cfg->q.n_layers; ++l) rc |= oalloc(h, &h->cql_acts[k][l], R * (size_t)maxw);
    rc |= oalloc(h, &h->cql_row_p, 2 * B);
    rc |= oalloc(h, &h->cql_sync, 2);
    rc |= oalloc(h, &h->cql_gap, 2 * S);
    rc |= oalloc(h, &h->cql_ap, S + 1);
    rc |= oalloc(h, &h->cql_ap_state, 3);
    rc |= oalloc(h, &h->cql_zero, 1);
  }
  if (redq) {
    const size_t M = (size_t)rq->n_min;
    rc |= oalloc(h, &h->redq_sub, S * M);
    for (int l = 1; l <= cfg->q.n_layers; ++l) {
      rc |= oalloc(h, &h->redq_acts[l], RN * B * (size_t)maxw);
      rc |= oalloc(h, &h->redq_tacts[l], M * B * (size_t)maxw);
    }
    rc |= oalloc(h, &h->redq_d0, RN * B * (size_t)maxw);
    rc |= oalloc(h, &h->redq_d1, RN * B * (size_t)maxw);
    rc |= oalloc(h, &h->redq_dq, RN * B);
    rc |= oalloc(h, &h->redq_dx, RN * B * (size_t)(O + A));
    rc |= oalloc(h, &h->redq_qmin, B);
  }
  if (ec != nullptr && ec->eta > 0.0) {
    for (int l = 1; l < cfg->q.n_layers; ++l) {
      rc |= oalloc(h, &h->edac_e[l], RN * B * (size_t)maxw);
      rc |= oalloc(h, &h->edac_t[l], RN * B * (size_t)maxw);
    }
    rc |= oalloc(h, &h->edac_ones, B);
    rc |= oalloc(h, &h->edac_g, RN * B * (size_t)A);
    rc |= oalloc(h, &h->edac_u, RN * B * (size_t)A);
    rc |= oalloc(h, &h->edac_grad, RN * (size_t)state_pad(h->net[1].P));
  }
  if (ec != nullptr) rc |= oalloc(h, &h->edac_div, S);
  if (iql) {
    rc |= oalloc(h, &h->dbuf4, B * (size_t)maxw);
    rc |= oalloc(h, &h->dbuf5, B * (size_t)maxw);
    rc |= oalloc(h, &h->iql_dv, B);
    rc |= oalloc(h, &h->iql_dout, B * (size_t)(2 * A));
    rc |= oalloc(h, &h->iql_zero, B);
    rc |= oalloc(h, &h->out_vl, S);
    rc |= oalloc(h, &h->out_vm, S);
    rc |= oalloc(h, &h->out_wm, S);
  }
  if (dsac) {
    rc |= oalloc(h, &h->sac_logp, B);
    rc |= oalloc(h, &h->sac_dout, B * n_dq);
    rc |= oalloc(h, &h->sac_alpha, S + 1);
    rc |= oalloc(h, &h->sac_state, 3);
    rc |= oalloc(h, &h->out_logp, S);
    rc |= oalloc(h, &h->dqn_bad, S);
  }
  if (dqn) {
    rc |= oalloc(h, &h->dqn_dout, B * (size_t)cfg->q.sizes[cfg->q.n_layers] * (iqn ? IN : 1));
    rc |= oalloc(h, &h->dqn_bad, S);
    rc |= oalloc(h, &h->per_w, S * B);
    rc |= oalloc(h, &h->per_newp, S * B);
    rc |= oalloc(h, &h->per_absd, B);
    rc |= oalloc(h, &h->per_bad, S);
    rc |= oalloc(h, &h->nstep_disc, S * B);
    rc |= oalloc(h, &h->nstep_rows, S * B);
    rc |= oalloc(h, &h->c51_row_loss, B);  // C51's and QR-DQN's heads
    rc |= oalloc(h, &h->c51_sync, 2);
  }
  if (d4pg) {
    rc |= oalloc(h, &h->dqn_bad, S);  // the head's invalid-row count, always 0 (no action column)
    rc |= oalloc(h, &h->per_w, S * B);
    rc |= oalloc(h, &h->per_newp, S * B);
    rc |= oalloc(h, &h->per_absd, B);
    rc |= oalloc(h, &h->per_bad, S);
    rc |= oalloc(h, &h->nstep_disc, S * B);
    rc |= oalloc(h, &h->nstep_rows, S * B);
    rc |= oalloc(h, &h->c51_row_loss, B);
    rc |= oalloc(h, &h->c51_sync, 2);
  }
  if (c51 || d4pg) rc |= oalloc(h, &h->c51_support, C51_MAX_ATOMS);
  if (iqn) {
    const size_t D = cfg->q.sizes[1], H = cfg->q.sizes[2], n = cfg->q.sizes[3];
    rc |= oalloc(h, &h->iqn_taus, S * B * (IN + INt + IK));
    rc |= oalloc(h, &h->iqn_cos_q, B * IN * (size_t)IC);
    rc |= oalloc(h, &h->iqn_cos_t, B * (INt + IK) * (size_t)IC);
    rc |= oalloc(h, &h->iqn_cos_n, B * IK * (size_t)IC);
    const int M[3] = {IN, INt + IK, IK};
    for (int k = 0; k < 3; ++k) {
      const size_t R = B * M[k];
      IqnPass& p = h->iqn_pass[k];
      rc |= oalloc(h, &p.psi, B * D);
      rc |= oalloc(h, &p.phi, R * D);
      rc |= oalloc(h, &p.z, R * D);
      rc |= oalloc(h, &p.hid, R * H);
      rc |= oalloc(h, &p.out, R * n);
    }
    rc |= oalloc(h, &h->iqn_dhid, B * IN * H);
    rc |= oalloc(h, &h->iqn_dz, B * IN * D);
    rc |= oalloc(h, &h->iqn_dphi, B * IN * D);
    rc |= oalloc(h, &h->iqn_dpsi, B * D);
  }
  rc |= arena_commit(h);
  if (rc == 0) {
    float* q = h->state;
    for (int i = 0; i < n_nets(h); ++i) {
      NetBuf& nb = h->net[i];
      if (!nb.present) continue;
      nb.flat = q;
      if (nb.P_flat == nb.P) nb.params = q, nb.flat_grad = nb.grad;
      q += state_pad(nb.P_flat);
    }
    for (int i = 0; i < n_opt(h); ++i)
      if (h->net[i].present) {
        h->net[i].m = q;
        q += state_pad(h->net[i].P_flat);
        h->net[i].v = q;
        q += state_pad(h->net[i].P_flat);
      }
  }
  if (!rc && cudaMallocHost(reinterpret_cast<void**>(&h->h_adam_tab), h->K * adam_tab_len(h) * sizeof(float2)) != cudaSuccess)
    rc = 1;
  if (!rc && cudaStreamCreateWithFlags(&h->gs, cudaStreamNonBlocking) != cudaSuccess) rc = 1;
  if (!rc && cudaEventCreateWithFlags(&h->ev, cudaEventDisableTiming) != cudaSuccess) rc = 1;
  if (!rc && cudaStreamCreateWithFlags(&h->s2, cudaStreamNonBlocking) != cudaSuccess) rc = 1;
  if (!rc && cudaStreamCreateWithFlags(&h->s3, cudaStreamNonBlocking) != cudaSuccess) rc = 1;
  if (!rc && cudaStreamCreateWithFlags(&h->s4, cudaStreamNonBlocking) != cudaSuccess) rc = 1;
  if (!rc && cudaEventCreateWithFlags(&h->ev_side, cudaEventDisableTiming) != cudaSuccess) rc = 1;
  if (!rc && cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming) != cudaSuccess) rc = 1;
  if (!rc && cudaEventCreateWithFlags(&h->ev_join, cudaEventDisableTiming) != cudaSuccess) rc = 1;
  if (!rc && d4pg) {  // the support, z_i = float32(v_min + i dz) in double as set_c51 writes it, in every arena
    const double dz = (dc->v_max - dc->v_min) / (NA - 1);
    std::vector<float> z((size_t)h->K * C51_MAX_ATOMS, 0.f);
    for (int k = 0; k < h->K; ++k)
      for (int i = 0; i < NA; ++i) z[(size_t)k * C51_MAX_ATOMS + i] = (float)(dc->v_min + i * dz);
    if (cudaMemcpy2D(h->c51_support, h->lane_stride, z.data(), C51_MAX_ATOMS * sizeof(float),
                     C51_MAX_ATOMS * sizeof(float), h->K, cudaMemcpyHostToDevice) != cudaSuccess)
      rc = 1;
  }
  if (!rc && h->edac_ones) {  // EDAC's ones-backward reads dOut = 1 from every arena
    const size_t nb = (size_t)h->cfg.max_minibatch;
    const std::vector<float> ones((size_t)h->K * nb, 1.f);
    if (cudaMemcpy2D(h->edac_ones, h->lane_stride, ones.data(), nb * sizeof(float), nb * sizeof(float), h->K,
                     cudaMemcpyHostToDevice) != cudaSuccess)
      rc = 1;
  }
  if (rc) {
    b200rl_offpolicy_destroy(h);
    return 1;
  }
  *out = h;
  return 0;
}

extern "C" int b200rl_offpolicy_create(const b200rl_offpolicy_config* cfg, b200rl_offpolicy** out) {
  return create_engine(cfg, nullptr, nullptr, 1, out);
}

extern "C" int b200rl_offpolicy_create_group(const b200rl_offpolicy_config* cfg, int32_t n_learners,
                                             b200rl_offpolicy** out) {
  return create_engine(cfg, nullptr, nullptr, n_learners, out);
}

extern "C" int b200rl_offpolicy_create_iqn(const b200rl_offpolicy_config* cfg, const b200rl_iqn_config* iqn,
                                           int32_t n_learners, b200rl_offpolicy** out) {
  B200RL_REQUIRE(iqn, "offpolicy_create_iqn: NULL IQN counts");
  return create_engine(cfg, iqn, nullptr, n_learners, out);
}

extern "C" int b200rl_offpolicy_create_d4pg(const b200rl_offpolicy_config* cfg, const b200rl_d4pg_config* d4pg,
                                            int32_t n_learners, b200rl_offpolicy** out) {
  B200RL_REQUIRE(d4pg, "offpolicy_create_d4pg: NULL D4PG support");
  return create_engine(cfg, nullptr, d4pg, n_learners, out);
}

extern "C" int b200rl_offpolicy_create_tqc(const b200rl_offpolicy_config* cfg, const b200rl_tqc_config* tqc,
                                           int32_t n_learners, b200rl_offpolicy** out) {
  B200RL_REQUIRE(tqc, "offpolicy_create_tqc: NULL TQC counts");
  return create_engine(cfg, nullptr, nullptr, n_learners, out, tqc);
}

extern "C" int b200rl_offpolicy_create_cql(const b200rl_offpolicy_config* cfg, const b200rl_cql_config* cql,
                                           int32_t n_learners, b200rl_offpolicy** out) {
  B200RL_REQUIRE(cql, "offpolicy_create_cql: NULL CQL config");
  return create_engine(cfg, nullptr, nullptr, n_learners, out, nullptr, cql);
}

extern "C" int b200rl_offpolicy_create_redq(const b200rl_offpolicy_config* cfg, const b200rl_redq_config* redq,
                                            int32_t n_learners, b200rl_offpolicy** out) {
  B200RL_REQUIRE(redq, "offpolicy_create_redq: NULL argument");
  return create_engine(cfg, nullptr, nullptr, n_learners, out, nullptr, nullptr, nullptr, redq);
}

extern "C" int b200rl_offpolicy_create_edac(const b200rl_offpolicy_config* cfg, const b200rl_edac_config* edac,
                                            int32_t n_learners, b200rl_offpolicy** out) {
  B200RL_REQUIRE(cfg && edac && out, "offpolicy_create_edac: NULL argument");
  B200RL_REQUIRE(cfg->algo == 11, "offpolicy_create_edac: the config's algo must be 11 (EDAC), got %d", cfg->algo);
  const int N = edac->n_critics;
  B200RL_REQUIRE(N >= 2 && N <= REDQ_MAX_CRITICS, "offpolicy_create_edac: n_critics must be 2..%d, got %d",
                 REDQ_MAX_CRITICS, N);
  B200RL_REQUIRE(std::isfinite(edac->eta) && edac->eta >= 0.0, "offpolicy_create_edac: eta must be finite and >= 0, "
                 "got %g", edac->eta);
  B200RL_REQUIRE(cfg->n_q == 2, "offpolicy_create_edac: EDAC needs n_q = 2 (its first two critics are the train call's "
                 "q1 / q2), got %d", cfg->n_q);
  B200RL_REQUIRE(cfg->dueling_k == 0 && cfg->noisy_layers == 0, "offpolicy_create_edac: EDAC takes neither dueling_k "
                 "nor noisy_layers: dueling and noisy networks are not implemented for it");
  const b200rl_mlp_desc &p = cfg->policy, &q = cfg->q;
  const int O = p.sizes[0], A = q.sizes[0] - O;
  B200RL_REQUIRE(b200rl_mlp_param_count(&p) > 0 && A >= 1 && p.sizes[p.n_layers] == 2 * A, "offpolicy_create_edac: "
                 "the policy must map [obs %d] -> [mean | log_std] = 2 x %d values, got %d -> %d", O, A, O,
                 p.sizes[p.n_layers]);
  B200RL_REQUIRE(b200rl_mlp_param_count(&q) > 0 && q.sizes[q.n_layers] == 1, "offpolicy_create_edac: the critics must "
                 "map [obs %d + act %d] -> 1, got %d -> %d", O, A, q.sizes[0], q.sizes[q.n_layers]);
  // the diversity pass differentiates the critics twice; with ReLU masks the second derivative has no term of its own
  B200RL_REQUIRE(edac->eta == 0.0 || ((q.n_layers == 1 || q.hidden_act == B200RL_ACT_RELU) &&
                                      q.out_act == B200RL_ACT_IDENTITY),
                 "offpolicy_create_edac: eta > 0 needs ReLU hidden layers and an identity output in the critics (the "
                 "diversity term of other activations is not implemented); eta = 0 (SAC-N) takes any");
  const b200rl_redq_config rq{N, N};
  return create_engine(cfg, nullptr, nullptr, n_learners, out, nullptr, nullptr, nullptr, &rq, edac);
}

extern "C" int b200rl_offpolicy_create_iql(const b200rl_offpolicy_config* cfg, const b200rl_iql_config* iql,
                                           int32_t n_learners, b200rl_offpolicy** out) {
  B200RL_REQUIRE(iql, "offpolicy_create_iql: NULL IQL config");
  return create_engine(cfg, nullptr, nullptr, n_learners, out, nullptr, nullptr, iql);
}

extern "C" void b200rl_offpolicy_destroy(b200rl_offpolicy* h) {
  if (!h) return;
  if (h->graph) cudaGraphExecDestroy(h->graph);
  if (h->ev) cudaEventDestroy(h->ev);
  if (h->ev_fork) cudaEventDestroy(h->ev_fork);
  if (h->ev_join) cudaEventDestroy(h->ev_join);
  if (h->ev_side) cudaEventDestroy(h->ev_side);
  if (h->s2) cudaStreamDestroy(h->s2);
  if (h->s3) cudaStreamDestroy(h->s3);
  if (h->s4) cudaStreamDestroy(h->s4);
  if (h->gs) cudaStreamDestroy(h->gs);
  if (h->h_adam_tab) cudaFreeHost(h->h_adam_tab);
  for (void* p : h->allocs) cudaFree(p);
  delete h;
}

extern "C" int b200rl_offpolicy_set_params(b200rl_offpolicy* h, int which, const float* host_flat, int64_t n,
                                           void* stream) {
  B200RL_REQUIRE(h == nullptr || h->K == 1, "offpolicy_set_params: a learner group moves its state with get_state / set_state");
  B200RL_REQUIRE(h && host_flat && which >= 0 && which < n_nets(h) && h->net[which].flat, "offpolicy_set_params: bad net");
  B200RL_REQUIRE(n == h->net[which].P_flat, "offpolicy_set_params: expects %lld floats", (long long)h->net[which].P_flat);
  B200RL_CUDA(cudaMemcpyAsync(h->net[which].flat, host_flat, (size_t)n * 4, cudaMemcpyHostToDevice,
                              static_cast<cudaStream_t>(stream)));
  return 0;
}

extern "C" int b200rl_offpolicy_get_params(b200rl_offpolicy* h, int which, float* host_flat, int64_t n, void* stream) {
  B200RL_REQUIRE(h == nullptr || h->K == 1, "offpolicy_get_params: a learner group moves its state with get_state / set_state");
  B200RL_REQUIRE(h && host_flat && which >= 0 && which < n_nets(h) && h->net[which].flat, "offpolicy_get_params: bad net");
  B200RL_REQUIRE(n == h->net[which].P_flat, "offpolicy_get_params: expects %lld floats", (long long)h->net[which].P_flat);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200RL_CUDA(cudaMemcpyAsync(host_flat, h->net[which].flat, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
  B200RL_CUDA(cudaStreamSynchronize(s));
  return 0;
}

extern "C" int b200rl_offpolicy_set_adam(b200rl_offpolicy* h, int which, const float* exp_avg, const float* exp_avg_sq,
                                         int64_t n, int64_t step, void* stream) {
  B200RL_REQUIRE(h == nullptr || h->K == 1, "offpolicy_set_adam: a learner group moves its state with get_state / set_state");
  B200RL_REQUIRE(h && which >= 0 && which < n_opt(h) && h->net[which].m, "offpolicy_set_adam: bad net");
  NetBuf& nb = h->net[which];
  B200RL_REQUIRE(n == nb.P_flat && step >= 0, "offpolicy_set_adam: expects %lld floats", (long long)nb.P_flat);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (exp_avg) B200RL_CUDA(cudaMemcpyAsync(nb.m, exp_avg, (size_t)n * 4, cudaMemcpyHostToDevice, s));
  else B200RL_CUDA(cudaMemsetAsync(nb.m, 0, (size_t)n * 4, s));
  if (exp_avg_sq) B200RL_CUDA(cudaMemcpyAsync(nb.v, exp_avg_sq, (size_t)n * 4, cudaMemcpyHostToDevice, s));
  else B200RL_CUDA(cudaMemsetAsync(nb.v, 0, (size_t)n * 4, s));
  nb.step[0] = step;
  return 0;
}

extern "C" int b200rl_offpolicy_get_adam(b200rl_offpolicy* h, int which, float* exp_avg, float* exp_avg_sq, int64_t n,
                                         int64_t* step, void* stream) {
  B200RL_REQUIRE(h == nullptr || h->K == 1, "offpolicy_get_adam: a learner group moves its state with get_state / set_state");
  B200RL_REQUIRE(h && which >= 0 && which < n_opt(h) && h->net[which].m && exp_avg && exp_avg_sq && step,
                 "offpolicy_get_adam: bad arguments");
  NetBuf& nb = h->net[which];
  B200RL_REQUIRE(n == nb.P_flat, "offpolicy_get_adam: expects %lld floats", (long long)nb.P_flat);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200RL_CUDA(cudaMemcpyAsync(exp_avg, nb.m, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
  B200RL_CUDA(cudaMemcpyAsync(exp_avg_sq, nb.v, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
  B200RL_CUDA(cudaStreamSynchronize(s));
  *step = nb.step[0];
  return 0;
}

// Whole learner state in ONE call and ONE synchronisation: blob = for every present network 0..5 (REDQ: 0..2N) its
// parameters, then for every optimizer 0..2 (policy, Q1, Q2; IQL: 0..3, V last; REDQ: 0..N) exp_avg and exp_avg_sq;
// steps[n_opt] = Adam step counts.
// A group moves [K][blob] and steps[K][n_opt] with one strided copy (the slab heads every learner's arena).
static int64_t state_floats(const b200rl_offpolicy* h) { return h->K * h->state_n; }

extern "C" int64_t b200rl_offpolicy_state_floats(b200rl_offpolicy* h) { return h ? state_floats(h) : -1; }

// One copy each way: the slab IS the blob.  With a page-locked `blob` the copy is a plain DMA transfer.
extern "C" int b200rl_offpolicy_get_state(b200rl_offpolicy* h, float* blob, int64_t n_floats, int64_t* steps,
                                          void* stream) {
  B200RL_REQUIRE(h && blob && steps && n_floats == state_floats(h), "offpolicy_get_state: bad arguments");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200RL_CUDA(cudaMemcpy2DAsync(blob, (size_t)h->state_n * 4, h->state, h->lane_stride, (size_t)h->state_n * 4, h->K,
                                cudaMemcpyDeviceToHost, s));
  const int no = n_opt(h);
  for (int z = 0; z < h->K; ++z)
    for (int i = 0; i < no; ++i) steps[no * z + i] = h->net[i].m ? h->net[i].step[z] : 0;
  B200RL_CUDA(cudaStreamSynchronize(s));
  return 0;
}

extern "C" int b200rl_offpolicy_set_state(b200rl_offpolicy* h, const float* blob, int64_t n_floats, const int64_t* steps,
                                          void* stream) {
  B200RL_REQUIRE(h && blob && steps && n_floats == state_floats(h), "offpolicy_set_state: bad arguments");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int no = n_opt(h);
  for (int z = 0; z < h->K; ++z)
    for (int i = 0; i < no; ++i)
      if (h->net[i].m) B200RL_REQUIRE(steps[no * z + i] >= 0, "offpolicy_set_state: negative step count");
  B200RL_CUDA(cudaMemcpy2DAsync(h->state, h->lane_stride, blob, (size_t)h->state_n * 4, (size_t)h->state_n * 4, h->K,
                                cudaMemcpyHostToDevice, s));
  for (int z = 0; z < h->K; ++z)
    for (int i = 0; i < no; ++i)
      if (h->net[i].m) h->net[i].step[z] = steps[no * z + i];
  B200RL_CUDA(cudaStreamSynchronize(s));  // `blob` may be reused by the caller right away
  return 0;
}

extern "C" int b200rl_offpolicy_set_sac(b200rl_offpolicy* h, const b200rl_sac_hparams* sp) {
  B200RL_REQUIRE(h && sp, "offpolicy_set_sac: NULL argument");
  B200RL_REQUIRE(!h->iql, "offpolicy_set_sac: an IQL engine (algo = 9) takes b200rl_offpolicy_set_iql, not set_sac");
  B200RL_REQUIRE(h->sac || h->dsac, "offpolicy_set_sac: the engine was not created with algo = 1 (SAC) or 5 (discrete "
                 "SAC)");
  B200RL_REQUIRE(sp->learn_alpha == 0 || sp->learn_alpha == 1, "offpolicy_set_sac: learn_alpha must be 0 or 1");
  B200RL_REQUIRE(sp->log_std_min <= sp->log_std_max, "offpolicy_set_sac: log_std_min > log_std_max");
  h->sac_hp = *sp;
  h->sac_hp.reserved = 0;  // part of the graph cache key
  h->sac_set = true;
  return 0;
}

extern "C" int b200rl_offpolicy_set_dqn(b200rl_offpolicy* h, const b200rl_dqn_hparams* dp) {
  B200RL_REQUIRE(h && dp, "offpolicy_set_dqn: NULL argument");
  B200RL_REQUIRE(!h->dsac, "offpolicy_set_dqn: a discrete SAC engine (algo = 5) takes b200rl_offpolicy_set_sac, not "
                 "set_dqn");
  B200RL_REQUIRE(!h->edac, "offpolicy_set_dqn: an EDAC engine (algo = 11) takes b200rl_offpolicy_set_sac, not set_dqn");
  B200RL_REQUIRE(!h->redq, "offpolicy_set_dqn: a REDQ engine (algo = 10) takes b200rl_offpolicy_set_sac, not set_dqn");
  B200RL_REQUIRE(!h->tqc, "offpolicy_set_dqn: a TQC engine (algo = 7) takes b200rl_offpolicy_set_sac, not set_dqn");
  B200RL_REQUIRE(!h->iql, "offpolicy_set_dqn: an IQL engine (algo = 9) takes b200rl_offpolicy_set_iql, not set_dqn");
  B200RL_REQUIRE(h->dqn, "offpolicy_set_dqn: the engine was not created with algo = 2 (DQN)");
  B200RL_REQUIRE(dp->target_update_interval >= 1, "offpolicy_set_dqn: target_update_interval must be >= 1, got %d",
                 dp->target_update_interval);
  B200RL_REQUIRE(dp->double_q == 0 || dp->double_q == 1, "offpolicy_set_dqn: double_q must be 0 or 1");
  h->dqn_hp = *dp;
  h->dqn_set = true;
  return 0;
}

extern "C" int b200rl_offpolicy_set_c51(b200rl_offpolicy* h, const b200rl_c51_hparams* cp) {
  B200RL_REQUIRE(h && cp, "offpolicy_set_c51: NULL argument");
  B200RL_REQUIRE(!h->dsac, "offpolicy_set_c51: a discrete SAC engine (algo = 5) has no categorical head");
  B200RL_REQUIRE(!h->edac, "offpolicy_set_c51: an EDAC engine (algo = 11) has no categorical head");
  B200RL_REQUIRE(!h->redq, "offpolicy_set_c51: a REDQ engine (algo = 10) has no categorical head");
  B200RL_REQUIRE(!h->tqc, "offpolicy_set_c51: a TQC engine (algo = 7) has no categorical head");
  B200RL_REQUIRE(!h->iql, "offpolicy_set_c51: an IQL engine (algo = 9) has no categorical head");
  B200RL_REQUIRE(!h->d4pg, "offpolicy_set_c51: a D4PG engine (algo = 6) takes its support at create "
                 "(b200rl_offpolicy_create_d4pg)");
  B200RL_REQUIRE(h->c51, "offpolicy_set_c51: the engine was not created with algo = 3 (C51)");
  const int N = cp->n_atoms, width = h->net[1].d.sizes[h->net[1].d.n_layers];
  B200RL_REQUIRE(N >= 2 && N <= C51_MAX_ATOMS, "offpolicy_set_c51: n_atoms must be 2..%d, got %d", C51_MAX_ATOMS, N);
  B200RL_REQUIRE(std::isfinite(cp->v_min) && std::isfinite(cp->v_max) && cp->v_min < cp->v_max,
                 "offpolicy_set_c51: the support needs finite v_min < v_max, got [%g, %g]", cp->v_min, cp->v_max);
  B200RL_REQUIRE(width % N == 0, "offpolicy_set_c51: the Q network's output width %d is not n_actions x n_atoms for "
                 "n_atoms = %d", width, N);
  B200RL_REQUIRE(c51_warps(width / N, N) >= 1, "offpolicy_set_c51: %d actions x %d atoms is too wide for the head's "
                 "shared memory", width / N, N);
  b200rl_c51_hparams hp = *cp;
  hp.reserved = 0;  // part of the graph cache key
  if (h->c51_set && memcmp(&hp, &h->c51_hp, sizeof(hp)) == 0) return 0;  // the support is already in place
  // z_i = float32(v_min + i dz), dz = (v_max - v_min) / (N - 1), in double (not linspace's rounding)
  const double dz = (cp->v_max - cp->v_min) / (N - 1);
  std::vector<float> z((size_t)h->K * C51_MAX_ATOMS, 0.f);  // one row per learner
  for (int k = 0; k < h->K; ++k)
    for (int i = 0; i < N; ++i) z[(size_t)k * C51_MAX_ATOMS + i] = (float)(cp->v_min + i * dz);
  B200RL_CUDA(cudaMemcpy2DAsync(h->c51_support, h->lane_stride, z.data(), C51_MAX_ATOMS * sizeof(float),
                                C51_MAX_ATOMS * sizeof(float), h->K, cudaMemcpyHostToDevice, h->gs));
  B200RL_CUDA(cudaStreamSynchronize(h->gs));
  h->c51_hp = hp;
  h->c51_set = true;
  return 0;
}

extern "C" int b200rl_offpolicy_set_qr(b200rl_offpolicy* h, const b200rl_qr_hparams* qp) {
  B200RL_REQUIRE(h && qp, "offpolicy_set_qr: NULL argument");
  B200RL_REQUIRE(!h->dsac, "offpolicy_set_qr: a discrete SAC engine (algo = 5) has no quantile head");
  B200RL_REQUIRE(!h->iql, "offpolicy_set_qr: an IQL engine (algo = 9) has no quantile head");
  B200RL_REQUIRE(!h->edac, "offpolicy_set_qr: an EDAC engine (algo = 11) has no quantile critics");
  B200RL_REQUIRE(!h->redq, "offpolicy_set_qr: a REDQ engine (algo = 10) has no quantile critics");
  B200RL_REQUIRE(!h->tqc, "offpolicy_set_qr: a TQC engine (algo = 7) takes its quantile counts at create "
                 "(b200rl_offpolicy_create_tqc)");
  B200RL_REQUIRE(h->dqn && !h->c51 && !h->iqn, "offpolicy_set_qr: the engine was not created with algo = 2 (DQN)");
  const int N = qp->n_quantiles, width = h->net[1].d.sizes[h->net[1].d.n_layers];
  B200RL_REQUIRE(N >= 1 && N <= QR_MAX_QUANTILES, "offpolicy_set_qr: n_quantiles must be 1..%d, got %d",
                 QR_MAX_QUANTILES, N);
  B200RL_REQUIRE(width % N == 0, "offpolicy_set_qr: the Q network's output width %d is not n_actions x n_quantiles "
                 "for n_quantiles = %d", width, N);
  B200RL_REQUIRE(qr_smem_floats(width / N, N) <= C51_SMEM_FLOATS, "offpolicy_set_qr: %d actions x %d quantiles is too wide for the "
                 "head's shared memory", width / N, N);
  h->qr_hp = *qp;
  h->qr_hp.reserved = 0;  // part of the graph cache key
  h->qr = true;
  return 0;
}

extern "C" int b200rl_offpolicy_set_per(b200rl_offpolicy* h, const b200rl_per_hparams* pp) {
  B200RL_REQUIRE(h && pp, "offpolicy_set_per: NULL argument");
  B200RL_REQUIRE(!h->dsac, "offpolicy_set_per: prioritized replay is not implemented for discrete SAC engines (algo = "
                 "5)");
  B200RL_REQUIRE(!h->c51, "offpolicy_set_per: prioritized replay is not implemented for C51 engines");
  B200RL_REQUIRE(!h->edac, "offpolicy_set_per: prioritized replay is not implemented for EDAC engines (algo = 11)");
  B200RL_REQUIRE(!h->redq, "offpolicy_set_per: prioritized replay is not implemented for REDQ engines (algo = 10)");
  B200RL_REQUIRE(!h->tqc, "offpolicy_set_per: prioritized replay is not implemented for TQC engines (algo = 7)");
  B200RL_REQUIRE(!h->iql, "offpolicy_set_per: prioritized replay is not implemented for IQL engines (algo = 9)");
  B200RL_REQUIRE(h->dqn || h->d4pg, "offpolicy_set_per: prioritized replay is implemented for DQN engines (algo = 2) "
                 "and D4PG engines (algo = 6) only");
  B200RL_REQUIRE(pp->alpha >= 0.0 && std::isfinite(pp->alpha), "offpolicy_set_per: alpha must be >= 0");
  B200RL_REQUIRE(pp->eps > 0.0 && std::isfinite(pp->eps), "offpolicy_set_per: eps must be > 0");
  B200RL_REQUIRE(pp->beta_start >= 0.0 && pp->beta_start <= 1.0, "offpolicy_set_per: beta_start must be in [0, 1]");
  B200RL_REQUIRE(pp->beta_anneal_steps >= 1, "offpolicy_set_per: beta_anneal_steps must be >= 1");
  h->per_hp = *pp;
  h->per_set = true;
  return 0;
}

extern "C" int b200rl_offpolicy_set_nstep(b200rl_offpolicy* h, int32_t n_step, const float* const* episode_ends) {
  B200RL_REQUIRE(h, "offpolicy_set_nstep: NULL engine");
  B200RL_REQUIRE(!h->dsac, "offpolicy_set_nstep: n-step returns are not implemented for discrete SAC engines (algo = "
                 "5)");
  B200RL_REQUIRE(!h->edac, "offpolicy_set_nstep: n-step returns are not implemented for EDAC engines (algo = 11)");
  B200RL_REQUIRE(!h->redq, "offpolicy_set_nstep: n-step returns are not implemented for REDQ engines (algo = 10)");
  B200RL_REQUIRE(!h->tqc, "offpolicy_set_nstep: n-step returns are not implemented for TQC engines (algo = 7)");
  B200RL_REQUIRE(!h->iql, "offpolicy_set_nstep: n-step returns are not implemented for IQL engines (algo = 9)");
  B200RL_REQUIRE(h->dqn || h->d4pg, "offpolicy_set_nstep: n-step returns are implemented for DQN and C51 engines "
                 "(algo = 2 or 3) and D4PG engines (algo = 6) only");
  B200RL_REQUIRE(n_step >= 1 && n_step <= NSTEP_MAX, "offpolicy_set_nstep: n_step must be 1..%d, got %d", NSTEP_MAX,
                 n_step);
  LaneSrc<true> ends{};
  if (n_step > 1) {
    B200RL_REQUIRE(episode_ends != nullptr, "offpolicy_set_nstep: n_step = %d needs the episode-end columns", n_step);
    for (int z = 0; z < h->K; ++z) {
      B200RL_REQUIRE(episode_ends[z] != nullptr, "offpolicy_set_nstep: learner %d: NULL episode-end column", z);
      ends.p[z] = episode_ends[z];
    }
  }
  h->nstep = n_step;
  h->nstep_ends = ends;
  return 0;
}

extern "C" int b200rl_offpolicy_set_noise_keys(b200rl_offpolicy* h, const uint64_t* seed, const uint64_t* call) {
  B200RL_REQUIRE(h && seed && call, "offpolicy_set_noise_keys: NULL argument");
  B200RL_REQUIRE(!h->dsac, "offpolicy_set_noise_keys: a discrete SAC engine (algo = 5) draws no noise");
  B200RL_REQUIRE(!h->edac, "offpolicy_set_noise_keys: an EDAC engine (algo = 11) has no noisy layers; its policy's "
                 "draws come with the train call");
  B200RL_REQUIRE(!h->redq, "offpolicy_set_noise_keys: a REDQ engine (algo = 10) has no noisy layers; its subsets come "
                 "with set_redq_subsets or are drawn by train_gather_rng");
  B200RL_REQUIRE(!h->tqc, "offpolicy_set_noise_keys: a TQC engine (algo = 7) has no noisy layers; its policy's draws "
                 "come with the train call");
  B200RL_REQUIRE(!h->iql, "offpolicy_set_noise_keys: an IQL engine (algo = 9) draws no noise");
  B200RL_REQUIRE(h->noisy || h->iqn, "offpolicy_set_noise_keys: the engine has no noisy layers (config noisy_layers = "
                 "0)");
  const size_t n = adam_tab_len(h);
  for (int z = 0; z < h->K; ++z) {  // uploaded with the table by run_staged
    unsigned long long* keys = reinterpret_cast<unsigned long long*>(h->h_adam_tab + z * n + n - 2);
    keys[0] = seed[z], keys[1] = call[z];
  }
  h->noisy_keys = true;
  return 0;
}

extern "C" int b200rl_offpolicy_get_noisy_draws(b200rl_offpolicy* h, int32_t S, float* eps) {
  B200RL_REQUIRE(h && eps && S >= 0 && S <= h->cfg.max_steps, "offpolicy_get_noisy_draws: bad arguments");
  B200RL_REQUIRE(h->noisy, "offpolicy_get_noisy_draws: the engine has no noisy layers (config noisy_layers = 0)");
  const size_t w = (size_t)S * 2 * h->noisy_lay.E * 4;
  if (w) B200RL_CUDA(cudaMemcpy2DAsync(eps, w, h->noisy_draws, h->lane_stride, w, h->K, cudaMemcpyDeviceToHost, h->gs));
  B200RL_CUDA(cudaStreamSynchronize(h->gs));
  return 0;
}

extern "C" int b200rl_offpolicy_get_iqn_draws(b200rl_offpolicy* h, int32_t S, float* taus) {
  B200RL_REQUIRE(h && taus && S >= 0 && S <= h->cfg.max_steps, "offpolicy_get_iqn_draws: bad arguments");
  B200RL_REQUIRE(h->iqn, "offpolicy_get_iqn_draws: the engine was not created with algo = 4 (IQN)");
  B200RL_REQUIRE(h->iqn_last_B > 0, "offpolicy_get_iqn_draws: the engine has not run a train step yet");
  const size_t w = (size_t)S * h->iqn_last_B * (h->iqn_cfg.n + h->iqn_cfg.n_target + h->iqn_cfg.k) * 4;
  if (w) B200RL_CUDA(cudaMemcpy2DAsync(taus, w, h->iqn_taus, h->lane_stride, w, h->K, cudaMemcpyDeviceToHost, h->gs));
  B200RL_CUDA(cudaStreamSynchronize(h->gs));
  return 0;
}

extern "C" int b200rl_offpolicy_set_alpha_group(b200rl_offpolicy* h, const float* log_alpha, const float* exp_avg,
                                                const float* exp_avg_sq, const int64_t* step) {
  B200RL_REQUIRE(h && (h->sac || h->dsac), "offpolicy_set_alpha: not a SAC engine");
  B200RL_REQUIRE(log_alpha && exp_avg && exp_avg_sq && step, "offpolicy_set_alpha: NULL argument");
  float v[B200RL_MAX_LEARNERS][3];
  for (int z = 0; z < h->K; ++z) {
    B200RL_REQUIRE(step[z] >= 0, "offpolicy_set_alpha: negative step count");
    v[z][0] = log_alpha[z], v[z][1] = exp_avg[z], v[z][2] = exp_avg_sq[z];
  }
  B200RL_CUDA(cudaMemcpy2DAsync(h->sac_state, h->lane_stride, v, sizeof(v[0]), sizeof(v[0]), h->K,
                                cudaMemcpyHostToDevice, h->gs));
  B200RL_CUDA(cudaStreamSynchronize(h->gs));
  for (int z = 0; z < h->K; ++z) h->alpha_step[z] = step[z];
  return 0;
}

extern "C" int b200rl_offpolicy_get_alpha_group(b200rl_offpolicy* h, float* log_alpha, float* exp_avg,
                                                float* exp_avg_sq, int64_t* step) {
  B200RL_REQUIRE(h && (h->sac || h->dsac) && log_alpha && exp_avg && exp_avg_sq && step,
                 "offpolicy_get_alpha: bad arguments");
  float v[B200RL_MAX_LEARNERS][3];
  B200RL_CUDA(cudaMemcpy2DAsync(v, sizeof(v[0]), h->sac_state, h->lane_stride, sizeof(v[0]), h->K,
                                cudaMemcpyDeviceToHost, h->gs));
  B200RL_CUDA(cudaStreamSynchronize(h->gs));
  for (int z = 0; z < h->K; ++z) {
    log_alpha[z] = v[z][0], exp_avg[z] = v[z][1], exp_avg_sq[z] = v[z][2];
    step[z] = h->alpha_step[z];
  }
  return 0;
}

extern "C" int b200rl_offpolicy_set_alpha(b200rl_offpolicy* h, float log_alpha, float exp_avg, float exp_avg_sq,
                                          int64_t step) {
  B200RL_REQUIRE(h == nullptr || h->K == 1, "offpolicy_set_alpha: a learner group takes offpolicy_set_alpha_group");
  return b200rl_offpolicy_set_alpha_group(h, &log_alpha, &exp_avg, &exp_avg_sq, &step);
}

extern "C" int b200rl_offpolicy_get_alpha(b200rl_offpolicy* h, float* log_alpha, float* exp_avg, float* exp_avg_sq,
                                          int64_t* step) {
  B200RL_REQUIRE(h == nullptr || h->K == 1, "offpolicy_get_alpha: a learner group takes offpolicy_get_alpha_group");
  return b200rl_offpolicy_get_alpha_group(h, log_alpha, exp_avg, exp_avg_sq, step);
}

extern "C" int b200rl_offpolicy_sac_outputs(b200rl_offpolicy* h, int32_t S, float* log_prob_means, float* alphas) {
  B200RL_REQUIRE(h && (h->sac || h->dsac) && log_prob_means && alphas && S >= 0 && S <= h->cfg.max_steps,
                 "offpolicy_sac_outputs: bad arguments");
  const size_t w = (size_t)S * 4;
  if (S > 0) {
    B200RL_CUDA(cudaMemcpy2DAsync(log_prob_means, w, h->out_logp, h->lane_stride, w, h->K, cudaMemcpyDeviceToHost, h->gs));
    B200RL_CUDA(cudaMemcpy2DAsync(alphas, w, h->sac_alpha, h->lane_stride, w, h->K, cudaMemcpyDeviceToHost, h->gs));
  }
  B200RL_CUDA(cudaStreamSynchronize(h->gs));
  return 0;
}

extern "C" int b200rl_offpolicy_set_cql(b200rl_offpolicy* h, const b200rl_cql_hparams* cp) {
  B200RL_REQUIRE(h && cp, "offpolicy_set_cql: NULL argument");
  B200RL_REQUIRE(!h->iql, "offpolicy_set_cql: an IQL engine (algo = 9) takes b200rl_offpolicy_set_iql, not set_cql");
  B200RL_REQUIRE(!h->edac, "offpolicy_set_cql: an EDAC engine (algo = 11) takes b200rl_offpolicy_set_sac, not set_cql");
  B200RL_REQUIRE(!h->redq, "offpolicy_set_cql: a REDQ engine (algo = 10) takes b200rl_offpolicy_set_sac, not set_cql");
  B200RL_REQUIRE(h->cql, "offpolicy_set_cql: the engine was not created with algo = 8 (CQL)");
  B200RL_REQUIRE(std::isfinite(cp->weight) && cp->weight >= 0.0, "offpolicy_set_cql: weight must be finite and >= 0, "
                 "got %g", cp->weight);
  B200RL_REQUIRE(std::isfinite(cp->temperature) && cp->temperature > 0.0, "offpolicy_set_cql: temperature must be "
                 "finite and > 0, got %g", cp->temperature);
  B200RL_REQUIRE(std::isfinite(cp->target_action_gap) && std::isfinite(cp->alpha_lr) && std::isfinite(cp->alpha_beta1) &&
                 std::isfinite(cp->alpha_beta2) && std::isfinite(cp->alpha_eps), "offpolicy_set_cql: non-finite "
                 "Lagrange settings");
  B200RL_REQUIRE(cp->backup_entropy == 0 || cp->backup_entropy == 1, "offpolicy_set_cql: backup_entropy must be 0 or 1");
  h->cql_hp = *cp;
  h->cql_hp.reserved = 0;  // part of the graph cache key
  h->cql_set = true;
  return 0;
}

extern "C" int b200rl_offpolicy_set_alpha_prime_group(b200rl_offpolicy* h, const float* log_alpha_prime,
                                                      const float* exp_avg, const float* exp_avg_sq,
                                                      const int64_t* step) {
  B200RL_REQUIRE(h && h->cql, "offpolicy_set_alpha_prime: not a CQL engine (algo = 8)");
  B200RL_REQUIRE(log_alpha_prime && exp_avg && exp_avg_sq && step, "offpolicy_set_alpha_prime: NULL argument");
  float v[B200RL_MAX_LEARNERS][3];
  for (int z = 0; z < h->K; ++z) {
    B200RL_REQUIRE(step[z] >= 0, "offpolicy_set_alpha_prime: negative step count");
    v[z][0] = log_alpha_prime[z], v[z][1] = exp_avg[z], v[z][2] = exp_avg_sq[z];
  }
  B200RL_CUDA(cudaMemcpy2DAsync(h->cql_ap_state, h->lane_stride, v, sizeof(v[0]), sizeof(v[0]), h->K,
                                cudaMemcpyHostToDevice, h->gs));
  B200RL_CUDA(cudaStreamSynchronize(h->gs));
  for (int z = 0; z < h->K; ++z) h->ap_step[z] = step[z];
  return 0;
}

extern "C" int b200rl_offpolicy_get_alpha_prime_group(b200rl_offpolicy* h, float* log_alpha_prime, float* exp_avg,
                                                      float* exp_avg_sq, int64_t* step) {
  B200RL_REQUIRE(h && h->cql && log_alpha_prime && exp_avg && exp_avg_sq && step,
                 "offpolicy_get_alpha_prime: bad arguments");
  float v[B200RL_MAX_LEARNERS][3];
  B200RL_CUDA(cudaMemcpy2DAsync(v, sizeof(v[0]), h->cql_ap_state, h->lane_stride, sizeof(v[0]), h->K,
                                cudaMemcpyDeviceToHost, h->gs));
  B200RL_CUDA(cudaStreamSynchronize(h->gs));
  for (int z = 0; z < h->K; ++z) {
    log_alpha_prime[z] = v[z][0], exp_avg[z] = v[z][1], exp_avg_sq[z] = v[z][2];
    step[z] = h->ap_step[z];
  }
  return 0;
}

extern "C" int b200rl_offpolicy_cql_outputs(b200rl_offpolicy* h, int32_t S, float* gaps, float* alpha_primes) {
  B200RL_REQUIRE(h && h->cql && gaps && alpha_primes && S >= 0 && S <= h->cfg.max_steps,
                 "offpolicy_cql_outputs: bad arguments");
  const size_t w = (size_t)S * 4, maxS = (size_t)h->cfg.max_steps;
  for (int k = 0; k < 2 && S > 0; ++k)
    B200RL_CUDA(cudaMemcpy2DAsync(gaps + (size_t)k * S, 2 * w, h->cql_gap + k * maxS, h->lane_stride, w, h->K,
                                  cudaMemcpyDeviceToHost, h->gs));
  if (S > 0)
    B200RL_CUDA(cudaMemcpy2DAsync(alpha_primes, w, h->cql_ap, h->lane_stride, w, h->K, cudaMemcpyDeviceToHost, h->gs));
  B200RL_CUDA(cudaStreamSynchronize(h->gs));
  if (!h->cql_cfg.lagrange)
    for (size_t i = 0; i < (size_t)h->K * S; ++i) alpha_primes[i] = 1.f;
  return 0;
}

extern "C" int b200rl_offpolicy_set_iql(b200rl_offpolicy* h, const b200rl_iql_hparams* ip) {
  B200RL_REQUIRE(h && ip, "offpolicy_set_iql: NULL argument");
  B200RL_REQUIRE(!h->edac, "offpolicy_set_iql: an EDAC engine (algo = 11) takes b200rl_offpolicy_set_sac, not set_iql");
  B200RL_REQUIRE(!h->redq, "offpolicy_set_iql: a REDQ engine (algo = 10) takes b200rl_offpolicy_set_sac, not set_iql");
  B200RL_REQUIRE(h->iql, "offpolicy_set_iql: the engine was not created with algo = 9 (IQL)");
  B200RL_REQUIRE(ip->expectile > 0.0 && ip->expectile < 1.0, "offpolicy_set_iql: expectile must be in (0, 1), got %g",
                 ip->expectile);
  B200RL_REQUIRE(std::isfinite(ip->beta) && ip->beta >= 0.0, "offpolicy_set_iql: beta must be finite and >= 0, got %g",
                 ip->beta);
  B200RL_REQUIRE(std::isfinite(ip->max_weight) && ip->max_weight > 0.0, "offpolicy_set_iql: max_weight must be finite "
                 "and > 0, got %g", ip->max_weight);
  B200RL_REQUIRE(std::isfinite(ip->log_std_min) && std::isfinite(ip->log_std_max) && ip->log_std_min < ip->log_std_max,
                 "offpolicy_set_iql: the log-std bounds need finite log_std_min < log_std_max, got [%g, %g]",
                 ip->log_std_min, ip->log_std_max);
  B200RL_REQUIRE(std::isfinite(ip->v_lr) && std::isfinite(ip->v_beta1) && std::isfinite(ip->v_beta2) &&
                 std::isfinite(ip->v_eps), "offpolicy_set_iql: non-finite Adam settings of the value network");
  h->iql_hp = *ip;
  h->iql_set = true;
  return 0;
}

extern "C" int b200rl_offpolicy_iql_outputs(b200rl_offpolicy* h, int32_t S, float* value_losses, float* value_means,
                                            float* weight_means) {
  B200RL_REQUIRE(h && h->iql && value_losses && value_means && weight_means && S >= 0 && S <= h->cfg.max_steps,
                 "offpolicy_iql_outputs: bad arguments");
  const size_t w = (size_t)S * 4;
  float* dst[3] = {value_losses, value_means, weight_means};
  const float* src[3] = {h->out_vl, h->out_vm, h->out_wm};
  for (int k = 0; k < 3 && S > 0; ++k)
    B200RL_CUDA(cudaMemcpy2DAsync(dst[k], w, src[k], h->lane_stride, w, h->K, cudaMemcpyDeviceToHost, h->gs));
  B200RL_CUDA(cudaStreamSynchronize(h->gs));
  return 0;
}

static size_t cql_draw_floats(const b200rl_offpolicy* h, int S, int B) {
  return (size_t)S * 3 * B * h->cql_cfg.n_actions * h->A;
}

// A CQL call with host draws consumes the ones b200rl_offpolicy_set_cql_draws staged for its (S, B)
static int cql_take_draws(b200rl_offpolicy* h, int S, int B, const char* what) {
  if (!h->cql) return 0;
  B200RL_REQUIRE(h->cql_staged_S == S && h->cql_staged_B == B, "%s: a CQL engine needs its draws [S=%d, 3, B=%d, N, A] "
                 "from b200rl_offpolicy_set_cql_draws before a call with host draws", what, S, B);
  h->cql_staged_S = h->cql_staged_B = -1;
  return 0;
}

extern "C" int b200rl_offpolicy_set_cql_draws(b200rl_offpolicy* h, int32_t S, int32_t B, const float* draws) {
  B200RL_REQUIRE(h && draws && h->cql, "offpolicy_set_cql_draws: bad arguments (a CQL engine, algo = 8, takes them)");
  B200RL_REQUIRE(S >= 0 && S <= h->cfg.max_steps && B >= 1 && B <= h->cfg.max_minibatch,
                 "offpolicy_set_cql_draws: S=%d B=%d exceed the capacities", S, B);
  const size_t w = cql_draw_floats(h, S, B) * 4;
  if (w) B200RL_CUDA(cudaMemcpy2DAsync(h->cql_draws, h->lane_stride, draws, w, w, h->K, cudaMemcpyHostToDevice, h->gs));
  B200RL_CUDA(cudaStreamSynchronize(h->gs));
  h->cql_staged_S = S, h->cql_staged_B = B;
  return 0;
}

extern "C" int b200rl_offpolicy_get_cql_draws(b200rl_offpolicy* h, int32_t S, int32_t B, float* draws) {
  B200RL_REQUIRE(h && draws && h->cql, "offpolicy_get_cql_draws: bad arguments (a CQL engine, algo = 8, has them)");
  B200RL_REQUIRE(S >= 0 && S <= h->cfg.max_steps && B >= 1 && B <= h->cfg.max_minibatch,
                 "offpolicy_get_cql_draws: S=%d B=%d exceed the capacities", S, B);
  const size_t w = cql_draw_floats(h, S, B) * 4;
  if (w) B200RL_CUDA(cudaMemcpy2DAsync(draws, w, h->cql_draws, h->lane_stride, w, h->K, cudaMemcpyDeviceToHost, h->gs));
  B200RL_CUDA(cudaStreamSynchronize(h->gs));
  return 0;
}

// A REDQ call with host subsets consumes the ones b200rl_offpolicy_set_redq_subsets staged for its S
static int redq_take_subsets(b200rl_offpolicy* h, int S, const char* what) {
  if (!h->redq || h->edac) return 0;  // EDAC's target takes every critic
  B200RL_REQUIRE(h->redq_staged_S == S, "%s: a REDQ engine needs its subsets [S=%d, M] from "
                 "b200rl_offpolicy_set_redq_subsets before a call with host draws", what, S);
  h->redq_staged_S = -1;
  return 0;
}

extern "C" int b200rl_offpolicy_set_redq_subsets(b200rl_offpolicy* h, int32_t S, const int32_t* subsets) {
  B200RL_REQUIRE(h && subsets, "offpolicy_set_redq_subsets: NULL argument");
  B200RL_REQUIRE(!h->edac, "offpolicy_set_redq_subsets: an EDAC engine (algo = 11) takes the min over all its target "
                 "critics and draws no subsets");
  B200RL_REQUIRE(h->redq, "offpolicy_set_redq_subsets: the engine was not created with algo = 10 (REDQ)");
  B200RL_REQUIRE(S >= 0 && S <= h->cfg.max_steps, "offpolicy_set_redq_subsets: S=%d exceeds the capacity %d", S,
                 h->cfg.max_steps);
  const int N = h->redq_cfg.n_critics, M = h->redq_cfg.n_min;
  for (long long r = 0; r < (long long)h->K * S; ++r) {
    const int32_t* e = subsets + r * M;
    unsigned long long seen = 0;
    for (int j = 0; j < M; ++j) {
      B200RL_REQUIRE(e[j] >= 0 && e[j] < N && !((seen >> e[j]) & 1ull), "offpolicy_set_redq_subsets: learner %d, step "
                     "%d: a subset needs %d distinct critics in 0..%d, got %d at position %d", (int)(r / (S ? S : 1)),
                     (int)(r % (S ? S : 1)), M, N - 1, e[j], j);
      seen |= 1ull << e[j];
    }
  }
  const size_t w = (size_t)S * M * 4;
  if (w) B200RL_CUDA(cudaMemcpy2DAsync(h->redq_sub, h->lane_stride, subsets, w, w, h->K, cudaMemcpyHostToDevice, h->gs));
  B200RL_CUDA(cudaStreamSynchronize(h->gs));
  h->redq_staged_S = S;
  return 0;
}

extern "C" int b200rl_offpolicy_get_redq_subsets(b200rl_offpolicy* h, int32_t S, int32_t* subsets) {
  B200RL_REQUIRE(h && subsets && h->redq && !h->edac, "offpolicy_get_redq_subsets: bad arguments (a REDQ engine, algo "
                 "= 10, has them)");
  B200RL_REQUIRE(S >= 0 && S <= h->cfg.max_steps, "offpolicy_get_redq_subsets: S=%d exceeds the capacity", S);
  const size_t w = (size_t)S * h->redq_cfg.n_min * 4;
  if (w) B200RL_CUDA(cudaMemcpy2DAsync(subsets, w, h->redq_sub, h->lane_stride, w, h->K, cudaMemcpyDeviceToHost, h->gs));
  B200RL_CUDA(cudaStreamSynchronize(h->gs));
  return 0;
}

extern "C" int b200rl_offpolicy_edac_outputs(b200rl_offpolicy* h, int32_t S, float* diversity) {
  B200RL_REQUIRE(h && h->edac && diversity, "offpolicy_edac_outputs: bad arguments (an EDAC engine, algo = 11, has "
                 "them)");
  B200RL_REQUIRE(S == h->redq_last_S, "offpolicy_edac_outputs: the last call ran S=%d steps, asked for %d",
                 h->redq_last_S, S);
  const size_t w = (size_t)S * 4;
  if (w) B200RL_CUDA(cudaMemcpy2DAsync(diversity, w, h->edac_div, h->lane_stride, w, h->K, cudaMemcpyDeviceToHost, h->gs));
  B200RL_CUDA(cudaStreamSynchronize(h->gs));
  return 0;
}

extern "C" int b200rl_offpolicy_redq_outputs(b200rl_offpolicy* h, int32_t S, float* q_values, float* q_losses) {
  B200RL_REQUIRE(h && h->redq && q_values && q_losses, "offpolicy_redq_outputs: bad arguments (a REDQ engine, algo = "
                 "10, has them)");
  B200RL_REQUIRE(S == h->redq_last_S, "offpolicy_redq_outputs: the last call ran S=%d steps, asked for %d",
                 h->redq_last_S, S);
  const size_t N = (size_t)h->redq_cfg.n_critics, wv = N * S * h->redq_last_B * 4, wl = N * S * 4;
  if (wv) {
    B200RL_CUDA(cudaMemcpy2DAsync(q_values, wv, h->out_q1, h->lane_stride, wv, h->K, cudaMemcpyDeviceToHost, h->gs));
    B200RL_CUDA(cudaMemcpy2DAsync(q_losses, wl, h->out_l1, h->lane_stride, wl, h->K, cudaMemcpyDeviceToHost, h->gs));
  }
  B200RL_CUDA(cudaStreamSynchronize(h->gs));
  return 0;
}

// c51_loss_kernel<LANES, WEIGHTED, NSTEP> of a call: WEIGHTED for prioritized replay (D4PG engines), NSTEP for n-step
// returns
template <bool LANES>
static auto c51_head(bool weighted, bool nstep) {
  return weighted ? (nstep ? c51_loss_kernel<LANES, true, true> : c51_loss_kernel<LANES, true, false>)
                  : (nstep ? c51_loss_kernel<LANES, false, true> : c51_loss_kernel<LANES, false, false>);
}

// Enqueue the S train steps on `s` (plain launches or under stream capture).  Everything that varies between calls
// with the same (S, B, hyper-parameters) is read from device buffers: staged minibatches, Adam scalar tables.
// A D4PG engine (h->d4pg) differs in its heads and staging only: the critic's head is c51_loss_kernel on its N logits
// (act = NULL, n = 1; the target logits from Q1targ at [s' | mu_targ(s')]), the policy's d4pg_policy_loss_kernel, the
// dOut of both backward passes N wide.  A prioritized call (h->per_run) opens each step with the draw on s (draw,
// weights, gather or n-step walk) and runs the priority update on s4 beside the critic's backward pass; the next
// step's draw joins it.
static int enqueue_steps(b200rl_offpolicy* h, const b200rl_offpolicy_hparams* hp, int S, int B, cudaStream_t s,
                         int* n_pol_out) {
  const bool td3 = h->cfg.n_q == 2;
  const int O = h->O, A = h->A;
  const int maxS = h->cfg.max_steps;
  NetBuf &pi = h->net[0], &q1 = h->net[1], &q2 = h->net[2], &pit = h->net[3], &q1t = h->net[4], &q2t = h->net[5];
  const int Lq = q1.d.n_layers, Lp = pi.d.n_layers;
  const int ew = 256;
  cudaStream_t s2 = h->s2, s3 = h->s3, s4 = h->s4;
  int n_pol = 0;
  const bool d4pg = h->d4pg, per = h->per_run, nstep = h->nstep > 1;
  const int NQ = d4pg ? h->d4pg_cfg.n_atoms : 1;  // the critics' output width
  const int W = d4pg ? c51_warps(1, NQ) : 1;      // the D4PG heads' warps per CTA
  const size_t head_smem = sizeof(float) * (size_t)(NQ + W * (3 * NQ + 1));
  const float vmin = (float)h->d4pg_cfg.v_min, vmax = (float)h->d4pg_cfg.v_max;
  const float dz = d4pg ? (float)((h->d4pg_cfg.v_max - h->d4pg_cfg.v_min) / (NQ - 1)) : 0.f;
  const float2* betas = h->adam_tab + (size_t)3 * maxS;
  const unsigned long long* keys = reinterpret_cast<const unsigned long long*>(h->adam_tab + (size_t)4 * maxS);
  // A step is a dependency graph, not a sequence; the branches below are what the kernels actually need:
  //   s  : target policy -> Q1 target ---------+-> Q1 loss -> Q1 dX chain -----+-> Adam(Q1) -> [policy step] -> polyak
  //   s2 :               -> Q2 target ---------+-> Q2 loss -> Q2 dX chain -----+-> Adam(Q2)
  //   s3 : Q1 forward on [s | a] (independent of the targets) ..... Q1's dW products (pi's in the policy step)
  //   s4 : Q2 forward on [s | a] .................................. Q2's dW products
  // Critical path per step: 6 + 1 + 3 + 1 kernels (was 7 + 10 in a single chain), policy steps 14 more (was 19).
  for (int st = 0; st < S; ++st) {
    float* s_obs = h->obs + (size_t)st * B * O;
    float* s_act = h->act + (size_t)st * B * A;
    float* s_rew = h->rew + (size_t)st * B;
    float* s_nobs = h->nobs + (size_t)st * B * O;
    float* s_done = h->done + (size_t)st * B;
    float* s_disc = d4pg ? h->nstep_disc + (size_t)st * B : nullptr;
    long long* s_idx = h->idx + (size_t)st * B;
    float* s_w = per ? h->per_w + (size_t)st * B : nullptr;
    if (per) {  // D4PG: the step's prioritized draw ahead of everything that reads its minibatch
      if (st > 0 && edge(h, s4, s)) return 1;  // the previous step's priorities are in the tree
      if (launch(h, nstep ? per_draw_kernel<false, true> : per_draw_kernel<false, false>,
                 nstep ? per_draw_kernel<true, true> : per_draw_kernel<true, false>, 1, GTHREADS, 0, s, h->replay,
                 betas, keys, st, B, O, A, h->nstep, (float)hp->gamma, s_idx, s_w, s_obs, s_act, s_rew, s_nobs, s_done,
                 s_disc, h->nstep_rows + (size_t)st * B))
        return 1;
    }
    // ---- the critics' forward passes on [s | a]: their values are also the logged Q-values (td3.py:231-235) ----
    float* qa[2][B200RL_MAX_LAYERS + 1];
    for (int qi = 0; qi < (td3 ? 2 : 1); ++qi) {
      qa[qi][0] = const_cast<float*>(s_obs);
      for (int l = 1; l <= Lq; ++l) qa[qi][l] = h->acts[qi == 0 ? 1 : 4][l];
      cudaStream_t qs = qi == 0 ? s3 : s4;
      if (edge(h, s, qs)) return 1;
      if (net_forward(h, qi == 0 ? q1 : q2, qa[qi], B, qs, s_act, A, O)) return 1;
    }
    // ---- targets (td3.py:325-341 / ddpg.py:275-282): the smoothing noise rides on the last layer's epilogue;
    //      [s' | a'] is read in place by the target critics' first layer ----
    float* ta[B200RL_MAX_LAYERS + 1];
    ta[0] = const_cast<float*>(s_nobs);
    for (int l = 1; l <= Lp; ++l) ta[l] = h->acts[0][l];
    if (net_forward(h, pit, ta, B, s, nullptr, 0, 0, hp->use_target_noise ? h->eps + (size_t)st * B * A : nullptr, hp))
      return 1;
    float* tq[B200RL_MAX_LAYERS + 1];
    tq[0] = const_cast<float*>(s_nobs);
    for (int l = 1; l < Lq; ++l) tq[l] = h->acts_tq[l];  // apart from the target policy's stack, whose output it reads
    tq[Lq] = h->qt1;
    if (td3) {
      if (edge(h, s, s2)) return 1;
      float* tq2[B200RL_MAX_LAYERS + 1];
      tq2[0] = const_cast<float*>(s_nobs);
      for (int l = 1; l < Lq; ++l) tq2[l] = h->acts[3][l];
      tq2[Lq] = h->qt2;
      if (net_forward(h, q2t, tq2, B, s2, ta[Lp], A, O)) return 1;
    }
    if (net_forward(h, q1t, tq, B, s, ta[Lp], A, O)) return 1;
    if (td3 && edge(h, s2, s)) return 1;  // both target values are complete on `s`
    // ---- Q steps (td3.py:343-358): TD target + MSE + dq in one kernel, backward, Adam ----
    if (td3) {
      if (edge(h, s, s2)) return 1;   // the targets
      if (edge(h, s4, s2)) return 1;  // Q2's forward pass
    }
    if (edge(h, s3, s)) return 1;     // Q1's forward pass
    for (int qi = (td3 ? 1 : 0); qi >= 0; --qi) {
      NetBuf& qn = qi == 0 ? q1 : q2;
      cudaStream_t qs = qi == 0 ? s : s2;
      float* dq = qi == 0 ? h->dq : h->dq2;
      if (d4pg) {  // the projected cross-entropy on the critic's logits; Q1targ's logits are in qt1
        if (launch(h, c51_head<false>(per, nstep), c51_head<true>(per, nstep), (B + W - 1) / W, W * 32, head_smem, s,
                   qa[0][Lq], h->qt1, nullptr, nullptr, s_rew, s_done, s_disc, h->c51_support, (float)hp->gamma, vmin,
                   vmax, dz, B, 1, NQ, h->dq, h->c51_row_loss, h->out_q1 + (size_t)st * B, h->c51_sync,
                   h->out_l1 + st, h->dqn_bad + st, s_w, h->per_absd))
          return 1;
        if (per) {
          if (edge(h, s, s4)) return 1;
          if (launch(h, per_update_kernel<false>, per_update_kernel<true>, 1, GTHREADS, 0, s4, h->replay, s_idx,
                     h->per_absd, B, (float)h->per_hp.alpha, (float)h->per_hp.eps, h->per_newp + (size_t)st * B,
                     h->per_bad + st))
            return 1;
        }
      } else if (launch(h, q_loss_kernel<false>, q_loss_kernel<true>, 1, GTHREADS, 0, qs, qa[qi][Lq], s_rew, s_done,
                        h->qt1, td3 ? h->qt2 : nullptr, (float)hp->gamma, B, dq,
                        (qi == 0 ? h->out_l1 : h->out_l2) + st, (qi == 0 ? h->out_q1 : h->out_q2) + (size_t)st * B)) {
        return 1;
      }
      if (net_backward(h, qn, qa[qi], dq, NQ, B, true, nullptr, qs, qi != 0, s_act, A, O, qi == 0 ? s3 : s4)) return 1;
      if (adam_net(h, qn, h->adam_tab + (size_t)(1 + qi) * maxS, st, hp->q_beta1, hp->q_beta2, hp->q_eps, qs)) return 1;
    }
    if (td3 && edge(h, s2, s)) return 1;
    // ---- delayed policy step + polyak (td3.py:244-263, 301-323; ddpg: every step) ----
    if (st % hp->policy_delay == 0) {
      float* pa[B200RL_MAX_LAYERS + 1];
      pa[0] = const_cast<float*>(s_obs);
      for (int l = 1; l <= Lp; ++l) pa[l] = h->acts[2][l];
      if (net_forward(h, pi, pa, B, s)) return 1;
      float* qp[B200RL_MAX_LAYERS + 1];
      qp[0] = const_cast<float*>(s_obs);
      for (int l = 1; l <= Lq; ++l) qp[l] = h->acts[1][l];
      if (net_forward(h, q1, qp, B, s, pa[Lp], A, O)) return 1;  // Q1 with its freshly updated parameters (td3.py:309)
      if (d4pg) {  // -mean of the expected values; the logit gradient -(1/B) p_k (z_k - Q)
        if (launch(h, d4pg_policy_loss_kernel<false>, d4pg_policy_loss_kernel<true>, (B + W - 1) / W, W * 32,
                   sizeof(float) * (size_t)(NQ + W * NQ), s, qp[Lq], h->c51_support, B, NQ, h->dq, h->c51_row_loss,
                   h->c51_sync, h->out_lp + n_pol))
          return 1;
      } else if (launch(h, q_loss_kernel<false>, q_loss_kernel<true>, 1, GTHREADS, 0, s, qp[Lq], nullptr, nullptr,
                        nullptr, nullptr, 0.f, B, h->dq, h->out_lp + n_pol, nullptr)) {
        return 1;
      }
      // gradient w.r.t. Q1's input; its action columns are the gradient w.r.t. pi(s) (Q parameters frozen)
      if (net_backward(h, q1, qp, h->dq, NQ, B, false, h->x_cat, s)) return 1;
      if (net_backward(h, pi, pa, h->x_cat + O, O + A, B, true, nullptr, s, false, nullptr, 0, 0, s3)) return 1;
      if (adam_net(h, pi, h->adam_tab, n_pol, hp->policy_beta1, hp->policy_beta2, hp->policy_eps, s)) return 1;
      PolyakArgs pk{};
      pk.n_nets = td3 ? 3 : 2;
      int nmax = 0;
      for (int k = 0; k < pk.n_nets; ++k) {
        pk.target[k] = h->net[3 + k].params;
        pk.param[k] = h->net[k].params;
        pk.n[k] = (int)h->net[k].P;
        nmax = pk.n[k] > nmax ? pk.n[k] : nmax;
      }
      if (launch(h, polyak_kernel<false>, polyak_kernel<true>, (nmax + ew - 1) / ew, ew, 0, s, pk,
                 (float)hp->polyak_rho, (float)(1.0 - hp->polyak_rho)))
        return 1;
      ++n_pol;
    }
  }
  if (per && edge(h, s4, s)) return 1;
  *n_pol_out = n_pol;
  return 0;
}

// The S SAC steps (sac/sac.py update(): one critic step, one policy step, the optional temperature step and polyak).
// Per step the branches are:
//   s  : pi(s') -> squash -> Q1targ ----+-> soft Q1 loss -> Q1 bwd, Adam -+-> Q1(s, a_pi) -+-> policy loss -> Q1 dX -+->
//   s2 :                    -> Q2targ --+-> soft Q2 loss -> Q2 bwd, Adam -+-> Q2(s, a_pi) -+                -> Q2 dX -+
//   s3 : Q1 on [s | a] -> pi(s) -> squash ............ Q1's dW products ......... (then pi's dW products)
//   s4 : Q2 on [s | a] ............................... Q2's dW products -> polyak (both critic pairs)
//        ... -> squash backward -> pi bwd, Adam on s; the temperature step rides on s2 behind Q2's dX chain.
// Step st reads alpha[st]; the temperature step writes alpha[st + 1], so nothing it writes is read in the same step.
// A TQC engine (h->tqc) differs in its heads only: tqc_target_kernel on s behind both target critics (the truncated
// pooled atoms y), tqc_critic_loss_kernel in place of each soft Q loss, tqc_policy_loss_kernel in place of the policy
// loss, and the critics' dOut M wide in every backward pass.
static int enqueue_sac_steps(b200rl_offpolicy* h, const b200rl_offpolicy_hparams* hp, int S, int B, cudaStream_t s) {
  const int O = h->O, A = h->A;
  const int maxS = h->cfg.max_steps;
  const b200rl_sac_hparams& sp = h->sac_hp;
  NetBuf &pi = h->net[0], &q1 = h->net[1], &q2 = h->net[2], &q1t = h->net[4], &q2t = h->net[5];
  const int Lq = q1.d.n_layers, Lp = pi.d.n_layers;
  const float lmin = (float)sp.log_std_min, lmax = (float)sp.log_std_max, limit = (float)hp->action_limit;
  const int ew = 256, rows_grid = (B + 127) / 128;
  cudaStream_t s2 = h->s2, s3 = h->s3, s4 = h->s4;
  const bool tqc = h->tqc;
  const int NQ = tqc ? h->tqc_cfg.n_quantiles : 1;             // the critics' output width, M
  const int kN = tqc ? 2 * (NQ - h->tqc_cfg.n_drop_per_net) : 0;  // target atoms kept
  const bool cql = h->cql, lag = cql && h->cql_cfg.lagrange;
  const b200rl_cql_hparams& cq = h->cql_hp;
  const int CN = cql ? h->cql_cfg.n_actions : 0, R = B * (1 + 3 * CN);  // the critic step's stacked rows
  const int rows = cql ? R : B;
  if (launch(h, sac_alpha_init_kernel<false>, sac_alpha_init_kernel<true>, (S + 1 + ew - 1) / ew, ew, 0, s,
             h->sac_alpha, S + 1, h->sac_state, sp.learn_alpha, (float)sp.alpha))
    return 1;
  if (lag && launch(h, sac_alpha_init_kernel<false>, sac_alpha_init_kernel<true>, 1, ew, 0, s, h->cql_ap, S + 1,
                    h->cql_ap_state, 1, 0.f))
    return 1;
  PolyakArgs pk{};  // 1 -> 4, 2 -> 5
  pk.n_nets = 2;
  for (int k = 0; k < 2; ++k) {
    pk.target[k] = h->net[4 + k].params;
    pk.param[k] = h->net[1 + k].params;
    pk.n[k] = (int)h->net[1 + k].P;
  }
  for (int st = 0; st < S; ++st) {
    const float* s_obs = h->obs + (size_t)st * B * O;
    const float* s_act = h->act + (size_t)st * B * A;
    const float* s_rew = h->rew + (size_t)st * B;
    const float* s_nobs = h->nobs + (size_t)st * B * O;
    const float* s_done = h->done + (size_t)st * B;
    const float* eps_next = h->eps + (size_t)(2 * st) * B * A;  // [S, 2, B, A]: the draw for s', then the one for s
    const float* eps_cur = eps_next + (size_t)B * A;
    const float* alpha = h->sac_alpha + st;
    // ---- the critics on [s | a] (the logged Q-values); pi(s) with the pre-update policy behind Q1's.  CQL: pi(s)
    // first, the critics on the stacked rows once both policy outputs are in ----
    float* qa[2][B200RL_MAX_LAYERS + 1];
    for (int qi = 0; qi < 2; ++qi) {
      qa[qi][0] = cql ? h->cql_x : const_cast<float*>(s_obs);
      for (int l = 1; l <= Lq; ++l) qa[qi][l] = cql ? h->cql_acts[qi][l] : h->acts[qi == 0 ? 1 : 4][l];
      cudaStream_t qs = qi == 0 ? s3 : s4;
      if (cql) continue;
      if (edge(h, s, qs)) return 1;
      if (net_forward(h, qi == 0 ? q1 : q2, qa[qi], B, qs, s_act, A, O)) return 1;
    }
    if (cql && edge(h, s, s3)) return 1;
    float* pa[B200RL_MAX_LAYERS + 1];
    pa[0] = const_cast<float*>(s_obs);
    for (int l = 1; l <= Lp; ++l) pa[l] = h->acts[2][l];
    if (net_forward(h, pi, pa, B, s3)) return 1;
    if (launch(h, sac_squash_kernel<false>, sac_squash_kernel<true>, rows_grid, 128, 0, s3, pa[Lp], eps_cur, B, A, lmin,
               lmax, limit, h->sac_act, h->sac_logp))
      return 1;
    // ---- soft targets: a', log pi' from the current policy at s'; the target critics read [s' | a'] in place ----
    float* ta[B200RL_MAX_LAYERS + 1];
    ta[0] = const_cast<float*>(s_nobs);
    for (int l = 1; l <= Lp; ++l) ta[l] = h->acts[0][l];
    if (net_forward(h, pi, ta, B, s)) return 1;
    if (launch(h, sac_squash_kernel<false>, sac_squash_kernel<true>, rows_grid, 128, 0, s, ta[Lp], eps_next, B, A, lmin,
               lmax, limit, h->sac_act_next, h->sac_logp_next))
      return 1;
    if (cql) {  // the stacked operand [s | a] ++ [s_i | sampled actions], then both critics on it
      if (edge(h, s3, s)) return 1;
      const float lu = (float)(-(double)A * std::log(2.0 * hp->action_limit));
      if (launch(h, cql_stage_kernel<false>, cql_stage_kernel<true>, (R + 127) / 128, 128, 0, s, s_obs, s_act, ta[Lp],
                 pa[Lp], h->cql_draws + (size_t)st * 3 * B * CN * A, B, CN, O, A, lmin, lmax, limit, lu, h->cql_x,
                 h->cql_logp))
        return 1;
      for (int qi = 0; qi < 2; ++qi) {
        cudaStream_t qs = qi == 0 ? s3 : s4;
        if (edge(h, s, qs)) return 1;
        if (net_forward(h, qi == 0 ? q1 : q2, qa[qi], R, qs)) return 1;
      }
    }
    float* tq[2][B200RL_MAX_LAYERS + 1];
    for (int qi = 0; qi < 2; ++qi) {
      tq[qi][0] = const_cast<float*>(s_nobs);
      for (int l = 1; l < Lq; ++l) tq[qi][l] = qi == 0 ? h->acts_tq[l] : h->acts[3][l];
      tq[qi][Lq] = qi == 0 ? h->qt1 : h->qt2;
    }
    if (edge(h, s, s2)) return 1;
    if (net_forward(h, q2t, tq[1], B, s2, h->sac_act_next, A, O)) return 1;
    if (net_forward(h, q1t, tq[0], B, s, h->sac_act_next, A, O)) return 1;
    if (edge(h, s2, s)) return 1;
    if (tqc && launch(h, tqc_target_kernel<false>, tqc_target_kernel<true>, B,
                      (2 * NQ + 31) / 32 * 32, 0, s, h->qt1, h->qt2, s_rew, s_done,
                      h->sac_logp_next, alpha, (float)hp->gamma, NQ, kN, h->tqc_y))
      return 1;
    // ---- critic step: soft TD target + MSE + dq, backward, Adam (Q2 on s2, Q1 on s) ----
    if (edge(h, s, s2)) return 1;
    if (edge(h, s4, s2)) return 1;
    if (edge(h, s3, s)) return 1;
    for (int qi = 1; qi >= 0; --qi) {
      NetBuf& qn = qi == 0 ? q1 : q2;
      cudaStream_t qs = qi == 0 ? s : s2;
      float* dq = qi == 0 ? h->dq : h->dq2;
      if (tqc) {  // the quantile Huber loss of the critic's M quantiles against the kN kept target atoms
        if (launch(h, tqc_critic_loss_kernel<false>, tqc_critic_loss_kernel<true>, B,
                   (NQ + 31) / 32 * 32, 0, qs, qa[qi][Lq], h->tqc_y, B, NQ, kN, dq,
                   h->tqc_row_loss + (size_t)qi * B, (qi == 0 ? h->out_q1 : h->out_q2) + (size_t)st * B,
                   h->tqc_sync + qi, (qi == 0 ? h->out_l1 : h->out_l2) + st))
          return 1;
      } else if (launch(h, sac_q_loss_kernel<false>, sac_q_loss_kernel<true>, 1, GTHREADS, 0, qs, qa[qi][Lq], s_rew,
                        s_done, h->qt1, h->qt2, h->sac_logp_next,
                        cql && !cq.backup_entropy ? (const float*)h->cql_zero : alpha, (float)hp->gamma, B, dq,
                        (qi == 0 ? h->out_l1 : h->out_l2) + st, (qi == 0 ? h->out_q1 : h->out_q2) + (size_t)st * B)) {
        return 1;
      }
      if (cql && launch(h, cql_penalty_kernel<false>, cql_penalty_kernel<true>, (B + CQL_WARPS - 1) / CQL_WARPS,
                        CQL_WARPS * 32, 0, qs, qa[qi][Lq], h->cql_logp, B, CN, (float)cq.temperature,
                        (float)cq.weight, lag ? (const float*)(h->cql_ap + st) : nullptr,
                        (float)cq.target_action_gap, dq, h->cql_row_p + (size_t)qi * B, h->cql_sync + qi,
                        (qi == 0 ? h->out_l1 : h->out_l2) + st, h->cql_gap + (size_t)qi * maxS + st))
        return 1;
      if (net_backward(h, qn, qa[qi], dq, NQ, rows, true, nullptr, qs, qi != 0, cql ? nullptr : s_act, cql ? 0 : A,
                       cql ? 0 : O, qi == 0 ? s3 : s4))
        return 1;
      if (adam_net(h, qn, h->adam_tab + (size_t)(1 + qi) * maxS, st, hp->q_beta1, hp->q_beta2, hp->q_eps, qs)) return 1;
    }
    if (edge(h, s2, s)) return 1;
    if (lag && launch(h, cql_alpha_prime_kernel<false>, cql_alpha_prime_kernel<true>, 1, 1, 0, s, h->cql_gap + st,
                      h->cql_gap + maxS + st, (float)cq.weight, (float)cq.target_action_gap, h->cql_ap_state,
                      h->adam_tab + (size_t)4 * maxS, st, (float)(1.0 - cq.alpha_beta1), (float)cq.alpha_beta2,
                      (float)(1.0 - cq.alpha_beta2), (float)cq.alpha_eps, h->cql_ap + st + 1))
      return 1;
    // ---- polyak beside the policy step: the targets are next read by the next step ----
    if (edge(h, s, s4)) return 1;
    if (launch(h, polyak_kernel<false>, polyak_kernel<true>, (pk.n[0] + ew - 1) / ew, ew, 0, s4, pk,
               (float)hp->polyak_rho, (float)(1.0 - hp->polyak_rho)))
      return 1;
    // ---- policy step: both updated critics on [s | a_pi], differentiated w.r.t. their input only ----
    float* qp[2][B200RL_MAX_LAYERS + 1];
    for (int qi = 0; qi < 2; ++qi) {
      qp[qi][0] = const_cast<float*>(s_obs);
      for (int l = 1; l <= Lq; ++l) qp[qi][l] = h->acts[qi == 0 ? 1 : 4][l];
    }
    if (edge(h, s, s2)) return 1;
    if (net_forward(h, q2, qp[1], B, s2, h->sac_act, A, O)) return 1;
    if (net_forward(h, q1, qp[0], B, s, h->sac_act, A, O)) return 1;
    if (edge(h, s2, s)) return 1;
    if (tqc) {  // every quantile of both critics carries -1 / (2 M B)
      if (launch(h, tqc_policy_loss_kernel<false>, tqc_policy_loss_kernel<true>, 1, GTHREADS, 0, s, qp[0][Lq],
                 qp[1][Lq], h->sac_logp, alpha, B, NQ, h->dq, h->dq2, h->out_lp + st, h->out_logp + st))
        return 1;
    } else if (launch(h, sac_policy_loss_kernel<false>, sac_policy_loss_kernel<true>, 1, GTHREADS, 0, s, qp[0][Lq],
                      qp[1][Lq], h->sac_logp, alpha, B, h->dq, h->dq2, h->out_lp + st, h->out_logp + st)) {
      return 1;
    }
    if (edge(h, s, s2)) return 1;
    if (net_backward(h, q2, qp[1], h->dq2, NQ, B, false, h->x_cat2, s2, true)) return 1;
    if (sp.learn_alpha) {  // -mean(log_alpha (log pi + target_entropy)), one Adam step; alpha[st + 1] = exp(log_alpha)
      if (launch(h, sac_alpha_step_kernel<false>, sac_alpha_step_kernel<true>, 1, GTHREADS, 0, s2, h->sac_logp, B,
                 (float)sp.target_entropy, h->sac_state, h->adam_tab + (size_t)3 * maxS, st,
                 (float)(1.0 - sp.alpha_beta1), (float)sp.alpha_beta2, (float)(1.0 - sp.alpha_beta2),
                 (float)sp.alpha_eps, h->sac_alpha + st + 1))
        return 1;
    }
    if (net_backward(h, q1, qp[0], h->dq, NQ, B, false, h->x_cat, s)) return 1;
    if (edge(h, s2, s)) return 1;
    if (launch(h, sac_squash_backward_kernel<false>, sac_squash_backward_kernel<true>, (B * A + ew - 1) / ew, ew, 0, s,
               pa[Lp], eps_cur, h->x_cat + O, h->x_cat2 + O, O + A, B, A, lmin, lmax, limit, alpha, h->sac_dout))
      return 1;
    if (net_backward(h, pi, pa, h->sac_dout, 2 * A, B, true, nullptr, s, false, nullptr, 0, 0, s3)) return 1;
    if (adam_net(h, pi, h->adam_tab, st, hp->policy_beta1, hp->policy_beta2, hp->policy_eps, s)) return 1;
    if (edge(h, s4, s)) return 1;
  }
  return 0;
}

// The S discrete SAC steps (Christodoulou 2019: one critic step, one policy step, the optional temperature step and
// polyak; the order of enqueue_sac_steps).  Per step the branches are:
//   s  : pi(s') -> Q1targ(s') ---+-> Q1 head -> Q1 bwd, Adam -+-> Q1(s) -+-> policy head -> pi bwd, Adam -+->
//   s2 :           Q2targ(s') ---+-> Q2 head -> Q2 bwd, Adam -+-> Q2(s) -+   -> temperature step --------+
//   s3 : Q1(s) -> pi(s) ........... Q1's dW products ....................... pi's dW products
//   s4 : Q2(s) .................... Q2's dW products -> polyak (both critic pairs)
// The heads need no input gradient of any network: every backward pass is the weight-gradient products and the dX
// chain down to the first hidden layer.  pi(s) is the policy at the start of the step (it is updated last); the
// policy head reads the critics just updated, with no gradient into them.  Step st reads alpha[st]; the temperature
// step writes alpha[st + 1] from the policy head's E_i.
static int enqueue_dsac_steps(b200rl_offpolicy* h, const b200rl_offpolicy_hparams* hp, int S, int B, cudaStream_t s) {
  const int O = h->O;
  const int maxS = h->cfg.max_steps;
  const b200rl_sac_hparams& sp = h->sac_hp;
  NetBuf &pi = h->net[0], &q1 = h->net[1], &q2 = h->net[2], &q1t = h->net[4], &q2t = h->net[5];
  const int Lq = q1.d.n_layers, Lp = pi.d.n_layers, n = q1.d.sizes[Lq];
  const int ew = 256;
  cudaStream_t s2 = h->s2, s3 = h->s3, s4 = h->s4;
  if (launch(h, sac_alpha_init_kernel<false>, sac_alpha_init_kernel<true>, (S + 1 + ew - 1) / ew, ew, 0, s,
             h->sac_alpha, S + 1, h->sac_state, sp.learn_alpha, (float)sp.alpha))
    return 1;
  PolyakArgs pk{};  // 1 -> 4, 2 -> 5
  pk.n_nets = 2;
  for (int k = 0; k < 2; ++k) {
    pk.target[k] = h->net[4 + k].params;
    pk.param[k] = h->net[1 + k].params;
    pk.n[k] = (int)h->net[1 + k].P;
  }
  for (int st = 0; st < S; ++st) {
    float* s_obs = h->obs + (size_t)st * B * O;
    const float* s_act = h->act + (size_t)st * B;
    const float* s_rew = h->rew + (size_t)st * B;
    float* s_nobs = h->nobs + (size_t)st * B * O;
    const float* s_done = h->done + (size_t)st * B;
    const float* alpha = h->sac_alpha + st;
    // ---- the critics on s (the logged Q-values); pi(s) with the pre-update policy behind Q1's ----
    float* qa[2][B200RL_MAX_LAYERS + 1];
    for (int qi = 0; qi < 2; ++qi) {
      qa[qi][0] = s_obs;
      for (int l = 1; l <= Lq; ++l) qa[qi][l] = h->acts[qi == 0 ? 1 : 4][l];
      cudaStream_t qs = qi == 0 ? s3 : s4;
      if (edge(h, s, qs)) return 1;
      if (net_forward(h, qi == 0 ? q1 : q2, qa[qi], B, qs)) return 1;
    }
    float* pa[B200RL_MAX_LAYERS + 1];
    pa[0] = s_obs;
    for (int l = 1; l <= Lp; ++l) pa[l] = h->acts[2][l];
    if (net_forward(h, pi, pa, B, s3)) return 1;
    // ---- soft targets: pi(s') and both target critics on s' ----
    float* ta[B200RL_MAX_LAYERS + 1];
    ta[0] = s_nobs;
    for (int l = 1; l <= Lp; ++l) ta[l] = h->acts[0][l];
    float* tq[2][B200RL_MAX_LAYERS + 1];
    for (int qi = 0; qi < 2; ++qi) {
      tq[qi][0] = s_nobs;
      for (int l = 1; l <= Lq; ++l) tq[qi][l] = qi == 0 ? h->acts_tq[l] : h->acts[3][l];
    }
    if (edge(h, s, s2)) return 1;
    if (net_forward(h, q2t, tq[1], B, s2)) return 1;
    if (net_forward(h, pi, ta, B, s)) return 1;
    if (net_forward(h, q1t, tq[0], B, s)) return 1;
    if (edge(h, s2, s)) return 1;
    // ---- critic step: V(s'), y, MSE and dOut in each head, weight-gradient backward, Adam (Q2 on s2, Q1 on s) ----
    if (edge(h, s, s2)) return 1;
    if (edge(h, s4, s2)) return 1;
    if (edge(h, s3, s)) return 1;
    for (int qi = 1; qi >= 0; --qi) {
      NetBuf& qn = qi == 0 ? q1 : q2;
      cudaStream_t qs = qi == 0 ? s : s2;
      float* dq = qi == 0 ? h->dq : h->dq2;
      if (launch(h, dsac_q_loss_kernel<false>, dsac_q_loss_kernel<true>, 1, GTHREADS, 0, qs, qa[qi][Lq], ta[Lp],
                 tq[0][Lq], tq[1][Lq], s_act, s_rew, s_done, alpha, (float)hp->gamma, B, n, dq,
                 (qi == 0 ? h->out_l1 : h->out_l2) + st, (qi == 0 ? h->out_q1 : h->out_q2) + (size_t)st * B,
                 qi == 0 ? h->dqn_bad + st : nullptr))
        return 1;
      if (net_backward(h, qn, qa[qi], dq, n, B, true, nullptr, qs, qi != 0, nullptr, 0, 0, qi == 0 ? s3 : s4)) return 1;
      if (adam_net(h, qn, h->adam_tab + (size_t)(1 + qi) * maxS, st, hp->q_beta1, hp->q_beta2, hp->q_eps, qs)) return 1;
    }
    if (edge(h, s2, s)) return 1;
    // ---- polyak beside the policy step: the targets are next read by the next step ----
    if (edge(h, s, s4)) return 1;
    if (launch(h, polyak_kernel<false>, polyak_kernel<true>, (pk.n[0] + ew - 1) / ew, ew, 0, s4, pk,
               (float)hp->polyak_rho, (float)(1.0 - hp->polyak_rho)))
      return 1;
    // ---- policy step: both updated critics on s, the head, pi's backward pass and Adam ----
    float* qp[2][B200RL_MAX_LAYERS + 1];
    for (int qi = 0; qi < 2; ++qi) {
      qp[qi][0] = s_obs;
      for (int l = 1; l <= Lq; ++l) qp[qi][l] = h->acts[qi == 0 ? 1 : 4][l];
    }
    if (edge(h, s, s2)) return 1;
    if (net_forward(h, q2, qp[1], B, s2)) return 1;
    if (net_forward(h, q1, qp[0], B, s)) return 1;
    if (edge(h, s2, s)) return 1;
    if (launch(h, dsac_policy_loss_kernel<false>, dsac_policy_loss_kernel<true>, 1, GTHREADS, 0, s, pa[Lp], qp[0][Lq],
               qp[1][Lq], alpha, B, n, h->sac_dout, h->sac_logp, h->out_lp + st, h->out_logp + st))
      return 1;
    if (sp.learn_alpha) {  // -mean(log_alpha (E_i + target_entropy)), one Adam step; alpha[st + 1] = exp(log_alpha)
      if (edge(h, s, s2)) return 1;
      if (launch(h, sac_alpha_step_kernel<false>, sac_alpha_step_kernel<true>, 1, GTHREADS, 0, s2, h->sac_logp, B,
                 (float)sp.target_entropy, h->sac_state, h->adam_tab + (size_t)3 * maxS, st,
                 (float)(1.0 - sp.alpha_beta1), (float)sp.alpha_beta2, (float)(1.0 - sp.alpha_beta2),
                 (float)sp.alpha_eps, h->sac_alpha + st + 1))
        return 1;
    }
    if (net_backward(h, pi, pa, h->sac_dout, n, B, true, nullptr, s, false, nullptr, 0, 0, s3)) return 1;
    if (adam_net(h, pi, h->adam_tab, st, hp->policy_beta1, hp->policy_beta2, hp->policy_eps, s)) return 1;
    if (sp.learn_alpha && edge(h, s2, s)) return 1;
    if (edge(h, s4, s)) return 1;
  }
  return 0;
}

// The S IQL steps (b200rl.h, "IQL": value step, policy step with the new V, critic step with the new V, polyak).  Per
// step the branches are:
//   s  : Q1targ(s, a) -> V(s) -+-> value head -> V bwd, Adam -> V'(s) -+----------------+-> Q1 head -> Q1 bwd, Adam -+->
//   s2 : Q2targ(s, a) ---------+   (V's dW products)  -> V'(s') ------|----------------+-> Q2 head -> Q2 bwd, Adam -+
//   s3 : pi(s) ........................................................+-> AWR head -> pi bwd, Adam ..................+
//   s4 : Q1(s, a) -> Q2(s, a) (pre-update, the logged Q-values) ........................ Q2's dW products
// then polyak on s.  No network needs an input gradient: every backward pass is the weight-gradient products and the
// dX chain down to the first hidden layer.  The policy and critic branches share nothing but what they read, so each
// backward pass has a gradient ping-pong of its own (pi dbuf0/1, Q2 dbuf2/3, Q1 dbuf4/5).
static int enqueue_iql_steps(b200rl_offpolicy* h, const b200rl_offpolicy_hparams* hp, int S, int B, cudaStream_t s) {
  const int O = h->O, A = h->A;
  const int maxS = h->cfg.max_steps;
  const b200rl_iql_hparams& ip = h->iql_hp;
  NetBuf &pi = h->net[0], &q1 = h->net[1], &q2 = h->net[2], &vn = h->net[3], &q1t = h->net[4], &q2t = h->net[5];
  const int Lq = q1.d.n_layers, Lp = pi.d.n_layers, Lv = vn.d.n_layers;
  const int ew = 256;
  cudaStream_t s2 = h->s2, s3 = h->s3, s4 = h->s4;
  PolyakArgs pk{};  // 1 -> 4, 2 -> 5
  pk.n_nets = 2;
  for (int k = 0; k < 2; ++k) {
    pk.target[k] = h->net[4 + k].params;
    pk.param[k] = h->net[1 + k].params;
    pk.n[k] = (int)h->net[1 + k].P;
  }
  for (int st = 0; st < S; ++st) {
    float* s_obs = h->obs + (size_t)st * B * O;
    const float* s_act = h->act + (size_t)st * B * A;
    const float* s_rew = h->rew + (size_t)st * B;
    float* s_nobs = h->nobs + (size_t)st * B * O;
    const float* s_done = h->done + (size_t)st * B;
    float *qa[2][B200RL_MAX_LAYERS + 1], *tq[2][B200RL_MAX_LAYERS + 1];
    float *pa[B200RL_MAX_LAYERS + 1], *va[B200RL_MAX_LAYERS + 1], *vn2[B200RL_MAX_LAYERS + 1];
    for (int qi = 0; qi < 2; ++qi) {
      qa[qi][0] = tq[qi][0] = s_obs;
      for (int l = 1; l <= Lq; ++l) qa[qi][l] = h->acts[qi == 0 ? 1 : 4][l];
      for (int l = 1; l < Lq; ++l) tq[qi][l] = qi == 0 ? h->acts_tq[l] : h->acts[3][l];
      tq[qi][Lq] = qi == 0 ? h->qt1 : h->qt2;
    }
    pa[0] = va[0] = s_obs;
    vn2[0] = s_nobs;
    for (int l = 1; l <= Lp; ++l) pa[l] = h->acts[2][l];
    for (int l = 1; l <= Lv; ++l) va[l] = h->acts[0][l], vn2[l] = h->acts[3][l];  // stack 3 is free once Q2targ is read
    // ---- the step's start: the critics (logged), pi(s), both target critics and V(s), all at (s, a) ----
    if (edge(h, s, s2) || edge(h, s, s3) || edge(h, s, s4)) return 1;
    if (net_forward(h, q1, qa[0], B, s4, s_act, A, O) || net_forward(h, q2, qa[1], B, s4, s_act, A, O)) return 1;
    if (net_forward(h, pi, pa, B, s3)) return 1;
    if (net_forward(h, q2t, tq[1], B, s2, s_act, A, O)) return 1;
    if (net_forward(h, q1t, tq[0], B, s, s_act, A, O) || net_forward(h, vn, va, B, s)) return 1;
    if (edge(h, s2, s)) return 1;
    // ---- value step: expectile head, V's backward pass and Adam, then V'(s) and V'(s') ----
    if (launch(h, iql_value_loss_kernel<false>, iql_value_loss_kernel<true>, 1, GTHREADS, 0, s, h->qt1, h->qt2, va[Lv],
               (float)ip.expectile, (float)(1.0 - ip.expectile), B, h->iql_dv, h->out_vl + st, h->out_vm + st))
      return 1;
    if (net_backward(h, vn, va, h->iql_dv, 1, B, true, nullptr, s, 0, nullptr, 0, 0, s2)) return 1;
    if (adam_net(h, vn, h->adam_tab + (size_t)3 * maxS, st, ip.v_beta1, ip.v_beta2, ip.v_eps, s)) return 1;
    if (edge(h, s, s2)) return 1;
    if (net_forward(h, vn, vn2, B, s2)) return 1;
    if (net_forward(h, vn, va, B, s)) return 1;
    // ---- policy step on s3: the AWR head with V'(s), pi's backward pass and Adam ----
    if (edge(h, s, s3)) return 1;
    if (launch(h, iql_policy_loss_kernel<false>, iql_policy_loss_kernel<true>, 1, GTHREADS, 0, s3, pa[Lp], s_act,
               h->qt1, h->qt2, va[Lv], B, A, (float)ip.beta, (float)ip.max_weight, (float)ip.log_std_min,
               (float)ip.log_std_max, (float)hp->action_limit, h->iql_dout, h->out_lp + st, h->out_wm + st))
      return 1;
    if (net_backward(h, pi, pa, h->iql_dout, 2 * A, B, true, nullptr, s3, 0)) return 1;
    if (adam_net(h, pi, h->adam_tab, st, hp->policy_beta1, hp->policy_beta2, hp->policy_eps, s3)) return 1;
    // ---- critic step: y = r + gamma (1 - d) V'(s') in each head (both target inputs V'(s'), temperature 0),
    // weight-gradient backward, Adam (Q2 on s2, Q1 on s) ----
    if (edge(h, s4, s) || edge(h, s2, s) || edge(h, s, s2)) return 1;
    for (int qi = 1; qi >= 0; --qi) {
      NetBuf& qn = qi == 0 ? q1 : q2;
      cudaStream_t qs = qi == 0 ? s : s2;
      float* dq = qi == 0 ? h->dq : h->dq2;
      if (launch(h, sac_q_loss_kernel<false>, sac_q_loss_kernel<true>, 1, GTHREADS, 0, qs, qa[qi][Lq], s_rew, s_done,
                 vn2[Lv], vn2[Lv], h->iql_zero, h->iql_zero, (float)hp->gamma, B, dq,
                 (qi == 0 ? h->out_l1 : h->out_l2) + st, (qi == 0 ? h->out_q1 : h->out_q2) + (size_t)st * B))
        return 1;
      if (net_backward(h, qn, qa[qi], dq, 1, B, true, nullptr, qs, qi == 0 ? 2 : 1, s_act, A, O,
                       qi == 0 ? nullptr : s4))
        return 1;
      if (adam_net(h, qn, h->adam_tab + (size_t)(1 + qi) * maxS, st, hp->q_beta1, hp->q_beta2, hp->q_eps, qs)) return 1;
    }
    if (edge(h, s2, s)) return 1;
    if (launch(h, polyak_kernel<false>, polyak_kernel<true>, (pk.n[0] + ew - 1) / ew, ew, 0, s, pk,
               (float)hp->polyak_rho, (float)(1.0 - hp->polyak_rho)))
      return 1;
    if (edge(h, s3, s)) return 1;
  }
  return 0;
}

// dqn_loss_kernel<LANES, WEIGHTED, NSTEP> of a call: WEIGHTED for prioritized replay, NSTEP for n-step returns
template <bool LANES>
static auto dqn_head(bool weighted, bool nstep) {
  return weighted ? (nstep ? dqn_loss_kernel<LANES, true, true> : dqn_loss_kernel<LANES, true, false>)
                  : (nstep ? dqn_loss_kernel<LANES, false, true> : dqn_loss_kernel<LANES, false, false>);
}

// the same choice of qr_loss_kernel
template <bool LANES>
static auto qr_head(bool weighted, bool nstep) {
  return weighted ? (nstep ? qr_loss_kernel<LANES, true, true> : qr_loss_kernel<LANES, true, false>)
                  : (nstep ? qr_loss_kernel<LANES, false, true> : qr_loss_kernel<LANES, false, false>);
}

// and of iqn_loss_kernel
template <bool LANES>
static auto iqn_head(bool weighted, bool nstep) {
  return weighted ? (nstep ? iqn_loss_kernel<LANES, true, true> : iqn_loss_kernel<LANES, true, false>)
                  : (nstep ? iqn_loss_kernel<LANES, false, true> : iqn_loss_kernel<LANES, false, false>);
}

// The S DQN steps.  Per step:
//   s  : Q_targ(s') ---------------+-> loss -> dX chain -> Adam(Q) -> target copy (on the steps the flag table marks)
//   s2 : Q(s') (Double DQN only) --+
//   s3 : Q(s) ---------------------+   ........ Q's dW products
// Q(s') reads the parameters at the start of the step: the step's Adam waits for the loss kernel, which joins it.
// A C51 engine (h->c51) takes c51_loss_kernel as its loss head, a QR-DQN engine (h->qr) qr_loss_kernel; nothing else
// in the step differs.  A dueling Q network (q.duel_k) runs dueling_forward / dueling_backward in place of
// net_forward / net_backward.  An IQN engine (h->iqn) opens each step with iqn_draw_kernel on s, runs iqn_forward for
// Q(s) with the N online fractions, Q_targ(s') with the N' target and K argmax fractions and Double DQN's Q(s') with
// the K argmax fractions, takes iqn_loss_kernel as its loss head and iqn_backward as its backward pass.
// A prioritized call (h->per_run) opens each step with the draw on s (draw, weights, gather), takes the weighted loss
// head, and runs the priority update on s4 beside the backward pass; the next step's draw joins it.
static int enqueue_dqn_steps(b200rl_offpolicy* h, const b200rl_offpolicy_hparams* hp, int S, int B, cudaStream_t s) {
  const int O = h->O;
  const int maxS = h->cfg.max_steps;
  const bool dbl = h->dqn_hp.double_q != 0;
  NetBuf &q = h->net[1], &qt = h->net[4];
  const int L = q.d.n_layers, n = q.d.sizes[L];
  const int top = q.duel_k ? L + 1 : L;  // a dueling network's stack also holds [V | A] (dueling_forward)
  auto forward = [&](float* const* acts, cudaStream_t st) {
    return q.duel_k ? dueling_forward(h, q, acts, B, st) : net_forward(h, q, acts, B, st);
  };
  const int ew = 256;
  cudaStream_t s2 = h->s2, s3 = h->s3, s4 = h->s4;
  const bool per = h->per_run;
  const bool nstep = h->nstep > 1;  // the loss heads read each row's staged discount
  const float2* betas = h->adam_tab + (size_t)3 * maxS;
  const unsigned long long* keys = reinterpret_cast<const unsigned long long*>(h->adam_tab + (size_t)4 * maxS);
  const float alpha = (float)h->per_hp.alpha, eps = (float)h->per_hp.eps;
  const NoisyLayout& lay = h->noisy_lay;
  const unsigned long long* noise_keys = keys + 2;
  const unsigned compose_ctas = (unsigned)(lay.tiles[lay.n] + ((lay.E + 3) / 4 + GTHREADS - 1) / GTHREADS);  // + draws
  for (int st = 0; st < S; ++st) {
    // noisy layers: both networks' weights drawn and composed behind the previous step's Adam and target copy, ahead
    // of every forward pass of this one
    if (h->noisy && launch(h, noisy_compose_kernel<false>, noisy_compose_kernel<true>, dim3(compose_ctas, 2), GTHREADS,
                           0, s, lay, q.flat, qt.flat, q.params, qt.params, noise_keys, st, h->noisy_draws))
      return 1;
    float* s_obs = h->obs + (size_t)st * B * O;
    float* s_act = h->act + (size_t)st * B;
    float* s_rew = h->rew + (size_t)st * B;
    float* s_nobs = h->nobs + (size_t)st * B * O;
    float* s_done = h->done + (size_t)st * B;
    float* s_disc = h->nstep_disc + (size_t)st * B;
    long long* s_idx = h->idx + (size_t)st * B;
    float* s_w = h->per_w + (size_t)st * B;
    if (per) {
      if (st > 0 && edge(h, s4, s)) return 1;  // the previous step's priorities are in the tree
      if (launch(h, nstep ? per_draw_kernel<false, true> : per_draw_kernel<false, false>,
                 nstep ? per_draw_kernel<true, true> : per_draw_kernel<true, false>, 1, GTHREADS, 0, s, h->replay,
                 betas, keys, st, B, O, 1, h->nstep, (float)hp->gamma, s_idx, s_w, s_obs, s_act, s_rew, s_nobs, s_done,
                 s_disc, h->nstep_rows + (size_t)st * B))
        return 1;
    }
    if (h->iqn) {
      const int N = h->iqn_cfg.n, Nt = h->iqn_cfg.n_target, K = h->iqn_cfg.k, C = h->iqn_cfg.n_cos;
      float* taus = h->iqn_taus + (size_t)st * B * (N + Nt + K);
      if (launch(h, iqn_draw_kernel<false>, iqn_draw_kernel<true>,
                 (unsigned)(((long long)B * (N + Nt + K) * C + GTHREADS - 1) / GTHREADS), GTHREADS, 0, s, B, N, Nt, K, C,
                 noise_keys, st, taus, h->iqn_cos_q, h->iqn_cos_t, h->iqn_cos_n))
        return 1;
      if (edge(h, s, s3) || iqn_forward(h, q, s_obs, h->iqn_cos_q, B, N, h->iqn_pass[0], s3)) return 1;
      if (dbl && (edge(h, s, s2) || iqn_forward(h, q, s_nobs, h->iqn_cos_n, B, K, h->iqn_pass[2], s2))) return 1;
      if (iqn_forward(h, qt, s_nobs, h->iqn_cos_t, B, Nt + K, h->iqn_pass[1], s)) return 1;
      if (dbl && edge(h, s2, s)) return 1;
      if (edge(h, s3, s)) return 1;
      if (launch(h, iqn_head<false>(per, nstep), iqn_head<true>(per, nstep), B, (std::max(N, 32) + 31) / 32 * 32,
                 sizeof(float) * (size_t)iqn_smem_floats(n, N, Nt), s, h->iqn_pass[0].out, h->iqn_pass[1].out,
                 dbl ? h->iqn_pass[2].out : nullptr, taus, s_act, s_rew, s_done, s_disc, (float)hp->gamma, B, n, N, Nt,
                 K, h->dqn_dout, h->c51_row_loss, h->out_q1 + (size_t)st * B, h->c51_sync, h->out_l1 + st,
                 h->dqn_bad + st, s_w, h->per_absd))
        return 1;
      if (per) {
        if (edge(h, s, s4)) return 1;
        if (launch(h, per_update_kernel<false>, per_update_kernel<true>, 1, GTHREADS, 0, s4, h->replay, s_idx,
                   h->per_absd, B, alpha, eps, h->per_newp + (size_t)st * B, h->per_bad + st))
          return 1;
      }
      if (iqn_backward(h, q, s_obs, h->iqn_cos_q, B, h->iqn_pass[0], h->dqn_dout, s, s3)) return 1;
      if (adam_net(h, q, h->adam_tab + (size_t)maxS, st, hp->q_beta1, hp->q_beta2, hp->q_eps, s)) return 1;
      if (launch(h, dqn_target_copy_kernel<false>, dqn_target_copy_kernel<true>, (unsigned)((q.P_flat + ew - 1) / ew),
                 ew, 0, s, qt.flat, q.flat, (int)q.P_flat, h->adam_tab + (size_t)3 * maxS, st))
        return 1;
      continue;
    }
    float* qa[B200RL_MAX_LAYERS + 1];  // Q(s): its stack is what the backward pass reads
    qa[0] = s_obs;
    for (int l = 1; l <= top; ++l) qa[l] = h->acts[1][l];
    if (edge(h, s, s3)) return 1;
    if (forward(qa, s3)) return 1;
    float* qn[B200RL_MAX_LAYERS + 1];
    if (dbl) {
      qn[0] = s_nobs;
      for (int l = 1; l <= top; ++l) qn[l] = h->acts[3][l];
      if (edge(h, s, s2)) return 1;
      if (forward(qn, s2)) return 1;
    }
    float* tq[B200RL_MAX_LAYERS + 1];
    tq[0] = s_nobs;
    for (int l = 1; l <= top; ++l) tq[l] = h->acts_tq[l];
    if (q.duel_k ? dueling_forward(h, qt, tq, B, s) : net_forward(h, qt, tq, B, s)) return 1;
    if (dbl && edge(h, s2, s)) return 1;
    if (edge(h, s3, s)) return 1;
    if (h->c51) {
      const int N = h->c51_hp.n_atoms, W = c51_warps(n / N, N);
      const size_t smem = sizeof(float) * (size_t)(N + W * (3 * N + n / N));
      const float vmin = (float)h->c51_hp.v_min, vmax = (float)h->c51_hp.v_max;
      const float dz = (float)((h->c51_hp.v_max - h->c51_hp.v_min) / (N - 1));
      if (launch(h, c51_head<false>(false, nstep), c51_head<true>(false, nstep), (B + W - 1) / W, W * 32, smem, s,
                 qa[L], tq[L], dbl ? qn[L] : nullptr, s_act, s_rew, s_done, s_disc, h->c51_support, (float)hp->gamma,
                 vmin, vmax, dz, B, n / N, N, h->dqn_dout, h->c51_row_loss, h->out_q1 + (size_t)st * B, h->c51_sync,
                 h->out_l1 + st, h->dqn_bad + st, nullptr, nullptr))
        return 1;
    } else if (h->qr) {
      const int N = h->qr_hp.n_quantiles;
      if (launch(h, qr_head<false>(per, nstep), qr_head<true>(per, nstep), B, (N + 31) / 32 * 32,
                 sizeof(float) * (size_t)qr_smem_floats(n / N, N), s, qa[L], tq[L], dbl ? qn[L] : nullptr, s_act, s_rew, s_done,
                 s_disc, (float)hp->gamma, B, n / N, N, h->dqn_dout, h->c51_row_loss, h->out_q1 + (size_t)st * B,
                 h->c51_sync, h->out_l1 + st, h->dqn_bad + st, s_w, h->per_absd))
        return 1;
    } else if (launch(h, dqn_head<false>(per, nstep), dqn_head<true>(per, nstep), 1, GTHREADS, 0, s, qa[L], tq[L],
                      dbl ? qn[L] : nullptr, s_act, s_rew, s_done, s_disc, (float)hp->gamma, B, n, h->dqn_dout,
                      h->out_l1 + st, h->out_q1 + (size_t)st * B, h->dqn_bad + st, s_w, h->per_absd)) {
      return 1;
    }
    if (per) {
      if (edge(h, s, s4)) return 1;
      if (launch(h, per_update_kernel<false>, per_update_kernel<true>, 1, GTHREADS, 0, s4, h->replay, s_idx,
                 h->per_absd, B, alpha, eps, h->per_newp + (size_t)st * B, h->per_bad + st))
        return 1;
    }
    if (q.duel_k ? dueling_backward(h, q, qa, h->dqn_dout, B, s, s3)
                 : net_backward(h, q, qa, h->dqn_dout, n, B, true, nullptr, s, false, nullptr, 0, 0, s3))
      return 1;
    if (h->noisy && launch(h, noisy_expand_kernel<false>, noisy_expand_kernel<true>, (unsigned)lay.tiles[lay.n],
                           GTHREADS, 0, s, lay, q.grad, h->noisy_draws, st, q.flat_grad))
      return 1;
    if (adam_net(h, q, h->adam_tab + (size_t)maxS, st, hp->q_beta1, hp->q_beta2, hp->q_eps, s)) return 1;
    if (launch(h, dqn_target_copy_kernel<false>, dqn_target_copy_kernel<true>, (unsigned)((q.P_flat + ew - 1) / ew), ew,
               0, s, qt.flat, q.flat, (int)q.P_flat, h->adam_tab + (size_t)3 * maxS, st))
      return 1;
  }
  if (per && edge(h, s4, s)) return 1;
  return 0;
}

// The step program of the engine's algorithm on `s` (plain launches or under stream capture); *n_pol = its policy steps
// One launch of gemm_ens_kernel<MODE>: nm slots per learner (sub != NULL: their members from that table)
template <int MODE>
static int gemm_ens(const b200rl_offpolicy* h, const GemmArgs& g, const EnsStrides& es, const int* sub, int nm,
                    cudaStream_t s) {
  const dim3 grid((g.N + GT - 1) / GT, (g.M + GT - 1) / GT, (unsigned)(nm * h->K));
  if (h->K == 1) gemm_ens_kernel<MODE, false><<<grid, GTHREADS, 0, s>>>(g, es, sub, nm, (size_t)0);
  else gemm_ens_kernel<MODE, true><<<grid, GTHREADS, 0, s>>>(g, es, sub, nm, h->lane_stride);
  B200RL_CUDA(cudaGetLastError());
  count_launch(1);
  return 0;
}

// net_forward of nm critics of the ensemble that starts at network `first` (1: the critics, N + 1: the targets) on
// the shared input [x | a]: slot k's activations at acts[l] + k act_stride floats, its member k (sub == NULL) or sub[k].
// Every member's GemmArgs are those net_forward gives a solo critic.
static int ens_forward(const b200rl_offpolicy* h, int first, float* const* acts, size_t act_stride, const float* x,
                       const float* a, int B, const int* sub, int nm, cudaStream_t s) {
  const NetBuf& nb = h->net[first];
  const int L = nb.d.n_layers;
  const unsigned ps = (unsigned)(state_pad(nb.P) * 4), as = (unsigned)(act_stride * 4);
  for (int l = 0; l < L; ++l) {
    GemmArgs g{};
    EnsStrides es{};
    if (l == 0) {
      g.A = x; g.lda = h->O;
      g.A2 = a; g.lda2 = h->A; g.ksplit = h->O;
    } else {
      g.A = acts[l]; g.lda = nb.d.sizes[l]; es.a = as;
    }
    g.B = nb.params + nb.w_off[l]; g.ldb = nb.d.sizes[l]; es.b = ps;
    g.C = acts[l + 1]; g.ldc = nb.d.sizes[l + 1]; es.c = as;
    g.bias = nb.params + nb.b_off[l];
    g.act = (l == L - 1) ? nb.d.out_act : nb.d.hidden_act;
    g.M = B; g.N = nb.d.sizes[l + 1]; g.K = nb.d.sizes[l];
    if (gemm_ens<0>(h, g, es, sub, nm, s)) return 1;
  }
  return 0;
}

// net_backward of all N critics on [x | a] from dOut (critic k's [B, 1] at dOut + k B): the weight gradients into the
// critics' gradient block (want_grads; on s_dw beside the dX chain, at most 3 layers, as net_backward), the input
// gradient into dx_out (critic k's [B, O + A] at dx_out + k B (O + A)) when dx_out != NULL
static int ens_backward(b200rl_offpolicy* h, float* const* acts, const float* x, const float* a, const float* dOut,
                        int B, bool want_grads, float* dx_out, cudaStream_t s, cudaStream_t s_dw) {
  const NetBuf& nb = h->net[1];
  const int L = nb.d.n_layers, N = h->redq_cfg.n_critics;
  const bool side = s_dw != nullptr && want_grads && L <= 3;
  const unsigned ps = (unsigned)(state_pad(nb.P) * 4), as = (unsigned)((size_t)h->cfg.max_minibatch * h->maxw * 4);
  const float* dY = dOut;
  int ldd = 1;
  unsigned ds = (unsigned)B * 4;
  float* pp[2] = {h->redq_d0, h->redq_d1};
  for (int l = L - 1; l >= 0; --l) {
    const int nout = nb.d.sizes[l + 1], nin = nb.d.sizes[l];
    const int act = (l == L - 1) ? nb.d.out_act : nb.d.hidden_act;
    if (want_grads) {
      GemmArgs g{};
      EnsStrides es{};
      g.A = dY; g.lda = ldd; es.a = ds; g.Y = acts[l + 1]; g.ldy = nout; es.y = as; g.act = act;
      if (l == 0) {
        g.B = x; g.ldb = h->O;
        g.A2 = a; g.lda2 = h->A; g.ksplit = h->O;
      } else {
        g.B = acts[l]; g.ldb = nin; es.b = as;
      }
      g.C = nb.grad + nb.w_off[l]; g.ldc = nin; es.c = ps;
      g.M = nout; g.N = nin; g.K = B;
      g.dbias = nb.grad + nb.b_off[l];
      if (side) {
        B200RL_CUDA(cudaEventRecord(h->ev_side, s));
        B200RL_CUDA(cudaStreamWaitEvent(s_dw, h->ev_side, 0));
      }
      if (gemm_ens<2>(h, g, es, nullptr, N, side ? s_dw : s)) return 1;
    }
    if (l > 0 || dx_out) {
      float* dst = (l == 0) ? dx_out : pp[l & 1];
      const unsigned dst_s = (l == 0) ? (unsigned)(B * (h->O + h->A) * 4) : as;
      GemmArgs g{};
      EnsStrides es{};
      g.A = dY; g.lda = ldd; es.a = ds; g.Y = acts[l + 1]; g.ldy = nout; es.y = as; g.act = act;
      g.B = nb.params + nb.w_off[l]; g.ldb = nin; es.b = ps;
      g.C = dst; g.ldc = nin; es.c = dst_s;
      g.M = B; g.N = nin; g.K = nout;
      if (gemm_ens<1>(h, g, es, nullptr, N, s)) return 1;
      dY = dst, ldd = nin, ds = dst_s;
    }
  }
  if (side) {
    B200RL_CUDA(cudaEventRecord(h->ev_side, s_dw));
    B200RL_CUDA(cudaStreamWaitEvent(s, h->ev_side, 0));
  }
  return 0;
}

// The S REDQ steps (b200rl.h, "REDQ"), SAC's order: critic step, then on policy steps the policy step and the
// temperature step; polyak every step.  Per step the branches are:
//   s  : pi(s') -> M target critics(s') -> target head -+-> critic head -> critics' bwd, Adam -+-> [policy step] -+->
//   s3 : N critics(s, a) -> [pi(s)] --------------------+   ... pi's dW products              |                   |
//   s4 :                     the critics' dW products ... -> polyak (all N targets) ----------+-------------------+
//   s2 :                                                          [temperature step beside the policy's backward]
// The critic ensemble is one launch per layer whatever N; the target ensemble reads its M members from the step's
// subset table.  On a policy step the critics just updated run on [s | a_pi] and are differentiated w.r.t. their input
// only; pi(s) is the policy at the start of the step.
static int enqueue_redq_steps(b200rl_offpolicy* h, const b200rl_offpolicy_hparams* hp, int S, int B, cudaStream_t s) {
  const int O = h->O, A = h->A, N = h->redq_cfg.n_critics, M = h->redq_cfg.n_min, G = hp->policy_delay;
  const int maxS = h->cfg.max_steps;
  const b200rl_sac_hparams& sp = h->sac_hp;
  NetBuf &pi = h->net[0], &q1 = h->net[1];
  const int Lq = q1.d.n_layers, Lp = pi.d.n_layers;
  const float lmin = (float)sp.log_std_min, lmax = (float)sp.log_std_max, limit = (float)hp->action_limit;
  const int ew = 256, rows_grid = (B + 127) / 128;
  const size_t astr = (size_t)h->cfg.max_minibatch * h->maxw;  // floats between two members' activations
  const int pst = (int)state_pad(q1.P);                         // floats between two members' parameters
  cudaStream_t s2 = h->s2, s3 = h->s3, s4 = h->s4;
  if (launch(h, sac_alpha_init_kernel<false>, sac_alpha_init_kernel<true>, (S + 1 + ew - 1) / ew, ew, 0, s,
             h->sac_alpha, S + 1, h->sac_state, sp.learn_alpha, (float)sp.alpha))
    return 1;
  PolyakArgs pk{};  // the critics' block onto the targets' block, padding included (zeros stay zeros)
  pk.n_nets = 1;
  pk.target[0] = h->net[N + 1].params;
  pk.param[0] = q1.params;
  pk.n[0] = N * pst;
  float *qa[B200RL_MAX_LAYERS + 1], *pa[B200RL_MAX_LAYERS + 1], *ta[B200RL_MAX_LAYERS + 1];
  for (int l = 1; l <= Lq; ++l) qa[l] = h->redq_acts[l];
  for (int l = 1; l <= Lp; ++l) pa[l] = h->acts[2][l], ta[l] = h->acts[0][l];
  int pol = 0;
  for (int st = 0; st < S; ++st) {
    float* s_obs = h->obs + (size_t)st * B * O;
    const float* s_act = h->act + (size_t)st * B * A;
    const float* s_rew = h->rew + (size_t)st * B;
    float* s_nobs = h->nobs + (size_t)st * B * O;
    const float* s_done = h->done + (size_t)st * B;
    const float* eps_next = h->eps + (size_t)(2 * st) * B * A;  // [S, 2, B, A]: the draw for s', then the one for s
    const float* eps_cur = eps_next + (size_t)B * A;
    const float* alpha = h->sac_alpha + st;
    const bool pstep = (st + 1) % G == 0 || st == S - 1;
    pa[0] = s_obs, ta[0] = s_nobs;
    // ---- the critics on [s | a] (the logged values) and, on a policy step, pi(s) with the pre-update policy ----
    if (edge(h, s, s3)) return 1;
    if (ens_forward(h, 1, qa, astr, s_obs, s_act, B, nullptr, N, s3)) return 1;
    if (pstep) {
      if (net_forward(h, pi, pa, B, s3)) return 1;
      if (launch(h, sac_squash_kernel<false>, sac_squash_kernel<true>, rows_grid, 128, 0, s3, pa[Lp], eps_cur, B, A,
                 lmin, lmax, limit, h->sac_act, h->sac_logp))
        return 1;
    }
    // ---- soft target: a', log pi' from the current policy at s', the M drawn target critics on [s' | a'] ----
    if (net_forward(h, pi, ta, B, s)) return 1;
    if (launch(h, sac_squash_kernel<false>, sac_squash_kernel<true>, rows_grid, 128, 0, s, ta[Lp], eps_next, B, A, lmin,
               lmax, limit, h->sac_act_next, h->sac_logp_next))
      return 1;
    if (ens_forward(h, N + 1, h->redq_tacts, astr, s_nobs, h->sac_act_next, B, h->redq_sub + (size_t)st * M, M, s))
      return 1;
    if (launch(h, redq_target_kernel<false>, redq_target_kernel<true>, rows_grid, 128, 0, s,
               (const float*)h->redq_tacts[Lq], (int)astr, M, B, h->redq_qmin, h->sac_alpha + st))
      return 1;
    // ---- critic step: every critic's head, backward pass and Adam, one launch each for the ensemble ----
    if (edge(h, s3, s)) return 1;
    if (launch(h, redq_q_loss_kernel<false>, redq_q_loss_kernel<true>, N, GTHREADS, 0, s, (const float*)qa[Lq],
               (int)astr, s_rew, s_done, (const float*)h->redq_qmin, (const float*)h->sac_logp_next, alpha,
               (float)hp->gamma, B, h->redq_dq, h->out_l1 + st, S, h->out_q1 + (size_t)st * B, S * B))
      return 1;
    if (ens_backward(h, qa, s_obs, s_act, h->redq_dq, B, true, nullptr, s, s4)) return 1;
    if (launch(h, redq_adam_kernel<false>, redq_adam_kernel<true>, dim3((unsigned)((q1.P + 255) / 256), N), 256, 0, s,
               q1.flat, (const float*)q1.flat_grad, (const float*)nullptr, q1.m, q1.v, (long long)q1.P, (size_t)pst * 4, (size_t)2 * pst * 4,
               (const float2*)(h->adam_tab + maxS), st, (float)(1.0 - hp->q_beta1), (float)hp->q_beta2,
               (float)(1.0 - hp->q_beta2), (float)hp->q_eps))
      return 1;
    // ---- polyak beside the policy step: the targets are next read by the next step ----
    if (edge(h, s, s4)) return 1;
    if (launch(h, polyak_kernel<false>, polyak_kernel<true>, (pk.n[0] + ew - 1) / ew, ew, 0, s4, pk,
               (float)hp->polyak_rho, (float)(1.0 - hp->polyak_rho)))
      return 1;
    if (pstep) {  // ---- policy step: the N updated critics on [s | a_pi], differentiated w.r.t. their input only ----
      if (ens_forward(h, 1, qa, astr, s_obs, h->sac_act, B, nullptr, N, s)) return 1;
      if (launch(h, redq_policy_loss_kernel<false>, redq_policy_loss_kernel<true>, 1, GTHREADS, 0, s,
                 (const float*)qa[Lq], (int)astr, N, (const float*)h->sac_logp, alpha, B, h->redq_dq,
                 h->out_lp + pol, h->out_logp + pol))
        return 1;
      if (sp.learn_alpha) {  // SAC's temperature step; alpha[st + 1] = exp(log_alpha)
        if (edge(h, s, s2)) return 1;
        if (launch(h, sac_alpha_step_kernel<false>, sac_alpha_step_kernel<true>, 1, GTHREADS, 0, s2, h->sac_logp, B,
                   (float)sp.target_entropy, h->sac_state, h->adam_tab + (size_t)3 * maxS, pol,
                   (float)(1.0 - sp.alpha_beta1), (float)sp.alpha_beta2, (float)(1.0 - sp.alpha_beta2),
                   (float)sp.alpha_eps, h->sac_alpha + st + 1))
          return 1;
      }
      if (ens_backward(h, qa, s_obs, h->sac_act, h->redq_dq, B, false, h->redq_dx, s, nullptr)) return 1;
      if (launch(h, redq_squash_backward_kernel<false>, redq_squash_backward_kernel<true>, (B * A + ew - 1) / ew, ew, 0,
                 s, (const float*)pa[Lp], eps_cur, (const float*)(h->redq_dx + O), B * (O + A), N, O + A, B, A, lmin,
                 lmax, limit, alpha, h->sac_dout))
        return 1;
      if (net_backward(h, pi, pa, h->sac_dout, 2 * A, B, true, nullptr, s, 0, nullptr, 0, 0, s3)) return 1;
      if (adam_net(h, pi, h->adam_tab, pol, hp->policy_beta1, hp->policy_beta2, hp->policy_eps, s)) return 1;
      if (sp.learn_alpha && edge(h, s2, s)) return 1;
      ++pol;
    }
    if (edge(h, s4, s)) return 1;
  }
  return 0;
}

// EDAC's diversity pass (b200rl.h, "EDAC") on the critics' forward activations at [s | a]: 3 Lq launches for the whole
// ensemble, the weight gradient of eta D into h->edac_grad and D into *div_out.  Layers are 0-based here: W_l maps
// acts[l] to acts[l + 1], e[l] is the ungated input gradient of sum_b Q_k at acts[l] (l >= 1; the first layer's is g, on
// the action columns only) and t[l] the tangent at acts[l].
static int edac_diversity(b200rl_offpolicy* h, float* const* acts, int B, float* div_out, cudaStream_t s) {
  const NetBuf& nb = h->net[1];
  const int L = nb.d.n_layers, N = h->redq_cfg.n_critics, O = h->O, A = h->A;
  const int* sz = nb.d.sizes;
  const unsigned ps = (unsigned)(state_pad(nb.P) * 4), as = (unsigned)((size_t)h->cfg.max_minibatch * h->maxw * 4);
  const unsigned gs = (unsigned)((size_t)B * A * 4);
  // ones-backward: e[l] = (e[l + 1] (.) act'(acts[l + 1])) W_l from dOut = 1; the first layer's weight is read from its
  // action columns (B = W_0 + O, ld O + A), so its product is g [B, A] directly
  for (int l = L - 1; l >= 0; --l) {
    GemmArgs g{};
    EnsStrides es{};
    const bool top = l == L - 1;
    g.A = top ? h->edac_ones : h->edac_e[l + 1]; g.lda = top ? 1 : sz[l + 1]; es.a = top ? 0u : as;
    g.Y = acts[l + 1]; g.ldy = sz[l + 1]; es.y = as; g.act = top ? nb.d.out_act : nb.d.hidden_act;
    g.B = nb.params + nb.w_off[l] + (l == 0 ? O : 0); g.ldb = sz[l]; es.b = ps;
    g.C = l == 0 ? h->edac_g : h->edac_e[l]; g.ldc = l == 0 ? A : sz[l]; es.c = l == 0 ? gs : as;
    g.M = B; g.N = l == 0 ? A : sz[l]; g.K = sz[l + 1];
    if (gemm_ens<1>(h, g, es, nullptr, N, s)) return 1;
  }
  const double c = 2.0 * h->edac_eta / ((double)B * (double)(N - 1));
  if (launch(h, edac_diversity_kernel<false>, edac_diversity_kernel<true>, 1, EDAC_THREADS, 0, s,
             (const float*)h->edac_g, N, B, A, c, h->edac_u, div_out))
    return 1;
  // tangent forward: t[1] = act'(acts[1]) (.) u W_0a^T, t[l + 1] = act'(acts[l + 1]) (.) t[l] W_l^T
  for (int l = 0; l < L - 1; ++l) {
    GemmArgs g{};
    EnsStrides es{};
    g.A = l == 0 ? h->edac_u : h->edac_t[l]; g.lda = l == 0 ? A : sz[l]; es.a = l == 0 ? gs : as;
    g.B = nb.params + nb.w_off[l] + (l == 0 ? O : 0); g.ldb = sz[l]; es.b = ps;
    g.C = h->edac_t[l + 1]; g.ldc = sz[l + 1]; es.c = as;
    g.Y = acts[l + 1]; g.ldy = sz[l + 1]; es.y = as; g.act = nb.d.hidden_act;
    g.M = B; g.N = sz[l + 1]; g.K = l == 0 ? A : sz[l];
    if (gemm_ens<4>(h, g, es, nullptr, N, s)) return 1;
  }
  // weight gradients: dW_l = sum_b (e[l + 1] (.) act'(acts[l + 1]))^T t[l] (the first layer's action columns from u),
  // no bias gradient
  for (int l = 0; l < L; ++l) {
    GemmArgs g{};
    EnsStrides es{};
    const bool top = l == L - 1;
    g.A = top ? h->edac_ones : h->edac_e[l + 1]; g.lda = top ? 1 : sz[l + 1]; es.a = top ? 0u : as;
    g.Y = acts[l + 1]; g.ldy = sz[l + 1]; es.y = as; g.act = top ? nb.d.out_act : nb.d.hidden_act;
    g.B = l == 0 ? h->edac_u : h->edac_t[l]; g.ldb = l == 0 ? A : sz[l]; es.b = l == 0 ? gs : as;
    g.C = h->edac_grad + nb.w_off[l] + (l == 0 ? O : 0); g.ldc = sz[l]; es.c = ps;
    g.M = sz[l + 1]; g.N = l == 0 ? A : sz[l]; g.K = B;
    if (gemm_ens<2>(h, g, es, nullptr, N, s)) return 1;
  }
  return 0;
}

// The S EDAC / SAC-N steps (b200rl.h, "EDAC"): REDQ's step program with every target critic, a policy step every step
// on the min head, and (eta > 0) the diversity pass.  Per step the branches are:
//   s  : pi(s') -> N target critics(s') -> target head -+-> critic head -> critics' bwd -+-> Adam -> policy step -+->
//   s3 : N critics(s, a) -+-> pi(s) --------------------+   ... pi's dW products        |                       |
//   s2 :                  +-> diversity pass (eta > 0) ----------------------------------+  [temperature step]   |
//   s4 :                                       the critics' dW products ... -> polyak (all N targets) ----------+
static int enqueue_edac_steps(b200rl_offpolicy* h, const b200rl_offpolicy_hparams* hp, int S, int B, cudaStream_t s) {
  const int O = h->O, A = h->A, N = h->redq_cfg.n_critics;
  const int maxS = h->cfg.max_steps;
  const bool div = h->edac_eta > 0.0;
  const b200rl_sac_hparams& sp = h->sac_hp;
  NetBuf &pi = h->net[0], &q1 = h->net[1];
  const int Lq = q1.d.n_layers, Lp = pi.d.n_layers;
  const float lmin = (float)sp.log_std_min, lmax = (float)sp.log_std_max, limit = (float)hp->action_limit;
  const int ew = 256, rows_grid = (B + 127) / 128;
  const size_t astr = (size_t)h->cfg.max_minibatch * h->maxw;  // floats between two members' activations
  const int pst = (int)state_pad(q1.P);                         // floats between two members' parameters
  cudaStream_t s2 = h->s2, s3 = h->s3, s4 = h->s4;
  if (launch(h, sac_alpha_init_kernel<false>, sac_alpha_init_kernel<true>, (S + 1 + ew - 1) / ew, ew, 0, s,
             h->sac_alpha, S + 1, h->sac_state, sp.learn_alpha, (float)sp.alpha))
    return 1;
  PolyakArgs pk{};  // the critics' block onto the targets' block, padding included (zeros stay zeros)
  pk.n_nets = 1;
  pk.target[0] = h->net[N + 1].params;
  pk.param[0] = q1.params;
  pk.n[0] = N * pst;
  float *qa[B200RL_MAX_LAYERS + 1], *pa[B200RL_MAX_LAYERS + 1], *ta[B200RL_MAX_LAYERS + 1];
  for (int l = 1; l <= Lq; ++l) qa[l] = h->redq_acts[l];
  for (int l = 1; l <= Lp; ++l) pa[l] = h->acts[2][l], ta[l] = h->acts[0][l];
  for (int st = 0; st < S; ++st) {
    float* s_obs = h->obs + (size_t)st * B * O;
    const float* s_act = h->act + (size_t)st * B * A;
    const float* s_rew = h->rew + (size_t)st * B;
    float* s_nobs = h->nobs + (size_t)st * B * O;
    const float* s_done = h->done + (size_t)st * B;
    const float* eps_next = h->eps + (size_t)(2 * st) * B * A;  // [S, 2, B, A]: the draw for s', then the one for s
    const float* eps_cur = eps_next + (size_t)B * A;
    const float* alpha = h->sac_alpha + st;
    pa[0] = s_obs, ta[0] = s_nobs;
    // ---- the critics on [s | a] (the logged values, the diversity pass's masks) and pi(s) with the pre-update policy
    if (edge(h, s, s3)) return 1;
    if (ens_forward(h, 1, qa, astr, s_obs, s_act, B, nullptr, N, s3)) return 1;
    if (div) {
      if (edge(h, s3, s2)) return 1;
      if (edac_diversity(h, qa, B, h->edac_div + st, s2)) return 1;
    }
    if (net_forward(h, pi, pa, B, s3)) return 1;
    if (launch(h, sac_squash_kernel<false>, sac_squash_kernel<true>, rows_grid, 128, 0, s3, pa[Lp], eps_cur, B, A, lmin,
               lmax, limit, h->sac_act, h->sac_logp))
      return 1;
    // ---- soft target: a', log pi' from the current policy at s', all N target critics on [s' | a'] ----
    if (net_forward(h, pi, ta, B, s)) return 1;
    if (launch(h, sac_squash_kernel<false>, sac_squash_kernel<true>, rows_grid, 128, 0, s, ta[Lp], eps_next, B, A, lmin,
               lmax, limit, h->sac_act_next, h->sac_logp_next))
      return 1;
    if (ens_forward(h, N + 1, h->redq_tacts, astr, s_nobs, h->sac_act_next, B, nullptr, N, s)) return 1;
    if (launch(h, redq_target_kernel<false>, redq_target_kernel<true>, rows_grid, 128, 0, s,
               (const float*)h->redq_tacts[Lq], (int)astr, N, B, h->redq_qmin, h->sac_alpha + st))
      return 1;
    // ---- critic step: every critic's TD head and backward pass, then one Adam launch on g_td + g_div ----
    if (edge(h, s3, s)) return 1;
    if (launch(h, redq_q_loss_kernel<false>, redq_q_loss_kernel<true>, N, GTHREADS, 0, s, (const float*)qa[Lq],
               (int)astr, s_rew, s_done, (const float*)h->redq_qmin, (const float*)h->sac_logp_next, alpha,
               (float)hp->gamma, B, h->redq_dq, h->out_l1 + st, S, h->out_q1 + (size_t)st * B, S * B))
      return 1;
    if (ens_backward(h, qa, s_obs, s_act, h->redq_dq, B, true, nullptr, s, s4)) return 1;
    if (div && edge(h, s2, s)) return 1;
    if (launch(h, redq_adam_kernel<false>, redq_adam_kernel<true>, dim3((unsigned)((q1.P + 255) / 256), N), 256, 0, s,
               q1.flat, (const float*)q1.flat_grad, (const float*)(div ? h->edac_grad : nullptr), q1.m, q1.v,
               (long long)q1.P, (size_t)pst * 4, (size_t)2 * pst * 4, (const float2*)(h->adam_tab + maxS), st,
               (float)(1.0 - hp->q_beta1), (float)hp->q_beta2, (float)(1.0 - hp->q_beta2), (float)hp->q_eps))
      return 1;
    // ---- polyak beside the policy step: the targets are next read by the next step ----
    if (edge(h, s, s4)) return 1;
    if (launch(h, polyak_kernel<false>, polyak_kernel<true>, (pk.n[0] + ew - 1) / ew, ew, 0, s4, pk,
               (float)hp->polyak_rho, (float)(1.0 - hp->polyak_rho)))
      return 1;
    // ---- policy step: the N updated critics on [s | a_pi], differentiated w.r.t. their input only ----
    if (ens_forward(h, 1, qa, astr, s_obs, h->sac_act, B, nullptr, N, s)) return 1;
    if (launch(h, edac_policy_loss_kernel<false>, edac_policy_loss_kernel<true>, 1, GTHREADS, 0, s,
               (const float*)qa[Lq], (int)astr, N, (const float*)h->sac_logp, alpha, B, h->redq_dq, h->out_lp + st,
               h->out_logp + st))
      return 1;
    if (sp.learn_alpha) {  // SAC's temperature step; alpha[st + 1] = exp(log_alpha)
      if (edge(h, s, s2)) return 1;
      if (launch(h, sac_alpha_step_kernel<false>, sac_alpha_step_kernel<true>, 1, GTHREADS, 0, s2, h->sac_logp, B,
                 (float)sp.target_entropy, h->sac_state, h->adam_tab + (size_t)3 * maxS, st,
                 (float)(1.0 - sp.alpha_beta1), (float)sp.alpha_beta2, (float)(1.0 - sp.alpha_beta2),
                 (float)sp.alpha_eps, h->sac_alpha + st + 1))
        return 1;
    }
    if (ens_backward(h, qa, s_obs, h->sac_act, h->redq_dq, B, false, h->redq_dx, s, nullptr)) return 1;
    if (launch(h, redq_squash_backward_kernel<false>, redq_squash_backward_kernel<true>, (B * A + ew - 1) / ew, ew, 0,
               s, (const float*)pa[Lp], eps_cur, (const float*)(h->redq_dx + O), B * (O + A), N, O + A, B, A, lmin, lmax,
               limit, alpha, h->sac_dout))
      return 1;
    if (net_backward(h, pi, pa, h->sac_dout, 2 * A, B, true, nullptr, s, 0, nullptr, 0, 0, s3)) return 1;
    if (adam_net(h, pi, h->adam_tab, st, hp->policy_beta1, hp->policy_beta2, hp->policy_eps, s)) return 1;
    if (sp.learn_alpha && edge(h, s2, s)) return 1;
    if (edge(h, s4, s)) return 1;
  }
  return 0;
}

static int enqueue_program(b200rl_offpolicy* h, const b200rl_offpolicy_hparams* hp, int S, int B, cudaStream_t s,
                           int* n_pol) {
  if (h->edac) {
    *n_pol = S;
    return enqueue_edac_steps(h, hp, S, B, s);
  }
  if (h->redq) {
    *n_pol = (S + hp->policy_delay - 1) / hp->policy_delay;
    return enqueue_redq_steps(h, hp, S, B, s);
  }
  if (h->iql) {
    *n_pol = S;
    return enqueue_iql_steps(h, hp, S, B, s);
  }
  if (h->sac) {
    *n_pol = S;
    return enqueue_sac_steps(h, hp, S, B, s);
  }
  if (h->dsac) {
    *n_pol = S;
    return enqueue_dsac_steps(h, hp, S, B, s);
  }
  if (h->dqn) return enqueue_dqn_steps(h, hp, S, B, s);
  return enqueue_steps(h, hp, S, B, s, n_pol);
}

// Runs the S steps on minibatches ALREADY staged in h->obs ... h->eps (stream h->gs) and reads the logs back.
static int run_staged(b200rl_offpolicy* h, const b200rl_offpolicy_hparams* hp, int32_t S, int32_t B, float* q1_values,
                      float* q2_values, float* q1_losses, float* q2_losses, float* policy_losses,
                      int32_t* n_policy_updates) {
  const bool td3 = h->cfg.n_q == 2;
  cudaStream_t s = h->gs;
  const size_t SB = (size_t)S * B;
  h->per_last = h->per_run;  // what get_per_draws may report
  h->nstep_last = h->nstep > 1;  // and get_nstep_draws
  if (h->iqn) h->iqn_last_B = B;  // and get_iqn_draws
  if (h->redq) h->redq_last_S = S, h->redq_last_B = B;  // and redq_outputs

  // Adam's step-dependent scalars for the steps of this call (torch's host-side double arithmetic), one small upload
  // (a group: one table per learner, from that learner's step counts, uploaded with one strided copy)
  const int maxS = h->cfg.max_steps;
  const int n_pol_expected = h->dqn ? 0 : (h->redq && !h->edac) || !(h->sac || h->dsac || h->iql)
                                                 ? (S + hp->policy_delay - 1) / hp->policy_delay
                                                 : S;  // SAC: no delay
  const size_t tab_n = adam_tab_len(h);
  const bool learn_alpha = (h->sac || h->dsac) && h->sac_hp.learn_alpha;
  const bool lagrange = h->cql && h->cql_cfg.lagrange;
  for (int z = 0; z < h->K; ++z) {
    float2* tab = h->h_adam_tab + z * tab_n;
    for (int k = 0; k < n_pol_expected; ++k)
      adam_scalars(h->net[0].step[z] + k + 1, hp->policy_lr, hp->policy_beta1, hp->policy_beta2, &tab[k].x, &tab[k].y);
    for (int qi = 0; qi < (td3 ? 2 : 1); ++qi)
      for (int k = 0; k < S; ++k)
        adam_scalars(h->net[1 + qi].step[z] + k + 1, qi == 0 ? hp->q1_lr : hp->q2_lr, hp->q_beta1, hp->q_beta2,
                     &tab[(size_t)(1 + qi) * maxS + k].x, &tab[(size_t)(1 + qi) * maxS + k].y);
    if (learn_alpha)
      for (int k = 0; k < S; ++k)
        adam_scalars(h->alpha_step[z] + k + 1, h->sac_hp.alpha_lr, h->sac_hp.alpha_beta1, h->sac_hp.alpha_beta2,
                     &tab[(size_t)3 * maxS + k].x, &tab[(size_t)3 * maxS + k].y);
    if (h->iql)
      for (int k = 0; k < S; ++k)
        adam_scalars(h->net[3].step[z] + k + 1, h->iql_hp.v_lr, h->iql_hp.v_beta1, h->iql_hp.v_beta2,
                     &tab[(size_t)3 * maxS + k].x, &tab[(size_t)3 * maxS + k].y);
    if (lagrange)
      for (int k = 0; k < S; ++k)
        adam_scalars(h->ap_step[z] + k + 1, h->cql_hp.alpha_lr, h->cql_hp.alpha_beta1, h->cql_hp.alpha_beta2,
                     &tab[(size_t)4 * maxS + k].x, &tab[(size_t)4 * maxS + k].y);
    if (h->dqn)  // copy after the steps that bring the Q optimizer's count to a multiple of the interval
      for (int k = 0; k < S; ++k)
        tab[(size_t)3 * maxS + k] = make_float2((h->net[1].step[z] + k + 1) % h->dqn_hp.target_update_interval == 0, 0.f);
    if (h->per_run)  // beta = min(1, beta0 + (1 - beta0) t / anneal), t = the Q optimizer's count before the step
      for (int k = 0; k < S; ++k) {
        const double b0 = h->per_hp.beta_start;
        const double t = (double)(h->net[1].step[z] + k);
        tab[(size_t)3 * maxS + k].y = (float)std::min(1.0, b0 + (1.0 - b0) * t / (double)h->per_hp.beta_anneal_steps);
      }
  }
  B200RL_CUDA(cudaMemcpy2DAsync(h->adam_tab, h->lane_stride, h->h_adam_tab, tab_n * sizeof(float2),
                                tab_n * sizeof(float2), h->K, cudaMemcpyHostToDevice, s));

  int n_pol = 0;
  const char* genv = getenv("B200RL_OFFPOLICY_GRAPH");
  const bool use_graph = !(genv != nullptr && genv[0] == '0');
  if (!use_graph) {
    if (enqueue_program(h, hp, S, B, s, &n_pol)) return 1;
  } else {
    GraphKey key;
    memset(&key, 0, sizeof(key));
    key.S = S, key.B = B, key.nstep = h->nstep;
    key.hp = *hp, key.sac = h->sac_hp, key.dqn = h->dqn_hp, key.c51 = h->c51_hp, key.qr = h->qr_hp;
    key.cql = h->cql_hp;
    key.iql = h->iql_hp, key.iql.v_lr = 0.0;
    if (h->per_run) key.per = h->per_hp, key.replay = h->replay;
    if (h->graph == nullptr || memcmp(&key, &h->graph_key, sizeof(key)) != 0) {
      if (h->graph) {
        cudaGraphExecDestroy(h->graph);
        h->graph = nullptr;
      }
      const int64_t l0 = launches_total();
      B200RL_CUDA(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
      const int rc = enqueue_program(h, hp, S, B, s, &n_pol);
      cudaGraph_t g = nullptr;
      const cudaError_t ce = cudaStreamEndCapture(s, &g);
      if (rc || ce != cudaSuccess || g == nullptr) {
        if (g) cudaGraphDestroy(g);
        if (!rc) set_error("offpolicy_train: stream capture failed: %s", cudaGetErrorString(ce));
        return 1;
      }
      const cudaError_t ie = cudaGraphInstantiate(&h->graph, g, 0);
      cudaGraphDestroy(g);
      if (ie != cudaSuccess) {
        h->graph = nullptr;
        set_error("offpolicy_train: cudaGraphInstantiate failed: %s", cudaGetErrorString(ie));
        return 1;
      }
      h->graph_launches = (int)(launches_total() - l0);
      count_launch(-h->graph_launches);  // counted per replay below
      h->graph_key = key;
      h->graph_npol = n_pol;
    }
    n_pol = h->graph_npol;
    B200RL_CUDA(cudaGraphLaunch(h->graph, s));
    count_launch(h->graph_launches);
  }
  for (int z = 0; z < h->K; ++z) {
    h->net[0].step[z] += n_pol;
    h->net[1].step[z] += S;
    if (td3) h->net[2].step[z] += S;
    for (int k = 3; h->redq && k <= h->redq_cfg.n_critics; ++k) h->net[k].step[z] += S;
    if (learn_alpha) h->alpha_step[z] += h->redq ? n_pol : S;  // REDQ: one temperature step per policy step
    if (lagrange) h->ap_step[z] += S;
    if (h->iql) h->net[3].step[z] += S;
  }
  // one device -> host read of everything train() logs: [K, S, B] values, [K, S] losses
  const size_t ls = h->lane_stride, K = (size_t)h->K;
  B200RL_CUDA(cudaMemcpy2DAsync(q1_values, SB * 4, h->out_q1, ls, SB * 4, K, cudaMemcpyDeviceToHost, s));
  B200RL_CUDA(cudaMemcpy2DAsync(q1_losses, (size_t)S * 4, h->out_l1, ls, (size_t)S * 4, K, cudaMemcpyDeviceToHost, s));
  if (td3) {  // REDQ: critic 2's, right behind critic 1's
    B200RL_CUDA(cudaMemcpy2DAsync(q2_values, SB * 4, h->redq ? h->out_q1 + SB : h->out_q2, ls, SB * 4, K,
                                  cudaMemcpyDeviceToHost, s));
    B200RL_CUDA(cudaMemcpy2DAsync(q2_losses, (size_t)S * 4, h->redq ? h->out_l1 + S : h->out_l2, ls, (size_t)S * 4, K,
                                  cudaMemcpyDeviceToHost, s));
  }
  if (n_pol > 0 && policy_losses != nullptr)  // NULL: a prioritized call (get_policy_losses reads them)
    B200RL_CUDA(cudaMemcpy2DAsync(policy_losses, (size_t)S * 4, h->out_lp, ls, (size_t)n_pol * 4, K,
                                  cudaMemcpyDeviceToHost, s));
  h->last_npol = n_pol;
  std::vector<int> bad(h->dqn || h->dsac ? K * S : 0), per_bad(h->per_run ? K * S : 0);
  if (h->dqn || h->dsac)
    B200RL_CUDA(cudaMemcpy2DAsync(bad.data(), (size_t)S * 4, h->dqn_bad, ls, (size_t)S * 4, K, cudaMemcpyDeviceToHost, s));
  if (h->per_run)
    B200RL_CUDA(cudaMemcpy2DAsync(per_bad.data(), (size_t)S * 4, h->per_bad, ls, (size_t)S * 4, K,
                                  cudaMemcpyDeviceToHost, s));
  B200RL_CUDA(cudaStreamSynchronize(s));
  *n_policy_updates = n_pol;
  const int n_actions = h->net[1].d.sizes[h->net[1].d.n_layers] /
                        (h->c51 ? h->c51_hp.n_atoms : h->qr ? h->qr_hp.n_quantiles : 1);
  const char* algo = h->c51 ? "C51" : h->qr ? "QR-DQN" : h->iqn ? "IQN" : h->dsac ? "discrete SAC" : h->d4pg ? "D4PG"
                                                                                                       : "DQN";
  for (size_t i = 0; i < bad.size(); ++i)
    B200RL_REQUIRE(bad[i] == 0, "offpolicy_train: %s learner %d, step %d: %d minibatch rows hold an action that is not "
                   "an integer in [0, %d); those rows were left out of the update", algo, (int)(i / S), (int)(i % S),
                   bad[i], n_actions);
  for (size_t i = 0; i < per_bad.size(); ++i)
    B200RL_REQUIRE(per_bad[i] == 0, "offpolicy_train_prioritized: %s learner %d, step %d: %d minibatch rows gave a "
                   "non-finite priority; their leaves were left unchanged", algo, (int)(i / S), (int)(i % S),
                   per_bad[i]);
  return 0;
}

// The front matter of every train call after its NULL checks: the checks all calls share, then `own` (the call's own
// checks), then -1 for S = 0 (nothing to run) or the engine's stream joined to the caller's `stream`.  noise_given: the
// call hands over (or draws) the noise its engine needs.
template <typename Own>
static int train_begin(b200rl_offpolicy* h, const b200rl_offpolicy_hparams* hp, int32_t S, int32_t B, bool noise_given,
                       bool q2_given, int32_t* n_policy_updates, void* stream, const char* what, Own own) {
  B200RL_REQUIRE(S >= 0 && S <= h->cfg.max_steps && B >= 1 && B <= h->cfg.max_minibatch,
                 "%s: S=%d B=%d exceed the capacities", what, S, B);
  B200RL_REQUIRE(h->cfg.n_q != 2 || q2_given, "%s: TD3 needs the Q2 outputs", what);
  B200RL_REQUIRE(h->dqn || h->dsac || !hp->use_target_noise || noise_given, "%s: target noise requested but no noise "
                 "given", what);
  B200RL_REQUIRE(h->dqn || h->dsac || hp->policy_delay >= 1, "%s: policy_delay must be >= 1", what);
  B200RL_REQUIRE(!h->d4pg || !hp->use_target_noise, "%s: D4PG has no target-policy smoothing: use_target_noise must be "
                 "0", what);
  if (h->sac) {
    B200RL_REQUIRE(h->sac_set, "%s: a SAC engine needs b200rl_offpolicy_set_sac before it trains", what);
    B200RL_REQUIRE(noise_given, "%s: SAC needs the noise draws [S, 2, B, A]", what);
  }
  B200RL_REQUIRE(!h->cql || h->cql_set, "%s: a CQL engine needs b200rl_offpolicy_set_cql before it trains", what);
  if (h->redq) {  // one Adam table row serves every critic
    B200RL_REQUIRE(hp->q1_lr == hp->q2_lr, "%s: REDQ's critics share one learning rate: q1_lr %g != q2_lr %g", what,
                   hp->q1_lr, hp->q2_lr);
    for (int z = 0; z < h->K; ++z)
      for (int k = 2; k <= h->redq_cfg.n_critics; ++k)
        B200RL_REQUIRE(h->net[k].step[z] == h->net[1].step[z], "%s: REDQ's critics share one Adam step count: learner "
                       "%d, critic %d has %lld steps, critic 1 %lld", what, z, k, (long long)h->net[k].step[z],
                       (long long)h->net[1].step[z]);
  }
  if (h->iql) {
    B200RL_REQUIRE(h->iql_set, "%s: an IQL engine needs b200rl_offpolicy_set_iql before it trains", what);
    B200RL_REQUIRE(!hp->use_target_noise && !noise_given, "%s: an IQL engine draws no noise: use_target_noise must be "
                   "0 and the noise NULL", what);
  }
  B200RL_REQUIRE(!h->dsac || h->sac_set, "%s: a discrete SAC engine needs b200rl_offpolicy_set_sac before it trains",
                 what);
  if (h->dqn) {
    B200RL_REQUIRE(h->dqn_set, "%s: a DQN engine needs b200rl_offpolicy_set_dqn before it trains", what);
    B200RL_REQUIRE(!h->c51 || h->c51_set, "%s: a C51 engine needs b200rl_offpolicy_set_c51 before it trains", what);
  }
  B200RL_REQUIRE(!h->noisy || h->noisy_keys, "%s: an engine with noisy layers needs fresh keys from "
                 "b200rl_offpolicy_set_noise_keys before every train call", what);
  B200RL_REQUIRE(!h->iqn || h->noisy_keys, "%s: an IQN engine needs fresh keys for its fraction draws from "
                 "b200rl_offpolicy_set_noise_keys before every train call", what);
  if (int rc = own()) return rc;
  h->noisy_keys = false;  // this call consumes them
  *n_policy_updates = 0;
  if (S == 0) return -1;
  B200RL_CUDA(cudaEventRecord(h->ev, static_cast<cudaStream_t>(stream)));
  B200RL_CUDA(cudaStreamWaitEvent(h->gs, h->ev, 0));
  return 0;
}

extern "C" int b200rl_offpolicy_train(b200rl_offpolicy* h, const b200rl_offpolicy_hparams* hp, int32_t S, int32_t B,
                                      const float* obs, const float* act, const float* rew, const float* next_obs,
                                      const float* done, const float* noise, float* q1_values, float* q2_values,
                                      float* q1_losses, float* q2_losses, float* policy_losses,
                                      int32_t* n_policy_updates, void* stream) {
  B200RL_REQUIRE(h && hp && obs && act && rew && next_obs && done && q1_values && q1_losses &&
                     (policy_losses || h->dqn) && n_policy_updates, "offpolicy_train: NULL argument");
  const auto own = [&] {
    B200RL_REQUIRE(h->nstep == 1, "offpolicy_train: n-step returns (n_step = %d) need the device replay columns: use "
                   "train_gather, train_gather_rng or train_prioritized", h->nstep);
    return 0;
  };
  if (int rc = train_begin(h, hp, S, B, noise != nullptr, q2_values && q2_losses, n_policy_updates, stream,
                           "offpolicy_train", own))
    return rc < 0 ? 0 : rc;
  cudaStream_t s = h->gs;  // everything runs on the engine's stream, ordered after the caller's
  const int O = h->O, A = h->A;
  const size_t SB = (size_t)S * B;
  // one host -> device upload of every minibatch of this train() call ([K, S, B, ...] into the K arenas)
  auto up = [&](void* dst, const void* src, size_t bytes) -> int {
    B200RL_CUDA(cudaMemcpy2DAsync(dst, h->lane_stride, src, bytes, bytes, h->K, cudaMemcpyHostToDevice, s));
    return 0;
  };
  if (up(h->obs, obs, SB * O * 4) || up(h->act, act, SB * A * 4) || up(h->rew, rew, SB * 4) ||
      up(h->nobs, next_obs, SB * O * 4) || up(h->done, done, SB * 4))
    return 1;
  if (h->sac && up(h->eps, noise, 2 * SB * A * 4)) return 1;
  if (cql_take_draws(h, S, B, "offpolicy_train") || redq_take_subsets(h, S, "offpolicy_train")) return 1;
  if (!h->sac && !h->dqn && !h->dsac && hp->use_target_noise && up(h->eps, noise, SB * A * 4)) return 1;

  return run_staged(h, hp, S, B, q1_values, q2_values, q1_losses, q2_losses, policy_losses, n_policy_updates);
}

// The five staged columns (obs, act, rew, next_obs, done) gathered from the call's replay table at the rows in h->idx:
// one launch per column for all learners; with n-step returns one nstep_gather_kernel launch, which also stages the
// discounts and last rows
static int gather_columns(b200rl_offpolicy* h, const b200rl_offpolicy_hparams* hp, long long SB, cudaStream_t s) {
  const int O = h->O, A = h->A;
  const ReplayLanes<true>& r = h->replay;
  if (h->nstep > 1)
    return launch(h, nstep_gather_kernel<false>, nstep_gather_kernel<true>, (unsigned)((SB + GTHREADS - 1) / GTHREADS),
                  GTHREADS, 0, s, r, h->idx, SB, O, A, h->nstep, (float)hp->gamma, h->obs, h->act, h->rew, h->nobs,
                  h->done, h->nstep_disc, h->nstep_rows);
  const LaneSrc<true>* src[5] = {&r.obs, &r.act, &r.rew, &r.next_obs, &r.done};
  float* dst[5] = {h->obs, h->act, h->rew, h->nobs, h->done};
  const int w[5] = {O, A, 1, O, 1};
  for (int c = 0; c < 5; ++c)
    if (launch(h, gather_rows_kernel<false>, gather_rows_kernel<true>, (unsigned)((SB * w[c] + 255) / 256), 256, 0, s,
               *src[c], h->idx, w[c], SB, dst[c]))
      return 1;
  return 0;
}

// The call's replay table: each learner's columns, row count, episode-end column (set_nstep) and tree (trees NULL:
// none)
static void set_replay(b200rl_offpolicy* h, const b200rl_offpolicy_replay* rb, float* const* trees) {
  ReplayLanes<true>& r = h->replay;
  r = ReplayLanes<true>{};
  for (int z = 0; z < h->K; ++z) {
    r.obs.p[z] = rb[z].obs, r.act.p[z] = rb[z].act, r.rew.p[z] = rb[z].rew, r.next_obs.p[z] = rb[z].next_obs;
    r.done.p[z] = rb[z].done, r.ends.p[z] = h->nstep_ends.p[z];
    r.tree[z] = trees != nullptr ? trees[z] : nullptr;
    r.rows[z] = rb[z].rows;
  }
}

static int check_replay(const b200rl_offpolicy* h, const b200rl_offpolicy_replay* rb, const char* what) {
  B200RL_REQUIRE(rb != nullptr, "%s: NULL replay columns", what);
  for (int z = 0; z < h->K; ++z)
    B200RL_REQUIRE(rb[z].obs && rb[z].act && rb[z].rew && rb[z].next_obs && rb[z].done && rb[z].rows >= 1,
                   "%s: learner %d: NULL replay column or no rows", what, z);
  return 0;
}

extern "C" int b200rl_offpolicy_train_gather_group(b200rl_offpolicy* h, const b200rl_offpolicy_hparams* hp, int32_t S,
                                                   int32_t B, const b200rl_offpolicy_replay* rb, const int64_t* idx,
                                                   const float* noise, float* q1_values, float* q2_values,
                                                   float* q1_losses, float* q2_losses, float* policy_losses,
                                                   int32_t* n_policy_updates, void* stream) {
  B200RL_REQUIRE(h && hp && idx && q1_values && q1_losses && (policy_losses || h->dqn) && n_policy_updates,
                 "offpolicy_train_gather: NULL argument");
  if (int rc = check_replay(h, rb, "offpolicy_train_gather")) return rc;
  const size_t SB = (size_t)S * B;
  const auto own = [&] {
    for (int z = 0; z < h->K; ++z)
      for (size_t i = 0; i < SB; ++i)
        B200RL_REQUIRE(idx[z * SB + i] >= 0 && idx[z * SB + i] < rb[z].rows,
                       "offpolicy_train_gather: index %lld outside the %lld replay rows", (long long)idx[z * SB + i],
                       (long long)rb[z].rows);
    return 0;
  };
  if (int rc = train_begin(h, hp, S, B, noise != nullptr, q2_values && q2_losses, n_policy_updates, stream,
                           "offpolicy_train_gather", own))
    return rc < 0 ? 0 : rc;
  set_replay(h, rb, nullptr);
  cudaStream_t s = h->gs;
  const int A = h->A;
  // the minibatches are gathered on the device from the replay columns: only the indices (and noise) cross PCIe
  const size_t ls = h->lane_stride;
  B200RL_CUDA(cudaMemcpy2DAsync(h->idx, ls, idx, SB * 8, SB * 8, h->K, cudaMemcpyHostToDevice, s));
  const size_t n_eps = h->sac ? 2 * SB * A : (hp->use_target_noise && !h->dqn && !h->dsac ? SB * A : 0);
  if (n_eps) B200RL_CUDA(cudaMemcpy2DAsync(h->eps, ls, noise, n_eps * 4, n_eps * 4, h->K, cudaMemcpyHostToDevice, s));
  if (cql_take_draws(h, S, B, "offpolicy_train_gather") || redq_take_subsets(h, S, "offpolicy_train_gather"))
    return 1;
  if (gather_columns(h, hp, (long long)SB, s)) return 1;
  return run_staged(h, hp, S, B, q1_values, q2_values, q1_losses, q2_losses, policy_losses, n_policy_updates);
}

extern "C" int b200rl_offpolicy_train_gather(b200rl_offpolicy* h, const b200rl_offpolicy_hparams* hp, int32_t S,
                                             int32_t B, const float* d_obs, const float* d_act, const float* d_rew,
                                             const float* d_next_obs, const float* d_done, int64_t rows,
                                             const int64_t* idx, const float* noise, float* q1_values,
                                             float* q2_values, float* q1_losses, float* q2_losses,
                                             float* policy_losses, int32_t* n_policy_updates, void* stream) {
  B200RL_REQUIRE(h == nullptr || h->K == 1, "offpolicy_train_gather: a learner group takes train_gather_group");
  B200RL_REQUIRE(d_obs && d_act && d_rew && d_next_obs && d_done, "offpolicy_train_gather: NULL argument");
  const b200rl_offpolicy_replay rb = {d_obs, d_act, d_rew, d_next_obs, d_done, rows};
  return b200rl_offpolicy_train_gather_group(h, hp, S, B, &rb, idx, noise, q1_values, q2_values, q1_losses, q2_losses,
                                             policy_losses, n_policy_updates, stream);
}

/* Opt-in: the minibatch indices and the target-smoothing noise are DRAWN ON THE DEVICE (Philox4x32-10 keyed by `seed`,
 * block `call`), so nothing but the hyper-parameters crosses PCIe on the way in.  The streams are not the reference's
 * (numpy's MT19937 / torch's CPU generator): same distributions, different numbers -- callers that need the reference's
 * draws use b200rl_offpolicy_train_gather.  The ring: `size` live rows, logical row u at physical (start + u) % rows. */
extern "C" int b200rl_offpolicy_train_gather_rng_group(b200rl_offpolicy* h, const b200rl_offpolicy_hparams* hp,
                                                       int32_t S, int32_t B, const b200rl_offpolicy_replay* rb,
                                                       const int64_t* ring_start, const int64_t* ring_size,
                                                       const uint64_t* seed, const uint64_t* call, float* q1_values,
                                                       float* q2_values, float* q1_losses, float* q2_losses,
                                                       float* policy_losses, int32_t* n_policy_updates, void* stream) {
  B200RL_REQUIRE(h && hp && ring_start && ring_size && seed && call && q1_values && q1_losses &&
                     (policy_losses || h->dqn) && n_policy_updates, "offpolicy_train_gather_rng: NULL argument");
  if (int rc = check_replay(h, rb, "offpolicy_train_gather_rng")) return rc;
  const auto own = [&] {
    for (int z = 0; z < h->K; ++z) {
      const long long rows = rb[z].rows;
      B200RL_REQUIRE(ring_size[z] >= 1 && ring_size[z] <= rows && ring_start[z] >= 0 && ring_start[z] < rows,
                     "offpolicy_train_gather_rng: bad ring (rows %lld, start %lld, size %lld)", rows,
                     (long long)ring_start[z], (long long)ring_size[z]);
    }
    return 0;
  };
  if (int rc = train_begin(h, hp, S, B, !h->iql, q2_values && q2_losses, n_policy_updates, stream,  // IQL: indices only
                           "offpolicy_train_gather_rng", own))
    return rc < 0 ? 0 : rc;
  set_replay(h, rb, nullptr);
  cudaStream_t s = h->gs;
  const int A = h->A;
  const long long SB = (long long)S * B;
  // DQN and discrete SAC: indices only
  const long long n_eps = h->sac ? 2 * SB * A : (hp->use_target_noise && !h->dqn && !h->dsac ? SB * A : 0);
  const long long n_thr = ((SB > n_eps ? SB : n_eps) + 3) / 4;
  DrawKeys<true> keys{};
  for (int z = 0; z < h->K; ++z)
    keys.seed[z] = seed[z], keys.call[z] = call[z], keys.start[z] = ring_start[z], keys.size[z] = ring_size[z],
    keys.capacity[z] = rb[z].rows;
  if (launch(h, draw_minibatches_kernel<false>, draw_minibatches_kernel<true>, (unsigned)((n_thr + 255) / 256), 256, 0,
             s, h->idx, SB, n_eps ? h->eps : nullptr, n_eps, keys))
    return 1;
  if (h->cql) {  // CQL's draws under their own Philox tag
    const long long n_cql = (long long)cql_draw_floats(h, S, B);
    if (launch(h, cql_draw_kernel<false>, cql_draw_kernel<true>, (unsigned)((n_cql / 4 + 1 + 255) / 256), 256, 0, s,
               h->cql_draws, n_cql, (long long)B * h->cql_cfg.n_actions * A, keys))
      return 1;
  }
  if (h->redq && !h->edac && launch(h, redq_draw_kernel<false>, redq_draw_kernel<true>, (unsigned)((S + 127) / 128), 128, 0, s,
                        h->redq_sub, (int)S, h->redq_cfg.n_critics, h->redq_cfg.n_min, keys))
    return 1;
  if (gather_columns(h, hp, SB, s)) return 1;
  return run_staged(h, hp, S, B, q1_values, q2_values, q1_losses, q2_losses, policy_losses, n_policy_updates);
}

extern "C" int b200rl_offpolicy_train_gather_rng(b200rl_offpolicy* h, const b200rl_offpolicy_hparams* hp, int32_t S,
                                                 int32_t B, const float* d_obs, const float* d_act, const float* d_rew,
                                                 const float* d_next_obs, const float* d_done, int64_t rows,
                                                 int64_t ring_start, int64_t ring_size, uint64_t seed, uint64_t call,
                                                 float* q1_values, float* q2_values, float* q1_losses,
                                                 float* q2_losses, float* policy_losses, int32_t* n_policy_updates,
                                                 void* stream) {
  B200RL_REQUIRE(h == nullptr || h->K == 1, "offpolicy_train_gather_rng: a learner group takes train_gather_rng_group");
  B200RL_REQUIRE(d_obs && d_act && d_rew && d_next_obs && d_done, "offpolicy_train_gather_rng: NULL argument");
  const b200rl_offpolicy_replay rb = {d_obs, d_act, d_rew, d_next_obs, d_done, rows};
  return b200rl_offpolicy_train_gather_rng_group(h, hp, S, B, &rb, &ring_start, &ring_size, &seed, &call, q1_values,
                                                 q2_values, q1_losses, q2_losses, policy_losses, n_policy_updates,
                                                 stream);
}

/* The draws of the last train_gather / train_gather_rng call (physical rows [S*B], noise [S*B*A] or NULL): what a test
 * replays through the oracle. */
extern "C" int b200rl_offpolicy_get_draws(b200rl_offpolicy* h, int32_t S, int32_t B, int64_t* idx, float* noise,
                                          void* stream) {
  B200RL_REQUIRE(h && idx && S >= 0 && S <= h->cfg.max_steps && B >= 1 && B <= h->cfg.max_minibatch,
                 "offpolicy_get_draws: bad arguments");
  cudaStream_t s = h->gs;
  (void)stream;
  const size_t SB = (size_t)S * B;
  static_assert(sizeof(long long) == sizeof(int64_t), "index width");
  const size_t n_eps = (h->sac ? 2 : 1) * SB * h->A;
  B200RL_REQUIRE(!h->iql || noise == nullptr, "offpolicy_get_draws: an IQL engine draws no noise: noise must be NULL");
  B200RL_CUDA(cudaMemcpy2DAsync(idx, SB * 8, h->idx, h->lane_stride, SB * 8, h->K, cudaMemcpyDeviceToHost, s));
  if (noise)
    B200RL_CUDA(cudaMemcpy2DAsync(noise, n_eps * 4, h->eps, h->lane_stride, n_eps * 4, h->K, cudaMemcpyDeviceToHost, s));
  B200RL_CUDA(cudaStreamSynchronize(s));
  return 0;
}

/* Prioritized replay (DQN engines): each step draws its minibatch from the learner's sum tree, weighs the rows, and
 * writes the new priorities back into the tree, all inside the step program (see b200rl.h). */
extern "C" int b200rl_offpolicy_train_prioritized_group(b200rl_offpolicy* h, const b200rl_offpolicy_hparams* hp,
                                                        int32_t S, int32_t B, const b200rl_offpolicy_replay* rb,
                                                        float* const* trees, const uint64_t* seed, const uint64_t* call,
                                                        float* q1_values, float* q1_losses, void* stream) {
  B200RL_REQUIRE(h && hp && trees && seed && call && q1_values && q1_losses,
                 "offpolicy_train_prioritized: NULL argument");
  B200RL_REQUIRE(!h->c51, "offpolicy_train_prioritized: prioritized replay is not implemented for C51 engines");
  B200RL_REQUIRE(!h->dsac, "offpolicy_train_prioritized: prioritized replay is not implemented for discrete SAC "
                 "engines (algo = 5)");
  B200RL_REQUIRE(!h->edac, "offpolicy_train_prioritized: prioritized replay is not implemented for EDAC engines "
                 "(algo = 11)");
  B200RL_REQUIRE(!h->redq, "offpolicy_train_prioritized: prioritized replay is not implemented for REDQ engines "
                 "(algo = 10)");
  B200RL_REQUIRE(!h->tqc, "offpolicy_train_prioritized: prioritized replay is not implemented for TQC engines (algo = "
                 "7)");
  B200RL_REQUIRE(!h->iql, "offpolicy_train_prioritized: prioritized replay is not implemented for IQL engines (algo = "
                 "9)");
  B200RL_REQUIRE(h->dqn || h->d4pg, "offpolicy_train_prioritized: prioritized replay is implemented for DQN engines "
                 "(algo = 2) and D4PG engines (algo = 6) only");
  B200RL_REQUIRE(h->per_set, "offpolicy_train_prioritized: call b200rl_offpolicy_set_per first");
  if (int rc = check_replay(h, rb, "offpolicy_train_prioritized")) return rc;
  const auto own = [&] {
    for (int z = 0; z < h->K; ++z) {
      B200RL_REQUIRE(trees[z] != nullptr, "offpolicy_train_prioritized: learner %d: NULL tree", z);
      B200RL_REQUIRE(rb[z].rows < ((int64_t)1 << 31),
                     "offpolicy_train_prioritized: learner %d: more than 2^31 - 1 rows", z);
      // every learner's update kernel rewrites its tree's leaves and interior nodes concurrently with the others: two
      // learners on one tree would race (stale interior sums, a lost running max)
      for (int y = 0; y < z; ++y)
        B200RL_REQUIRE(trees[y] != trees[z], "offpolicy_train_prioritized: learners %d and %d share one tree: every "
                       "learner of a group needs its own prioritized replay buffer", y, z);
    }
    return 0;
  };
  int32_t n_pol = 0;
  if (int rc = train_begin(h, hp, S, B, true, false, &n_pol, stream, "offpolicy_train_prioritized", own))
    return rc < 0 ? 0 : rc;
  set_replay(h, rb, trees);
  const size_t tab_n = adam_tab_len(h);
  for (int z = 0; z < h->K; ++z) {
    unsigned long long* keys =
        reinterpret_cast<unsigned long long*>(h->h_adam_tab + z * tab_n + (size_t)4 * h->cfg.max_steps);
    keys[0] = seed[z], keys[1] = call[z];  // uploaded with the table by run_staged
  }
  h->per_run = true;
  const int rc = run_staged(h, hp, S, B, q1_values, nullptr, q1_losses, nullptr, nullptr, &n_pol);
  h->per_run = false;
  return rc;
}

extern "C" int b200rl_offpolicy_train_prioritized(b200rl_offpolicy* h, const b200rl_offpolicy_hparams* hp, int32_t S,
                                                  int32_t B, const float* d_obs, const float* d_act, const float* d_rew,
                                                  const float* d_next_obs, const float* d_done, int64_t rows,
                                                  float* tree, uint64_t seed, uint64_t call, float* q1_values,
                                                  float* q1_losses, void* stream) {
  B200RL_REQUIRE(h == nullptr || h->K == 1,
                 "offpolicy_train_prioritized: a learner group takes train_prioritized_group");
  const b200rl_offpolicy_replay rb = {d_obs, d_act, d_rew, d_next_obs, d_done, rows};
  return b200rl_offpolicy_train_prioritized_group(h, hp, S, B, &rb, &tree, &seed, &call, q1_values, q1_losses, stream);
}

extern "C" int b200rl_offpolicy_get_per_draws(b200rl_offpolicy* h, int32_t S, int32_t B, int64_t* idx, float* weights,
                                              float* priorities, void* stream) {
  B200RL_REQUIRE(h && (h->dqn || h->d4pg) && idx && weights && priorities && S >= 0 && S <= h->cfg.max_steps && B >= 1 &&
                     B <= h->cfg.max_minibatch, "offpolicy_get_per_draws: bad arguments");
  B200RL_REQUIRE(h->per_last, "offpolicy_get_per_draws: the engine's last train call was not a prioritized one");
  (void)stream;
  cudaStream_t s = h->gs;
  const size_t SB = (size_t)S * B, ls = h->lane_stride;
  B200RL_CUDA(cudaMemcpy2DAsync(idx, SB * 8, h->idx, ls, SB * 8, h->K, cudaMemcpyDeviceToHost, s));
  B200RL_CUDA(cudaMemcpy2DAsync(weights, SB * 4, h->per_w, ls, SB * 4, h->K, cudaMemcpyDeviceToHost, s));
  B200RL_CUDA(cudaMemcpy2DAsync(priorities, SB * 4, h->per_newp, ls, SB * 4, h->K, cudaMemcpyDeviceToHost, s));
  B200RL_CUDA(cudaStreamSynchronize(s));
  return 0;
}

extern "C" int b200rl_offpolicy_get_policy_losses(b200rl_offpolicy* h, int32_t S, float* policy_losses,
                                                  int32_t* n_policy_updates) {
  B200RL_REQUIRE(h && policy_losses && n_policy_updates && S >= 0 && S <= h->cfg.max_steps,
                 "offpolicy_get_policy_losses: bad arguments");
  B200RL_REQUIRE(!h->dqn, "offpolicy_get_policy_losses: a DQN engine has no policy");
  const int n = std::min(S, h->last_npol);
  if (n > 0)
    B200RL_CUDA(cudaMemcpy2DAsync(policy_losses, (size_t)S * 4, h->out_lp, h->lane_stride, (size_t)n * 4, h->K,
                                  cudaMemcpyDeviceToHost, h->gs));
  B200RL_CUDA(cudaStreamSynchronize(h->gs));
  *n_policy_updates = n;
  return 0;
}

extern "C" int b200rl_offpolicy_get_nstep_draws(b200rl_offpolicy* h, int32_t S, int32_t B, int64_t* last_rows,
                                                float* returns, float* discounts, void* stream) {
  B200RL_REQUIRE(h && (h->dqn || h->d4pg) && last_rows && returns && discounts && S >= 0 && S <= h->cfg.max_steps &&
                     B >= 1 &&
                     B <= h->cfg.max_minibatch, "offpolicy_get_nstep_draws: bad arguments");
  B200RL_REQUIRE(h->nstep_last, "offpolicy_get_nstep_draws: the engine's last train call was not an n-step one");
  (void)stream;
  cudaStream_t s = h->gs;
  const size_t SB = (size_t)S * B, ls = h->lane_stride;
  B200RL_CUDA(cudaMemcpy2DAsync(last_rows, SB * 8, h->nstep_rows, ls, SB * 8, h->K, cudaMemcpyDeviceToHost, s));
  B200RL_CUDA(cudaMemcpy2DAsync(returns, SB * 4, h->rew, ls, SB * 4, h->K, cudaMemcpyDeviceToHost, s));
  B200RL_CUDA(cudaMemcpy2DAsync(discounts, SB * 4, h->nstep_disc, ls, SB * 4, h->K, cudaMemcpyDeviceToHost, s));
  B200RL_CUDA(cudaStreamSynchronize(s));
  return 0;
}

extern "C" int64_t b200rl_per_tree_floats(int64_t leaves) {
  if (leaves < 1 || leaves >= ((int64_t)1 << 31)) return -1;
  long long off[PER_MAX_LEVELS + 1];
  const int top = per_levels(leaves, off);
  return off[top] + PER_FAN;
}

// parents of the leaves [lo, hi), level by level up to the root
static int per_tree_ancestors(float* tree, long long leaves, long long lo, long long hi, cudaStream_t s) {
  long long off[PER_MAX_LEVELS + 1];
  const int top = per_levels(leaves, off);
  for (int k = 1; k <= top; ++k) {
    lo /= PER_FAN;
    hi = (hi + PER_FAN - 1) / PER_FAN;
    per_tree_level_kernel<<<(unsigned)((hi - lo + 255) / 256), 256, 0, s>>>(tree, off[k - 1], off[k], lo, hi);
    B200RL_CUDA(cudaGetLastError());
    count_launch(1);
  }
  return 0;
}

extern "C" int b200rl_per_tree_build(float* tree, int64_t leaves, void* stream) {
  B200RL_REQUIRE(tree && b200rl_per_tree_floats(leaves) > 0, "per_tree_build: bad arguments (leaves %lld)",
                 (long long)leaves);
  return per_tree_ancestors(tree, leaves, 0, leaves, static_cast<cudaStream_t>(stream));
}

extern "C" int b200rl_per_tree_set_range(float* tree, int64_t leaves, int64_t start, int64_t count, void* stream) {
  B200RL_REQUIRE(tree && b200rl_per_tree_floats(leaves) > 0 && start >= 0 && start < leaves && count >= 0 &&
                     count <= leaves, "per_tree_set_range: bad arguments (leaves %lld, start %lld, count %lld)",
                 (long long)leaves, (long long)start, (long long)count);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const long long max_at = b200rl_per_tree_floats(leaves) - PER_FAN + 1;
  const long long first = std::min<long long>(count, leaves - start);
  const long long seg[2][2] = {{start, first}, {0, count - first}};  // wrap-aware
  for (const auto& g : seg) {
    if (g[1] == 0) continue;
    per_tree_fill_kernel<<<(unsigned)((g[1] + 255) / 256), 256, 0, s>>>(tree, g[0], g[1], max_at);
    B200RL_CUDA(cudaGetLastError());
    count_launch(1);
    if (per_tree_ancestors(tree, leaves, g[0], g[0] + g[1], s)) return 1;
  }
  return 0;
}
