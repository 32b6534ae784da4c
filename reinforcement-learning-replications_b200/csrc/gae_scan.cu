// gae_scan: bootstrapped rewards + discounted returns + TD residuals + GAE as ONE segmented reverse scan.
//
// Replaces (reference: /root/reference/src/rl_replicas/): utils.py:14-28 discounted_cumulative_sums,
// utils.py:31-44 gae, utils.py:74-87 bootstrap_rewards_with_last_values and the per-episode Python loops of
// algorithms/ppo.py:142-161.
//
// Both recurrences are first-order linear:  y_i = b_i + a_i * y_{i+1}  scanned from the END of the flat transition
// array, with a_i = 0 on the last step of every episode (segment reset):
//   returns:    a = gamma,        b_i = r_i            (+ gamma * V(last_obs) on the last step of a NOT-done episode)
//   advantages: a = gamma*lambda, b_i = delta_i = r_i + f32(gamma*v_{i+1}) - v_i     (v_L = V(last_obs) even when done)
// The pair (a,b) composes associatively: (a1,b1) o (a2,b2) = (a1*a2, b1 + a1*b2), so the scan is
//   thread: 8 consecutive items sequentially (exactly the reference's float64 recurrence inside a thread),
//   warp:   suffix scan of the 32 thread aggregates with shuffles,
//   CTA:    8 warp aggregates through shared memory,
//   grid:   single-pass decoupled look-back over tile descriptors.  The kernel is persistent: grid = resident CTAs,
//           CTA c walks tiles T-1-c, T-1-c-G, ... from the END of the array, so the tile it waits on always belongs to
//           a running CTA; a tile that contains an episode end has a == 0 and cuts the chain.  A producer warp
//           prefetches the next tile (cp.async) and finds its episode range while the scan warps work.
// HBM traffic = algorithmic traffic: read r (4 or 8 B) + v (4 B), write adv (4 B) + ret (4 B) per transition.
// All carries are float64 (the reference scans in float64, utils.py:28); outputs are cast to float32 like ppo.py:151,160.
#include <type_traits>

#include "common.cuh"

namespace b200rl {

constexpr int SCAN_CONSUMERS = 256;                 // 8 scan warps
constexpr int SCAN_THREADS = SCAN_CONSUMERS + 32;   // + 1 producer warp (cp.async prefetch + episode search)
constexpr int SCAN_ITEMS = 8;
constexpr int SCAN_TILE = SCAN_CONSUMERS * SCAN_ITEMS;  // 2048 transitions per tile

// Look-back records.  Each tile owns 8 x 16-byte records {value, tag}; a record is valid iff tag == launch tag.
// Value and tag travel in ONE 16-byte transaction, so no fence / release-acquire pair is needed to publish or to
// consume them (the trick CUB's decoupled look-back uses for its packed tile descriptors):
//   0 a_ret  1 b_ret  2 a_adv  3 b_adv   tile aggregate
//   4 y_ret  5 y_adv                      recurrence values at the tile's FIRST element ("inclusive")
struct __align__(16) ScanRec {
  double val, tag;
};
constexpr int SCAN_RECS = 8;
constexpr int SCAN_MAXE = 48;  // episodes per tile staged in shared memory (more: global-memory path)

// Workspace header.  The workspace is zeroed ONCE (at allocation); after that every launch cleans up after itself:
// look-back records carry the negated launch epoch as their tag (a stale record from an earlier launch, or statistics an
// earlier launch of another n left in the same bytes, read as "not ready"), and the last
// CTA to finish resets the done counter and bumps the epoch.  => one kernel launch per scan, no memset.
struct ScanHeader {
  int reserved0;
  int done;
  int epoch;
  int error;
  int pad[12];
};

struct Aff {
  double a, b;
};
__device__ __forceinline__ Aff compose(const Aff first, const Aff later) {
  return Aff{first.a * later.a, first.b + first.a * later.b};
}

struct ScanArgs {
  const void* rew;
  const float* values;
  const float* last_values;
  const long long* off;
  const unsigned char* done;
  long long n, n_ep;
  double gamma, gl;
  float gamma_f;
  float* adv;
  float* ret;
  ScanHeader* hdr;
  ScanRec* recs;
  double2* partial;
  double* stats;
  int num_tiles;
  double pw_r[5], pw_a[5];  // gamma^(8*2^k), (gamma*lambda)^(8*2^k): warp-scan multipliers of uncut chunks
};

// one pipeline slot: a tile's rewards and values (+ the first value of the next tile) and its episode range
template <typename RewT>
struct __align__(16) TileBuf {
  RewT r[SCAN_TILE];
  float v[SCAN_TILE + 4];
  long long e0, e1;
  long long soff[SCAN_MAXE + 2];  // off[e0 .. e1 + 1] when staged
  float slv[SCAN_MAXE];           // last_values[e0 .. e1]
  int sdone[SCAN_MAXE];           // done[e0 .. e1]
  int staged, pad;
};

__device__ __forceinline__ uint32_t sm_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void ld_rec(const ScanRec* p, double& v, double& t) {
  asm volatile("ld.volatile.global.v2.f64 {%0, %1}, [%2];" : "=d"(v), "=d"(t) : "l"(p) : "memory");
}
__device__ __forceinline__ void st_rec(ScanRec* p, double v, double t) {
  asm volatile("st.volatile.global.v2.f64 [%0], {%1, %2};" ::"l"(p), "d"(v), "d"(t) : "memory");
}
__device__ __forceinline__ void sbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void sbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool sbar_wait(uint32_t bar, uint32_t parity) {  // bounded: false = protocol failure
  for (uint32_t it = 0; it < (1u << 24); ++it) {
    uint32_t done;
    asm volatile(
        "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done) : "r"(bar), "r"(parity) : "memory");
    if (done) return true;
  }
  return false;
}
__device__ __forceinline__ void scan_cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, %0;" ::"n"(SCAN_CONSUMERS) : "memory"); }

// suffix scan of per-thread aggregates inside a warp; returns the EXCLUSIVE suffix (composition of lanes > lane)
// and leaves the inclusive aggregate of the whole warp in lane 0's `incl`.
__device__ __forceinline__ Aff warp_suffix_exclusive(Aff& incl, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const double a2 = __shfl_down_sync(0xffffffffu, incl.a, o);
    const double b2 = __shfl_down_sync(0xffffffffu, incl.b, o);
    if (lane + o < 32) {
      incl.b = incl.b + incl.a * b2;
      incl.a = incl.a * a2;
    }
  }
  Aff ex;
  ex.a = __shfl_down_sync(0xffffffffu, incl.a, 1);
  ex.b = __shfl_down_sync(0xffffffffu, incl.b, 1);
  if (lane == 31) {
    ex.a = 1.0;
    ex.b = 0.0;
  }
  return ex;
}

// Warp-cooperative 32-ary search: max e in [0, n_ep) with off[e] <= target (requires off[0] <= target < off[n_ep]).
__device__ __forceinline__ long long warp_find_episode(const long long* __restrict__ off, long long n_ep,
                                                       long long target, int lane) {
  long long lo = 0, hi = n_ep;  // invariant: off[lo] <= target < off[hi]
  while (hi - lo > 1) {
    const long long step = (hi - lo + 31) / 32;
    const long long idx = lo + (long long)lane * step;
    const bool ok = (idx < hi) && (__ldg(off + idx) <= target);  // monotone in lane; lane 0 is always true
    const int cnt = __popc(__ballot_sync(0xffffffffu, ok));
    lo = lo + (long long)(cnt - 1) * step;
    hi = (lo + step < hi) ? lo + step : hi;
  }
  return lo;
}

// Persistent kernel: CTA c owns tiles T-1-c, T-1-c-G, ... (from the END of the array; G = gridDim.x <= resident
// CTAs, so the tile a CTA waits on always belongs to a CTA that is running).  Warp 8 prefetches the next tile's
// rewards / values with cp.async and finds its episode range while warps 0..7 scan the current tile.
template <typename RewT>
__global__ void __launch_bounds__(SCAN_THREADS, 3) gae_scan_kernel(const ScanArgs p) {
  extern __shared__ __align__(16) unsigned char scan_smem[];
  TileBuf<RewT>* buf = reinterpret_cast<TileBuf<RewT>*>(scan_smem);
  __shared__ __align__(8) unsigned long long bars[4];  // full[0], full[1], empty[0], empty[1]
  __shared__ int s_epoch, s_last;
  __shared__ Aff s_wret[SCAN_CONSUMERS / 32], s_wadv[SCAN_CONSUMERS / 32];
  __shared__ Aff s_xret[SCAN_CONSUMERS / 32], s_xadv[SCAN_CONSUMERS / 32];  // composition of the warps AFTER w
  __shared__ double s_carry[2];
  __shared__ double s_red[2][SCAN_CONSUMERS / 32];

  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);  // provably warp-uniform role branch
  const int G = gridDim.x, c = blockIdx.x, T = p.num_tiles;
  const long long n = p.n;
  const int n_mine = (T - 1 - c) / G + 1;  // host guarantees G <= T
  if (tid == 0) {
    s_epoch = *reinterpret_cast<volatile int*>(&p.hdr->epoch);  // constant for the whole launch
    sbar_init(sm_addr(&bars[0]), 32);
    sbar_init(sm_addr(&bars[1]), 32);
    sbar_init(sm_addr(&bars[2]), 1);
    sbar_init(sm_addr(&bars[3]), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == SCAN_CONSUMERS / 32) {
    // ================================ producer warp ================================
    const RewT* rew = static_cast<const RewT*>(p.rew);
    for (int k = 0; k < n_mine; ++k) {
      const int tile = T - 1 - c - k * G, b = k & 1;
      if (k >= 2 && !sbar_wait(sm_addr(&bars[2 + b]), ((k >> 1) - 1) & 1)) {
        p.hdr->error = 1;
        return;
      }
      const long long t0 = (long long)tile * SCAN_TILE;
      const int cnt = (int)((n - t0) < SCAN_TILE ? (n - t0) : SCAN_TILE);
      const int cntv = cnt + ((t0 + cnt < n) ? 1 : 0);  // + first value of the next tile (v_{i+1} of the last item)
      // whole 16-byte chunks with cp.async (tile starts are 16-byte aligned), the ragged tail with plain copies
      const int r16 = (int)((size_t)cnt * sizeof(RewT) / 16), v16 = cntv * 4 / 16;
      const char* gr = reinterpret_cast<const char*>(rew + t0);
      const char* gv = reinterpret_cast<const char*>(p.values + t0);
      const uint32_t sr = sm_addr(buf[b].r), sv = sm_addr(buf[b].v);
      for (int i = lane; i < r16; i += 32) scan_cp_async16(sr + 16 * i, gr + 16 * (size_t)i);
      for (int i = lane; i < v16; i += 32) scan_cp_async16(sv + 16 * i, gv + 16 * (size_t)i);
      for (int i = r16 * (int)(16 / sizeof(RewT)) + lane; i < cnt; i += 32) buf[b].r[i] = rew[t0 + i];
      for (int i = v16 * 4 + lane; i < cntv; i += 32) buf[b].v[i] = p.values[t0 + i];
      // episodes that overlap this tile (warp-cooperative; overlaps the copies in flight)
      const long long e0 = warp_find_episode(p.off, p.n_ep, t0, lane);
      const long long e1 = warp_find_episode(p.off, p.n_ep, t0 + cnt - 1, lane);
      const int ne = (int)(e1 - e0 + 1);
      if (lane == 0) {
        buf[b].e0 = e0;
        buf[b].e1 = e1;
        buf[b].staged = ne <= SCAN_MAXE ? 1 : 0;
      }
      if (ne <= SCAN_MAXE) {  // the scan warps then never touch global memory for episode boundaries
        for (int i = lane; i <= ne; i += 32) buf[b].soff[i] = __ldg(p.off + e0 + i);
        for (int i = lane; i < ne; i += 32) {
          buf[b].slv[i] = __ldg(p.last_values + e0 + i);
          buf[b].sdone[i] = (int)__ldg(p.done + e0 + i);
        }
      }
      asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
      sbar_arrive(sm_addr(&bars[b]));  // 32 arrivals (release): this lane's copies and stores are visible
    }
    return;
  }

  // ================================== scan warps ====================================
  // Records of THIS launch carry this tag (0 = never written).  It is negative because record slots share workspace
  // bytes with the per-tile / per-episode statistics of earlier launches of a different n, and those land sums of
  // squares (>= 0) in the tag slot: a positive tag could equal one and a stale slot would read as published.
  const double tag = -(double)(s_epoch + 1);
  for (int k = 0; k < n_mine; ++k) {
    const int tile = T - 1 - c - k * G, b = k & 1;
    if (!sbar_wait(sm_addr(&bars[b]), (k >> 1) & 1)) {
      if (tid == 0) p.hdr->error = 1;
      break;
    }
    const long long t0 = (long long)tile * SCAN_TILE;
    const long long i0 = t0 + (long long)tid * SCAN_ITEMS;
    const TileBuf<RewT>* tb = &buf[b];
    const long long te0 = tb->e0, te1 = tb->e1;
    const bool staged = tb->staged != 0;
    const bool fast = staged && (t0 + SCAN_TILE <= n);  // whole tile in range, episode data in shared memory
    double r[SCAN_ITEMS];
    float v[SCAN_ITEMS + 1];
    double b_ret[SCAN_ITEMS], b_adv[SCAN_ITEMS];
    unsigned cut = 0;  // bit j set: a_j == 0 (episode end, or out of range)
    if (fast) {
      // ---- hot path: vector shared loads, 32-bit tile-relative indices, no bounds checks ----
      const int base = tid * SCAN_ITEMS;
      if (sizeof(RewT) == 8) {
#pragma unroll
        for (int q = 0; q < SCAN_ITEMS / 2; ++q) {
          const double2 x = *reinterpret_cast<const double2*>(reinterpret_cast<const double*>(tb->r) + base + 2 * q);
          r[2 * q] = x.x;
          r[2 * q + 1] = x.y;
        }
      } else {
#pragma unroll
        for (int q = 0; q < SCAN_ITEMS / 4; ++q) {
          const float4 x = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(tb->r) + base + 4 * q);
          r[4 * q] = x.x; r[4 * q + 1] = x.y; r[4 * q + 2] = x.z; r[4 * q + 3] = x.w;
        }
      }
      {
        const float4 x0 = *reinterpret_cast<const float4*>(tb->v + base);
        const float4 x1 = *reinterpret_cast<const float4*>(tb->v + base + 4);
        v[0] = x0.x; v[1] = x0.y; v[2] = x0.z; v[3] = x0.w;
        v[4] = x1.x; v[5] = x1.y; v[6] = x1.z; v[7] = x1.w;
        v[8] = tb->v[base + 8];  // the producer staged values[t0 + 2048] when it exists (else unused: episode end)
      }
      const int ne = (int)(te1 - te0 + 1);
      int el = 0;  // local episode index of item `base`: last k with off[k] - t0 <= base
      for (int k = 1; k < ne; ++k)
        if ((int)(tb->soff[k] - t0) <= base) el = k;
      int next_rel = (int)(tb->soff[el + 1] - t0);
#pragma unroll
      for (int j = 0; j < SCAN_ITEMS; ++j) {
        const bool last = (base + j == next_rel - 1);
        float vnext = v[j + 1];
        double boot = 0.0;
        if (last) {
          const float vl = tb->slv[el];
          vnext = vl;                                        // utils.py:41: delta_{L-1} uses V(last_obs) even when done
          if (!tb->sdone[el]) boot = p.gamma * (double)vl;   // utils.py:81-85 + ppo.py:149: ret_{L-1} = r + gamma*R_L
          cut |= 1u << j;
          ++el;
          next_rel = (el < ne) ? (int)(tb->soff[el + 1] - t0) : 0x7fffffff;
        }
        // utils.py:41: rewards[:-1] (f64) + gamma*values[1:] (evaluated in float32) - values[:-1]
        b_adv[j] = (r[j] + (double)__fmul_rn(p.gamma_f, vnext)) - (double)v[j];
        b_ret[j] = r[j] + boot;
      }
    } else {
      // ---- general path: partial last tile and / or more episodes than the staging area holds ----
#pragma unroll
      for (int j = 0; j < SCAN_ITEMS; ++j) {
        const bool in = i0 + j < n;
        r[j] = in ? (double)tb->r[tid * SCAN_ITEMS + j] : 0.0;
        v[j] = in ? tb->v[tid * SCAN_ITEMS + j] : 0.f;
      }
      v[SCAN_ITEMS] = (i0 + SCAN_ITEMS < n) ? tb->v[tid * SCAN_ITEMS + SCAN_ITEMS] : 0.f;
      auto off_at = [&](long long ee) { return staged ? tb->soff[ee - te0] : __ldg(p.off + ee); };
      long long e = 0, next_off = 0;
      if (i0 < n) {  // e = max{e : off[e] <= i0}, within the tile's episode range
        long long lo = te0, hi = te1 + 1;
        while (hi - lo > 1) {
          const long long mid = (lo + hi) >> 1;
          if (off_at(mid) <= i0) lo = mid; else hi = mid;
        }
        e = lo;
        next_off = off_at(e + 1);
      }
#pragma unroll
      for (int j = 0; j < SCAN_ITEMS; ++j) {
        const long long i = i0 + j;
        if (i < n) {
          while (i >= next_off) {
            ++e;
            next_off = off_at(e + 1);
          }
          const bool last = (i == next_off - 1);
          float vnext = v[j + 1];
          double boot = 0.0;
          if (last) {
            const float vl = staged ? tb->slv[e - te0] : __ldg(p.last_values + e);
            const int dn = staged ? tb->sdone[e - te0] : (int)__ldg(p.done + e);
            vnext = vl;
            if (!dn) boot = p.gamma * (double)vl;
            cut |= 1u << j;
          }
          b_adv[j] = (r[j] + (double)__fmul_rn(p.gamma_f, vnext)) - (double)v[j];
          b_ret[j] = r[j] + boot;
        } else {
          cut |= 1u << j;
          b_ret[j] = 0.0;
          b_adv[j] = 0.0;
        }
      }
    }
    // every consumer has taken what it needs from the slot: hand it back to the producer (runs two tiles ahead)
    consumer_sync();
    if (tid == 0) sbar_arrive(sm_addr(&bars[2 + b]));

    // ---- thread aggregate: compose items 7..0 ----
    Aff tr{1.0, 0.0}, ta{1.0, 0.0};
#pragma unroll
    for (int j = SCAN_ITEMS - 1; j >= 0; --j) {
      const bool cj = (cut >> j) & 1u;
      const double ar = cj ? 0.0 : p.gamma, aa = cj ? 0.0 : p.gl;
      tr.b = b_ret[j] + ar * tr.b;
      tr.a = ar * tr.a;
      ta.b = b_adv[j] + aa * ta.b;
      ta.a = aa * ta.a;
    }

    // ---- warp + CTA suffix scans ----
    const Aff ex_r = warp_suffix_exclusive(tr, lane);
    const Aff ex_a = warp_suffix_exclusive(ta, lane);
    if (lane == 0) {
      s_wret[warp] = tr;
      s_wadv[warp] = ta;
    }
    consumer_sync();

    // ---- warp 0: publish the tile aggregate, look back over later tiles for the carry-in, publish inclusive.
    //      Records are self-validating 16-byte {value, tag} pairs: six lanes poll six records in one round trip. ----
    if (warp == 0) {
      Aff agg_r{1.0, 0.0}, agg_a{1.0, 0.0};
      for (int w = SCAN_CONSUMERS / 32 - 1; w >= 0; --w) {
        agg_r = compose(s_wret[w], agg_r);
        agg_a = compose(s_wadv[w], agg_a);
      }
      if (lane < SCAN_CONSUMERS / 32) {  // lane w: composition of warps w+1 .. 7 (what follows warp w inside the tile)
        Aff xr{1.0, 0.0}, xa{1.0, 0.0};
        for (int w = SCAN_CONSUMERS / 32 - 1; w > lane; --w) {
          xr = compose(s_wret[w], xr);
          xa = compose(s_wadv[w], xa);
        }
        s_xret[lane] = xr;
        s_xadv[lane] = xa;
      }
      ScanRec* mine = p.recs + (size_t)tile * SCAN_RECS;
      if (lane < 4) st_rec(mine + lane, lane == 0 ? agg_r.a : lane == 1 ? agg_r.b : lane == 2 ? agg_a.a : agg_a.b, tag);

      Aff acc_r{1.0, 0.0}, acc_a{1.0, 0.0};
      bool failed = false;
      for (int j = tile + 1; j < T && !failed; ++j) {
        if (acc_r.a == 0.0 && acc_a.a == 0.0) break;  // an episode end in between: nothing further matters
        const ScanRec* theirs = p.recs + (size_t)j * SCAN_RECS;
        double val = 0.0, tg = 0.0;
        unsigned m = 0;
        for (int spins = 0;; ++spins) {
          if (lane < 6) ld_rec(theirs + lane, val, tg);
          m = __ballot_sync(0xffffffffu, lane < 6 && tg == tag);
          if ((m & 0x0fu) == 0x0fu || (m & 0x30u) == 0x30u) break;
          if (spins > (1 << 20)) {  // bounded: never hang the GPU; flag and bail out
            failed = true;
            break;
          }
          __nanosleep(20);
        }
        if (failed) break;
        if ((m & 0x30u) == 0x30u) {  // their inclusive values are known: the chain ends here
          const double yr = __shfl_sync(0xffffffffu, val, 4), ya = __shfl_sync(0xffffffffu, val, 5);
          acc_r = Aff{0.0, acc_r.b + acc_r.a * yr};
          acc_a = Aff{0.0, acc_a.b + acc_a.a * ya};
          break;
        }
        const double ar = __shfl_sync(0xffffffffu, val, 0), br = __shfl_sync(0xffffffffu, val, 1);
        const double aa = __shfl_sync(0xffffffffu, val, 2), ba = __shfl_sync(0xffffffffu, val, 3);
        acc_r = compose(acc_r, Aff{ar, br});
        acc_a = compose(acc_a, Aff{aa, ba});
      }
      // beyond the end of the array the recurrence value is 0
      if (lane == 4) st_rec(mine + 4, agg_r.b + agg_r.a * acc_r.b, tag);
      if (lane == 5) st_rec(mine + 5, agg_a.b + agg_a.a * acc_a.b, tag);
      if (lane == 0) {
        s_carry[0] = acc_r.b;
        s_carry[1] = acc_a.b;
        if (failed) p.hdr->error = 1;
      }
    }
    consumer_sync();

    // ---- carry-in of this thread = (lanes after me in my warp) o (warps after mine) applied to the tile carry ----
    const Aff xw_r = s_xret[warp], xw_a = s_xadv[warp];
    const Aff x_r = compose(ex_r, xw_r), x_a = compose(ex_a, xw_a);
    double y_r = x_r.b + x_r.a * s_carry[0];
    double y_a = x_a.b + x_a.a * s_carry[1];

    // ---- final sequential recurrence over the thread's items (the reference's own float64 loop) ----
    float o_ret[SCAN_ITEMS], o_adv[SCAN_ITEMS];
    double s1 = 0.0, s2 = 0.0;
#pragma unroll
    for (int j = SCAN_ITEMS - 1; j >= 0; --j) {
      const bool cj = (cut >> j) & 1u;
      y_r = b_ret[j] + (cj ? 0.0 : p.gamma) * y_r;
      y_a = b_adv[j] + (cj ? 0.0 : p.gl) * y_a;
      o_ret[j] = (float)y_r;
      o_adv[j] = (float)y_a;
      if (fast || i0 + j < n) {
        const double af = (double)o_adv[j];  // statistics of the float32 tensor, like normalize_tensor's input
        s1 += af;
        s2 += af * af;
      }
    }
    if (fast || i0 + SCAN_ITEMS <= n) {
      *reinterpret_cast<float4*>(p.ret + i0) = make_float4(o_ret[0], o_ret[1], o_ret[2], o_ret[3]);
      *reinterpret_cast<float4*>(p.ret + i0 + 4) = make_float4(o_ret[4], o_ret[5], o_ret[6], o_ret[7]);
      *reinterpret_cast<float4*>(p.adv + i0) = make_float4(o_adv[0], o_adv[1], o_adv[2], o_adv[3]);
      *reinterpret_cast<float4*>(p.adv + i0 + 4) = make_float4(o_adv[4], o_adv[5], o_adv[6], o_adv[7]);
    } else {
#pragma unroll
      for (int j = 0; j < SCAN_ITEMS; ++j)
        if (i0 + j < n) {
          p.ret[i0 + j] = o_ret[j];
          p.adv[i0 + j] = o_adv[j];
        }
    }

    // ---- per-tile advantage statistics (fixed order => deterministic) ----
    s1 = warp_sum(s1);
    s2 = warp_sum(s2);
    if (lane == 0) {
      s_red[0][warp] = s1;
      s_red[1][warp] = s2;
    }
    consumer_sync();
    if (tid == 0) {
      double t1 = 0.0, t2 = 0.0;
      for (int w = 0; w < SCAN_CONSUMERS / 32; ++w) {
        t1 += s_red[0][w];
        t2 += s_red[1][w];
      }
      p.partial[tile] = make_double2(t1, t2);
    }
  }

  // ---- the last CTA to finish sums the per-tile statistics in a fixed order and resets the header ----
  if (tid == 0) {
    __threadfence();
    s_last = (atomicAdd(&p.hdr->done, 1) == G - 1) ? 1 : 0;
  }
  consumer_sync();
  if (!s_last) return;
  __threadfence();
  __shared__ double f1[SCAN_CONSUMERS], f2[SCAN_CONSUMERS];
  double fa = 0.0, fb = 0.0;
  for (int i = tid; i < T; i += SCAN_CONSUMERS) {
    const double2 x = __ldcg(p.partial + i);
    fa += x.x;
    fb += x.y;
  }
  f1[tid] = fa;
  f2[tid] = fb;
  consumer_sync();
  for (int o = SCAN_CONSUMERS / 2; o > 0; o >>= 1) {
    if (tid < o) {
      f1[tid] += f1[tid + o];
      f2[tid] += f2[tid + o];
    }
    consumer_sync();
  }
  if (tid == 0) {
    const bool bad = p.hdr->error != 0;
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    p.stats[0] = bad ? nan : f1[0];
    p.stats[1] = bad ? nan : f2[0];
    p.stats[2] = (double)n;
    p.hdr->done = 0;
    p.hdr->error = 0;
    p.hdr->epoch = (s_epoch + 1) & 0x0fffffff;
  }
}


// ---------------------------------------------------------------------------------------------------------------
// Episode-parallel variant: ONE WARP PER EPISODE, walking 256-transition chunks (aligned to the flat array) from the
// episode's end to its start with the recurrence carries in registers.  No CTA barrier, no look-back, no per-item
// boundary search: the only special element is the episode's last step.  This is the regime RL batches live in
// (hundreds to millions of episodes of up to a few thousand steps); the tile kernel above covers few / very long
// episodes.  Per-episode advantage statistics go to ep_partial[e]; the last CTA sums them in a fixed order.
// ---------------------------------------------------------------------------------------------------------------
#ifndef B200RL_EP_WARPS  // overridable for A/B builds (tools/scan_variants.sh)
#define B200RL_EP_WARPS 8
#endif
#ifndef B200RL_EP_STAGES
#define B200RL_EP_STAGES 4
#endif
#ifndef B200RL_EP_CTAS
#define B200RL_EP_CTAS 2
#endif
constexpr int EP_WARPS = B200RL_EP_WARPS;
constexpr int EP_STAGES = B200RL_EP_STAGES;  // chunks in flight per warp (cp.async ring)
constexpr int EP_CTAS = B200RL_EP_CTAS;      // CTAs per SM the grid is sized for
#ifndef B200RL_EP_MINB
#define B200RL_EP_MINB 2                     // min resident CTAs per SM the compiler must fit (register cap)
#endif

template <typename RewT>
__global__ void __launch_bounds__(EP_WARPS * 32, B200RL_EP_MINB) gae_scan_episode_kernel(const ScanArgs p, double2* ep_partial) {
  extern __shared__ __align__(16) unsigned char ep_smem[];
  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);  // provably warp-uniform: episode loops and bounds stay uniform
  const long long n_warps = (long long)gridDim.x * EP_WARPS;
  const RewT* __restrict__ rew = static_cast<const RewT*>(p.rew);
  double lp_r = 1.0, lp_a = 1.0;  // gamma^(8*(31-lane)): coefficient of the incoming carry for this lane
  for (int k = 0; k < 31 - lane; ++k) {
    lp_r *= p.pw_r[0];
    lp_a *= p.pw_a[0];
  }
  // Chunks of an episode [beg, end): 256 items each, anchored at top = round_up(end, 8) and walked downwards until
  // bot = round_down(beg, 8) is covered; chunk starts are multiples of 8 items, so every lane's 8 rewards / 8 values
  // are 16-byte aligned.  Items outside [beg, end) are masked (their recurrence inputs are zeroed, which makes the
  // constant-coefficient recurrence exact at the episode's last step) and never stored.
  // Per-warp ring of EP_STAGES chunks filled with cp.async: every lane copies exactly the items it will consume, so
  // the ring needs no barrier -- the lane's own wait_group orders its copies before its reads.  The issue side runs
  // EP_STAGES chunks ahead of the consumer ACROSS episode boundaries (episodes w, w + n_warps, ... belong to warp w).
  constexpr int STAGE_BYTES = 256 * (int)sizeof(RewT) + 256 * 4;
  unsigned char* wbase = ep_smem + (size_t)warp * EP_STAGES * STAGE_BYTES;
  long long ie = (long long)blockIdx.x * EP_WARPS + warp, ics = 0, ibot = 0;  // issue-side iterator
  long long nx_beg = 0, nx_end = 0;  // offsets of the issue side's NEXT episode, fetched one episode ahead (the loads
                                     // then complete under the current episode's chunks instead of stalling the switch)
  if (ie < p.n_ep) {
    ibot = __ldg(p.off + ie) & ~7LL;
    ics = ((__ldg(p.off + ie + 1) + 7) & ~7LL) - 256;
    if (ie + n_warps < p.n_ep) {
      nx_beg = __ldg(p.off + ie + n_warps);
      nx_end = __ldg(p.off + ie + n_warps + 1);
    }
  }
  auto issue_next = [&](int st) {
    if (ie < p.n_ep) {
      const long long j0 = ics + lane * SCAN_ITEMS;
      if (j0 >= ibot && j0 + SCAN_ITEMS <= p.n) {
        const uint32_t dr = sm_addr(wbase + st * STAGE_BYTES + lane * SCAN_ITEMS * (int)sizeof(RewT));
        const char* sr = reinterpret_cast<const char*>(rew + j0);
#pragma unroll
        for (int k = 0; k < SCAN_ITEMS * (int)sizeof(RewT) / 16; ++k) scan_cp_async16(dr + 16 * k, sr + 16 * k);
        const uint32_t dv = sm_addr(wbase + st * STAGE_BYTES + 256 * (int)sizeof(RewT) + lane * SCAN_ITEMS * 4);
        scan_cp_async16(dv, p.values + j0);
        scan_cp_async16(dv + 16, p.values + j0 + 4);
      }
      ics -= 256;
      if (ics + 256 <= ibot) {  // episode covered: move to this warp's next one
        ie += n_warps;
        if (ie < p.n_ep) {
          ibot = nx_beg & ~7LL;
          ics = ((nx_end + 7) & ~7LL) - 256;
          if (ie + n_warps < p.n_ep) {
            nx_beg = __ldg(p.off + ie + n_warps);
            nx_end = __ldg(p.off + ie + n_warps + 1);
          }
        }
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
#pragma unroll
  for (int st = 0; st < EP_STAGES; ++st) issue_next(st);
  int stage = 0;
  // episode metadata is fetched one episode ahead so its latency hides behind the current episode's chunks
  long long nbeg = 0, nend = 0;
  float nvl = 0.f;
  unsigned char ndn = 0;
  {
    const long long e0 = (long long)blockIdx.x * EP_WARPS + warp;
    if (e0 < p.n_ep) {
      nbeg = __ldg(p.off + e0);
      nend = __ldg(p.off + e0 + 1);
      nvl = __ldg(p.last_values + e0);
      ndn = __ldg(p.done + e0);
    }
  }
  for (long long e = (long long)blockIdx.x * EP_WARPS + warp; e < p.n_ep; e += n_warps) {
    const long long beg = nbeg, end = nend;
    const long long bot = beg & ~7LL;
    const bool aligned = ((beg | end) & 7LL) == 0;  // warp-uniform
    const float vl = nvl;
    const double boot = ndn ? 0.0 : p.gamma * (double)vl;  // utils.py:81-85 + ppo.py:149
    if (e + n_warps < p.n_ep) {
      nbeg = __ldg(p.off + e + n_warps);
      nend = __ldg(p.off + e + n_warps + 1);
      nvl = __ldg(p.last_values + e + n_warps);
      ndn = __ldg(p.done + e + n_warps);
    }
    double carry_r = 0.0, carry_a = 0.0;  // recurrence values at the first item of the chunk processed before
    float v_first_prev = vl;              // value of that item (v_{i+1} of this chunk's last item)
    double s1 = 0.0, s2 = 0.0;
    long long cs = ((end + 7) & ~7LL) - 256;
    // Two copies of the chunk loop: episodes whose bounds are multiples of 8 items (every fixed-horizon batch) never
    // need the per-item masks of the general one.
    auto run_chunks = [&](auto aligned_tag) {
    constexpr bool ALIGNED = decltype(aligned_tag)::value;
    do {
      const long long i0 = cs + lane * SCAN_ITEMS;
      double r[SCAN_ITEMS];
      float v[SCAN_ITEMS];
      asm volatile("cp.async.wait_group %0;" ::"n"(EP_STAGES - 1) : "memory");
      if (i0 >= bot && i0 + SCAN_ITEMS <= p.n) {
        const unsigned char* sb = wbase + stage * STAGE_BYTES;
        if (sizeof(RewT) == 8) {
          const double2* q = reinterpret_cast<const double2*>(sb) + lane * 4;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const double2 x = q[j];
            r[2 * j] = x.x;
            r[2 * j + 1] = x.y;
          }
        } else {
          const float4* q = reinterpret_cast<const float4*>(sb) + lane * 2;
          const float4 y0 = q[0], y1 = q[1];
          r[0] = y0.x; r[1] = y0.y; r[2] = y0.z; r[3] = y0.w;
          r[4] = y1.x; r[5] = y1.y; r[6] = y1.z; r[7] = y1.w;
        }
        const float4* qv = reinterpret_cast<const float4*>(sb + 256 * sizeof(RewT)) + lane * 2;
        const float4 x0 = qv[0], x1 = qv[1];
        v[0] = x0.x; v[1] = x0.y; v[2] = x0.z; v[3] = x0.w;
        v[4] = x1.x; v[5] = x1.y; v[6] = x1.z; v[7] = x1.w;
      } else {  // lane below the episode (all masked) or straddling the end of the arrays (not in the ring)
#pragma unroll
        for (int j = 0; j < SCAN_ITEMS; ++j) {
          const bool in = i0 + j >= bot && i0 + j < p.n;
          r[j] = in ? (double)rew[i0 + j] : 0.0;
          v[j] = in ? p.values[i0 + j] : 0.f;
        }
      }
      issue_next(stage);  // refill the slot just drained
      stage = stage + 1 == EP_STAGES ? 0 : stage + 1;

      float vn7 = __shfl_down_sync(0xffffffffu, v[0], 1);  // value of the next lane's first item
      if (lane == 31) vn7 = v_first_prev;
      double d[SCAN_ITEMS];
#pragma unroll
      for (int j = 0; j < SCAN_ITEMS; ++j) {
        const float vnext = j < SCAN_ITEMS - 1 ? v[j + 1] : vn7;  // utils.py:41: gamma * values[1:] in float32
        d[j] = (r[j] + (double)__fmul_rn(p.gamma_f, vnext)) - (double)v[j];
      }
      const bool edge = cs < beg || cs + 256 >= end;  // warp-uniform: chunk holds masked items or the last step
      int lo = 0, hi = SCAN_ITEMS;
      bool lane_off = false;
      if (ALIGNED && edge) {
        // episode bounds on multiples of 8 items (every fixed-horizon batch): a lane is wholly inside or wholly outside,
        // and the last step is item 7 of one lane -- no per-item masks
        lane_off = i0 < beg || i0 >= end;
        if (lane_off) lo = hi = SCAN_ITEMS;
        if (i0 + SCAN_ITEMS == end) {  // last step: delta uses V(last_obs) even when done; the return bootstraps if not done
          d[SCAN_ITEMS - 1] = (r[SCAN_ITEMS - 1] + (double)__fmul_rn(p.gamma_f, vl)) - (double)v[SCAN_ITEMS - 1];
          r[SCAN_ITEMS - 1] += boot;
        }
      } else if (!ALIGNED && edge) {
        lo = (int)min(max(beg - i0, 0LL), (long long)SCAN_ITEMS);
        hi = (int)max(min(end - i0, (long long)SCAN_ITEMS), 0LL);
        const long long jl64 = end - 1 - i0;
        const int jl = (jl64 >= 0 && jl64 < SCAN_ITEMS) ? (int)jl64 : -1;
#pragma unroll
        for (int j = 0; j < SCAN_ITEMS; ++j) {
          if (j < lo || j >= hi) {
            r[j] = 0.0;
            d[j] = 0.0;
          } else if (j == jl) {  // last step: delta uses V(last_obs) even when done; the return bootstraps if not done
            d[j] = (r[j] + (double)__fmul_rn(p.gamma_f, vl)) - (double)v[j];
            r[j] += boot;
          }
        }
      }
      double tr = r[SCAN_ITEMS - 1], ta = d[SCAN_ITEMS - 1];
#pragma unroll
      for (int j = SCAN_ITEMS - 2; j >= 0; --j) {
        tr = r[j] + p.gamma * tr;
        ta = d[j] + p.gl * ta;
      }
      if (ALIGNED && lane_off) {  // a lane outside the episode contributes nothing (select, not multiply: its data may be anything)
        tr = 0.0;
        ta = 0.0;
      }
#pragma unroll
      for (int k = 0; k < 5; ++k) {
        const double r2 = __shfl_down_sync(0xffffffffu, tr, 1 << k);
        const double a2 = __shfl_down_sync(0xffffffffu, ta, 1 << k);
        if (lane + (1 << k) < 32) {
          tr += p.pw_r[k] * r2;
          ta += p.pw_a[k] * a2;
        }
      }
      double y_r = __shfl_down_sync(0xffffffffu, tr, 1);
      double y_a = __shfl_down_sync(0xffffffffu, ta, 1);
      if (lane == 31) {
        y_r = 0.0;
        y_a = 0.0;
      }
      y_r += lp_r * carry_r;
      y_a += lp_a * carry_a;
      float o_ret[SCAN_ITEMS], o_adv[SCAN_ITEMS];
#pragma unroll
      for (int j = SCAN_ITEMS - 1; j >= 0; --j) {
        y_r = r[j] + p.gamma * y_r;
        y_a = d[j] + p.gl * y_a;
        o_ret[j] = (float)y_r;
        o_adv[j] = (float)y_a;
      }
      if (lo == 0 && hi == SCAN_ITEMS && i0 + SCAN_ITEMS <= p.n) {
#pragma unroll
        for (int j = 0; j < SCAN_ITEMS; ++j) {
          const double af = (double)o_adv[j];
          s1 += af;
          s2 += af * af;
        }
        *reinterpret_cast<float4*>(p.ret + i0) = make_float4(o_ret[0], o_ret[1], o_ret[2], o_ret[3]);
        *reinterpret_cast<float4*>(p.ret + i0 + 4) = make_float4(o_ret[4], o_ret[5], o_ret[6], o_ret[7]);
        *reinterpret_cast<float4*>(p.adv + i0) = make_float4(o_adv[0], o_adv[1], o_adv[2], o_adv[3]);
        *reinterpret_cast<float4*>(p.adv + i0 + 4) = make_float4(o_adv[4], o_adv[5], o_adv[6], o_adv[7]);
      } else {
#pragma unroll
        for (int j = 0; j < SCAN_ITEMS; ++j) {
          if (j >= lo && j < hi) {
            const double af = (double)o_adv[j];
            s1 += af;
            s2 += af * af;
            p.ret[i0 + j] = o_ret[j];
            p.adv[i0 + j] = o_adv[j];
          }
        }
      }
      // carries for the next (earlier) chunk: the recurrence values and the value at this chunk's first item
      carry_r = __shfl_sync(0xffffffffu, y_r, 0);
      carry_a = __shfl_sync(0xffffffffu, y_a, 0);
      v_first_prev = __shfl_sync(0xffffffffu, v[0], 0);
      cs -= 256;
    } while (cs + 256 > bot);
    };
    if (aligned) run_chunks(std::true_type{});
    else run_chunks(std::false_type{});
    s1 = warp_sum(s1);
    s2 = warp_sum(s2);
    if (lane == 0) ep_partial[e] = make_double2(s1, s2);
  }

  // ---- the last CTA to finish sums the per-episode statistics in a fixed order ----
  __shared__ int s_last;
  __shared__ double f1[EP_WARPS * 32], f2[EP_WARPS * 32];
  __syncthreads();
  if (tid == 0) {
    __threadfence();
    s_last = (atomicAdd(&p.hdr->done, 1) == (int)gridDim.x - 1) ? 1 : 0;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  double fa = 0.0, fb = 0.0;
  for (long long i = tid; i < p.n_ep; i += EP_WARPS * 32) {
    const double2 x = __ldcg(ep_partial + i);
    fa += x.x;
    fb += x.y;
  }
  f1[tid] = fa;
  f2[tid] = fb;
  __syncthreads();
  for (int o = EP_WARPS * 16; o > 0; o >>= 1) {
    if (tid < o) {
      f1[tid] += f1[tid + o];
      f2[tid] += f2[tid + o];
    }
    __syncthreads();
  }
  if (tid == 0) {
    p.stats[0] = f1[0];
    p.stats[1] = f2[0];
    p.stats[2] = (double)p.n;
    p.hdr->done = 0;
  }
}

static inline int scan_tiles(int64_t n) { return (int)((n + SCAN_TILE - 1) / SCAN_TILE); }

template <typename RewT>
static int launch_scan(const ScanArgs& a, cudaStream_t s) {
  const size_t smem = 2 * sizeof(TileBuf<RewT>);
  static int cached_blocks = 0;  // resident CTAs per device for this instantiation
  if (cached_blocks == 0) {
    B200RL_CUDA(cudaFuncSetAttribute(gae_scan_kernel<RewT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    B200RL_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gae_scan_kernel<RewT>, SCAN_THREADS, smem));
    const int sms = device_sm_count();
    B200RL_REQUIRE(per_sm > 0 && sms > 0, "gae_scan: kernel does not fit on this device");
    cached_blocks = per_sm * sms;
  }
  const int grid = a.num_tiles < cached_blocks ? a.num_tiles : cached_blocks;  // all CTAs co-resident (look-back)
  gae_scan_kernel<RewT><<<grid, SCAN_THREADS, smem, s>>>(a);
  B200RL_CUDA(cudaGetLastError());
  count_launch(1);
  return 0;
}

}  // namespace b200rl

using namespace b200rl;

extern "C" size_t b200rl_gae_scan_workspace_bytes(int64_t n) {
  const size_t t = (size_t)scan_tiles(n < 1 ? 1 : n);
  // header | look-back records | per-tile statistics | per-episode statistics (episode kernel, n_ep <= n / 16)
  return sizeof(ScanHeader) + t * SCAN_RECS * sizeof(ScanRec) + t * sizeof(double2) + (((size_t)(n < 1 ? 1 : n) + 15) & ~(size_t)15);
}

extern "C" int b200rl_gae_scan(const void* rewards, int rewards_f64, const float* values, const float* last_values,
                               const int64_t* ep_offsets, const uint8_t* ep_done, int64_t n, int64_t n_ep,
                               double gamma, double gae_lambda, float* adv_raw, float* ret, double* stats,
                               void* workspace, size_t workspace_bytes, void* stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200RL_REQUIRE(n >= 0 && n_ep >= 0, "gae_scan: negative size");
  B200RL_REQUIRE(stats != nullptr, "gae_scan: stats is NULL");
  if (n == 0) {
    B200RL_CUDA(cudaMemsetAsync(stats, 0, 3 * sizeof(double), s));
    return 0;
  }
  B200RL_REQUIRE(n_ep >= 1, "gae_scan: %lld transitions but no episode", (long long)n);
  B200RL_REQUIRE(rewards && values && last_values && ep_offsets && ep_done && adv_raw && ret && workspace,
                 "gae_scan: NULL pointer argument");
  B200RL_REQUIRE(aligned16(rewards) && aligned16(values) && aligned16(adv_raw) && aligned16(ret) &&
                     aligned16(workspace),
                 "gae_scan: rewards/values/adv/ret/workspace must be 16-byte aligned");
  B200RL_REQUIRE(workspace_bytes >= b200rl_gae_scan_workspace_bytes(n), "gae_scan: workspace too small");
  const int tiles = scan_tiles(n);
  ScanArgs a;
  a.rew = rewards;
  a.values = values;
  a.last_values = last_values;
  a.off = reinterpret_cast<const long long*>(ep_offsets);
  a.done = ep_done;
  a.n = n;
  a.n_ep = n_ep;
  a.gamma = gamma;
  a.gl = gamma * gae_lambda;
  a.gamma_f = (float)gamma;
  for (int k = 0; k < 5; ++k) {
    a.pw_r[k] = pow(a.gamma, 8.0 * (1 << k));
    a.pw_a[k] = pow(a.gl, 8.0 * (1 << k));
  }
  a.adv = adv_raw;
  a.ret = ret;
  a.hdr = static_cast<ScanHeader*>(workspace);
  a.recs = reinterpret_cast<ScanRec*>(static_cast<char*>(workspace) + sizeof(ScanHeader));
  a.partial = reinterpret_cast<double2*>(reinterpret_cast<char*>(a.recs) + (size_t)tiles * SCAN_RECS * sizeof(ScanRec));
  a.stats = stats;
  a.num_tiles = tiles;
  // Regime switch: many episodes of moderate length -> one warp per episode (no inter-CTA dependency at all);
  // few or very long episodes -> tile kernel with decoupled look-back.
  const bool by_episode = n_ep >= 256 && n_ep <= n / 16 && n / n_ep <= 32768;
  if (by_episode) {
    double2* ep_partial = reinterpret_cast<double2*>(reinterpret_cast<char*>(a.partial) + (size_t)tiles * sizeof(double2));
    const int grid = (int)std::min<long long>((n_ep + EP_WARPS - 1) / EP_WARPS, (long long)EP_CTAS * device_sm_count());
    const int smem64 = EP_WARPS * EP_STAGES * (256 * 8 + 1024), smem32 = EP_WARPS * EP_STAGES * (256 * 4 + 1024);
    static bool configured = false;
    if (!configured) {
      B200RL_CUDA(cudaFuncSetAttribute(gae_scan_episode_kernel<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem64));
      B200RL_CUDA(cudaFuncSetAttribute(gae_scan_episode_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem32));
      configured = true;
    }
    if (rewards_f64)
      gae_scan_episode_kernel<double><<<grid, EP_WARPS * 32, smem64, s>>>(a, ep_partial);
    else
      gae_scan_episode_kernel<float><<<grid, EP_WARPS * 32, smem32, s>>>(a, ep_partial);
    B200RL_CUDA(cudaGetLastError());
    count_launch(1);
    return 0;
  }
  return rewards_f64 ? launch_scan<double>(a, s) : launch_scan<float>(a, s);
}
