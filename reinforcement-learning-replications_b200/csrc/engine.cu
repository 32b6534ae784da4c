// On-policy update engine: device-resident batch + flat parameters + Adam state, and the whole per-epoch update
// (the reference's PPO.train / VPG.train, /root/reference/src/rl_replicas/algorithms/ppo.py:139-223, vpg.py:127-192)
// as a host-sync-free stream of kernel launches.  See include/b200rl.h for the C ABI.
#include <atomic>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <vector>

#include "common.cuh"
#include "tc_common.cuh"
#include "tc3.cuh"

namespace b200rl {

bool use_tc(const b200rl_mlp_desc& d);  // mlp_fused.cu: the tensor-core kernels take this network

static thread_local std::string g_error;
static std::atomic<int64_t> g_launches{0};  // engines of different host threads count into it

void set_error(const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_error = buf;
}
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
int64_t launches_total() { return g_launches.load(std::memory_order_relaxed); }

int device_sm_count() {
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return -1;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return -1;
  return sms;
}

// One buffer per (device, stream): launches on one stream run one after the other, so they can share it, and
// launches on different streams (data-parallel engines on one GPU) never do.  Every tensor-core grid is at most one
// CTA per SM, so the buffer is allocated once at that size (132 x 256 KB = 33 MB on an H100) and never resized or
// freed while the process runs.  Launches under stream capture are refused: a captured graph could be replayed on
// another stream while this one uses the same buffer.
int tc_grid(int64_t n_rows) {
  const int64_t tiles = (n_rows + 127) / 128;
  const int sms = device_sm_count();
  if (sms <= 0) return -1;
  return (int)(tiles < sms ? (tiles < 1 ? 1 : tiles) : sms);
}

int mlp3_offsets(const b200rl_mlp_desc& d, int w_off[3], int b_off[3]) {
  int off = 0;
  for (int l = 0; l < 3; ++l) {
    w_off[l] = off;
    off += d.sizes[l + 1] * d.sizes[l];
    b_off[l] = off;
    off += d.sizes[l + 1];
  }
  return off;
}

float* acc_mem(int grid, cudaStream_t s) {
  struct Entry {
    int dev;
    cudaStream_t stream;
    float* ptr;
  };
  static std::mutex mu;
  static std::vector<Entry> entries;
  int dev = 0;
  const int sms = device_sm_count();
  if (grid <= 0 || grid > sms || cudaGetDevice(&dev) != cudaSuccess) return nullptr;
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(s, &cap) != cudaSuccess || cap != cudaStreamCaptureStatusNone) return nullptr;
  std::lock_guard<std::mutex> lock(mu);
  for (const Entry& e : entries)
    if (e.dev == dev && e.stream == s) return e.ptr;
  float* p = nullptr;
  if (cudaMalloc(&p, (size_t)sms * ACC_CTA_FLOATS * sizeof(float)) != cudaSuccess) return nullptr;
  entries.push_back(Entry{dev, s, p});
  return p;
}

}  // namespace b200rl

using namespace b200rl;

extern "C" const char* b200rl_last_error(void) { return g_error.c_str(); }
extern "C" int b200rl_version(void) { return B200RL_VERSION; }
extern "C" int64_t b200rl_launch_count(void) { return launches_total(); }

struct b200rl_onpolicy {
  b200rl_onpolicy_config cfg;
  int64_t Pp = 0, Pv = 0;
  int grid_cap = 0;
  int obs_dim = 0, act_cols = 0;
  // batch
  float *obs = nullptr, *act = nullptr, *last_obs = nullptr;
  void* rew = nullptr;
  int64_t* off = nullptr;
  uint8_t* done = nullptr;
  int64_t n_rows = 0, n_ep = 0;
  float* absmax = nullptr;   // per-feature max |obs| [32], per-feature max |last_obs| [32], max |returns| [1]: range
                             // hints of the fp16 tensor-core kernels
  bool hints_valid = false;  // set by the preamble, cleared whenever the batch buffers may have been rewritten
  // derived
  float *values = nullptr, *last_values = nullptr, *adv_raw = nullptr, *ret = nullptr, *old_logp = nullptr;
  double* adv_stats = nullptr;
  void* scan_ws = nullptr;
  size_t scan_ws_bytes = 0;
  // parameters / optimiser state
  float *pol = nullptr, *old_pol = nullptr, *val = nullptr, *log_std = nullptr;
  float *pol_m = nullptr, *pol_v = nullptr, *val_m = nullptr, *val_v = nullptr;
  int64_t pol_step = 0, val_step = 0;
  // workspaces
  float* partials = nullptr;
  double* scalar_partials = nullptr;
  float *pol_grad = nullptr, *val_grad = nullptr;  // [P + N_SCALARS]
  double* slots = nullptr;                         // [n_slots][N_SCALARS] scalar history
  int n_slots = 0;
  int last_slots = 0;  // slots the last update wrote (and read back into h_slots)
  int* flags = nullptr;  // 0 stop flag, 1 policy steps applied, 2 value steps applied
  double* h_slots = nullptr;  // pinned
  int* h_flags = nullptr;     // pinned
  double* h_stats3 = nullptr; // pinned
  // TRPO (allocated on first use)
  int out_cols = 0;
  float* old_out = nullptr;  // [max_rows, out_cols] outputs of the old policy
  float *cg_x = nullptr, *cg_r = nullptr, *cg_p = nullptr, *cg_z = nullptr, *cg_prev = nullptr, *cg_descent = nullptr;
  double* cg_sc = nullptr;   // 8 doubles, see trpo.cu
  int* cg_flags = nullptr;   // 4 ints
  double* h_cg_sc = nullptr; // pinned
  int* h_cg_flags = nullptr; // pinned
  // fused policy + value step (mlp_tc3.cu)
  bool fused_ok = false;     // both networks fit the fused kernel's shape gate
  uint8_t* ximg = nullptr;   // packed observation tiles
  float* xscale = nullptr;   // [64]
  float* trip = nullptr;     // [2] floats: 0 observations out of range (pack_obs), 1 range trip inside a step
  float* grad_all = nullptr; // [Pp + Pv + 16]: both gradients + both scalar tails, the ONE all-reduce buffer per iteration
  float* snap = nullptr;     // snapshot [3 Pp + 3 Pv + Pp]: restored when a fused update must be redone
  float* h_trip = nullptr;   // pinned
  int last_fused = 0;        // the last update / gradient stage ran on the fused path (which buffer device_view shows)
  // trainable log_std (policies/gaussian_policy.py:25-37 with log_std inside the optimizer): the policy vector is then
  // [network parameters | log_std] for set / get_params, Adam and the gradient; policy steps run on the fp32 kernel
  int train_log_std = 0;
  int n_ls = 0;              // entries appended to the policy vector (= action width when train_log_std)
  // one-shot gradient exchange over peer-mapped memory (data-parallel runs on one node)
  float* xchg = nullptr;     // this rank's exchange buffer: [2][xchg_stride] floats + 2 sequence words
  int64_t xchg_stride = 0;
  float** peers_dev = nullptr;  // device copy of the ranks' buffer pointers
  unsigned* done_counter = nullptr;
  int comm_world = 0, comm_rank = 0;
  unsigned comm_seq = 0;
  std::vector<void*> allocs;
};

namespace {

template <typename T>
int dev_alloc(b200rl_onpolicy* h, T** p, size_t count) {
  void* q = nullptr;
  B200RL_CUDA(cudaMalloc(&q, (count ? count : 1) * sizeof(T)));
  B200RL_CUDA(cudaMemset(q, 0, (count ? count : 1) * sizeof(T)));
  h->allocs.push_back(q);
  *p = static_cast<T*>(q);
  return 0;
}

int ensure_slots(b200rl_onpolicy* h, int n) {
  if (n <= h->n_slots) return 0;
  if (h->h_slots) cudaFreeHost(h->h_slots);
  h->h_slots = nullptr;
  double* d = nullptr;
  if (dev_alloc(h, &d, (size_t)n * B200RL_N_SCALARS)) return 1;
  h->slots = d;
  B200RL_CUDA(cudaMallocHost(reinterpret_cast<void**>(&h->h_slots), (size_t)n * B200RL_N_SCALARS * sizeof(double)));
  h->n_slots = n;
  return 0;
}

struct Net {
  const b200rl_mlp_desc* mlp;
  float* params;
  int64_t P;
};

// one fused launch over the loaded batch
int launch_fused(b200rl_onpolicy* h, const b200rl_mlp_desc& mlp, int loss, int dist, const float* params,
                 const float* obs, int64_t n_rows, int64_t n_global, double clip, bool use_adv, bool use_old,
                 float* row_out, bool want_scalars, const int* skip, cudaStream_t s) {
  b200rl_mlp_loss_grad_args a;
  memset(&a, 0, sizeof(a));
  a.mlp = mlp;
  a.loss = loss;
  a.dist = dist;
  a.n_rows = n_rows;
  a.n_global = n_global;
  a.clip_range = (float)clip;
  a.params = params;
  a.obs = obs;
  if (dist != B200RL_DIST_NONE) {
    a.actions = h->act;
    // trainable log_std lives behind the network parameters of the (old) policy vector
    a.log_std = !h->train_log_std ? h->log_std : (params == h->old_pol ? h->old_pol + h->Pp : h->pol + h->Pp);
    a.train_log_std = h->train_log_std && loss != B200RL_LOSS_EVAL && loss != B200RL_LOSS_MSE;
  }
  if (use_adv) {
    a.adv_raw = h->adv_raw;
    a.adv_stats = h->adv_stats;
  }
  if (use_old) a.old_logp = h->old_logp;
  if (loss == B200RL_LOSS_MSE) a.target = h->ret;
  a.row_out = row_out;
  a.partials = h->partials;
  a.scalar_partials = want_scalars ? h->scalar_partials : nullptr;
  a.skip_flag = skip;
  if (h->hints_valid) {
    if (obs == h->obs) a.obs_absmax = h->absmax;
    if (obs == h->last_obs) a.obs_absmax = h->absmax + 32;
    if (loss == B200RL_LOSS_MSE) a.target_absmax = h->absmax + 64;
  }
  return b200rl_mlp_loss_grad(&a, s);
}

}  // namespace

extern "C" int b200rl_onpolicy_create(const b200rl_onpolicy_config* cfg, b200rl_onpolicy** out) {
  B200RL_REQUIRE(cfg && out, "onpolicy_create: NULL argument");
  B200RL_REQUIRE(cfg->max_rows > 0 && cfg->max_episodes > 0, "onpolicy_create: capacities must be positive");
  const int64_t Pp = b200rl_mlp_param_count(&cfg->policy), Pv = b200rl_mlp_param_count(&cfg->value);
  B200RL_REQUIRE(Pp > 0 && Pv > 0, "onpolicy_create: invalid MLP description");
  B200RL_REQUIRE(cfg->policy.sizes[0] == cfg->value.sizes[0], "onpolicy_create: policy/value observation widths differ");
  B200RL_REQUIRE(cfg->value.sizes[cfg->value.n_layers] == 1, "onpolicy_create: value network must have one output");
  B200RL_REQUIRE(cfg->dist == B200RL_DIST_GAUSSIAN || cfg->dist == B200RL_DIST_CATEGORICAL,
                 "onpolicy_create: dist must be GAUSSIAN or CATEGORICAL");
  // log_std and the loss epilogues are sized for 16 action dimensions (set_log_std would otherwise write past them)
  B200RL_REQUIRE(cfg->dist != B200RL_DIST_GAUSSIAN || cfg->policy.sizes[cfg->policy.n_layers] <= 16,
                 "onpolicy_create: a Gaussian policy supports at most 16 action dimensions, got %d",
                 cfg->policy.sizes[cfg->policy.n_layers]);
  const int sms = device_sm_count();
  B200RL_REQUIRE(sms > 0, "onpolicy_create: no CUDA device (%s)", cudaGetErrorString(cudaGetLastError()));
  b200rl_onpolicy* h = new b200rl_onpolicy();
  h->cfg = *cfg;
  h->Pp = Pp;
  h->Pv = Pv;
  h->grid_cap = sms;
  h->obs_dim = cfg->policy.sizes[0];
  const int A = cfg->policy.sizes[cfg->policy.n_layers];
  h->act_cols = cfg->dist == B200RL_DIST_GAUSSIAN ? A : 1;
  const size_t N = (size_t)cfg->max_rows, E = (size_t)cfg->max_episodes;
  const size_t N_tiles = (N + 127) / 128 * 128;  // the fused step copies its per-row loss inputs in whole 128-row tiles
  const size_t Pmax = (size_t)(Pp > Pv ? Pp : Pv);
  int rc = 0;
  rc |= dev_alloc(h, &h->obs, N * h->obs_dim + 64);  // + slack: the tc kernel stages whole 16-byte chunks
  rc |= dev_alloc(h, &h->act, N_tiles * h->act_cols);
  rc |= dev_alloc(h, &h->last_obs, E * h->obs_dim + 64);
  rc |= dev_alloc(h, reinterpret_cast<char**>(&h->rew), N * (cfg->rewards_f64 ? 8 : 4));
  rc |= dev_alloc(h, &h->off, E + 1);
  rc |= dev_alloc(h, &h->done, E);
  rc |= dev_alloc(h, &h->values, N);
  rc |= dev_alloc(h, &h->last_values, E);
  rc |= dev_alloc(h, &h->adv_raw, N_tiles);
  rc |= dev_alloc(h, &h->ret, N_tiles);
  rc |= dev_alloc(h, &h->old_logp, N_tiles);
  rc |= dev_alloc(h, &h->adv_stats, 4);
  h->scan_ws_bytes = b200rl_gae_scan_workspace_bytes(cfg->max_rows);
  rc |= dev_alloc(h, reinterpret_cast<char**>(&h->scan_ws), h->scan_ws_bytes);
  rc |= dev_alloc(h, &h->pol, (size_t)Pp + 16);
  rc |= dev_alloc(h, &h->old_pol, (size_t)Pp + 16);
  rc |= dev_alloc(h, &h->val, (size_t)Pv);
  rc |= dev_alloc(h, &h->log_std, 16);
  rc |= dev_alloc(h, &h->pol_m, (size_t)Pp + 16);
  rc |= dev_alloc(h, &h->pol_v, (size_t)Pp + 16);
  rc |= dev_alloc(h, &h->val_m, (size_t)Pv);
  rc |= dev_alloc(h, &h->val_v, (size_t)Pv);
  h->fused_ok = tc3_shape_ok(cfg->policy, cfg->value);
  // mlp_tc2 emits two partial rows per CTA; the fused step's rows hold both networks' gradients side by side
  rc |= dev_alloc(h, &h->partials, (size_t)2 * sms * (h->fused_ok ? (size_t)(Pp + Pv) : Pmax + 16));
  rc |= dev_alloc(h, &h->scalar_partials, (size_t)2 * sms * 2 * B200RL_N_SCALARS);
  if (h->fused_ok) {
    rc |= dev_alloc(h, &h->ximg, tc3_ximg_bytes(cfg->max_rows));
    rc |= dev_alloc(h, &h->xscale, 64);
    rc |= dev_alloc(h, &h->trip, 4);
    rc |= dev_alloc(h, &h->grad_all, (size_t)(Pp + Pv) + 2 * B200RL_N_SCALARS);
    rc |= dev_alloc(h, &h->snap, (size_t)(4 * Pp + 3 * Pv));
    if (!rc && cudaMallocHost(reinterpret_cast<void**>(&h->h_trip), 4 * sizeof(float)) != cudaSuccess) rc = 1;
  }
  rc |= dev_alloc(h, &h->absmax, 72);
  rc |= dev_alloc(h, &h->pol_grad, (size_t)Pp + 16 + B200RL_N_SCALARS);
  rc |= dev_alloc(h, &h->val_grad, (size_t)Pv + B200RL_N_SCALARS);
  rc |= dev_alloc(h, &h->flags, 8);
  if (!rc) rc |= ensure_slots(h, 256);
  if (!rc && cudaMallocHost(reinterpret_cast<void**>(&h->h_flags), 8 * sizeof(int)) != cudaSuccess) rc = 1;
  if (!rc && cudaMallocHost(reinterpret_cast<void**>(&h->h_stats3), 4 * sizeof(double)) != cudaSuccess) rc = 1;
  if (rc) {
    std::string keep = g_error.empty() ? std::string("onpolicy_create: allocation failed") : g_error;
    b200rl_onpolicy_destroy(h);
    g_error = keep;
    return 1;
  }
  *out = h;
  return 0;
}

extern "C" void b200rl_onpolicy_destroy(b200rl_onpolicy* h) {
  if (!h) return;
  for (void* p : h->allocs) cudaFree(p);
  if (h->h_cg_sc) cudaFreeHost(h->h_cg_sc);
  if (h->h_cg_flags) cudaFreeHost(h->h_cg_flags);
  if (h->h_slots) cudaFreeHost(h->h_slots);
  if (h->h_flags) cudaFreeHost(h->h_flags);
  if (h->h_stats3) cudaFreeHost(h->h_stats3);
  if (h->h_trip) cudaFreeHost(h->h_trip);
  delete h;
}

static float* param_ptr(b200rl_onpolicy* h, int which, int64_t* n) {
  switch (which) {
    case 0: *n = h->Pp + h->n_ls; return h->pol;
    case 1: *n = h->Pp + h->n_ls; return h->old_pol;
    case 2: *n = h->Pv; return h->val;
    default: *n = 0; return nullptr;
  }
}

extern "C" int b200rl_onpolicy_set_params(b200rl_onpolicy* h, int which, const float* host_flat, int64_t n,
                                          void* stream) {
  B200RL_REQUIRE(h && host_flat, "set_params: NULL argument");
  int64_t cnt;
  float* d = param_ptr(h, which, &cnt);
  B200RL_REQUIRE(d && n == cnt, "set_params: which=%d expects %lld floats, got %lld", which, (long long)cnt, (long long)n);
  B200RL_CUDA(cudaMemcpyAsync(d, host_flat, (size_t)n * 4, cudaMemcpyHostToDevice, static_cast<cudaStream_t>(stream)));
  return 0;
}

extern "C" int b200rl_onpolicy_get_params(b200rl_onpolicy* h, int which, float* host_flat, int64_t n, void* stream) {
  B200RL_REQUIRE(h && host_flat, "get_params: NULL argument");
  int64_t cnt;
  float* d = param_ptr(h, which, &cnt);
  B200RL_REQUIRE(d && n == cnt, "get_params: which=%d expects %lld floats, got %lld", which, (long long)cnt, (long long)n);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200RL_CUDA(cudaMemcpyAsync(host_flat, d, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
  B200RL_CUDA(cudaStreamSynchronize(s));
  return 0;
}

extern "C" int b200rl_onpolicy_set_adam(b200rl_onpolicy* h, int which, const float* exp_avg, const float* exp_avg_sq,
                                        int64_t n, int64_t step, void* stream) {
  B200RL_REQUIRE(h && (which == 0 || which == 2), "set_adam: which must be 0 (policy) or 2 (value)");
  const int64_t cnt = which == 0 ? h->Pp + h->n_ls : h->Pv;
  B200RL_REQUIRE(n == cnt && step >= 0, "set_adam: expects %lld floats, got %lld", (long long)cnt, (long long)n);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  float* m = which == 0 ? h->pol_m : h->val_m;
  float* v = which == 0 ? h->pol_v : h->val_v;
  if (exp_avg) B200RL_CUDA(cudaMemcpyAsync(m, exp_avg, (size_t)n * 4, cudaMemcpyHostToDevice, s));
  else B200RL_CUDA(cudaMemsetAsync(m, 0, (size_t)n * 4, s));
  if (exp_avg_sq) B200RL_CUDA(cudaMemcpyAsync(v, exp_avg_sq, (size_t)n * 4, cudaMemcpyHostToDevice, s));
  else B200RL_CUDA(cudaMemsetAsync(v, 0, (size_t)n * 4, s));
  (which == 0 ? h->pol_step : h->val_step) = step;
  return 0;
}

extern "C" int b200rl_onpolicy_get_adam(b200rl_onpolicy* h, int which, float* exp_avg, float* exp_avg_sq, int64_t n,
                                        int64_t* step, void* stream) {
  B200RL_REQUIRE(h && (which == 0 || which == 2) && exp_avg && exp_avg_sq && step, "get_adam: bad arguments");
  const int64_t cnt = which == 0 ? h->Pp + h->n_ls : h->Pv;
  B200RL_REQUIRE(n == cnt, "get_adam: expects %lld floats, got %lld", (long long)cnt, (long long)n);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200RL_CUDA(cudaMemcpyAsync(exp_avg, which == 0 ? h->pol_m : h->val_m, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
  B200RL_CUDA(cudaMemcpyAsync(exp_avg_sq, which == 0 ? h->pol_v : h->val_v, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
  B200RL_CUDA(cudaStreamSynchronize(s));
  *step = which == 0 ? h->pol_step : h->val_step;
  return 0;
}

extern "C" int b200rl_onpolicy_set_train_log_std(b200rl_onpolicy* h, int32_t on) {
  B200RL_REQUIRE(h, "set_train_log_std: NULL handle");
  B200RL_REQUIRE(!on || h->cfg.dist == B200RL_DIST_GAUSSIAN, "set_train_log_std: only Gaussian policies have a log_std");
  h->train_log_std = on ? 1 : 0;
  h->n_ls = on ? h->act_cols : 0;
  return 0;
}

extern "C" int b200rl_onpolicy_set_log_std(b200rl_onpolicy* h, const float* host_log_std, int64_t n, void* stream) {
  B200RL_REQUIRE(h && host_log_std, "set_log_std: NULL argument");
  B200RL_REQUIRE(h->cfg.dist == B200RL_DIST_GAUSSIAN && n == h->act_cols, "set_log_std: expects %d floats", h->act_cols);
  B200RL_CUDA(cudaMemcpyAsync(h->log_std, host_log_std, (size_t)n * 4, cudaMemcpyHostToDevice,
                              static_cast<cudaStream_t>(stream)));
  return 0;
}

extern "C" int b200rl_onpolicy_load_batch(b200rl_onpolicy* h, const float* obs, const float* actions,
                                          const void* rewards, const float* last_obs, const int64_t* ep_offsets,
                                          const uint8_t* ep_done, int64_t n_rows, int64_t n_episodes,
                                          int src_on_device, void* stream) {
  B200RL_REQUIRE(h && obs && actions && rewards && last_obs && ep_offsets && ep_done, "load_batch: NULL argument");
  B200RL_REQUIRE(n_rows >= 1 && n_rows <= h->cfg.max_rows, "load_batch: n_rows %lld exceeds capacity %lld",
                 (long long)n_rows, (long long)h->cfg.max_rows);
  B200RL_REQUIRE(n_episodes >= 1 && n_episodes <= h->cfg.max_episodes,
                 "load_batch: n_episodes %lld exceeds capacity %lld", (long long)n_episodes,
                 (long long)h->cfg.max_episodes);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const cudaMemcpyKind k = src_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
  if (!src_on_device) {  // host-side validation of the CSR structure (cheap; the scan relies on it)
    B200RL_REQUIRE(ep_offsets[0] == 0 && ep_offsets[n_episodes] == n_rows,
                   "load_batch: ep_offsets must start at 0 and end at n_rows");
    for (int64_t e = 0; e < n_episodes; ++e)
      B200RL_REQUIRE(ep_offsets[e + 1] > ep_offsets[e], "load_batch: episode %lld is empty", (long long)e);
  }
  B200RL_CUDA(cudaMemcpyAsync(h->obs, obs, (size_t)n_rows * h->obs_dim * 4, k, s));
  B200RL_CUDA(cudaMemcpyAsync(h->act, actions, (size_t)n_rows * h->act_cols * 4, k, s));
  B200RL_CUDA(cudaMemcpyAsync(h->rew, rewards, (size_t)n_rows * (h->cfg.rewards_f64 ? 8 : 4), k, s));
  B200RL_CUDA(cudaMemcpyAsync(h->last_obs, last_obs, (size_t)n_episodes * h->obs_dim * 4, k, s));
  B200RL_CUDA(cudaMemcpyAsync(h->off, ep_offsets, (size_t)(n_episodes + 1) * 8, k, s));
  B200RL_CUDA(cudaMemcpyAsync(h->done, ep_done, (size_t)n_episodes, k, s));
  h->n_rows = n_rows;
  h->n_ep = n_episodes;
  h->hints_valid = false;
  return 0;
}

// ---- the shared preamble of PPO / VPG / TRPO train(): value inference -> scan -> (all-reduce of 3 scalars) ----
static int run_preamble(b200rl_onpolicy* h, const b200rl_ppo_hparams* hp, b200rl_allreduce_fn ar, void* user,
                        cudaStream_t s) {
  // range hints for the fp16 tensor-core kernel: one pass over the observations per update instead of per launch
  h->hints_valid = false;
  if (h->obs_dim <= 32) {
    if (b200rl_absmax_cols(h->obs, h->n_rows, h->obs_dim, h->absmax, s)) return 1;
    if (b200rl_absmax_cols(h->last_obs, h->n_ep, h->obs_dim, h->absmax + 32, s)) return 1;
    h->hints_valid = true;
  }
  // utils.py:60-71 compute_values: V(obs_t) for every step and V(last_observation) for every episode
  if (launch_fused(h, h->cfg.value, B200RL_LOSS_EVAL, B200RL_DIST_NONE, h->val, h->obs, h->n_rows, h->n_rows, 0.0,
                   false, false, h->values, false, nullptr, s)) return 1;
  if (launch_fused(h, h->cfg.value, B200RL_LOSS_EVAL, B200RL_DIST_NONE, h->val, h->last_obs, h->n_ep, h->n_ep, 0.0,
                   false, false, h->last_values, false, nullptr, s)) return 1;
  if (b200rl_gae_scan(h->rew, h->cfg.rewards_f64, h->values, h->last_values, h->off, h->done, h->n_rows, h->n_ep,
                      hp->gamma, hp->gae_lambda, h->adv_raw, h->ret, h->adv_stats, h->scan_ws, h->scan_ws_bytes, s))
    return 1;
  if (b200rl_absmax(h->ret, h->n_rows, h->absmax + 64, s)) return 1;
  // normalize_tensor (utils.py:90-92) is over the GLOBAL batch: one 3-scalar all-reduce per update
  if (ar && ar(user, h->adv_stats, 3, 1, s)) {
    set_error("allreduce callback failed (advantage statistics)");
    return 1;
  }
  return 0;
}

static int run_value_loop(b200rl_onpolicy* h, const b200rl_ppo_hparams* hp, b200rl_allreduce_fn ar, void* user,
                          int64_t n_glob, int slot0, cudaStream_t s, int j0 = 0) {
  const int grid = b200rl_mlp_grid(&h->cfg.value, h->n_rows, 1);
  for (int j = j0; j < hp->num_value_gradients; ++j) {  // ppo.py:186-192
    double* slot = h->slots + (size_t)(slot0 + j) * B200RL_N_SCALARS;
    if (launch_fused(h, h->cfg.value, B200RL_LOSS_MSE, B200RL_DIST_NONE, h->val, h->obs, h->n_rows, n_glob, 0.0,
                     false, false, nullptr, true, nullptr, s)) return 1;
    if (b200rl_reduce_partials(h->partials, h->scalar_partials, grid, h->Pv, h->val_grad, slot, ar ? 1 : 0, nullptr, s))
      return 1;
    if (ar && ar(user, h->val_grad, h->Pv + B200RL_N_SCALARS, 0, s)) {
      set_error("allreduce callback failed (value gradient)");
      return 1;
    }
    if (b200rl_adam_step(h->val, h->val_grad, h->val_m, h->val_v, h->Pv, h->val_step + j + 1, hp->value_lr,
                         hp->value_beta1, hp->value_beta2, hp->value_eps, nullptr, 0, (double)n_glob, 0.0, nullptr,
                         h->flags + 2, ar ? h->val_grad + h->Pv : nullptr, ar ? slot : nullptr, s))
      return 1;
  }
  return 0;
}

// ---- fused policy + value iterations (mlp_tc3.cu): step i of both loops in one pass over the batch ----------------
static void fill_tc3_net(const b200rl_mlp_desc& d, Tc3Net* n, int* P) {
  n->n_out = d.sizes[3];
  n->h1 = d.sizes[1];
  n->h2 = d.sizes[2];
  *P = mlp3_offsets(d, n->w_off, n->b_off);
}

// both chains of the step kernel on the engine's buffers; no early-stop flag (stop_flag = NULL)
static Tc3Args tc3_args(const b200rl_onpolicy* h, const b200rl_ppo_hparams* hp, int64_t n_glob) {
  Tc3Args k;
  memset(&k, 0, sizeof(k));
  k.n_in = h->obs_dim;
  k.dist = h->cfg.dist;
  fill_tc3_net(h->cfg.policy, &k.net[0], &k.P[0]);
  fill_tc3_net(h->cfg.value, &k.net[1], &k.P[1]);
  k.params[0] = h->pol;
  k.params[1] = h->val;
  k.n_rows = h->n_rows;
  k.inv_n = 1.0f / (float)n_glob;
  k.n_glob_f = (float)n_glob;
  k.clip_lo = (float)(1.0 - hp->clip_range);
  k.clip_hi = (float)(1.0 + hp->clip_range);
  k.ximg = h->ximg;
  k.xscale = h->xscale;
  k.actions = h->act;
  k.log_std = h->log_std;
  k.adv_raw = h->adv_raw;
  k.adv_stats = h->adv_stats;
  k.old_logp = h->old_logp;
  k.target = h->ret;
  k.target_absmax = h->absmax + 64;
  k.partials = h->partials;
  k.scalar_partials = h->scalar_partials;
  k.x_bad = h->trip;
  k.status = h->trip + 1;
  k.run_policy = k.run_value = 1;
  return k;
}

static void fill_seg(Ra3Seg* g, float* params, float* m, float* v, int64_t step, double lr, double b1, double b2,
                     double eps) {
  g->params = params;
  g->m = m;
  g->v = v;
  g->one_minus_b1 = (float)(1.0 - b1);
  g->b2 = (float)b2;
  g->one_minus_b2 = (float)(1.0 - b2);
  adam_scalars(step, lr, b1, b2, &g->step_size, &g->bc2_sqrt);
  g->eps = (float)eps;
}

// Iterations [0, n_iter) of the policy AND the value loop.  Every `poll` iterations the host looks at the early-stop
// flag (one 4-byte read-back): once the policy loop has stopped, the remaining value steps are faster on the
// two-tiles-in-flight value kernel than as the lone chain of the fused one.  Returns the iterations done in *done.
static int run_fused_iterations(b200rl_onpolicy* h, const b200rl_ppo_hparams* hp, b200rl_allreduce_fn ar, void* user,
                                int64_t n_glob, int K, int n_iter, cudaStream_t s, int* done) {
  Tc3Args k = tc3_args(h, hp, n_glob);
  k.stop_flag = h->flags;
  Ra3Args a;
  memset(&a, 0, sizeof(a));
  a.partials = h->partials;
  a.scalar_partials = h->scalar_partials;
  a.rows = 2 * tc_grid(h->n_rows);
  a.P[0] = h->Pp;
  a.P[1] = h->Pv;
  a.grad = h->grad_all;
  a.n_global = (double)n_glob;
  a.kl_limit = 1.5 * hp->max_kl_divergence;
  a.kl_limit_on = 1;
  a.stop_flag = h->flags;
  a.applied_p = h->flags + 1;
  a.applied_v = h->flags + 2;
  a.run_policy = 1;
  a.run_value = 1;
  const int64_t n_all = h->Pp + h->Pv + 2 * B200RL_N_SCALARS;
  constexpr int poll = 8;
  // B200RL_PEER_ONE_LAUNCH=0 keeps publish / wait / gather as three launches (A/B runs)
  const char* e1 = getenv("B200RL_PEER_ONE_LAUNCH");
  const bool one_launch = !(e1 != nullptr && e1[0] == '0') && ra3_one_wave(h->Pp + h->Pv);
  int i = 0;
  for (; i < n_iter; ++i) {
    if (launch_mlp_tc3(k, s)) return 1;
    fill_seg(&a.seg[0], h->pol, h->pol_m, h->pol_v, h->pol_step + i + 1, hp->policy_lr, hp->policy_beta1,
             hp->policy_beta2, hp->policy_eps);
    fill_seg(&a.seg[1], h->val, h->val_m, h->val_v, h->val_step + i + 1, hp->value_lr, hp->value_beta1, hp->value_beta2,
             hp->value_eps);
    a.slot_p = h->slots + (size_t)i * B200RL_N_SCALARS;
    a.slot_v = h->slots + (size_t)(K + 1 + i) * B200RL_N_SCALARS;
    if (!ar) {
      a.mode = 0;
      if (launch_reduce_adam3(a, s)) return 1;
    } else if (h->comm_world > 1) {  // one-shot exchange over NVLink peer memory, no collective call
      a.peers = h->peers_dev;
      a.world = h->comm_world;
      a.rank = h->comm_rank;
      a.xchg_stride = h->xchg_stride;
      a.seq = ++h->comm_seq;
      a.done_counter = h->done_counter;
      a.comm_error = h->flags + 4;
      if (one_launch) {
        a.mode = 5;
        if (launch_reduce_adam3(a, s)) return 1;
      } else {
        a.mode = 3;
        if (launch_reduce_adam3(a, s)) return 1;
        if (launch_wait_peers(a, s)) return 1;
        a.mode = 4;
        if (launch_reduce_adam3(a, s)) return 1;
      }
    } else {
      a.mode = 1;
      if (launch_reduce_adam3(a, s)) return 1;
      if (ar(user, h->grad_all, n_all, 0, s)) {  // ONE all-reduce: both gradients + both scalar tails
        set_error("allreduce callback failed (fused policy + value gradient)");
        return 1;
      }
      a.mode = 2;
      if (launch_reduce_adam3(a, s)) return 1;
    }
    if ((i % poll) == poll - 1 && i + 1 < n_iter) {
      B200RL_CUDA(cudaMemcpyAsync(h->h_flags, h->flags, sizeof(int), cudaMemcpyDeviceToHost, s));
      B200RL_CUDA(cudaStreamSynchronize(s));
      if (h->h_flags[0] != 0) {
        ++i;
        break;
      }
    }
  }
  *done = i;
  return 0;
}

static int run_update_impl(b200rl_onpolicy* h, const b200rl_ppo_hparams* hp, b200rl_allreduce_fn ar, void* user,
                           b200rl_update_stats* stats, cudaStream_t s, int policy_loss, bool fused, bool* tripped) {
  const int64_t launches0 = launches_total();
  const int64_t n_glob = hp->n_global_rows > 0 ? hp->n_global_rows : h->n_rows;
  const bool ppo = policy_loss == B200RL_LOSS_PPO_CLIP;
  const int K = ppo ? hp->num_policy_gradients : 1;
  const int Kv = hp->num_value_gradients;
  if (ensure_slots(h, K + Kv + 4)) return 1;
  B200RL_CUDA(cudaMemsetAsync(h->flags, 0, 8 * sizeof(int), s));
  B200RL_CUDA(cudaMemsetAsync(h->slots, 0, (size_t)(K + Kv + 4) * B200RL_N_SCALARS * sizeof(double), s));
  const size_t Pp = (size_t)h->Pp, Pv = (size_t)h->Pv;
  if (fused) {  // what a redo on the wide-range path starts from
    B200RL_CUDA(cudaMemsetAsync(h->trip, 0, 4 * sizeof(float), s));
    float* q = h->snap;
    const float* src[7] = {h->pol, h->pol_m, h->pol_v, h->old_pol, h->val, h->val_m, h->val_v};
    for (int t = 0; t < 7; ++t) {
      const size_t n = t < 4 ? Pp : Pv;
      B200RL_CUDA(cudaMemcpyAsync(q, src[t], n * 4, cudaMemcpyDeviceToDevice, s));
      q += n;
    }
  }

  if (run_preamble(h, hp, ar, user, s)) return 1;

  const int dist = h->cfg.dist;
  const int grid_p = b200rl_mlp_grid(&h->cfg.policy, h->n_rows, 1);
  const int grid_e = b200rl_mlp_grid(&h->cfg.policy, h->n_rows, 0);
  int* stop = ppo ? h->flags : nullptr;
  if (ppo) {
    // ppo.py:241-243: old_policy is frozen for the whole epoch => its log-probs are computed once
    if (launch_fused(h, h->cfg.policy, B200RL_LOSS_EVAL, dist, h->old_pol, h->obs, h->n_rows, n_glob, 0.0, false,
                     false, h->old_logp, false, nullptr, s)) return 1;
  }
  int i0 = 0;  // iterations of both loops already done by the fused kernel
  if (fused) {
    if (launch_pack_obs(h->obs, h->n_rows, h->obs_dim, h->absmax, h->ximg, h->xscale, h->trip, s)) return 1;
    if (run_fused_iterations(h, hp, ar, user, n_glob, K, K < Kv ? K : Kv, s, &i0)) return 1;
  }
  const int64_t Pe = h->Pp + h->n_ls;  // policy vector incl. a trainable log_std
  const int grid_pp = h->train_log_std ? b200rl_mlp_grid(&h->cfg.policy, h->n_rows, 4) : grid_p;
  for (int i = i0; i < K; ++i) {  // ppo.py:173-181 / vpg.py:194-207
    double* slot = h->slots + (size_t)i * B200RL_N_SCALARS;
    if (launch_fused(h, h->cfg.policy, policy_loss, dist, h->pol, h->obs, h->n_rows, n_glob, hp->clip_range, true,
                     ppo, nullptr, true, stop, s)) return 1;
    if (b200rl_reduce_partials(h->partials, h->scalar_partials, grid_pp, Pe, h->pol_grad, slot, ar ? 1 : 0, stop, s))
      return 1;
    if (ar && ar(user, h->pol_grad, Pe + B200RL_N_SCALARS, 0, s)) {
      set_error("allreduce callback failed (policy gradient)");
      return 1;
    }
    // KL carried by this forward pass = approx KL after the previous update (ppo.py:176-181), checked on device
    const void* kl = !ppo ? nullptr : (ar ? static_cast<const void*>(h->pol_grad + Pe + 1)
                                          : static_cast<const void*>(slot + 1));
    if (b200rl_adam_step(h->pol, h->pol_grad, h->pol_m, h->pol_v, Pe, h->pol_step + i + 1, hp->policy_lr,
                         hp->policy_beta1, hp->policy_beta2, hp->policy_eps, kl, ar ? 1 : 0, (double)n_glob,
                         1.5 * hp->max_kl_divergence, stop, h->flags + 1, ar ? h->pol_grad + Pe : nullptr,
                         ar ? slot : nullptr, s))
      return 1;
  }
  if (ppo) {
    // KL after the last update (only reached when no early stop fired): forward-only pass, slot K
    double* slot = h->slots + (size_t)K * B200RL_N_SCALARS;
    if (launch_fused(h, h->cfg.policy, B200RL_LOSS_EVAL, dist, h->pol, h->obs, h->n_rows, n_glob, 0.0, false, true,
                     nullptr, true, stop, s)) return 1;
    if (b200rl_reduce_partials(nullptr, h->scalar_partials, grid_e, h->Pp, nullptr, slot, 0, stop, s)) return 1;
    if (ar && ar(user, slot, B200RL_N_SCALARS, 1, s)) {
      set_error("allreduce callback failed (final KL)");
      return 1;
    }
    // ppo.py:183: old_policy.load_state_dict(policy.state_dict())
    B200RL_CUDA(cudaMemcpyAsync(h->old_pol, h->pol, (size_t)Pe * 4, cudaMemcpyDeviceToDevice, s));
  }

  if (run_value_loop(h, hp, ar, user, n_glob, K + 1, s, i0)) return 1;

  // ---- one device->host read of the statistics ----
  if (fused) {
    // a range trip on ANY rank sends every rank through the redo (the collective keeps them in step)
    if (ar && ar(user, h->trip, 2, 0, s)) {
      set_error("allreduce callback failed (range flags)");
      return 1;
    }
    B200RL_CUDA(cudaMemcpyAsync(h->h_trip, h->trip, 2 * sizeof(float), cudaMemcpyDeviceToHost, s));
  }
  B200RL_CUDA(cudaMemcpyAsync(h->h_slots, h->slots, (size_t)(K + Kv + 2) * B200RL_N_SCALARS * sizeof(double),
                              cudaMemcpyDeviceToHost, s));
  h->last_slots = K + Kv + 2;
  B200RL_CUDA(cudaMemcpyAsync(h->h_flags, h->flags, 8 * sizeof(int), cudaMemcpyDeviceToHost, s));
  B200RL_CUDA(cudaMemcpyAsync(h->h_stats3, h->adv_stats, 3 * sizeof(double), cudaMemcpyDeviceToHost, s));
  B200RL_CUDA(cudaStreamSynchronize(s));
  if (fused && (h->h_trip[0] != 0.f || h->h_trip[1] != 0.f)) {
    // fp16 operands left their range somewhere in this update: put everything back; the caller redoes it
    const float* q = h->snap;
    float* dst[7] = {h->pol, h->pol_m, h->pol_v, h->old_pol, h->val, h->val_m, h->val_v};
    for (int t = 0; t < 7; ++t) {
      const size_t n = t < 4 ? Pp : Pv;
      B200RL_CUDA(cudaMemcpyAsync(dst[t], q, n * 4, cudaMemcpyDeviceToDevice, s));
      q += n;
    }
    *tripped = true;
    return 0;
  }

  B200RL_REQUIRE(h->h_flags[4] == 0, "update: a peer's gradient did not arrive within 10 s (peer exchange over NVLink)");
  memset(stats, 0, sizeof(*stats));
  const double ng = (double)n_glob;
  const int applied_p = h->h_flags[1], applied_v = h->h_flags[2];
  const double* s0 = h->h_slots;
  stats->policy_loss_before = K > 0 ? s0[0] / ng : NAN;
  stats->entropy_before = K > 0 ? s0[2] / ng : NAN;
  {
    const double mean = s0[3] / ng;
    stats->logp_std_before = K > 0 ? sqrt(fmax(0.0, (s0[4] - ng * mean * mean) / (ng - 1.0))) : NAN;
  }
  stats->kl_divergence = ppo ? h->h_slots[(size_t)applied_p * B200RL_N_SCALARS + 1] / ng : NAN;
  double vsum = 0.0;
  for (int j = 0; j < Kv; ++j) vsum += h->h_slots[(size_t)(K + 1 + j) * B200RL_N_SCALARS] / ng;
  stats->value_loss_mean = Kv > 0 ? vsum / Kv : NAN;
  stats->value_loss_first = Kv > 0 ? h->h_slots[(size_t)(K + 1) * B200RL_N_SCALARS] / ng : NAN;
  stats->value_loss_last = Kv > 0 ? h->h_slots[(size_t)(K + Kv) * B200RL_N_SCALARS] / ng : NAN;
  stats->policy_steps_applied = applied_p;
  stats->value_steps_applied = applied_v;
  {
    const double cnt = h->h_stats3[2], mean = h->h_stats3[0] / cnt;
    stats->adv_mean = mean;
    stats->adv_std = sqrt((h->h_stats3[1] - cnt * mean * mean) / (cnt - 1.0));
  }
  h->pol_step += applied_p;
  h->val_step += applied_v;
  stats->kernel_launches = (int32_t)(launches_total() - launches0);
  stats->fused = fused ? 1 : 0;  // 1 = the fused policy + value step kernel did the iterations
  h->last_fused = fused ? 1 : 0;
  return 0;
}

static bool fused_step_enabled() {  // B200RL_FUSED_STEP=0 keeps the two-loop path (A/B parity runs)
  const char* e = getenv("B200RL_FUSED_STEP");
  return !(e != nullptr && e[0] == '0');
}

static int run_update(b200rl_onpolicy* h, const b200rl_ppo_hparams* hp, b200rl_allreduce_fn ar, void* user,
                      b200rl_update_stats* stats, void* stream, int policy_loss) {
  B200RL_REQUIRE(h && hp && stats, "update: NULL argument");
  B200RL_REQUIRE(h->n_rows > 0, "update: no batch loaded");
  B200RL_REQUIRE(hp->num_policy_gradients >= 0 && hp->num_value_gradients >= 0, "update: negative step count");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const bool fused = policy_loss == B200RL_LOSS_PPO_CLIP && h->fused_ok && !h->train_log_std && fused_step_enabled() &&
                     use_tc(h->cfg.policy) && use_tc(h->cfg.value) &&
                     hp->num_policy_gradients > 0 && hp->num_value_gradients > 0;
  bool tripped = false;
  if (run_update_impl(h, hp, ar, user, stats, s, policy_loss, fused, &tripped)) return 1;
  if (tripped) return run_update_impl(h, hp, ar, user, stats, s, policy_loss, false, &tripped);
  return 0;
}

extern "C" int b200rl_ppo_update(b200rl_onpolicy* h, const b200rl_ppo_hparams* hp, b200rl_allreduce_fn allreduce,
                                 void* user, b200rl_update_stats* stats, void* stream) {
  return run_update(h, hp, allreduce, user, stats, stream, B200RL_LOSS_PPO_CLIP);
}

extern "C" int b200rl_vpg_update(b200rl_onpolicy* h, const b200rl_ppo_hparams* hp, b200rl_allreduce_fn allreduce,
                                 void* user, b200rl_update_stats* stats, void* stream) {
  return run_update(h, hp, allreduce, user, stats, stream, B200RL_LOSS_VPG);
}

// ------------------------------------------------------------------------------------------------------------------
// TRPO
// ------------------------------------------------------------------------------------------------------------------
static int ensure_trpo(b200rl_onpolicy* h) {
  if (h->cg_x) return 0;
  h->out_cols = h->cfg.policy.sizes[h->cfg.policy.n_layers];
  int rc = 0;
  rc |= dev_alloc(h, &h->old_out, (size_t)h->cfg.max_rows * h->out_cols);
  rc |= dev_alloc(h, &h->cg_x, (size_t)h->Pp);
  rc |= dev_alloc(h, &h->cg_r, (size_t)h->Pp);
  rc |= dev_alloc(h, &h->cg_p, (size_t)h->Pp);
  rc |= dev_alloc(h, &h->cg_z, (size_t)h->Pp + B200RL_N_SCALARS);
  rc |= dev_alloc(h, &h->cg_prev, (size_t)h->Pp);
  rc |= dev_alloc(h, &h->cg_descent, (size_t)h->Pp);
  rc |= dev_alloc(h, &h->cg_sc, 8);
  rc |= dev_alloc(h, &h->cg_flags, 4);
  if (!rc && cudaMallocHost(reinterpret_cast<void**>(&h->h_cg_sc), 8 * sizeof(double)) != cudaSuccess) rc = 1;
  if (!rc && cudaMallocHost(reinterpret_cast<void**>(&h->h_cg_flags), 4 * sizeof(int)) != cudaSuccess) rc = 1;
  if (rc && g_error.empty()) set_error("trpo: allocation failed");
  return rc;
}

// out[P] = F v (without damping): one B200RL_LOSS_FVP launch + fixed-order reduction of the partials
static int launch_fvp(b200rl_onpolicy* h, const float* direction, float* out, int64_t n_glob, cudaStream_t s) {
  b200rl_mlp_loss_grad_args a;
  memset(&a, 0, sizeof(a));
  a.mlp = h->cfg.policy;
  a.loss = B200RL_LOSS_FVP;
  a.dist = h->cfg.dist;
  a.n_rows = h->n_rows;
  a.n_global = n_glob;
  a.params = h->pol;
  a.obs = h->obs;
  a.log_std = h->log_std;
  a.direction = direction;
  a.partials = h->partials;
  if (h->hints_valid) a.obs_absmax = h->absmax;
  if (b200rl_mlp_loss_grad(&a, s)) return 1;
  return b200rl_reduce_partials(h->partials, nullptr, b200rl_mlp_grid(&h->cfg.policy, h->n_rows, 2), h->Pp, out,
                                nullptr, 0, nullptr, s);
}

extern "C" int b200rl_onpolicy_fvp(b200rl_onpolicy* h, const float* host_v, float* host_out, int64_t n, double damping,
                                   void* stream) {
  B200RL_REQUIRE(h && host_v && host_out && n == h->Pp, "fvp: bad arguments");
  B200RL_REQUIRE(h->n_rows > 0, "fvp: no batch loaded");
  if (ensure_trpo(h)) return 1;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  B200RL_CUDA(cudaMemcpyAsync(h->cg_p, host_v, (size_t)n * 4, cudaMemcpyHostToDevice, s));
  if (launch_fvp(h, h->cg_p, h->cg_z, h->n_rows, s)) return 1;
  B200RL_CUDA(cudaMemcpyAsync(host_out, h->cg_z, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
  B200RL_CUDA(cudaStreamSynchronize(s));
  for (int64_t i = 0; i < n; ++i) host_out[i] += (float)damping * host_v[i];  // H -> H + damping I (cg optimizer :165)
  return 0;
}

extern "C" int b200rl_trpo_update(b200rl_onpolicy* h, const b200rl_ppo_hparams* hp, const b200rl_trpo_hparams* cg,
                                  b200rl_update_stats* stats, b200rl_trpo_stats* ts, void* stream) {
  return b200rl_trpo_update_dp(h, hp, cg, nullptr, nullptr, stats, ts, stream);
}

// Data-parallel TRPO (each rank holds a block of episodes, hp->n_global_rows = the global row count): every quantity the
// step derives from the batch is a sum over rows, so it is all-reduced where it is formed -- the advantage statistics,
// the surrogate gradient with its scalar sums, every Fisher-vector product, the scalar sums of every line-search
// evaluation, the value gradients -- and the conjugate-gradient / line-search decisions, taken on the device from those
// reduced values, come out identical on every rank.  ~30 small all-reduces per update.
extern "C" int b200rl_trpo_update_dp(b200rl_onpolicy* h, const b200rl_ppo_hparams* hp, const b200rl_trpo_hparams* cg,
                                     b200rl_allreduce_fn ar, void* user, b200rl_update_stats* stats,
                                     b200rl_trpo_stats* ts, void* stream) {
  B200RL_REQUIRE(h && hp && cg && stats && ts, "trpo_update: NULL argument");
  B200RL_REQUIRE(h->n_rows > 0, "trpo_update: no batch loaded");
  B200RL_REQUIRE(cg->n_conjugate_gradients >= 1 && cg->max_backtracks >= 1, "trpo_update: bad CG parameters");
  B200RL_REQUIRE(!h->train_log_std, "trpo_update: a trainable log_std is not part of the conjugate-gradient step");
  if (ensure_trpo(h)) return 1;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int64_t launches0 = launches_total();
  const int64_t n = h->n_rows;
  const int64_t n_glob = hp->n_global_rows > 0 ? hp->n_global_rows : n;
  const int Kv = hp->num_value_gradients, nb = cg->max_backtracks;
  const int n_slots = 1 + nb + Kv + 2;
  if (ensure_slots(h, n_slots)) return 1;
  B200RL_CUDA(cudaMemsetAsync(h->flags, 0, 8 * sizeof(int), s));
  B200RL_CUDA(cudaMemsetAsync(h->slots, 0, (size_t)n_slots * B200RL_N_SCALARS * sizeof(double), s));
  B200RL_CUDA(cudaMemsetAsync(h->cg_sc, 0, 8 * sizeof(double), s));
  if (run_preamble(h, hp, ar, user, s)) return 1;
  const int dist = h->cfg.dist;
  const int P = (int)h->Pp;
  const float delta = (float)cg->max_constraint, damping = (float)cg->hvp_damping_coefficient;

  b200rl_mlp_loss_grad_args a;
  // (1) old policy: log-probs and raw outputs (trpo.py:158-159, 171); frozen for the whole step
  memset(&a, 0, sizeof(a));
  a.mlp = h->cfg.policy;
  a.loss = B200RL_LOSS_EVAL;
  a.dist = dist;
  a.n_rows = n;
  a.n_global = n;
  a.params = h->old_pol;
  a.obs = h->obs;
  a.actions = h->act;
  a.log_std = h->log_std;
  a.row_out = h->old_logp;
  a.out_full = h->old_out;
  if (h->hints_valid) a.obs_absmax = h->absmax;
  if (b200rl_mlp_loss_grad(&a, s)) return 1;
  // (2) surrogate loss and its gradient at theta (trpo.py:228-239); slot 0 also carries the logged statistics
  if (launch_fused(h, h->cfg.policy, B200RL_LOSS_TRPO_SURROGATE, dist, h->pol, h->obs, n, n_glob, 0.0, true, true, nullptr,
                   true, nullptr, s)) return 1;
  if (b200rl_reduce_partials(h->partials, h->scalar_partials, b200rl_mlp_grid(&h->cfg.policy, n, 1), h->Pp, h->pol_grad,
                             h->slots, ar ? 1 : 0, nullptr, s)) return 1;
  if (ar) {  // gradient and scalar sums in one buffer
    if (ar(user, h->pol_grad, h->Pp + B200RL_N_SCALARS, 0, s)) {
      set_error("allreduce callback failed (surrogate gradient)");
      return 1;
    }
    if (trpo_tail_to_slot(h->pol_grad + h->Pp, h->slots, s)) return 1;
  }
  if (trpo_set_scalar(h->cg_sc + 1, h->slots, 0, 1.0 / (double)n_glob, s)) return 1;  // loss_before
  // (3) conjugate gradient: x ~ H^-1 g
  if (trpo_cg_init(h->pol_grad, h->cg_x, h->cg_r, h->cg_p, P, h->cg_sc, h->cg_flags, s)) return 1;
  int fvps = 0;
  auto fvp_allreduce = [&]() -> int {
    if (ar && ar(user, h->cg_z, h->Pp, 0, s)) {
      set_error("allreduce callback failed (Fisher-vector product)");
      return 1;
    }
    return 0;
  };
  for (int it = 0; it < cg->n_conjugate_gradients; ++it) {
    if (launch_fvp(h, h->cg_p, h->cg_z, n_glob, s)) return 1;
    if (fvp_allreduce()) return 1;
    ++fvps;
    if (trpo_cg_update(h->cg_z, damping, h->cg_x, h->cg_r, h->cg_p, P, h->cg_sc, h->cg_flags, s)) return 1;
  }
  // (4) step size and descent step
  if (trpo_nan_to_zero(h->cg_x, P, s)) return 1;
  if (launch_fvp(h, h->cg_x, h->cg_z, n_glob, s)) return 1;
  if (fvp_allreduce()) return 1;
  ++fvps;
  if (trpo_step_size(h->cg_x, h->cg_z, damping, delta, h->cg_descent, h->pol, h->cg_prev, P, h->cg_sc, s)) return 1;
  // (5) backtracking line search (device-side accept flag: later iterations become no-ops)
  const int grid_f = b200rl_mlp_grid(&h->cfg.policy, n, 3);
  for (int k = 0; k < nb; ++k) {
    const float ratio = (float)pow(cg->backtrack_ratio, (double)k);
    double* slot = h->slots + (size_t)(1 + k) * B200RL_N_SCALARS;
    if (trpo_ls_set_params(h->pol, h->cg_prev, h->cg_descent, ratio, P, h->cg_flags, s)) return 1;
    memset(&a, 0, sizeof(a));
    a.mlp = h->cfg.policy;
    a.loss = B200RL_LOSS_TRPO_SURROGATE;
    a.flags = B200RL_FLAG_FORWARD_ONLY;
    a.dist = dist;
    a.n_rows = n;
    a.n_global = n_glob;
    a.params = h->pol;
    a.obs = h->obs;
    a.actions = h->act;
    a.log_std = h->log_std;
    a.adv_raw = h->adv_raw;
    a.adv_stats = h->adv_stats;
    a.old_logp = h->old_logp;
    a.old_out = h->old_out;
    if (h->hints_valid) a.obs_absmax = h->absmax;
    a.scalar_partials = h->scalar_partials;
    a.skip_flag = h->cg_flags + 1;
    if (b200rl_mlp_loss_grad(&a, s)) return 1;
    if (b200rl_reduce_partials(nullptr, h->scalar_partials, grid_f, h->Pp, nullptr, slot, 0, h->cg_flags + 1, s)) return 1;
    if (ar && ar(user, slot, B200RL_N_SCALARS, 1, s)) {  // zeros once the search has accepted (skipped launches)
      set_error("allreduce callback failed (line-search evaluation)");
      return 1;
    }
    if (trpo_ls_check(slot, (double)n_glob, delta, h->cg_sc, h->cg_flags, k, s)) return 1;
  }
  if (trpo_ls_final(h->pol, h->cg_prev, P, delta, h->cg_sc, h->cg_flags, s)) return 1;
  // (6) trpo.py:192 old_policy.load_state_dict(policy.state_dict()); then the value steps (:195-201)
  B200RL_CUDA(cudaMemcpyAsync(h->old_pol, h->pol, (size_t)h->Pp * 4, cudaMemcpyDeviceToDevice, s));
  const int vslot0 = 1 + nb;
  if (run_value_loop(h, hp, ar, user, n_glob, vslot0, s)) return 1;

  B200RL_CUDA(cudaMemcpyAsync(h->h_slots, h->slots, (size_t)n_slots * B200RL_N_SCALARS * sizeof(double),
                              cudaMemcpyDeviceToHost, s));
  h->last_slots = n_slots;
  B200RL_CUDA(cudaMemcpyAsync(h->h_flags, h->flags, 8 * sizeof(int), cudaMemcpyDeviceToHost, s));
  B200RL_CUDA(cudaMemcpyAsync(h->h_stats3, h->adv_stats, 3 * sizeof(double), cudaMemcpyDeviceToHost, s));
  B200RL_CUDA(cudaMemcpyAsync(h->h_cg_sc, h->cg_sc, 8 * sizeof(double), cudaMemcpyDeviceToHost, s));
  B200RL_CUDA(cudaMemcpyAsync(h->h_cg_flags, h->cg_flags, 4 * sizeof(int), cudaMemcpyDeviceToHost, s));
  B200RL_CUDA(cudaStreamSynchronize(s));

  memset(stats, 0, sizeof(*stats));
  memset(ts, 0, sizeof(*ts));
  const double ng = (double)n_glob;
  const double* s0 = h->h_slots;
  stats->policy_loss_before = s0[0] / ng;
  stats->entropy_before = s0[2] / ng;
  {
    const double mean = s0[3] / ng;
    stats->logp_std_before = sqrt(fmax(0.0, (s0[4] - ng * mean * mean) / (ng - 1.0)));
  }
  stats->kl_divergence = h->h_cg_sc[4];
  double vsum = 0.0;
  for (int j = 0; j < Kv; ++j) vsum += h->h_slots[(size_t)(vslot0 + j) * B200RL_N_SCALARS] / ng;
  stats->value_loss_mean = Kv > 0 ? vsum / Kv : NAN;
  stats->value_loss_first = Kv > 0 ? h->h_slots[(size_t)vslot0 * B200RL_N_SCALARS] / ng : NAN;
  stats->value_loss_last = Kv > 0 ? h->h_slots[(size_t)(vslot0 + Kv - 1) * B200RL_N_SCALARS] / ng : NAN;
  stats->policy_steps_applied = h->h_cg_flags[2] ? 0 : 1;
  stats->value_steps_applied = h->h_flags[2];
  {
    const double cnt = h->h_stats3[2], mean = h->h_stats3[0] / cnt;
    stats->adv_mean = mean;
    stats->adv_std = sqrt((h->h_stats3[1] - cnt * mean * mean) / (cnt - 1.0));
  }
  h->val_step += h->h_flags[2];
  stats->kernel_launches = (int32_t)(launches_total() - launches0);
  ts->step_size = h->h_cg_sc[2];
  ts->xhx = h->h_cg_sc[5];
  ts->loss_before = h->h_cg_sc[1];
  ts->new_loss = h->h_cg_sc[3];
  ts->kl = h->h_cg_sc[4];
  ts->accepted_index = (int32_t)h->h_cg_sc[6];
  ts->rejected = h->h_cg_flags[2];
  ts->cg_converged = h->h_cg_flags[0];
  ts->fvp_launches = fvps;
  return 0;
}

extern "C" int b200rl_onpolicy_device_view(b200rl_onpolicy* h, const char* name, void** ptr, int64_t* count,
                                           int32_t* dtype) {
  B200RL_REQUIRE(h && name && ptr && count && dtype, "device_view: NULL argument");
  h->hints_valid = false;  // the caller may write through the view
  struct V { const char* n; void* p; int64_t c; int32_t d; };
  const V views[] = {
      {"values", h->values, h->n_rows, 0},        {"last_values", h->last_values, h->n_ep, 0},
      {"adv_raw", h->adv_raw, h->n_rows, 0},      {"ret", h->ret, h->n_rows, 0},
      {"old_logp", h->old_logp, h->n_rows, 0},    {"adv_stats", h->adv_stats, 3, 1},
      // after a fused update both gradients sit side by side in the all-reduce buffer
      {"policy_grad", h->last_fused ? h->grad_all : h->pol_grad, h->last_fused ? h->Pp : h->Pp + B200RL_N_SCALARS, 0},
      {"value_grad", h->last_fused ? h->grad_all + h->Pp : h->val_grad, h->last_fused ? h->Pv : h->Pv + B200RL_N_SCALARS, 0},
      {"policy_params", h->pol, h->Pp, 0},        {"old_policy_params", h->old_pol, h->Pp, 0},
      {"value_params", h->val, h->Pv, 0},         {"obs", h->obs, h->n_rows * h->obs_dim, 0},
      {"cg_x", h->cg_x, h->cg_x ? h->Pp : 0, 0},  {"cg_descent", h->cg_descent, h->cg_descent ? h->Pp : 0, 0},
      // the conjugate-gradient state after the last update: residual, direction, and F x of the step-size product
      {"cg_r", h->cg_r, h->cg_r ? h->Pp : 0, 0},  {"cg_p", h->cg_p, h->cg_p ? h->Pp : 0, 0},
      {"cg_z", h->cg_z, h->cg_z ? h->Pp : 0, 0},
      // the fused step kernel's per-slot partial rows [2 slots][P0 + P1] and scalar rows [2 slots][16]
      {"fused_partials", h->partials, h->fused_ok ? 2 * (int64_t)tc_grid(h->n_rows) * (h->Pp + h->Pv) : 0, 0},
      {"fused_scalar_partials", h->scalar_partials, h->fused_ok ? 2 * (int64_t)tc_grid(h->n_rows) * 2 * B200RL_N_SCALARS : 0, 1},
  };
  for (const V& v : views)
    if (strcmp(v.n, name) == 0) {
      *ptr = v.p;
      *count = v.c;
      *dtype = v.d;
      return 0;
    }
  set_error("device_view: unknown view '%s'", name);
  return 2;
}

// ---- peer exchange set-up -----------------------------------------------------------------------------------------
extern "C" int b200rl_onpolicy_comm_export(b200rl_onpolicy* h, void* handle64, void** local_ptr) {
  B200RL_REQUIRE(h && handle64 && local_ptr, "comm_export: NULL argument");
  B200RL_REQUIRE(h->fused_ok, "comm_export: the networks do not fit the fused step kernel (no peer exchange)");
  if (!h->xchg) {
    h->xchg_stride = ((h->Pp + h->Pv + 2 * B200RL_N_SCALARS + 31) / 32) * 32;
    // a dedicated allocation (cudaIpcGetMemHandle exports whole allocations)
    B200RL_CUDA(cudaMalloc(reinterpret_cast<void**>(&h->xchg), (size_t)(2 * h->xchg_stride) * 4 + 64));
    B200RL_CUDA(cudaMemset(h->xchg, 0, (size_t)(2 * h->xchg_stride) * 4 + 64));
    h->allocs.push_back(h->xchg);
    if (dev_alloc(h, &h->peers_dev, RA3_MAX_WORLD)) return 1;
    if (dev_alloc(h, &h->done_counter, 4)) return 1;
  }
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  cudaIpcMemHandle_t hd;
  B200RL_CUDA(cudaIpcGetMemHandle(&hd, h->xchg));
  memcpy(handle64, &hd, 64);
  *local_ptr = h->xchg;
  return 0;
}

extern "C" int b200rl_ipc_open(const void* handle64, void** ptr) {
  B200RL_REQUIRE(handle64 && ptr, "ipc_open: NULL argument");
  cudaIpcMemHandle_t hd;
  memcpy(&hd, handle64, 64);
  const cudaError_t e = cudaIpcOpenMemHandle(ptr, hd, cudaIpcMemLazyEnablePeerAccess);
  if (e != cudaSuccess) {
    (void)cudaGetLastError();  // the caller falls back to the collective path: do not leave the error for a later launch check
    set_error("cudaIpcOpenMemHandle failed: %s", cudaGetErrorString(e));
    return 1;
  }
  return 0;
}

extern "C" int b200rl_ipc_close(void* ptr) {
  if (ptr && cudaIpcCloseMemHandle(ptr) != cudaSuccess) {
    (void)cudaGetLastError();
    set_error("cudaIpcCloseMemHandle failed");
    return 1;
  }
  return 0;
}

extern "C" int b200rl_onpolicy_comm_attach(b200rl_onpolicy* h, int32_t rank, int32_t world, void* const* peer_ptrs) {
  B200RL_REQUIRE(h && peer_ptrs && h->xchg, "comm_attach: call comm_export first");
  B200RL_REQUIRE(world >= 1 && world <= RA3_MAX_WORLD && rank >= 0 && rank < world, "comm_attach: bad rank / world size");
  B200RL_REQUIRE(peer_ptrs[rank] == h->xchg, "comm_attach: peer_ptrs[rank] must be this engine's own buffer");
  B200RL_CUDA(cudaMemcpy(h->peers_dev, peer_ptrs, (size_t)world * sizeof(void*), cudaMemcpyHostToDevice));
  // every rank (re)starts its sequence at 1; stale sequence words cannot match before they are overwritten
  B200RL_CUDA(cudaMemset(reinterpret_cast<char*>(h->xchg) + (size_t)(2 * h->xchg_stride) * 4, 0, 64));
  h->comm_world = world;
  h->comm_rank = rank;
  h->comm_seq = 0;
  return 0;
}

extern "C" int b200rl_onpolicy_scalar_history(b200rl_onpolicy* h, double* out, int32_t max_slots, int32_t* n_slots) {
  B200RL_REQUIRE(h && out && n_slots && max_slots >= 0, "scalar_history: bad argument");
  const int n = h->last_slots < max_slots ? h->last_slots : max_slots;
  if (n > 0) memcpy(out, h->h_slots, (size_t)n * B200RL_N_SCALARS * sizeof(double));
  *n_slots = h->last_slots;
  return 0;
}

// Single stages on the loaded batch, for kernel-level timing (bench.py roofline) and ncu captures.
extern "C" int b200rl_onpolicy_run_stage(b200rl_onpolicy* h, const char* stage, const b200rl_ppo_hparams* hp,
                                         void* stream) {
  B200RL_REQUIRE(h && stage && hp, "run_stage: NULL argument");
  B200RL_REQUIRE(h->n_rows > 0, "run_stage: no batch loaded");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int64_t n_glob = hp->n_global_rows > 0 ? hp->n_global_rows : h->n_rows;
  if (strcmp(stage, "values") == 0)
    return launch_fused(h, h->cfg.value, B200RL_LOSS_EVAL, B200RL_DIST_NONE, h->val, h->obs, h->n_rows, h->n_rows, 0.0,
                        false, false, h->values, false, nullptr, s);
  if (strcmp(stage, "preamble") == 0) return run_preamble(h, hp, nullptr, nullptr, s);
  if (strcmp(stage, "scan") == 0)
    return b200rl_gae_scan(h->rew, h->cfg.rewards_f64, h->values, h->last_values, h->off, h->done, h->n_rows, h->n_ep,
                           hp->gamma, hp->gae_lambda, h->adv_raw, h->ret, h->adv_stats, h->scan_ws, h->scan_ws_bytes, s);
  if (strcmp(stage, "old_logp") == 0)
    return launch_fused(h, h->cfg.policy, B200RL_LOSS_EVAL, h->cfg.dist, h->old_pol, h->obs, h->n_rows, n_glob, 0.0,
                        false, false, h->old_logp, false, nullptr, s);
  // the gradient stages leave device_view("policy_grad" / "value_grad") on the buffer they write
  if (strcmp(stage, "policy_grad") == 0) {
    h->last_fused = 0;
    if (launch_fused(h, h->cfg.policy, B200RL_LOSS_PPO_CLIP, h->cfg.dist, h->pol, h->obs, h->n_rows, n_glob,
                     hp->clip_range, true, true, nullptr, true, nullptr, s)) return 1;
    return b200rl_reduce_partials(h->partials, h->scalar_partials, b200rl_mlp_grid(&h->cfg.policy, h->n_rows, 1),
                                  h->Pp, h->pol_grad, h->slots, 0, nullptr, s);
  }
  if (strcmp(stage, "policy_grad_kernel") == 0)
    return launch_fused(h, h->cfg.policy, B200RL_LOSS_PPO_CLIP, h->cfg.dist, h->pol, h->obs, h->n_rows, n_glob,
                        hp->clip_range, true, true, nullptr, true, nullptr, s);
  if (strcmp(stage, "value_grad") == 0) {
    h->last_fused = 0;
    if (launch_fused(h, h->cfg.value, B200RL_LOSS_MSE, B200RL_DIST_NONE, h->val, h->obs, h->n_rows, n_glob, 0.0, false,
                     false, nullptr, true, nullptr, s)) return 1;
    return b200rl_reduce_partials(h->partials, h->scalar_partials, b200rl_mlp_grid(&h->cfg.value, h->n_rows, 1), h->Pv,
                                  h->val_grad, h->slots, 0, nullptr, s);
  }
  if (strcmp(stage, "value_grad_kernel") == 0)
    return launch_fused(h, h->cfg.value, B200RL_LOSS_MSE, B200RL_DIST_NONE, h->val, h->obs, h->n_rows, n_glob, 0.0,
                        false, false, nullptr, true, nullptr, s);
  const bool fused_one = strcmp(stage, "fused_step_kernel_policy") == 0 || strcmp(stage, "fused_step_kernel_value") == 0;
  if (strcmp(stage, "pack_obs") == 0 || strcmp(stage, "fused_step_kernel") == 0 || strcmp(stage, "fused_step") == 0 ||
      fused_one) {
    B200RL_REQUIRE(h->fused_ok, "run_stage: the networks do not fit the fused step kernel");
    if (strcmp(stage, "pack_obs") == 0) {
      B200RL_CUDA(cudaMemsetAsync(h->trip, 0, 4 * sizeof(float), s));
      if (!h->hints_valid && b200rl_absmax_cols(h->obs, h->n_rows, h->obs_dim, h->absmax, s)) return 1;
      return launch_pack_obs(h->obs, h->n_rows, h->obs_dim, h->absmax, h->ximg, h->xscale, h->trip, s);
    }
    if (fused_one) {  // the step kernel with one network running: what each network's share of the launch costs
      Tc3Args k = tc3_args(h, hp, n_glob);
      k.run_policy = stage[18] == 'p';
      k.run_value = stage[18] == 'v';
      return launch_mlp_tc3(k, s);
    }
    // one iteration of both loops on the packed observations ("pack_obs" and "preamble" first): the step kernel
    // alone, or with the reduction of its partial rows (mode 1: parameters stay as they are)
    if (launch_mlp_tc3(tc3_args(h, hp, n_glob), s)) return 1;
    if (strcmp(stage, "fused_step_kernel") == 0) return 0;
    Ra3Args a;
    memset(&a, 0, sizeof(a));
    a.mode = 1;
    a.partials = h->partials;
    a.scalar_partials = h->scalar_partials;
    a.rows = 2 * tc_grid(h->n_rows);
    a.P[0] = h->Pp;
    a.P[1] = h->Pv;
    a.grad = h->grad_all;
    a.run_policy = a.run_value = 1;
    h->last_fused = 1;
    return launch_reduce_adam3(a, s);
  }
  if (strcmp(stage, "fvp") == 0) {  // one Fisher-vector product (kernel + fixed-order reduction) on the current direction
    if (ensure_trpo(h)) return 1;
    return launch_fvp(h, h->cg_p, h->cg_z, n_glob, s);
  }
  set_error("run_stage: unknown stage '%s'", stage);
  return 2;
}
