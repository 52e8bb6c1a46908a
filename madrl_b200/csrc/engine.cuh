// Host-side engine core shared by the three env families (waterworld.cu, pursuit.cu, hostage.cu).
//
// A family handle (madrl_ww, madrl_pursuit, madrl_hostage: opaque to C) derives from EngineCore and
// adds `cfg` (its config struct), `lay` (its state layout), a `step_bytes()` member giving the bytes of
// one lockstep step of each trajectory tensor, and whatever else is its own.  The `madrl_<family>_*`
// entry points forward to the functions below for everything that is not family-specific.
#pragma once
#include <math.h>
#include <cmath>
#include <mutex>
#include <new>

#include "common.cuh"
#include "host_pipeline.cuh"

namespace madrl {

struct EngineCore {
  char* state = nullptr;     // state blob (state_layout's total_bytes)
  bool owns_state = false;   // cudaMalloc'ed by create (not the caller's)
  int device = 0, sms = 0;
  int blocks_per_sm = 0;     // set_launch override of resident blocks per SM (0 = the family's default)
  HostPipe pipe;             // staging + streams of the host-buffer entry points (lazily created)
  void* term_obs = nullptr;  // set_terminal_obs (NULL = off)
  int obs_format = MADRL_OBS_NATIVE;   // set_obs_format: element type of every observation buffer
  int obs_cache = MADRL_OBS_CACHE_STREAM;   // set_obs_cache: L2 policy of the rollouts' observation stores

  // bytes of one observation element: `native` (the handle's real) or 2 (bfloat16)
  size_t obs_elem_bytes(size_t native) const { return obs_format == MADRL_OBS_BF16 ? 2 : native; }
};

// What the frame kernels of render.cu read of a family handle, which only its own source file can see into:
// the config, the state layout and the state blob.  Defined next to each family's handle.
template <class Cfg, class Layout>
struct HandleView {
  const Cfg* cfg;
  const Layout* lay;
  const char* state;
};
HandleView<madrl_ww_config, madrl_ww_layout> handle_view(const madrl_ww* h);
HandleView<madrl_pursuit_config, madrl_pursuit_layout> handle_view(const madrl_pursuit* h);
HandleView<madrl_hostage_config, madrl_hostage_layout> handle_view(const madrl_hostage* h);

template <class H>
int engine_destroy(H* h) {
  if (!h) return MADRL_OK;
  if (h->owns_state && h->state) cudaFree(h->state);
  h->pipe.destroy();
  delete h;
  return MADRL_OK;
}

// Record the current device and its SM count, take the caller's state blob (or cudaMalloc one of
// `bytes`) and zero it.
inline int engine_init(EngineCore* h, void* state_dev, size_t bytes) {
  cudaError_t e = cudaGetDevice(&h->device);
  if (e != cudaSuccess) { set_error("cudaGetDevice: %s", cudaGetErrorString(e)); return MADRL_ECUDA; }
  h->sms = sm_count(h->device);
  if (h->sms <= 0) return MADRL_ECUDA;
  if (state_dev) {
    h->state = (char*)state_dev;
  } else {
    e = cudaMalloc((void**)&h->state, bytes);
    if (e != cudaSuccess) { set_error("cudaMalloc(%zu): %s", bytes, cudaGetErrorString(e)); return MADRL_ENOMEM; }
    h->owns_state = true;
  }
  e = cudaMemset(h->state, 0, bytes);
  if (e != cudaSuccess) { set_error("cudaMemset: %s", cudaGetErrorString(e)); return MADRL_ECUDA; }
  return MADRL_OK;
}

// `*_create`: validate and lay out the config (the family's `state_layout`), engine_init, then
// `init(h)` uploads the family's constant tables.  On any failure the half-built handle is destroyed.
template <class H, class Cfg, class Layout, class Init>
int engine_create(const Cfg* c, void* state_dev, H** out, int (*state_layout)(const Cfg*, Layout*), Init init) {
  MADRL_REQUIRE(out != nullptr, "out is NULL");
  Layout lay;
  int rc = state_layout(c, &lay);
  if (rc) return rc;
  H* h = new (std::nothrow) H();
  if (!h) return MADRL_ENOMEM;
  h->cfg = *c;
  h->lay = lay;
  rc = engine_init(h, state_dev, lay.total_bytes);
  if (rc == MADRL_OK) rc = init(h);
  if (rc) {
    engine_destroy(h);
    return rc;
  }
  *out = h;
  return MADRL_OK;
}

// seed(): new key, draw counters reset to 0.
template <class H>
int engine_seed(H* h, uint64_t seed, void* stream) {
  MADRL_REQUIRE(h != nullptr, "handle is NULL");
  h->cfg.seed = seed;
  MADRL_CUDA_CHECK(cudaMemsetAsync(h->state + h->lay.rng_counter, 0, 8 * (size_t)h->cfg.n_envs, (cudaStream_t)stream));
  return MADRL_OK;
}

inline int engine_set_terminal_obs(EngineCore* h, void* term_obs_dev) {
  MADRL_REQUIRE(h != nullptr, "handle is NULL");
  h->term_obs = term_obs_dev;
  return MADRL_OK;
}

inline int engine_set_obs_format(EngineCore* h, int format, bool fp64) {
  MADRL_REQUIRE(h != nullptr, "handle is NULL");
  MADRL_REQUIRE(format == MADRL_OBS_NATIVE || format == MADRL_OBS_BF16, "unknown observation format %d", format);
  MADRL_REQUIRE(!(format == MADRL_OBS_BF16 && fp64), "bfloat16 observations need an fp32 handle (fp64 = 0)");
  h->obs_format = format;
  return MADRL_OK;
}

inline int engine_set_obs_cache(EngineCore* h, int mode, bool fp64) {
  MADRL_REQUIRE(h != nullptr, "handle is NULL");
  MADRL_REQUIRE(mode == MADRL_OBS_CACHE_STREAM || mode == MADRL_OBS_CACHE_KEEP, "unknown observation cache mode %d", mode);
  MADRL_REQUIRE(!(mode == MADRL_OBS_CACHE_KEEP && fp64), "MADRL_OBS_CACHE_KEEP needs an fp32 handle (fp64 = 0)");
  h->obs_cache = mode;
  return MADRL_OK;
}

// `warps_per_block` is range-checked for ABI stability and otherwise ignored: blocks are one warp.
inline int engine_set_launch(EngineCore* h, int warps_per_block, int blocks_per_sm) {
  MADRL_REQUIRE(h != nullptr, "handle is NULL");
  MADRL_REQUIRE(warps_per_block >= 0 && warps_per_block <= 4, "warps_per_block must be in [0,4]");
  MADRL_REQUIRE(blocks_per_sm >= 0 && blocks_per_sm <= 32, "blocks_per_sm must be in [0,32]");
  h->blocks_per_sm = blocks_per_sm;
  return MADRL_OK;
}

// One launch of a warp-per-env kernel over E envs: one 32-thread block per env, or a single
// persistent wave (SMs x resident blocks per SM, capped by set_launch, else by the family's
// `default_blocks_per_sm` when that is not 0) whose warps loop over the envs.  `grid_out`: the launch's grid.
template <class Kernel, class Params>
int engine_launch(const EngineCore* h, Kernel kfn, size_t smem, int E, cudaStream_t stream, const Params& p,
                  int default_blocks_per_sm = 0, int* grid_out = nullptr) {
  if (smem > 48 * 1024)
    MADRL_CUDA_CHECK(cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int resident = 0;
  MADRL_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident, kfn, 32, smem));
  if (resident < 1) resident = 1;
  const int cap = h->blocks_per_sm > 0 ? h->blocks_per_sm : default_blocks_per_sm;
  if (cap > 0 && cap < resident) resident = cap;
  int grid = E;
  if (grid > h->sms * resident) grid = h->sms * resident;
  MADRL_LAUNCH(kfn, grid, 32, smem, stream, p);
  g_launches.fetch_add(1);   // under stream capture: counted once, when recorded, not at each graph replay
  MADRL_CUDA_CHECK(cudaGetLastError());
  if (grid_out != nullptr) *grid_out = grid;
  return MADRL_OK;
}

// A family's launch log (madrl_ww_launch_log, madrl_pursuit_launch_log, madrl_hostage_launch_log): while it is on,
// every launch of the family's kernel appends the template arguments of the instantiation it ran and its grid, so
// that a test can check which kernel a launch path takes without a profiler.  Off, the default, it costs one
// relaxed load per launch.  `Fields` int32 per record.
template <int Fields>
struct LaunchLog {
  static constexpr int kMax = 4096;
  std::atomic<bool> on{false};
  std::mutex mu;
  int32_t recs[kMax][Fields];
  int n = 0;   // launches since the log was last read, including those past kMax

  void add(const int32_t (&rec)[Fields]) {
    if (!on.load(std::memory_order_relaxed)) return;
    std::lock_guard<std::mutex> lock(mu);
    if (n < kMax)
      for (int i = 0; i < Fields; ++i) recs[n][i] = rec[i];
    ++n;
  }

  // Copies the first min(n, max_records, kMax) records out, clears the log and turns it on or off -> n.
  int read(int enable, int32_t* records, int max_records) {
    MADRL_REQUIRE(max_records >= 0 && (max_records == 0 || records != nullptr), "bad launch-log buffer");
    std::lock_guard<std::mutex> lock(mu);
    const int got = n, keep = n < kMax ? n : kMax;
    for (int r = 0; r < keep && r < max_records; ++r)
      for (int i = 0; i < Fields; ++i) records[r * Fields + i] = recs[r][i];
    n = 0;
    on.store(enable != 0, std::memory_order_relaxed);
    return got;
  }
};

// `*_reset_host`: `reset(mask_dev, obs_dev)` is the family's device-pointer reset on the legacy default
// stream; the mask and the observations go through the staging buffer.
template <class H, class Reset>
int engine_reset_host(H* h, const uint8_t* mask_host, void* obs_host, Reset reset) {
  MADRL_REQUIRE(h != nullptr && obs_host != nullptr, "handle/obs is NULL");
  const StepBytes sb = h->step_bytes();
  const size_t E = sb.done, obs_b = sb.obs;   // one done byte per env; one step of observations
  const size_t mask_off = align_up(obs_b, 256);
  int rc = h->pipe.ensure(mask_off + E);
  if (rc) return rc;
  char* st = (char*)h->pipe.stage;
  uint8_t* mask_dev = nullptr;
  if (mask_host) {
    mask_dev = (uint8_t*)(st + mask_off);
    MADRL_CUDA_CHECK(cudaMemcpyAsync(mask_dev, mask_host, E, cudaMemcpyHostToDevice, 0));
    // rows of unmasked envs must survive: seed the staging buffer with the caller's obs
    MADRL_CUDA_CHECK(cudaMemcpyAsync(st, obs_host, obs_b, cudaMemcpyHostToDevice, 0));
  }
  rc = reset(mask_dev, st);
  if (rc) return rc;
  MADRL_CUDA_CHECK(cudaMemcpyAsync(obs_host, st, obs_b, cudaMemcpyDeviceToHost, 0));
  MADRL_CUDA_CHECK(cudaStreamSynchronize(0));
  return MADRL_OK;
}

// `*_rollout_host2`: `rollout(Tc, act, obs, rew, done, info, stream)` is the family's device-pointer
// rollout of Tc steps, run chunk by chunk through host_rollout.
template <class H, class Rollout>
int engine_rollout_host(H* h, int T, const void* act_h, void* obs_h, void* rew_h, void* done_h, void* info_h,
                        int flags, Rollout rollout) {
  MADRL_REQUIRE(h != nullptr, "handle is NULL");
  MADRL_REQUIRE(T >= 1, "T must be >= 1");
  MADRL_REQUIRE(act_h && obs_h && rew_h && done_h && info_h, "NULL trajectory buffer");
  MADRL_REQUIRE((flags & ~MADRL_HOST_OBS_LAST) == 0, "unknown flags %d", flags);
  void* const keep = h->term_obs;    // chunk-relative offsets: the side tensor is a device-API feature
  h->term_obs = nullptr;
  const int rc = host_rollout(h->pipe, T, h->step_bytes(), act_h, obs_h, rew_h, done_h, info_h,
                              flags & MADRL_HOST_OBS_LAST, rollout);
  h->term_obs = keep;
  return rc;
}

// Largest representable t with the double sqrt(t) <= thr_d: for a `real` d2, `sqrt(d2) <= thr_d` (what scipy's
// cdist + `<=` computes in the reference, in double) is then exactly `d2 <= t`.  The search is in double against
// the double threshold: a float sqrtf(t) against (float)thr_d rounds twice and admits up to two ulps more.
template <typename real>
real exact_sq_threshold(double thr_d) {
  real t = (real)(thr_d * thr_d);
  const real up = (real)INFINITY, dn = -(real)INFINITY;
  while (std::sqrt((double)t) <= thr_d) t = std::nextafter(t, up);
  while (std::sqrt((double)t) > thr_d) t = std::nextafter(t, dn);
  return t;
}

// The largest `real` at or below thr_d: for a `real` x, `x > round_down(thr_d)` is exactly `x > thr_d` (and `<=`
// likewise), the comparison the reference makes in double.  Rounding to nearest can land above thr_d
// ((float)0.2 = 0.20000000298), and an operand equal to it would then be sensed where the reference rejects it.
template <typename real>
real round_down(double thr_d) {
  const real t = (real)thr_d;
  return (double)t > thr_d ? std::nextafter(t, -(real)INFINITY) : t;
}

// Sensor unit vectors of the continuous families (Waterworld, Hostage): angles = linspace(0, 2pi, K+1)[:-1]
// (waterworld.py:29-31, hostage.py:27-29), stored at the layout's `sensors` offset as a cos row and a
// sin row of the handle's real type.
template <typename real>
int upload_sensor_table(char* dst, int K) {
  real* tab = new (std::nothrow) real[2 * (size_t)K];
  if (!tab) return MADRL_ENOMEM;
  const double step = (2.0 * M_PI - 0.0) / (double)K;
  for (int k = 0; k < K; ++k) {
    const double a = (double)k * step + 0.0;
    tab[k] = (real)cos(a);
    tab[K + k] = (real)sin(a);
  }
  cudaError_t e = cudaMemcpy(dst, tab, sizeof(real) * 2 * K, cudaMemcpyHostToDevice);
  delete[] tab;
  MADRL_CUDA_CHECK(e);
  return MADRL_OK;
}

template <class H>
int upload_sensors(H* h) {
  char* dst = h->state + h->lay.sensors;
  return h->cfg.fp64 ? upload_sensor_table<double>(dst, h->cfg.n_sensors) : upload_sensor_table<float>(dst, h->cfg.n_sensors);
}

}  // namespace madrl
