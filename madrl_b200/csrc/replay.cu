// rllab's DDPG replay pool on the device (rllab/rllab/algos/ddpg.py:85-145 MAReplayPool, fed by the decentralized
// branch of DDPG.train, :285-353).  A rollout's transitions are compacted, in (t, env, agent) order, into a ring of
// max_pool_size slots, and minibatches are gathered from it at Philox-drawn slots.  Every counter lives in device
// memory (ctl[4] = top, bottom, size, draw counter), so an add and a sample make no host synchronisation and can be
// captured in a CUDA graph.
//
//   replay_plan_kernel     one thread per env walks `done` with the path length and timestep counters; transition
//                          (t, e) is dropped at a horizon cut (the path reached max_path_length and the env did not
//                          terminate by itself) unless include_horizon.  Per step, a ballot gives each kept env its
//                          rank in its warp and each warp its count.
//   replay_scan_kernel     one block: exclusive scan of the [T][warps] counts in step-major order -> the index of
//                          each warp's first kept transition, the total K, the first index that lands (K may exceed
//                          the pool: only the last max_pool_size land), the first step with a landing transition,
//                          and the new top / bottom / size (add_sample's rule, :106-116).
//   replay_insert_kernel   one warp per source row u = (t', e, a), t' = -1 .. T-1 (obs_before, then obs[t']): the row
//                          is read once and written as the next observation of transition (t', e, a), unless done,
//                          and as the observation of (t'+1, e, a), each only where that transition lands.  A done
//                          step's next observation is term[t'].  The warp of u = t also writes transition t's action,
//                          scaled reward and terminal flag.  Warps start at the first step that lands, so a rollout
//                          far larger than the pool reads only what it keeps.
//   replay_sample_kernel   one warp per drawn row: slot = mulhi64(philox64(seed, counter + r), size - 1), i.e.
//                          uniform over [0, size - 1), which is the set MAReplayPool.random_batch's rejection loop
//                          (:118-128) accepts; gathers 2 D + Ad + 2 words.  replay_advance_kernel moves the counter.
// Observation rows are float32 or bfloat16 (O = uint16_t bits); they are moved, never converted, in the widest
// word (16, 8, 4 or 2 bytes) that the row length and every row pointer allow.  Slots and row offsets are 64-bit.
#include <algorithm>
#include <initializer_list>

#include "common.cuh"
#include "philox.cuh"

namespace madrl {

enum { kCtlTop = 0, kCtlBottom = 1, kCtlSize = 2, kCtlDraws = 3 };
// workspace info words: top before the add, first landing index, first step with a landing transition, K
enum { kInfoTop = 0, kInfoFirst = 1, kInfoStep = 2, kInfoK = 3 };
constexpr uint32_t kReplayTag = 2;   // Philox stream family of the sampler (0 env dynamics, 1 benchmark actions)
constexpr int kScanThreads = 1024;

__host__ __device__ __forceinline__ uint64_t mulhi64(uint64_t a, uint64_t b) {
  const uint64_t a_lo = (uint32_t)a, a_hi = a >> 32, b_lo = (uint32_t)b, b_hi = b >> 32;
  const uint64_t lo_lo = a_lo * b_lo, hi_lo = a_hi * b_lo, lo_hi = a_lo * b_hi, hi_hi = a_hi * b_hi;
  const uint64_t mid = (lo_lo >> 32) + (uint32_t)hi_lo + lo_hi;
  return hi_hi + (hi_lo >> 32) + (mid >> 32);
}

// The slot of draw n: a 64-bit Philox word scaled into [0, n_slots) by its multiply-high (bias < n_slots / 2^64).
__host__ __device__ __forceinline__ uint64_t replay_slot(uint64_t seed, uint64_t n, uint64_t n_slots) {
  const Philox4 b = philox4x32_10((uint32_t)n, (uint32_t)(n >> 32), 0u, kReplayTag, (uint32_t)seed,
                                  (uint32_t)(seed >> 32));
  return mulhi64(((uint64_t)b.w[1] << 32) | b.w[0], n_slots);
}

__global__ void replay_plan_kernel(int T, int E, const uint8_t* __restrict__ done, const int32_t* __restrict__ path_len0,
                                   const int32_t* __restrict__ timestep0, int max_path_length, int timestep_limit,
                                   int include_horizon, int8_t* __restrict__ rank, int32_t* __restrict__ wcnt) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if ((e & ~31) >= E) return;   // whole warps only: the ballot below needs every lane
  const bool live = e < E;
  const int lane = threadIdx.x & 31, W = (E + 31) / 32, w = e >> 5;
  int pl = live ? path_len0[e] : 0, ts = live ? timestep0[e] : 0;
  for (int t = 0; t < T; ++t) {
    bool keep = false;
    if (live) {
      const bool d = __ldcs(done + (size_t)t * E + e) != 0;
      ++pl;
      ++ts;
      // ddpg.py:310: a horizon cut is a done step at the path-length limit of an env that did not end by itself
      const bool cut = d && max_path_length > 0 && pl >= max_path_length && ts < timestep_limit;
      keep = !cut || include_horizon;
      if (d) pl = ts = 0;
    }
    const unsigned m = __ballot_sync(FULL_MASK, keep);
    if (live) rank[(size_t)t * E + e] = keep ? (int8_t)__popc(m & ((1u << lane) - 1u)) : (int8_t)-1;
    if (lane == 0) wcnt[(size_t)t * W + w] = __popc(m);
  }
}

__global__ void __launch_bounds__(kScanThreads) replay_scan_kernel(int W, int A, size_t cells, int64_t M,
                                                                   const int32_t* __restrict__ wcnt,
                                                                   int64_t* __restrict__ wbase,
                                                                   int64_t* __restrict__ ctl, int64_t* __restrict__ info) {
  __shared__ int64_t part[kScanThreads];
  __shared__ int64_t first_step[kScanThreads];
  const int i = threadIdx.x;
  const size_t per = (cells + kScanThreads - 1) / kScanThreads;
  const size_t lo = (size_t)i * per < cells ? (size_t)i * per : cells, hi = lo + per < cells ? lo + per : cells;
  int64_t s = 0;
  for (size_t c = lo; c < hi; ++c) s += wcnt[c];
  part[i] = s;
  __syncthreads();
  for (int o = 1; o < kScanThreads; o <<= 1) {   // inclusive Hillis-Steele scan of the per-thread sums
    const int64_t v = i >= o ? part[i - o] : 0;
    __syncthreads();
    part[i] += v;
    __syncthreads();
  }
  const int64_t K = part[kScanThreads - 1] * A;   // every kept (t, e) adds its A agents' transitions
  const int64_t first = K > M ? K - M : 0;   // transitions below `first` are overwritten within this add
  int64_t run = part[i] - s, step = INT64_MAX;
  for (size_t c = lo; c < hi; ++c) {
    const int32_t n = wcnt[c];
    wbase[c] = run;
    if (n > 0 && (run + n) * A > first && step == INT64_MAX) step = (int64_t)(c / W);
    run += n;
  }
  first_step[i] = step;
  __syncthreads();
  if (i == 0) {
    int64_t t0 = INT64_MAX;
    for (int k = 0; k < kScanThreads; ++k) t0 = first_step[k] < t0 ? first_step[k] : t0;
    const int64_t top = ctl[kCtlTop], bottom = ctl[kCtlBottom], size = ctl[kCtlSize];
    info[kInfoTop] = top;
    info[kInfoFirst] = first;
    info[kInfoStep] = t0;
    info[kInfoK] = K;
    // add_sample K times: top advances by K, bottom by every add made while the pool is full
    const int64_t over = size + K > M ? size + K - M : 0;
    ctl[kCtlTop] = (top + K) % M;
    ctl[kCtlBottom] = (bottom + over) % M;
    ctl[kCtlSize] = size + K < M ? size + K : M;
  }
}

// The pool slot of transition (t, e, a), or -1 when it is dropped or overwritten within this add.
__device__ __forceinline__ int64_t landing_slot(int t, int e, int a, int E, int A, int W, const int8_t* __restrict__ rank,
                                                const int64_t* __restrict__ wbase, int64_t top, int64_t first,
                                                int64_t M) {
  const int r = rank[(size_t)t * E + e];
  if (r < 0) return -1;
  const int64_t j = (wbase[(size_t)t * W + (e >> 5)] + r) * A + a;
  return j < first ? -1 : (top + j) % M;
}

// V: the word the rows are moved in (float4, float2, uint32_t, uint16_t); DV = row length in words.
template <typename V>
__global__ void replay_insert_kernel(int T, int E, int A, int DV, int Ad, int64_t M, const V* __restrict__ obs,
                                     const float* __restrict__ act, const float* __restrict__ rew,
                                     const uint8_t* __restrict__ done, const V* __restrict__ obs_before,
                                     const V* __restrict__ term, double scale_reward, const int8_t* __restrict__ rank,
                                     const int64_t* __restrict__ wbase, const int64_t* __restrict__ info,
                                     V* __restrict__ pool_obs, V* __restrict__ pool_next, float* __restrict__ pool_act,
                                     float* __restrict__ pool_rew, uint8_t* __restrict__ pool_term) {
  const int64_t t_first = info[kInfoStep];
  if (t_first == INT64_MAX) return;   // nothing lands
  const int64_t top = info[kInfoTop], first = info[kInfoFirst];
  const int W = (E + 31) / 32, lane = threadIdx.x & 31;
  const size_t EA = (size_t)E * A, rows = (size_t)(T + 1) * EA;
  const size_t warps = (size_t)gridDim.x * (blockDim.x / 32);
  for (size_t row = (size_t)t_first * EA + ((size_t)blockIdx.x * blockDim.x + threadIdx.x) / 32; row < rows;
       row += warps) {
    const int u = (int)(row / EA);   // source step + 1: u = 0 is obs_before
    const size_t ea = row % EA;
    const int e = (int)(ea / A), a = (int)(ea % A);
    // transition u - 1 takes this row as its next observation (or term[u - 1] when done); transition u as its
    // observation
    int64_t s_next = -1, s_obs = -1;
    bool d_prev = false;
    if (u >= 1) {
      s_next = landing_slot(u - 1, e, a, E, A, W, rank, wbase, top, first, M);
      d_prev = done[(size_t)(u - 1) * E + e] != 0;
    }
    if (u < T) s_obs = landing_slot(u, e, a, E, A, W, rank, wbase, top, first, M);
    const V* src = u == 0 ? obs_before + ea * DV : obs + ((size_t)(u - 1) * EA + ea) * DV;
    V* dn = (s_next >= 0 && !d_prev) ? pool_next + (size_t)s_next * DV : nullptr;
    V* dobs = s_obs >= 0 ? pool_obs + (size_t)s_obs * DV : nullptr;
    if (dn || dobs) {
      for (int k = lane; k < DV; k += 32) {
        const V v = __ldcs(src + k);
        if (dn) dn[k] = v;
        if (dobs) dobs[k] = v;
      }
    }
    if (s_next >= 0 && d_prev) {
      const V* ts = term + ((size_t)(u - 1) * EA + ea) * DV;
      V* dt = pool_next + (size_t)s_next * DV;
      for (int k = lane; k < DV; k += 32) dt[k] = __ldcs(ts + k);
    }
    if (s_obs >= 0) {
      const size_t k = (size_t)u * EA + ea;
      for (int c = lane; c < Ad; c += 32) pool_act[(size_t)s_obs * Ad + c] = __ldcs(act + k * Ad + c);
      if (lane == 0) {
        pool_rew[s_obs] = (float)((double)__ldcs(rew + k) * scale_reward);
        pool_term[s_obs] = done[(size_t)u * E + e] != 0 ? 1 : 0;
      }
    }
  }
}

template <typename V>
__global__ void replay_sample_kernel(size_t rows, int DV, int Ad, int64_t M, uint64_t seed,
                                     const V* __restrict__ pool_obs, const V* __restrict__ pool_next,
                                     const float* __restrict__ pool_act, const float* __restrict__ pool_rew,
                                     const uint8_t* __restrict__ pool_term, const int64_t* __restrict__ ctl,
                                     int64_t* __restrict__ idx, V* __restrict__ obs_out, V* __restrict__ next_out,
                                     float* __restrict__ act_out, float* __restrict__ rew_out,
                                     uint8_t* __restrict__ term_out) {
  const size_t r = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) / 32;
  if (r >= rows) return;
  const int lane = threadIdx.x & 31;
  const int64_t size = ctl[kCtlSize];
  // [0, size - 1), and slot 0 for a pool of at most one transition: the gather stays inside the pool
  const uint64_t n_slots = size > 1 ? (uint64_t)(size - 1) : 1;
  const int64_t s = (int64_t)replay_slot(seed, (uint64_t)ctl[kCtlDraws] + r, n_slots) % M;
  const V* so = pool_obs + (size_t)s * DV;
  const V* sn = pool_next + (size_t)s * DV;
  V* oo = obs_out + r * DV;
  V* on = next_out + r * DV;
  for (int k = lane; k < DV; k += 32) {
    __stcs(oo + k, so[k]);
    __stcs(on + k, sn[k]);
  }
  for (int c = lane; c < Ad; c += 32) __stcs(act_out + r * Ad + c, pool_act[(size_t)s * Ad + c]);
  if (lane == 0) {
    idx[r] = s;
    rew_out[r] = pool_rew[s];
    term_out[r] = pool_term[s];
  }
}

__global__ void replay_advance_kernel(int64_t* __restrict__ ctl, int64_t rows) {
  if (threadIdx.x == 0) ctl[kCtlDraws] += rows;
}

static size_t ws_rank_bytes(int T, int E) { return align_up((size_t)T * E, 16); }
static size_t ws_cnt_bytes(int T, int E) { return align_up((size_t)T * ((E + 31) / 32) * 4, 16); }

static int workspace_size(int T, int E, size_t* bytes) {
  MADRL_REQUIRE(T >= 1 && E >= 1, "bad shape");
  MADRL_REQUIRE(bytes, "NULL pointer");
  *bytes = ws_rank_bytes(T, E) + ws_cnt_bytes(T, E) + (size_t)T * ((E + 31) / 32) * 8 + 4 * 8;
  return MADRL_OK;
}

static bool aligned(const void* p, size_t a) { return ((uintptr_t)p % a) == 0; }

// The widest word in which rows of `row_bytes` can be moved between all of `ptrs`.
static size_t row_word(size_t row_bytes, std::initializer_list<const void*> ptrs) {
  for (size_t w : {(size_t)16, (size_t)8, (size_t)4}) {
    bool ok = row_bytes % w == 0;
    for (const void* p : ptrs) ok = ok && aligned(p, w);
    if (ok) return w;
  }
  return 2;
}

template <typename O>
static int replay_add(int T, int E, int A, int D, int Ad, size_t M, const O* obs, const float* act, const float* rew,
                      const uint8_t* done, const O* obs_before, const O* term, const int32_t* path_len0,
                      const int32_t* timestep0, int max_path_length, int timestep_limit, int include_horizon,
                      double scale_reward, O* pool_obs, O* pool_next, float* pool_act, float* pool_rew,
                      uint8_t* pool_term, int64_t* ctl, void* ws, void* stream) {
  MADRL_REQUIRE(T >= 1 && E >= 1 && A >= 1 && D >= 1 && Ad >= 1, "bad shape");
  MADRL_REQUIRE(M >= 1 && M < ((size_t)1 << 62), "max_pool_size must be in [1, 2^62), got %zu", M);
  MADRL_REQUIRE(obs && act && rew && done && obs_before && term && path_len0 && timestep0 && pool_obs && pool_next &&
                pool_act && pool_rew && pool_term && ctl && ws, "NULL pointer");
  MADRL_REQUIRE(timestep_limit >= 1 && max_path_length >= 0, "bad timestep_limit / max_path_length");
  MADRL_REQUIRE(aligned(ws, 16), "workspace must be 16-byte aligned");
  cudaStream_t s = (cudaStream_t)stream;
  const int W = (E + 31) / 32;
  char* w = (char*)ws;
  int8_t* rank = (int8_t*)w;
  int32_t* wcnt = (int32_t*)(w + ws_rank_bytes(T, E));
  int64_t* wbase = (int64_t*)(w + ws_rank_bytes(T, E) + ws_cnt_bytes(T, E));
  int64_t* info = wbase + (size_t)T * W;
  MADRL_LAUNCH(replay_plan_kernel, (E + 127) / 128, 128, 0, s, T, E, done, path_len0, timestep0, max_path_length,
               timestep_limit, include_horizon, rank, wcnt);
  MADRL_LAUNCH(replay_scan_kernel, 1, kScanThreads, 0, s, W, A, (size_t)T * W, (int64_t)M, wcnt, wbase, ctl, info);
  const size_t row_bytes = (size_t)D * sizeof(O);
  const size_t word = row_word(row_bytes, {obs, obs_before, term, pool_obs, pool_next});
  const int DV = (int)(row_bytes / word);
  const size_t warps = (size_t)(T + 1) * E * A;
  int dev = 0;
  MADRL_CUDA_CHECK(cudaGetDevice(&dev));
  const size_t blocks = std::min((warps + 7) / 8, (size_t)sm_count(dev) * 8);   // 8 warps per block, grid-stride
#define MADRL_INSERT(V)                                                                                             \
  MADRL_LAUNCH(replay_insert_kernel<V>, (unsigned)blocks, 256, 0, s, T, E, A, DV, Ad, (int64_t)M, (const V*)obs,    \
               act, rew, done, (const V*)obs_before, (const V*)term, scale_reward, rank, wbase, info, (V*)pool_obs, \
               (V*)pool_next, pool_act, pool_rew, pool_term)
  switch (word) {
    case 16: MADRL_INSERT(float4); break;
    case 8: MADRL_INSERT(float2); break;
    case 4: MADRL_INSERT(uint32_t); break;
    default: MADRL_INSERT(uint16_t); break;
  }
#undef MADRL_INSERT
  g_launches.fetch_add(3);
  MADRL_CUDA_CHECK(cudaGetLastError());
  return MADRL_OK;
}

template <typename O>
static int replay_sample(int n, int B, int D, int Ad, size_t M, uint64_t seed, const O* pool_obs, const O* pool_next,
                         const float* pool_act, const float* pool_rew, const uint8_t* pool_term, int64_t* ctl,
                         int64_t* idx, O* obs_out, O* next_out, float* act_out, float* rew_out, uint8_t* term_out,
                         void* stream) {
  MADRL_REQUIRE(n >= 1 && B >= 1 && D >= 1 && Ad >= 1, "bad shape");
  MADRL_REQUIRE(M >= 1 && M < ((size_t)1 << 62), "max_pool_size must be in [1, 2^62), got %zu", M);
  MADRL_REQUIRE(pool_obs && pool_next && pool_act && pool_rew && pool_term && ctl && idx && obs_out && next_out &&
                act_out && rew_out && term_out, "NULL pointer");
  cudaStream_t s = (cudaStream_t)stream;
  const size_t rows = (size_t)n * B;
  const size_t row_bytes = (size_t)D * sizeof(O);
  const size_t word = row_word(row_bytes, {pool_obs, pool_next, obs_out, next_out});
  const int DV = (int)(row_bytes / word);
  const size_t blocks = (rows + 7) / 8;
  MADRL_REQUIRE(blocks < ((size_t)1 << 31), "too many rows for one launch");
#define MADRL_SAMPLE(V)                                                                                          \
  MADRL_LAUNCH(replay_sample_kernel<V>, (unsigned)blocks, 256, 0, s, rows, DV, Ad, (int64_t)M, seed,             \
               (const V*)pool_obs, (const V*)pool_next, pool_act, pool_rew, pool_term, ctl, idx, (V*)obs_out, \
               (V*)next_out, act_out, rew_out, term_out)
  switch (word) {
    case 16: MADRL_SAMPLE(float4); break;
    case 8: MADRL_SAMPLE(float2); break;
    case 4: MADRL_SAMPLE(uint32_t); break;
    default: MADRL_SAMPLE(uint16_t); break;
  }
#undef MADRL_SAMPLE
  MADRL_LAUNCH(replay_advance_kernel, 1, 32, 0, s, ctl, (int64_t)rows);
  g_launches.fetch_add(2);
  MADRL_CUDA_CHECK(cudaGetLastError());
  return MADRL_OK;
}

}  // namespace madrl

using namespace madrl;

extern "C" int madrl_replay_workspace_size(int T, int E, size_t* bytes) { return workspace_size(T, E, bytes); }

extern "C" int madrl_replay_add_f32(int T, int E, int A, int D, int Ad, size_t M, const float* obs_dev,
                                    const float* act_dev, const float* rew_dev, const uint8_t* done_dev,
                                    const float* obs_before_dev, const float* term_dev, const int32_t* path_len0_dev,
                                    const int32_t* timestep0_dev, int max_path_length, int timestep_limit,
                                    int include_horizon, double scale_reward, float* pool_obs_dev,
                                    float* pool_next_dev, float* pool_act_dev, float* pool_rew_dev,
                                    uint8_t* pool_term_dev, int64_t* ctl_dev, void* ws_dev, void* stream) {
  return replay_add(T, E, A, D, Ad, M, obs_dev, act_dev, rew_dev, done_dev, obs_before_dev, term_dev, path_len0_dev,
                    timestep0_dev, max_path_length, timestep_limit, include_horizon, scale_reward, pool_obs_dev,
                    pool_next_dev, pool_act_dev, pool_rew_dev, pool_term_dev, ctl_dev, ws_dev, stream);
}

extern "C" int madrl_replay_add_bf16(int T, int E, int A, int D, int Ad, size_t M, const void* obs_dev,
                                     const float* act_dev, const float* rew_dev, const uint8_t* done_dev,
                                     const void* obs_before_dev, const void* term_dev, const int32_t* path_len0_dev,
                                     const int32_t* timestep0_dev, int max_path_length, int timestep_limit,
                                     int include_horizon, double scale_reward, void* pool_obs_dev,
                                     void* pool_next_dev, float* pool_act_dev, float* pool_rew_dev,
                                     uint8_t* pool_term_dev, int64_t* ctl_dev, void* ws_dev, void* stream) {
  return replay_add(T, E, A, D, Ad, M, (const uint16_t*)obs_dev, act_dev, rew_dev, done_dev,
                    (const uint16_t*)obs_before_dev, (const uint16_t*)term_dev, path_len0_dev, timestep0_dev,
                    max_path_length, timestep_limit, include_horizon, scale_reward, (uint16_t*)pool_obs_dev,
                    (uint16_t*)pool_next_dev, pool_act_dev, pool_rew_dev, pool_term_dev, ctl_dev, ws_dev, stream);
}

extern "C" int madrl_replay_sample_f32(int n, int B, int D, int Ad, size_t M, uint64_t seed, const float* pool_obs_dev,
                                       const float* pool_next_dev, const float* pool_act_dev,
                                       const float* pool_rew_dev, const uint8_t* pool_term_dev, int64_t* ctl_dev,
                                       int64_t* idx_dev, float* obs_out_dev, float* next_out_dev, float* act_out_dev,
                                       float* rew_out_dev, uint8_t* term_out_dev, void* stream) {
  return replay_sample(n, B, D, Ad, M, seed, pool_obs_dev, pool_next_dev, pool_act_dev, pool_rew_dev, pool_term_dev,
                       ctl_dev, idx_dev, obs_out_dev, next_out_dev, act_out_dev, rew_out_dev, term_out_dev, stream);
}

extern "C" int madrl_replay_sample_bf16(int n, int B, int D, int Ad, size_t M, uint64_t seed, const void* pool_obs_dev,
                                        const void* pool_next_dev, const float* pool_act_dev,
                                        const float* pool_rew_dev, const uint8_t* pool_term_dev, int64_t* ctl_dev,
                                        int64_t* idx_dev, void* obs_out_dev, void* next_out_dev, float* act_out_dev,
                                        float* rew_out_dev, uint8_t* term_out_dev, void* stream) {
  return replay_sample(n, B, D, Ad, M, seed, (const uint16_t*)pool_obs_dev, (const uint16_t*)pool_next_dev,
                       pool_act_dev, pool_rew_dev, pool_term_dev, ctl_dev, idx_dev, (uint16_t*)obs_out_dev,
                       (uint16_t*)next_out_dev, act_out_dev, rew_out_dev, term_out_dev, stream);
}
