// MAWaterWorld batched engine: persistent warp-per-env rollout kernel for sm_90a (H100).
//
// Reference semantics: madrl_environments/pursuit/waterworld.py (cited as ww:LINE).
//
// Design (see DESIGN.md):
//   * One WARP owns one env for the WHOLE T-step rollout.  The env's state lives in REGISTERS:
//     lane l holds objects l, l+32, ... (position + velocity); objects are ordered pursuers,
//     evaders, poisons.  There is no block barrier anywhere (blocks are one warp, and shared memory
//     is the warp's own; the WRITER instantiation's blocks add a warp that writes 8 env warps'
//     observations, see ww_obs_writer): warps are completely independent, so the SM's schedulers overlap the
//     phases of different envs.  HBM sees the state once per launch (a coalesced per-env record)
//     and, per step, only actions in and obs / reward / done / info out.
//   * Per step and pursuer, lanes act first as OBJECTS (relative position, squared distance,
//     collision test and exact conservative range cull, all reduced with __ballot_sync), then as
//     SENSORS (lane k = sensor k) looping over the few surviving candidates, whose geometry is
//     broadcast with __shfl_sync; nearest-object-per-sensor keeps the lowest index among equal
//     minima (np.argmin).  The pursuer's feature values are staged in shared memory and leave,
//     with the env-step's other rows or on their own, as TMA bulk stores (obs_row_stage).
//   * sqrt-free thresholds: every `cdist(...) <= thr` of the reference is evaluated as
//     d2 <= thr2 with thr2 the largest representable value whose correctly-rounded sqrt is
//     <= thr (computed on the host), which is exactly equivalent.
//   * fp32 production instantiation and fp64 verification instantiation of the same template.
#include <math.h>
#include <atomic>
#include <cmath>
#include <mutex>
#include <new>
#include <type_traits>

#include "common.cuh"
#include "engine.cuh"
#include "philox.cuh"

namespace madrl {

template <typename real, typename O = real>   // O: observation element type (see obs_cvt)
struct WWParams {
  int E, env_id_base, Np, Ne, Npo, K, n_coop, D, Nall;
  int reward_global, addid, speed_features, random_obstacle, timestep_limit, max_path_length;
  int T, mode, auto_reset;  // mode 0 = rollout, 1 = reset
  int stage_step;            // observation staging: 1 = the env-step's Np rows at once, 0 = row by row (obs_row_stage)
  // element strides of one lockstep step in the trajectory tensors (host-computed so that the
  // per-step pointer bumps are plain 64-bit adds on constant-bank operands)
  size_t obs_step, agent_step;   // E*Np*D and E*Np
  real r_p2, range, cull2;                           // sensing thresholds (ww:68-69)
  real range_up;                                     // nextafter(range, +inf): `sv < range_up` <=> `sv <= range`
  real coll2_e, coll2_po;                            // (r_p + r_obj) as exact squared thresholds
  real obst2_p, obst2_e, obst2_po;                   // (r_class + R_obst)       ww:251,259,267
  real resp2_p, resp2_e, resp2_po;                   // (2 r_class + R_obst)     ww:140
  real obst_x, obst_y, ev_speed, poison_speed, action_scale;
  real poison_reward, food_reward, encounter_reward, control_penalty;
  uint64_t seed;
  // state: per-env records
  real* objs;         // [E][4][Nall]  (x, y, vx, vy rows)
  real* obst;         // [E][2]
  int32_t *timestep, *path_len;
  uint64_t* ctr;
  const real* sensors;  // [2][K]
  // trajectory tensors
  const real* actions;
  O* obs;
  real* rew;
  uint8_t* done;
  int32_t* info;
  const uint8_t* mask;
  O* term_obs;      // optional [T][E][A][D]: terminal observations of done steps (see keep_terminal_rows)
  // in-kernel action source (POLICY instantiation, madrl_ww_rollout_heuristic): the reference's hand-written
  // policy (heuristics/waterworld.py:11-53) closes the loop inside the launch -- no action tensor is read
  const O* policy_obs0;      // [E][Np][D] the observation the FIRST action is computed from
  real* actions_out;         // [T][E][Np][2] the actions taken (NULL = not recorded)
  // fused per-rollout exchange (multi-GPU): every rank also stores its reward / done / info rows
  // into slot `peer_rank` of each destination gather buffer through NVLink peer mappings (CUDA
  // IPC).  Rows are staged in registers and written as coalesced runs (rewards every 32/Np steps,
  // done/info every 32 steps) into an ENV-major layout [slot][E][Tmax][...], because thousands of
  // 4-byte remote stores per step cost far more than the bytes they carry.
  int n_peers, peer_rank, peer_tmax;
  real* peer_rew[8];
  uint8_t* peer_done[8];
  int32_t* peer_info[8];
};

// 0 <= sv < best, zeros of both signs included, as the reference's `sv < 0` rejection leaves it: sx * jx + sy * jy
// is -0.0 when the candidate sits exactly at the pursuer's position (jx = jy = +0) and neither sensor component is
// positive, which happens when pursuers are clipped into the same corner, and the reference senses it there.  The
// strict `<` keeps the first index among equal values (np.argmin), -0.0 against +0.0 included.  (A one-comparison
// unsigned test of the bit patterns rejects -0.0, and once best = -0.0 would let a later +0.0 win.)
template <typename real>
__device__ __forceinline__ bool in_zero_to(real sv, real best) { return !(sv < (real)0) && sv < best; }

template <typename real>
struct Spawn { real x, y, vx, vy; uint64_t ctr; };

// ww:139-142 + ww:360-374: rejection-sample a position outside the obstacle's keep-out disc,
// then (optionally) a velocity.  Executed warp-uniformly (every lane runs the same stream), so
// no broadcast is needed; rare, hence not inlined into the hot loop.
template <typename real>
__device__ __noinline__ Spawn<real> spawn_object(uint64_t seed, uint32_t env_id, uint64_t ctr,
                                                 real obx, real oby, real thr2, real speed,
                                                 int with_velocity) {
  SeqStream rs;
  rs.init(seed, env_id, 0u, ctr);
  Spawn<real> s;
  s.x = rs.next_unit<real>();
  s.y = rs.next_unit<real>();
  while (true) {
    const real dx = s.x - obx, dy = s.y - oby;
    if (!(dx * dx + dy * dy <= thr2)) break;
    s.x = rs.next_unit<real>();
    s.y = rs.next_unit<real>();
  }
  s.vx = 0; s.vy = 0;
  if (with_velocity) {
    s.vx = (rs.next_unit<real>() - (real)0.5) * speed;
    s.vy = (rs.next_unit<real>() - (real)0.5) * speed;
  }
  s.ctr = rs.counter;
  return s;
}

// Observation rows leave through shared memory (after the candidate slots) and TMA bulk stores.  When an
// env-step's Np rows fit (stage_step), they are staged together, tail triples included, and leave as one
// bulk store at the end of the step.  Otherwise each row's feature values go through a two-slot ring:
// while one slot's bulk store still reads its source, the next row is staged in the other, and the tail
// triple, known only after every pursuer has sensed, is stored directly.  n values are staged at the
// global address modulo 16, so that their 16-byte-aligned global interior and its shared source are
// both 16-byte aligned; hence the 16 bytes of slack.
__host__ __device__ __forceinline__ uint32_t obs_stage_bytes(int n, int real_bytes) {
  return (((uint32_t)n * (uint32_t)real_bytes + 15u) & ~15u) + 16u;
}
// Staging an env-step keeps 32 one-warp blocks per SM: 32 x (6 KB + the 1 KB reserved per block) fit
// the H100's 227 KB of shared memory per SM.
constexpr size_t kStepStageMaxBytes = 6 * 1024;

// Writer-warp staging (ww_kernel's WRITER instantiations, DESIGN §4.1): a block of kWrEnvs env warps, which
// step adjacent envs, and one writer warp.  Every env-step's rows go into the env warp's part of a ring
// slot of the block's shared memory; the writer warp copies each full slot, one step of kWrEnvs adjacent envs
// and so one contiguous run of the [T][E][Np][D] tensor, to HBM.  The env warps then never wait on a store or
// issue one; they only fence their rows into the async proxy before handing a slot over.  The defaults are the
// fastest of scripts/ww_write_path.py's sweep (DESIGN §4.3); the macros exist for that sweep.
#ifndef MADRL_WW_WRITER_SLOTS
#define MADRL_WW_WRITER_SLOTS 2        // S: steps of the group in flight between the env warps and the writer
#endif
#ifndef MADRL_WW_WRITER_ENVS
#define MADRL_WW_WRITER_ENVS 8         // env warps (= adjacent envs) per block
#endif
#ifndef MADRL_WW_WRITER_WARPS_PER_SM
#define MADRL_WW_WRITER_WARPS_PER_SM 16   // resident env warps per SM
#endif
#ifndef MADRL_WW_WRITER_BULK
#define MADRL_WW_WRITER_BULK 1         // 0: the writer copies a slot with 16-byte stores instead of one cp.async.bulk
#endif
constexpr int kWrSlots = MADRL_WW_WRITER_SLOTS, kWrEnvs = MADRL_WW_WRITER_ENVS;
constexpr int kWrBlocksPerSm = MADRL_WW_WRITER_WARPS_PER_SM / MADRL_WW_WRITER_ENVS;
constexpr bool kWrBulk = MADRL_WW_WRITER_BULK != 0;
// A group's rows start 16-byte aligned in every step whenever the tensor's base and step stride are.
static_assert(kWrEnvs % 4 == 0 && kWrSlots >= 2 && kWrBlocksPerSm >= 1, "writer-warp geometry");
constexpr int kWrThreads = 32 * (kWrEnvs + 1);
// Shared memory of a writer block: the full / empty mbarriers of the S slots, each env warp's candidate slots,
// then the ring (slots of `slot` bytes).
__host__ __device__ __forceinline__ uint32_t wr_slot_bytes(int env_step_bytes) {
  return ((uint32_t)(kWrEnvs * env_step_bytes) + 15u) & ~15u;
}
constexpr uint32_t kWrBarBytes = (2 * 8 * kWrSlots + 15) & ~15;
// An env warp's view of the ring: the mbarriers (full s at bar + 8 s, empty s at bar + 8 (S + s)), the ring, the
// slot size, this warp's rows within a slot, and the slot s and phase parity of the current step.
struct WrRing {
  uint32_t bar, ring, slot, rows, phase;
  int s;
  __device__ __forceinline__ uint32_t empty() const { return bar + 8u * (uint32_t)(kWrSlots + s); }
  __device__ __forceinline__ uint32_t step_rows() const { return ring + (uint32_t)s * slot + rows; }
};
struct NoWrRing {};

// Shared address of element 0 of `row` (a row of the env-step starting at `obs_t`), after waiting for
// the bulk store that last read that memory: the previous step's (whole-step staging, first row of
// the step) or the one two rows ago (ring slot `slot_off`).
template <typename O>
__device__ __forceinline__ uint32_t obs_row_stage(bool whole_step, uint32_t stage, uint32_t slot_off,
                                                  const O* obs_t, const O* row, int lane) {
  if (whole_step) {
    if (row == obs_t) {
      if (lane == 0) bulk_wait_read_all();
      __syncwarp();
    }
    return stage + ((uint32_t)(uintptr_t)obs_t & 15u) + (uint32_t)((row - obs_t) * sizeof(O));
  }
  if (lane == 0) bulk_wait_read_all_but_1();
  __syncwarp();
  return stage + slot_off + ((uint32_t)(uintptr_t)row & 15u);
}

// The n values staged at `slot` -> global `row`: the 16-byte-aligned interior as one bulk store
// (HBM then sees whole sectors from one writer), the <= 16 bytes outside it on either side by
// direct stores of one lane per element.  Full writes, no read-back, so the rows are bit-identical
// to per-lane stores.
template <bool KEEP, typename O>
__device__ __forceinline__ void obs_row_store(uint32_t slot, O* row, int n, int lane) {
  fence_async_shared();   // this lane's shared stores -> visible to the async proxy ...
  __syncwarp();           // ... before lane 0 issues the copy; the edge lanes read other lanes' values
  const uintptr_t g0 = (uintptr_t)row, g1 = g0 + (uintptr_t)n * sizeof(O);
  const uintptr_t a0 = (g0 + 15u) & ~(uintptr_t)15u, a1 = g1 & ~(uintptr_t)15u;
  const bool bulk = a1 > a0;
  if (lane == 0 && bulk) bulk_store_obs<KEEP>((void*)a0, slot + (uint32_t)(a0 - (g0 & ~(uintptr_t)15u)), (uint32_t)(a1 - a0));
  const int head = bulk ? (int)((a0 - g0) / sizeof(O)) : n;
  const int tail = bulk ? (int)((g1 - a1) / sizeof(O)) : 0;
  if (lane < head + tail) {
    const int i = lane < head ? lane : n - tail + (lane - head);
    store_obs<KEEP>(row + i, lds_obs<O>(slot + ((uint32_t)g0 & 15u) + (uint32_t)(i * sizeof(O))));
  }
}

// WRITER: shared address of pursuer pi's row, `row_off` bytes into this env warp's part of the step's ring slot
// (`rows`), after waiting, at the step's first row, until the writer warp has released the slot (`empty`, completed
// phase parity `phase ^ 1`: the copy of what the slot held S steps ago; the first S steps find the slot free).
__device__ __forceinline__ uint32_t wr_row_stage(uint32_t empty, uint32_t phase, uint32_t rows, int pi, uint32_t row_off) {
  if (pi == 0) mbar_wait(empty, phase ^ 1u);
  return rows + row_off;
}

// The writer warp of a WRITER block: for every step of every env group of the block, wait until the group's
// env warps have staged the step in ring slot s ("full" mbarrier s), copy the slot to the group's contiguous run
// of the observation tensor (16-aligned: the host only selects WRITER when the base and step stride are), and
// release the slot ("empty" mbarrier s).  The copy is one cp.async.bulk (evict-first), and a slot is released
// once the next one's bulk store is issued and the slot's own has read its source.  Without kWrBulk it is
// 16-byte shared loads and evict-first global stores instead: the generic proxy, so the env warps need no
// proxy fence, but the writer issues two instructions per 16 bytes.  A group's run is always a whole number of
// 16-byte units, so `tail` below never selects an element: the host's stride rule makes E*Np*D a multiple of 4, and
// a partial last group's k envs satisfy k = E (mod kWrEnvs) with kWrEnvs a multiple of 4, so k*Np*D is one too.
// (The one-per-lane tail stores stay, since removing them changes this kernel's SASS.)
template <typename real, typename O>
__device__ __forceinline__ void ww_obs_writer(const WWParams<real, O>& p, uint32_t bar, uint32_t ring, uint32_t slot_bytes,
                                              uint32_t env_bytes, int lane) {
  static_assert(sizeof(O) == sizeof(float), "the writer warp stores float32 observations");
  int s = 0;
  [[maybe_unused]] int prev = -1;   // kWrBulk: the slot whose bulk store was issued last
  uint32_t phase = 0u;
  const size_t step_bytes = p.obs_step * sizeof(O);
  for (int g0 = (int)blockIdx.x * kWrEnvs; g0 < p.E; g0 += (int)gridDim.x * kWrEnvs) {
    const uint32_t n = (uint32_t)min(kWrEnvs, p.E - g0) * env_bytes, n16 = n & ~15u;
    char* dst = reinterpret_cast<char*>(p.obs + (size_t)g0 * p.Np * p.D);
    for (int t = 0; t < p.T; ++t, dst += step_bytes) {
      const uint32_t src = ring + (uint32_t)s * slot_bytes;
      mbar_wait(bar + 8u * s, phase);
      if constexpr (kWrBulk) {
        if (lane == 0) ring_bulk_store(dst, src, n16);
      } else {
#pragma unroll 4
        for (uint32_t i = 16u * (uint32_t)lane; i < n16; i += 512u) stcs_f32x4(dst + i, ring_lds_f32x4(src + i));
      }
      const uint32_t tail = n16 + (uint32_t)lane * (uint32_t)sizeof(O);
      if (tail < n) store_stream(reinterpret_cast<float*>(dst + tail), ring_lds_f32(src + tail));
      __syncwarp();   // every lane has read the slot before it is released
      if constexpr (kWrBulk) {
        if (lane == 0 && prev >= 0) { bulk_wait_read_all_but_1(); mbar_arrive(bar + 8u * (kWrSlots + prev), 1u); }
        prev = s;
      } else {
        if (lane == 0) mbar_arrive(bar + 8u * (kWrSlots + s), 1u);
      }
      if (++s == kWrSlots) { s = 0; phase ^= 1u; }
    }
  }
  if constexpr (kWrBulk)
    if (lane == 0) bulk_wait_all();   // the last bulk store has read its source before the block exits
}

// OPL = objects per lane (ceil(n_obj / 32)); KCH = sensors per lane (ceil(K / 32));
// KC = compile-time sensor count (0 = runtime p.K): with KC known the 7 feature-row stores of a
// pursuer use immediate offsets from one shared address.
// PEER = compile the fused multi-GPU exchange in (a separate instantiation, so the single-GPU kernel
// carries none of its registers).
// POLICY = the actions come from the in-kernel heuristic policy instead of the action tensor (again a
// separate instantiation: the open-loop kernel carries none of its instructions): kWwPolicyAgent divides each
// pursuer's action by its own norm, kWwPolicyEnv all of an env's actions by one norm (madrl_ww_set_heuristic_norm).
// KEEP = observation rows are stored at normal L2 priority instead of evict-first (store_obs).
// WRITER = writer-warp staging (kWrEnvs env warps + 1 writer warp per block; whole-step staging, 16-byte-aligned
// observation base and step stride, open loop, no PEER / POLICY / KEEP).
constexpr int kWwPolicyAgent = 1, kWwPolicyEnv = 2;
template <typename real, typename O, int OPL, int KCH, int KC, bool PEER, int POLICY = 0, bool KEEP = false,
          bool WRITER = false>
__global__ void __launch_bounds__(WRITER ? kWrThreads : 32, WRITER ? kWrBlocksPerSm : (OPL <= 4 ? 28 : 16))
ww_kernel(const __grid_constant__ WWParams<real, O> p) {
  const real INF = real_inf<real>();
  const int K = KC > 0 ? KC : p.K;
  // 32-thread blocks: the env index derives from blockIdx alone, so ptxas can prove every loop and
  // branch on it warp-uniform -- no BRA.DIV guards in front of the warp collectives, loop bookkeeping
  // on the uniform datapath, fewer registers.
  const int lane = WRITER ? (int)(threadIdx.x & 31u) : (int)threadIdx.x;
  // WRITER: env warp 0 .. kWrEnvs-1, or the writer; broadcast from lane 0 so that ptxas knows it is warp-uniform
  const int wr_warp = WRITER ? __shfl_sync(FULL_MASK, (int)(threadIdx.x >> 5), 0) : 0;
  const int warp_global = WRITER ? (int)blockIdx.x * kWrEnvs + wr_warp : (int)blockIdx.x;
  const int warp_stride = WRITER ? (int)gridDim.x * kWrEnvs : (int)gridDim.x;
  const int eLo = p.Np, eHi = p.Np + p.Ne, Nall = p.Nall;
  constexpr bool SMEM = OPL >= 2;
  const unsigned lt_mask = lanemask_lt();
  extern __shared__ __align__(16) unsigned char ww_smem[];
  // this warp's candidate slots (OPL >= 2), then its observation staging (32-bit shared address)
  uint32_t slots = smem_addr(ww_smem);
  asm volatile("" : "+r"(slots));   // keep it in a register: ptxas otherwise re-derives it from SR_CgaCtaId at every use
  // WRITER: the ring (an empty type otherwise, so that the other instantiations compile as they did without it)
  typename std::conditional<WRITER, WrRing, NoWrRing>::type wr;
  if constexpr (WRITER) {
    const uint32_t env_bytes = (uint32_t)(p.Np * p.D) * (uint32_t)sizeof(O);
    const uint32_t cand = SMEM ? (uint32_t)Nall * CandSlot<real>::kStride : 0u;
    wr.bar = slots;
    wr.slot = wr_slot_bytes((int)env_bytes);
    wr.ring = wr.bar + kWrBarBytes + kWrEnvs * cand;
    wr.rows = (uint32_t)wr_warp * env_bytes;
    wr.s = 0;
    wr.phase = 0u;
    if (threadIdx.x == 0)
      for (int s = 0; s < kWrSlots; ++s) { mbar_init(wr.bar + 8u * s, kWrEnvs); mbar_init(wr.bar + 8u * (kWrSlots + s), 1u); }
    __syncthreads();
    if (wr_warp == kWrEnvs) {
      ww_obs_writer(p, wr.bar, wr.ring, wr.slot, env_bytes, lane);
      return;
    }
    slots = wr.bar + kWrBarBytes + (uint32_t)wr_warp * cand;
  }

  // ---- per-lane constants: this lane as OBJECT (classes, thresholds) and as SENSOR -----------
  real cull2_l[OPL], coll2_l[OPL];
  unsigned mE[OPL], mP[OPL], mU[OPL];  // warp-uniform class masks of each object chunk
#pragma unroll
  for (int c = 0; c < OPL; ++c) {
    const int o = lane + 32 * c;
    const bool isU = o < eLo, isE = o >= eLo && o < eHi, isP = o >= eHi && o < Nall;
    cull2_l[c] = p.cull2;   // uniform: lanes beyond the last object hold a far-away sentinel position instead
    coll2_l[c] = isE ? p.coll2_e : (isP ? p.coll2_po : (real)-1);
    mU[c] = __ballot_sync(FULL_MASK, isU);
    mE[c] = __ballot_sync(FULL_MASK, isE);
    mP[c] = __ballot_sync(FULL_MASK, isP);
  }
  real sx_l[KCH], sy_l[KCH];
#pragma unroll
  for (int kc = 0; kc < KCH; ++kc) {
    const int k = lane + 32 * kc;
    sx_l[kc] = (k < K) ? p.sensors[k] : (real)0;
    sy_l[kc] = (k < K) ? p.sensors[K + k] : (real)0;
  }
  // the compile-time-K instantiation is also the speed_features = True one (the reference's defaults: K = 30, 7 rows
  // per sensor): no layout branch per pursuer; every other combination takes the KC = 0 instantiation
  const bool speed = KC > 0 ? true : (p.speed_features != 0);
  const int n_feat = speed ? 7 : 4;
  const uint32_t stage = slots + (SMEM ? (uint32_t)Nall * CandSlot<real>::kStride : 0u);
  const uint32_t slot_bytes = obs_stage_bytes(n_feat * K, sizeof(O));
  uint32_t slot_off = 0u;   // row-by-row staging: ring slot of the next row, 0 or slot_bytes
  typedef typename Vec2<real>::type V2;

  for (int e = warp_global; e < p.E; e += warp_stride) {
    if (p.mode == 1 && p.mask != nullptr && p.mask[e] == 0) continue;
    const uint32_t env_id = (uint32_t)(p.env_id_base + e);
    // ---- state: HBM record -> registers -----------------------------------------------------
    real x[OPL], y[OPL], vx[OPL], vy[OPL];
    unsigned col[OPL];  // per object: bit q set <=> pursuer q collides with it this step
    real* rec = p.objs + (size_t)e * 4 * Nall;
#pragma unroll
    for (int c = 0; c < OPL; ++c) {
      const int o = lane + 32 * c;
      const bool v = o < Nall;
      x[c] = v ? rec[o] : (real)1e18;            // sentinel: never in range of anything, never written back
      y[c] = v ? rec[Nall + o] : (real)1e18;
      vx[c] = v ? rec[2 * Nall + o] : (real)0;
      vy[c] = v ? rec[3 * Nall + o] : (real)0;
      col[c] = 0u;
    }
    real obx = p.obst[2 * (size_t)e], oby = p.obst[2 * (size_t)e + 1];
    int tt = p.timestep[e], ts = p.path_len[e];
    uint64_t ctr = p.ctr[e];

    // running output pointers: the env's first pursuer row at step t (warp-uniform), this lane's reward
    O* obs_t = p.obs + (size_t)e * p.Np * p.D;
    real* rew_t = p.rew + (size_t)e * p.Np + lane;
    size_t te = (size_t)e;   // index of (t, e) in the [T][E] done / info tensors
    int pass = (p.mode == 1) ? 1 : 0;  // pass 1 = reset pass: fresh draws, zero action, obs only
    const V2* act_t = reinterpret_cast<const V2*>(p.actions) + (size_t)e * p.Np + lane;

    // POLICY: un-normalised action of pursuer `lane` for the NEXT step (heuristics/waterworld.py:25-44),
    // first from the caller's observation, afterwards from the features this warp has just computed
    real pax = 0, pay = 0;
    if constexpr (POLICY) {
      // (bf16 obs0: the widened values -- the first decision after a launch boundary sees rounded features)
      const O* o0 = p.policy_obs0 + (size_t)e * p.Np * p.D;
      for (int pi = 0; pi < p.Np; ++pi, o0 += p.D) {
        const real cE = obs_widen<real>(o0[7 * K]) > (real)0 ? (real)1.5 : (real)1;        // heuristics/waterworld.py:41
        const real cP = obs_widen<real>(o0[7 * K + 1]) > (real)0 ? (real)1.5 : (real)1;    // :42
        real wx = 0, wy = 0;
#pragma unroll
        for (int kc = 0; kc < KCH; ++kc) {
          const int k = lane + 32 * kc;
          if (k < K) {
            const real w = (real)0.5 * obs_widen<real>(o0[5 * K + k]) +
                           (cE * obs_widen<real>(o0[K + k]) - obs_widen<real>(o0[k])) - cP * obs_widen<real>(o0[3 * K + k]);
            wx += w * sx_l[kc]; wy += w * sy_l[kc];
          }
        }
        wx = warp_allreduce_sum(wx); wy = warp_allreduce_sum(wy);
        if (lane == pi) { pax = wx; pay = wy; }
      }
    }

    // staging registers of the fused exchange
    const int rew_per = 32 / p.Np;                       // steps per coalesced reward run
    const int stage_src = lane % p.Np, stage_step = lane / p.Np;
    const size_t peer_env = (size_t)p.peer_rank * p.E + e;
    real st_rew = 0, r_stage = 0;
    int2 st_info = make_int2(0, 0);
    uint8_t st_done = 0;
    int sc_rew = 0;

    V2 act_nx;
    act_nx.x = 0; act_nx.y = 0;
    if (!POLICY && p.mode == 0 && lane < p.Np) act_nx = *act_t;
    for (int t = 0; t < p.T; ++t) {
      V2 act;
      act.x = 0; act.y = 0;
      if constexpr (POLICY == kWwPolicyEnv) {
        // heuristics/waterworld.py:47-51 on the env's Np x 2 batch: every action divided by the batch's Frobenius
        // norm, all zero when it is 0; scaled by the largest |component| first, as below
        const real m = warp_allreduce_max(lane < p.Np ? fmax(fabs(pax), fabs(pay)) : (real)0);
        const real ux = m > (real)0 ? pax / m : (real)0, uy = m > (real)0 ? pay / m : (real)0;
        const real n = sqrt(warp_allreduce_sum(lane < p.Np ? ux * ux + uy * uy : (real)0));
        if (lane < p.Np) {
          if (m > (real)0) { act.x = ux / n; act.y = uy / n; }
          if (p.actions_out != nullptr)
            reinterpret_cast<V2*>(p.actions_out)[(size_t)t * p.agent_step + (size_t)e * p.Np + lane] = act;
        }
      } else if constexpr (POLICY) {
        if (lane < p.Np) {   // heuristics/waterworld.py:44-50: unit vector, or zero when nothing is sensed
          // scaled by the larger component first: the squares of a tiny sum (cancellation leaves ~1e-21) would be
          // denormal in float32 and the "unit" vector off by 1e-4
          const real m = fmax(fabs(pax), fabs(pay));
          if (m > (real)0) {
            const real ux = pax / m, uy = pay / m, n = sqrt(ux * ux + uy * uy);
            act.x = ux / n; act.y = uy / n;
          }
          if (p.actions_out != nullptr)
            reinterpret_cast<V2*>(p.actions_out)[(size_t)t * p.agent_step + (size_t)e * p.Np + lane] = act;
        }
      } else if (p.mode == 0 && lane < p.Np) {
        // double-buffered in registers: the load for step t+1 is issued at the top of step t, so its HBM
        // latency hides behind a whole step (a prefetch.global.L1 left the first use of the action stalling)
        act = act_nx;
        if (t + 1 < p.T) act_nx = act_t[p.agent_step];
      }
      bool need_reset;
      do {
        if (pass) {
          // ---- reset draws, ww:144-170 (obstacle, pursuers, evaders, poisons) ----------------
          tt = 0; ts = 0;
          if (p.random_obstacle) {
            SeqStream rs;
            rs.init(p.seed, env_id, 0u, ctr);
            obx = rs.next_unit<real>();
            oby = rs.next_unit<real>();
            ctr = rs.counter;
          } else {
            obx = p.obst_x; oby = p.obst_y;
          }
          for (int o = 0; o < Nall; ++o) {
            const bool oU = o < eLo, oE = !oU && o < eHi;
            // ww:164,170 -- poisons also use ev_speed at reset
            const Spawn<real> s = spawn_object<real>(p.seed, env_id, ctr, obx, oby,
                                                     oU ? p.resp2_p : (oE ? p.resp2_e : p.resp2_po),
                                                     p.ev_speed, oU ? 0 : 1);
            ctr = s.ctr;
#pragma unroll
            for (int c = 0; c < OPL; ++c)
              if (o == lane + 32 * c) { x[c] = s.x; y[c] = s.y; vx[c] = s.vx; vy[c] = s.vy; }
          }
          act.x = 0; act.y = 0;
        }
        // ---- integrate pursuers, control penalty, walls: ww:221-245 (pursuers = chunk 0) -------
        real pen;
        {
          real sq = 0;
          if (lane < p.Np) {
            const real ax = act.x * p.action_scale, ay = act.y * p.action_scale;
            vx[0] += ax; vy[0] += ay;
            x[0] += vx[0]; y[0] += vy[0];
            sq = ax * ax + ay * ay;
            const real cx = clip01(x[0]), cy = clip01(y[0]);
            if (x[0] != cx) vx[0] = 0;
            if (y[0] != cy) vy[0] = 0;
            x[0] = cx; y[0] = cy;
          }
          pen = p.control_penalty * (p.reward_global ? warp_allreduce_sum(sq) : sq);
        }
        // ---- obstacle rebound (velocity only): ww:247-270 ----------------------------------------
#pragma unroll
        for (int c = 0; c < OPL; ++c) {
          const bool oE = (mE[c] >> lane) & 1u, oP = (mP[c] >> lane) & 1u, oU = (mU[c] >> lane) & 1u;
          const real thr = oU ? p.obst2_p : (oE ? p.obst2_e : (oP ? p.obst2_po : (real)-1));
          const real kf = oP ? (real)-1 : (real)-0.5;                  // ww:254,262,270
          const real dx = x[c] - obx, dy = y[c] - oby;
          if (dx * dx + dy * dy <= thr) { vx[c] = kf * vx[c]; vy[c] = kf * vy[c]; }
        }
        // ---- sense: one pursuer at a time -----------------------------------------------------
        // the pursuer's row: a global pointer (one-warp staging), or (WRITER) a 32-bit byte offset into the step's rows
        O* obs_row = obs_t;
        uint32_t row_off = 0u;
        for (int pi = 0; pi < p.Np; ++pi, obs_row += p.D, row_off += (uint32_t)(p.D * sizeof(O))) {
          const real mx = __shfl_sync(FULL_MASK, x[0], pi), my = __shfl_sync(FULL_MASK, y[0], pi);
          const real mvx = __shfl_sync(FULL_MASK, vx[0], pi), mvy = __shfl_sync(FULL_MASK, vy[0], pi);
          // nearest sensed object per class and sensor chunk (ww:64-72, 312-334)
          real bO[KCH], bE[KCH], bP[KCH], bU[KCH];
          int iE[KCH], iP[KCH], iU[KCH];
          const real orx = obx - mx, ory = oby - my;
          const real od2 = orx * orx + ory * ory;
          real pwx = 0, pwy = 0;       // POLICY: this lane's share of pursuer pi's next action
          unsigned tE = 0u, tP = 0u;   // POLICY: evaders / poisons pursuer pi touches this step (obs[7K], obs[7K+1])
#pragma unroll
          for (int kc = 0; kc < KCH; ++kc) {
            bO[kc] = bE[kc] = bP[kc] = bU[kc] = INF;
            iE[kc] = iP[kc] = iU[kc] = 0;
            if (od2 <= p.cull2) {   // the obstacle is sensed like a point object (pursuer radius only)
              const real sv = sx_l[kc] * orx + sy_l[kc] * ory;
              const bool ok = !((sv < (real)0) | (sv > p.range) | (od2 - sv * sv > p.r_p2));
              bO[kc] = ok ? sv : INF;
            }
          }
          if constexpr (SMEM) {
            constexpr uint32_t S = CandSlot<real>::kStride;
            uint32_t endU = slots, nEc = 0u, top = slots;
#pragma unroll
            for (int c = 0; c < OPL; ++c) {
              // lanes as OBJECTS: geometry, collisions (ww:278-293), conservative range cull, staging
              const real rx = x[c] - mx, ry = y[c] - my;
              const real d2 = rx * rx + ry * ry;
              const bool near = d2 <= cull2_l[c] && !(c == 0 && lane == pi);   // ww:70-71 `same`
              const unsigned cm = __ballot_sync(FULL_MASK, near);
              const bool hit = d2 <= coll2_l[c];
              if (hit) col[c] |= 1u << pi;
              if constexpr (POLICY) { const unsigned hm = __ballot_sync(FULL_MASK, hit); tE |= hm & mE[c]; tP |= hm & mP[c]; }
              // slot = rank among the candidates in ascending object index (= lane + 32 c)
              if (near) CandSlot<real>::put(top + (uint32_t)__popc(cm & lt_mask) * S, rx, ry, d2, vx[c], vy[c]);
              if (c == 0) endU = slots + (uint32_t)__popc(cm & mU[0]) * S;   // pursuers live in chunk 0 (Np <= 32)
              nEc += (uint32_t)__popc(cm & mE[c]);
              top += (uint32_t)__popc(cm) * S;
            }
            __syncwarp();
            // lanes as SENSORS: classes are contiguous in object index, hence in slot order U, E, P
            const uint32_t endE = endU + nEc * S, endP = top;   // the poisons end the list
            const real up = p.range_up;   // `sv < up` <=> `sv <= range`; a best below `up` <=> sensed
            uint32_t aE[KCH], aP[KCH], aU[KCH];
#pragma unroll
            for (int kc = 0; kc < KCH; ++kc) { bE[kc] = bP[kc] = bU[kc] = up; aE[kc] = aP[kc] = aU[kc] = slots; }
#define MADRL_WW_SCAN(A0, A1, BEST, AT)                                                  \
  _Pragma("unroll 2")                                                                  \
  for (uint32_t a = (A0); a != (A1); a += S) {                                           \
    real jx, jy, jd;                                                                     \
    CandSlot<real>::geom(a, jx, jy, jd);                                                 \
    _Pragma("unroll") for (int kc = 0; kc < KCH; ++kc) {                                 \
      const real sv = sx_l[kc] * jx + sy_l[kc] * jy;                                     \
      /* ww:64-72: 0 <= sv (<= range, through the initial best) and within the pursuer's radius of the ray */ \
      if (in_zero_to(sv, BEST[kc]) && !(jd - sv * sv > p.r_p2)) { BEST[kc] = sv; AT[kc] = a; } \
    }                                                                                    \
  }
            MADRL_WW_SCAN(slots, endU, bU, aU)
            MADRL_WW_SCAN(endU, endE, bE, aE)
            MADRL_WW_SCAN(endE, endP, bP, aP)
#undef MADRL_WW_SCAN
            uint32_t srow;
            if constexpr (WRITER) srow = wr_row_stage(wr.empty(), wr.phase, wr.step_rows(), pi, row_off);
            else srow = obs_row_stage(p.stage_step != 0, stage, slot_off, obs_t, obs_row, lane);
#pragma unroll
            for (int kc = 0; kc < KCH; ++kc) {
              const real sx = sx_l[kc], sy = sy_l[kc];
              // features ww:312-353, 388-395: feature-major, sensor-minor
              const int k = lane + 32 * kc;
              const bool hO = bO[kc] < INF, hE = bE[kc] < up, hP = bP[kc] < up, hU = bU[kc] < up;
              const real z = (real)0;
              const uint32_t o = srow + (uint32_t)(k * sizeof(O));   // this lane's column
              constexpr uint32_t R = sizeof(O);
              if constexpr (POLICY) {
                if (k < K) {
                  const real w = (real)0.5 * (hU ? bU[kc] : z) + ((tE ? (real)1.5 : (real)1) * (hE ? bE[kc] : z) - (hO ? bO[kc] : z)) -
                                 (tP ? (real)1.5 : (real)1) * (hP ? bP[kc] : z);
                  pwx += w * sx; pwy += w * sy;
                }
              }
              if (speed) {
                // slot 0 is read when nothing was sensed; its (possibly stale) value is masked below
                real oEx, oEy, oPx, oPy, oUx, oUy;
                CandSlot<real>::vel(aE[kc], oEx, oEy);
                CandSlot<real>::vel(aP[kc], oPx, oPy);
                CandSlot<real>::vel(aU[kc], oUx, oUy);
                if (k < K) {
                  stage_obs<O>(o + 0 * K * R, hO ? bO[kc] : z);
                  stage_obs<O>(o + 1 * K * R, hE ? bE[kc] : z);
                  stage_obs<O>(o + 2 * K * R, hE ? sx * (oEx - mvx) + sy * (oEy - mvy) : z);
                  stage_obs<O>(o + 3 * K * R, hP ? bP[kc] : z);
                  stage_obs<O>(o + 4 * K * R, hP ? sx * (oPx - mvx) + sy * (oPy - mvy) : z);
                  stage_obs<O>(o + 5 * K * R, hU ? bU[kc] : z);
                  stage_obs<O>(o + 6 * K * R, hU ? sx * (oUx - mvx) + sy * (oUy - mvy) : z);
                }
              } else if (k < K) {
                stage_obs<O>(o + 0 * K * R, hO ? bO[kc] : z);
                stage_obs<O>(o + 1 * K * R, hE ? bE[kc] : z);
                stage_obs<O>(o + 2 * K * R, hP ? bP[kc] : z);
                stage_obs<O>(o + 3 * K * R, hU ? bU[kc] : z);
              }
            }
            __syncwarp();   // the next pursuer's staging overwrites the slots
          } else {
            // OPL == 1 (objects are lanes): lanes as OBJECTS -- geometry, collisions (ww:278-293), conservative
            // range cull, and the velocity relative to pursuer pi, which the sensors shuffle for the speed features
            const real rx = x[0] - mx, ry = y[0] - my;
            const real d2 = rx * rx + ry * ry;
            const real rvx = vx[0] - mvx, rvy = vy[0] - mvy;
            const unsigned cm = __ballot_sync(FULL_MASK, d2 <= cull2_l[0]) & ~(1u << pi);   // ww:70-71 `same`
            const bool hit = d2 <= coll2_l[0];
            if (hit) col[0] |= 1u << pi;
            if constexpr (POLICY) { const unsigned hm = __ballot_sync(FULL_MASK, hit); tE |= hm & mE[0]; tP |= hm & mP[0]; }
            // lanes as SENSORS: one walk over the candidates in ascending index.  Classes are contiguous in object
            // index, so the (warp-uniform) index picks the class, and each class still sees its candidates in
            // ascending order: with the strict `<`, the lowest index among equal minima wins (np.argmin).
            const real up = p.range_up;   // `sv < up` <=> `sv <= range`; a best below `up` <=> sensed
#pragma unroll
            for (int kc = 0; kc < KCH; ++kc) bE[kc] = bP[kc] = bU[kc] = up;
            for (unsigned m = cm; m != 0u; m &= m - 1u) {
              const int j = __ffs(m) - 1;
              const real jx = __shfl_sync(FULL_MASK, rx, j), jy = __shfl_sync(FULL_MASK, ry, j);
              const real jd = __shfl_sync(FULL_MASK, d2, j);
#pragma unroll
              for (int kc = 0; kc < KCH; ++kc) {
                const real sv = sx_l[kc] * jx + sy_l[kc] * jy;
                // ww:64-72: 0 <= sv (<= range, through the initial best) and within the pursuer's radius of the ray.
                // `!(sv < 0)` as in the reference (and in_zero_to): a candidate exactly at the pursuer's position
                // (pursuers clipped into the same corner) gives sv = -0.0 for sensors with no positive component,
                // and the reference senses it at distance 0.
                const bool ok = !(sv < (real)0) & !(jd - sv * sv > p.r_p2);
                // a uniform branch on the class, then selects (no divergent branch on the sensor's test)
                auto take = [&](real& best, int& at) {
                  const bool t = ok & (sv < best);
                  best = t ? sv : best;
                  at = t ? j : at;
                };
                if (j < eLo) take(bU[kc], iU[kc]);
                else if (j < eHi) take(bE[kc], iE[kc]);
                else take(bP[kc], iP[kc]);
              }
            }
          uint32_t srow;
          if constexpr (WRITER) srow = wr_row_stage(wr.empty(), wr.phase, wr.step_rows(), pi, row_off);
          else srow = obs_row_stage(p.stage_step != 0, stage, slot_off, obs_t, obs_row, lane);
#pragma unroll
          for (int kc = 0; kc < KCH; ++kc) {
            const real sx = sx_l[kc], sy = sy_l[kc];
            // features ww:312-353, 388-395: feature-major, sensor-minor
            const int k = lane + 32 * kc;
            const bool hO = bO[kc] < INF, hE = bE[kc] < up, hP = bP[kc] < up, hU = bU[kc] < up;
            const real z = (real)0;
            const uint32_t o = srow + (uint32_t)(k * sizeof(O));   // this lane's column
            constexpr uint32_t R = sizeof(O);
            if constexpr (POLICY) {
              if (k < K) {
                const real w = (real)0.5 * (hU ? bU[kc] : z) + ((tE ? (real)1.5 : (real)1) * (hE ? bE[kc] : z) - (hO ? bO[kc] : z)) -
                               (tP ? (real)1.5 : (real)1) * (hP ? bP[kc] : z);
                pwx += w * sx; pwy += w * sy;
              }
            }
            if (speed) {
              // the winners' velocities relative to pursuer pi (index 0 when nothing was sensed, masked below)
              const real oEx = __shfl_sync(FULL_MASK, rvx, iE[kc]), oEy = __shfl_sync(FULL_MASK, rvy, iE[kc]);
              const real oPx = __shfl_sync(FULL_MASK, rvx, iP[kc]), oPy = __shfl_sync(FULL_MASK, rvy, iP[kc]);
              const real oUx = __shfl_sync(FULL_MASK, rvx, iU[kc]), oUy = __shfl_sync(FULL_MASK, rvy, iU[kc]);
              if (k < K) {
                stage_obs<O>(o + 0 * K * R, hO ? bO[kc] : z);
                stage_obs<O>(o + 1 * K * R, hE ? bE[kc] : z);
                stage_obs<O>(o + 2 * K * R, hE ? sx * oEx + sy * oEy : z);
                stage_obs<O>(o + 3 * K * R, hP ? bP[kc] : z);
                stage_obs<O>(o + 4 * K * R, hP ? sx * oPx + sy * oPy : z);
                stage_obs<O>(o + 5 * K * R, hU ? bU[kc] : z);
                stage_obs<O>(o + 6 * K * R, hU ? sx * oUx + sy * oUy : z);
              }
            } else if (k < K) {
              stage_obs<O>(o + 0 * K * R, hO ? bO[kc] : z);
              stage_obs<O>(o + 1 * K * R, hE ? bE[kc] : z);
              stage_obs<O>(o + 2 * K * R, hP ? bP[kc] : z);
              stage_obs<O>(o + 3 * K * R, hU ? bU[kc] : z);
            }
          }
          }
          if (!WRITER && !p.stage_step) {
            obs_row_store<KEEP>(stage + slot_off, obs_row, n_feat * K, lane);
            slot_off = slot_bytes - slot_off;
          }
          if constexpr (POLICY) {   // sum over the sensors; lane pi keeps pursuer pi's next action
            pwx = warp_allreduce_sum(pwx); pwy = warp_allreduce_sum(pwy);
            if (lane == pi) { pax = pwx; pay = pwy; }
          }
        }
        // ---- catches, respawn, rewards: ww:285,293,358-385 -----------------------------------------
        unsigned whoE = 0u, whoP = 0u, whoEnc = 0u;
        int nE = 0, nP = 0, nEnc = 0;
#pragma unroll
        for (int c = 0; c < OPL; ++c) {
          const int cnt = __popc(col[c]);
          // collisions needed to be caught: evaders n_coop (ww:285), poisons 1 (ww:293)
          const bool caught = ((mE[c] >> lane) & 1u) ? cnt >= p.n_coop : (((mP[c] >> lane) & 1u) && cnt >= 1);
          const unsigned cmk = __ballot_sync(FULL_MASK, caught);
          const unsigned enc = __ballot_sync(FULL_MASK, cnt >= 1) & mE[c];   // ww:376
          nE += __popc(cmk & mE[c]);
          nP += __popc(cmk & mP[c]);
          nEnc += __popc(enc);
          if (caught) { if ((mE[c] >> lane) & 1u) whoE |= col[c]; else whoP |= col[c]; }
          if ((enc >> lane) & 1u) whoEnc |= col[c];
          col[c] = 0u;
          for (unsigned m = cmk; m != 0u; m &= m - 1u) {   // ascending index: evaders, then poisons
            const int j = __ffs(m) - 1;
            const bool jE = (mE[c] >> j) & 1u;
            const Spawn<real> s = spawn_object<real>(p.seed, env_id, ctr, obx, oby,
                                                     jE ? p.resp2_e : p.resp2_po,
                                                     jE ? p.ev_speed : p.poison_speed, 1);
            ctr = s.ctr;
            if (lane == j) { x[c] = s.x; y[c] = s.y; vx[c] = s.vx; vy[c] = s.vy; }
          }
        }
        whoE = __reduce_or_sync(FULL_MASK, whoE);
        whoP = __reduce_or_sync(FULL_MASK, whoP);
        whoEnc = __reduce_or_sync(FULL_MASK, whoEnc);
        // ww:411-428 tail of every pursuer's row: [touched an evader, touched a poison, id]; lane i
        // writes pursuer i's.  whoEnc / whoP are exactly the any-collision masks (ww:376, ww:293).
        if (lane < p.Np) {
          const real vE = (real)((whoEnc >> lane) & 1u), vP = (real)((whoP >> lane) & 1u), id = (real)(lane + 1);
          const int i = lane * p.D + n_feat * K;
          if (WRITER || p.stage_step) {
            uint32_t a;
            if constexpr (WRITER) a = wr.step_rows() + (uint32_t)(i * sizeof(O));
            else a = stage + ((uint32_t)(uintptr_t)obs_t & 15u) + (uint32_t)(i * sizeof(O));
            stage_obs<O>(a, vE);
            stage_obs<O>(a + (uint32_t)sizeof(O), vP);
            if (p.addid) stage_obs<O>(a + 2 * (uint32_t)sizeof(O), id);
          } else {
            store_obs<KEEP>(obs_t + i, obs_cvt<O>(vE));
            store_obs<KEEP>(obs_t + i + 1, obs_cvt<O>(vP));
            if (p.addid) store_obs<KEEP>(obs_t + i + 2, obs_cvt<O>(id));
          }
        }
        if (!WRITER && p.stage_step) obs_row_store<KEEP>(stage, obs_t, p.Np * p.D, lane);
        if (!pass && lane < p.Np) {
          real r = pen;
          if (p.reward_global) {
            r += ((real)nE * p.food_reward + (real)nP * p.poison_reward) + (real)nEnc * p.encounter_reward;
          } else {   // fancy-index += : at most once per category (ww:383-385)
            if ((whoE >> lane) & 1u) r += p.food_reward;
            if ((whoP >> lane) & 1u) r += p.poison_reward;
            if ((whoEnc >> lane) & 1u) r += p.encounter_reward;
          }
          store_stream(rew_t, r);
          if (PEER) r_stage = r;
        }
        if (PEER && !pass && p.n_peers > 0) {   // stage this step's rewards: lane s*Np + a <- (step s, agent a)
          const real v = __shfl_sync(FULL_MASK, r_stage, stage_src);
          if (stage_step == sc_rew) st_rew = v;
          if (++sc_rew == rew_per) {
            if (lane < rew_per * p.Np) {
              const size_t off = (peer_env * p.peer_tmax + (size_t)(t + 1 - rew_per)) * p.Np + lane;
              for (int d = 0; d < p.n_peers; ++d) store_stream(p.peer_rew[d] + off, st_rew);
            }
            sc_rew = 0;
          }
        }
        // ---- evaders / poison drift; bounce only if BOTH coordinates left [0,1]: ww:397-409 ---------
#pragma unroll
        for (int c = 0; c < OPL; ++c) {
          if (((mE[c] | mP[c]) >> lane) & 1u) {
            x[c] += vx[c]; y[c] += vy[c];
            const bool ox = (x[c] < (real)0) || (x[c] > (real)1), oy = (y[c] < (real)0) || (y[c] > (real)1);
            if (ox && oy) { vx[c] = -vx[c]; vy[c] = -vy[c]; }
          }
        }
        // ---- bookkeeping ww:433-436 + VecEnvExecutor horizon ---------------------------------------
        tt += 1;
        need_reset = false;
        if (!pass) {
          ts += 1;
          const bool done = (tt >= p.timestep_limit) || (p.max_path_length > 0 && ts >= p.max_path_length);
          if (lane == 0) {
            p.done[te] = done ? 1 : 0;
            reinterpret_cast<int2*>(p.info)[te] = make_int2(nE, nP);
          }
          if (PEER && p.n_peers > 0) {  // stage done / info of step t in lane t % 32; flush every 32 steps
            if (lane == (t & 31)) { st_info = make_int2(nE, nP); st_done = done ? 1 : 0; }
            if ((t & 31) == 31 || t == p.T - 1) {
              if (lane <= (t & 31)) {
                const size_t off = peer_env * p.peer_tmax + (size_t)(t & ~31) + lane;
                for (int d = 0; d < p.n_peers; ++d) {
                  p.peer_done[d][off] = st_done;
                  reinterpret_cast<int2*>(p.peer_info[d])[off] = st_info;
                }
              }
            }
          }
          // VecEnvExecutor.step: a done env is reset in place and its obs slot receives the
          // reset observation (rllab/sandbox/rocky/tf/envs/vec_env_executor.py:24-27)
          need_reset = done && p.auto_reset;
          if (need_reset) {   // the rows' bulk stores must land before they are read back or rewritten by the reset pass
            if (!WRITER && lane == 0) bulk_wait_all();
            __syncwarp();
          }
          if (need_reset && p.term_obs != nullptr) {
            // WRITER: the terminal rows are still in the slot, which the reset pass overwrites before the writer
            // warp sees it, so HBM gets the reset rows once
            if constexpr (WRITER) keep_terminal_rows_staged<O>(wr.step_rows(), p.term_obs + (obs_t - p.obs), p.Np * p.D, lane);
            else keep_terminal_rows(obs_t, p.term_obs + (obs_t - p.obs), p.Np * p.D, lane);
          }
        }
        pass = need_reset ? 1 : 0;
      } while (need_reset);
      if constexpr (WRITER) {   // hand the slot to the writer warp; the last env of a partial group also arrives for the absent ones
        if constexpr (kWrBulk) fence_async_shared();
        __syncwarp();
        if (lane == 0) mbar_arrive(wr.bar + 8u * wr.s, e + 1 == p.E ? (uint32_t)(kWrEnvs - wr_warp) : 1u);
        if (++wr.s == kWrSlots) { wr.s = 0; wr.phase ^= 1u; }
      }
      obs_t += p.obs_step;
      act_t += p.agent_step;
      rew_t += p.agent_step;
      te += (size_t)p.E;
    }
    if (PEER && p.n_peers > 0 && sc_rew > 0 && lane < sc_rew * p.Np) {   // partial reward run at the end
      const size_t off = (peer_env * p.peer_tmax + (size_t)(p.T - sc_rew)) * p.Np + lane;
      for (int d = 0; d < p.n_peers; ++d) store_stream(p.peer_rew[d] + off, st_rew);
    }
    // ---- registers -> HBM record ------------------------------------------------------------------
#pragma unroll
    for (int c = 0; c < OPL; ++c) {
      const int o = lane + 32 * c;
      if (o < Nall) { rec[o] = x[c]; rec[Nall + o] = y[c]; rec[2 * Nall + o] = vx[c]; rec[3 * Nall + o] = vy[c]; }
    }
    if (lane == 0) {
      p.obst[2 * (size_t)e] = obx; p.obst[2 * (size_t)e + 1] = oby;
      p.timestep[e] = tt; p.path_len[e] = ts; p.ctr[e] = ctr;
    }
  }
  if (!WRITER && lane == 0) bulk_wait_all();   // the last bulk store has read its source before the block exits
}

}  // namespace madrl

// =================================================================================================
// Host side: C ABI
// =================================================================================================
using namespace madrl;

struct madrl_ww : EngineCore {
  madrl_ww_config cfg;
  madrl_ww_layout lay;
  // peer gather buffers (multi-GPU fused exchange); n_peers == 0: disabled
  int n_peers, peer_rank, peer_tmax;
  void* peer_rew[8];
  void* peer_done[8];
  void* peer_info[8];
  int obs_writer = MADRL_WW_OBS_WRITER_AUTO;   // set_obs_writer
  int heuristic_norm = MADRL_HEURISTIC_NORM_AGENT;   // set_heuristic_norm

  StepBytes step_bytes() const {
    const size_t E = cfg.n_envs, Np = cfg.n_pursuers, rb = lay.real_bytes;
    return {E * Np * 2 * rb, E * Np * lay.obs_dim * obs_elem_bytes(rb), E * Np * rb, E, E * 2 * 4};
  }
};

static int ww_validate(const madrl_ww_config* c) {
  MADRL_REQUIRE(c != nullptr, "config is NULL");
  MADRL_REQUIRE(c->n_envs > 0, "n_envs must be > 0");
  MADRL_REQUIRE(c->n_pursuers >= 1 && c->n_pursuers <= 32,
                "n_pursuers must be in [1,32] (collision rows are 32-bit masks), got %d", c->n_pursuers);
  MADRL_REQUIRE(c->n_evaders >= 1 && c->n_poison >= 1, "n_evaders and n_poison must be >= 1");
  MADRL_REQUIRE(c->n_sensors >= 1 && c->n_sensors <= 64, "n_sensors must be in [1,64], got %d", c->n_sensors);
  MADRL_REQUIRE(c->n_pursuers + c->n_evaders + c->n_poison <= 256,
                "n_pursuers + n_evaders + n_poison must be <= 256 (8 objects per lane)");
  MADRL_REQUIRE(c->n_coop >= 1, "n_coop must be >= 1");
  MADRL_REQUIRE(c->timestep_limit >= 1, "timestep_limit must be >= 1");
  return MADRL_OK;
}

extern "C" int madrl_ww_state_layout(const madrl_ww_config* c, madrl_ww_layout* out) {
  int rc = ww_validate(c);
  if (rc) return rc;
  MADRL_REQUIRE(out != nullptr, "layout out is NULL");
  const size_t rb = c->fp64 ? 8 : 4, E = (size_t)c->n_envs;
  const size_t nobj = (size_t)c->n_pursuers + c->n_evaders + c->n_poison;
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off = align_up(off + bytes, 256); return o; };
  out->rng_counter = take(8 * E);
  out->objs = take(rb * 4 * nobj * E);
  out->obst = take(rb * 2 * E);
  out->timestep = take(4 * E);
  out->path_len = take(4 * E);
  out->sensors = take(rb * 2 * (size_t)c->n_sensors);
  out->total_bytes = off;
  out->n_obj = (int32_t)nobj;
  out->obs_dim = c->n_sensors * (c->speed_features ? 7 : 4) + 2 + (c->addid ? 1 : 0);  // ww:18-24
  out->real_bytes = (int32_t)rb;
  out->_pad = 0;
  return MADRL_OK;
}

extern "C" int madrl_ww_create(const madrl_ww_config* c, void* state_dev, madrl_ww** out) {
  return engine_create(c, state_dev, out, madrl_ww_state_layout, upload_sensors<madrl_ww>);
}

extern "C" int madrl_ww_destroy(madrl_ww* h) { return engine_destroy(h); }

extern "C" void* madrl_ww_state_ptr(madrl_ww* h) { return h ? h->state : nullptr; }

HandleView<madrl_ww_config, madrl_ww_layout> madrl::handle_view(const madrl_ww* h) {
  return {&h->cfg, &h->lay, h->state};
}

extern "C" int madrl_ww_seed(madrl_ww* h, uint64_t seed, void* stream) { return engine_seed(h, seed, stream); }

extern "C" int madrl_ww_set_peers(madrl_ww* h, int n_peers, int rank, int t_max, void* const* rew_peers,
                                  void* const* done_peers, void* const* info_peers) {
  MADRL_REQUIRE(h != nullptr, "handle is NULL");
  MADRL_REQUIRE(n_peers >= 0 && n_peers <= 8, "n_peers must be in [0,8], got %d", n_peers);
  if (n_peers == 0) { h->n_peers = 0; return MADRL_OK; }
  MADRL_REQUIRE(rank >= 0 && t_max >= 1, "bad slot / t_max");
  MADRL_REQUIRE(rew_peers && done_peers && info_peers, "NULL peer pointer table");
  for (int d = 0; d < n_peers; ++d) {
    MADRL_REQUIRE(rew_peers[d] && done_peers[d] && info_peers[d], "NULL peer buffer %d", d);
    MADRL_REQUIRE(((uintptr_t)info_peers[d] & 7) == 0, "peer info buffer %d must be 8-byte aligned", d);
    h->peer_rew[d] = rew_peers[d]; h->peer_done[d] = done_peers[d]; h->peer_info[d] = info_peers[d];
  }
  h->n_peers = n_peers; h->peer_rank = rank; h->peer_tmax = t_max;
  return MADRL_OK;
}

extern "C" int madrl_ww_set_terminal_obs(madrl_ww* h, void* term_obs_dev) {
  return engine_set_terminal_obs(h, term_obs_dev);
}

extern "C" int madrl_ww_set_obs_format(madrl_ww* h, int format) {
  return engine_set_obs_format(h, format, h != nullptr && h->cfg.fp64);
}

extern "C" int madrl_ww_set_obs_cache(madrl_ww* h, int mode) {
  return engine_set_obs_cache(h, mode, h != nullptr && h->cfg.fp64);
}

extern "C" int madrl_ww_set_launch(madrl_ww* h, int warps_per_block, int blocks_per_sm) {
  return engine_set_launch(h, warps_per_block, blocks_per_sm);
}

extern "C" int madrl_ww_set_obs_writer(madrl_ww* h, int mode) {
  MADRL_REQUIRE(h != nullptr, "handle is NULL");
  MADRL_REQUIRE(mode == MADRL_WW_OBS_WRITER_AUTO || mode == MADRL_WW_OBS_WRITER_OFF || mode == MADRL_WW_OBS_WRITER_ON,
                "unknown observation writer mode %d", mode);
  h->obs_writer = mode;
  return MADRL_OK;
}

extern "C" int madrl_ww_set_heuristic_norm(madrl_ww* h, int norm) {
  MADRL_REQUIRE(h != nullptr, "handle is NULL");
  MADRL_REQUIRE(norm == MADRL_HEURISTIC_NORM_AGENT || norm == MADRL_HEURISTIC_NORM_ENV,
                "unknown heuristic norm %d", norm);
  h->heuristic_norm = norm;
  return MADRL_OK;
}

template <typename real>
static size_t ww_cand_bytes(int opl, int n_obj) { return opl >= 2 ? (size_t)n_obj * CandSlot<real>::kStride : 0; }

// The library's default cap on resident env warps per SM for an open-loop rollout of T steps with float32
// observations (0 = as many as fit; set_launch overrides it).  Where it caps, the writer-warp kernel runs if it
// can (ww_use_writer), with that many env warps per SM; else one-warp blocks.  See DESIGN §4.3 for the numbers
// behind each condition, measured on C2 (5 pursuers, 4096 envs: 2.17 -> 2.02 ms per 256-step launch):
//   * whole-step staging only: the C2 kernel computes about as fast with 16 warps per SM, each stepping two
//     envs in turn, as with 31, but its observation stores overlap the sensing better.  The ring staging of
//     larger env-steps (C4) and bfloat16 observations gain nothing or lose at 16;
//   * T >= 16: a launch of a step or a few has no later steps for the stores to overlap with;
//   * 16 x SMs warps split the envs into at least two rounds and the last is at least 4/5 full: a mostly
//     empty last round (e.g. 3000 envs on 132 SMs: 2112 + 888) costs more than the overlap saves.
static int ww_default_blocks_per_sm(const madrl_ww* h, int T) {
  const madrl_ww_config& c = h->cfg;
  if (c.fp64 || h->obs_format != MADRL_OBS_NATIVE || T < 16) return 0;
  const int opl = (h->lay.n_obj + 31) / 32;
  if (ww_cand_bytes<float>(opl, h->lay.n_obj) + obs_stage_bytes(c.n_pursuers * h->lay.obs_dim, sizeof(float)) >
      kStepStageMaxBytes)
    return 0;
  const long g = 16L * h->sms, E = c.n_envs, rounds = (E + g - 1) / g;
  return rounds >= 2 && 5 * (E - (rounds - 1) * g) >= 4 * g ? 16 : 0;
}

extern "C" int madrl_ww_default_blocks_per_sm(madrl_ww* h, int T) {
  MADRL_REQUIRE(h != nullptr, "handle is NULL");
  MADRL_REQUIRE(T >= 1, "T must be >= 1");
  return ww_default_blocks_per_sm(h, T);
}

// The launch log (madrl_ww_launch_log, see LaunchLog): one record per ww_kernel launch.
static LaunchLog<10> g_ww_log;

template <typename real, typename O, int OPL, int KCH, int KC, bool PEER, int POLICY, bool KEEP, bool WRITER>
static void ww_log_launch(int grid) {
  g_ww_log.add({(int32_t)sizeof(real), (int32_t)sizeof(O), OPL, KCH, KC, PEER, POLICY, KEEP, WRITER, grid});
}

extern "C" int madrl_ww_launch_log(int enable, int32_t* records, int max_records) {
  return g_ww_log.read(enable, records, max_records);
}

template <typename real, typename O, int OPL, int KCH, int KC, bool PEER, int POLICY, bool KEEP = false>
static int ww_launch_inst2(madrl_ww* h, const WWParams<real, O>& p, int cap, cudaStream_t stream) {
  const size_t smem = ww_cand_bytes<real>(OPL, p.Nall) + (p.stage_step ? obs_stage_bytes(p.Np * p.D, sizeof(O))
                                                                        : 2 * obs_stage_bytes(p.K * (p.speed_features ? 7 : 4), sizeof(O)));
  int grid = 0;
  const int rc = engine_launch(h, ww_kernel<real, O, OPL, KCH, KC, PEER, POLICY, KEEP>, smem, p.E, stream, p, cap, &grid);
  if (rc == MADRL_OK) ww_log_launch<real, O, OPL, KCH, KC, PEER, POLICY, KEEP, false>(grid);
  return rc;
}

// Whether a plain open-loop float32 rollout (no policy, peers or KEEP) of at most 32 objects runs on the writer-warp
// kernel.  It needs whole-step staging, and a 16-byte-aligned observation base and step stride, so that every group's rows start on a
// 16-byte boundary; otherwise, or with set_obs_writer(OFF), the one-warp kernel runs.  By default (AUTO) it replaces
// the launches ww_default_blocks_per_sm caps, unless set_launch chose a geometry; ON takes it wherever it can run.
static bool ww_use_writer(const madrl_ww* h, const WWParams<float, float>& p) {
  if (h->obs_writer == MADRL_WW_OBS_WRITER_OFF || p.mode != 0 || !p.stage_step) return false;
  if (((uintptr_t)p.obs | (uintptr_t)(p.obs_step * sizeof(float))) & 15u) return false;
  return h->obs_writer == MADRL_WW_OBS_WRITER_ON || (h->blocks_per_sm == 0 && ww_default_blocks_per_sm(h, p.T) > 0);
}

// The writer-warp kernel: kWrThreads-thread blocks, kWrBlocksPerSm of them per SM (fewer if they do not fit), each
// looping over groups of kWrEnvs adjacent envs.
template <int OPL, int KCH, int KC>
static int ww_launch_writer(madrl_ww* h, const WWParams<float, float>& p, cudaStream_t stream) {
  auto kfn = ww_kernel<float, float, OPL, KCH, KC, false, 0, false, true>;
  const size_t smem = kWrBarBytes + kWrEnvs * ww_cand_bytes<float>(OPL, p.Nall) +
                      kWrSlots * (size_t)wr_slot_bytes(p.Np * p.D * (int)sizeof(float));
  MADRL_CUDA_CHECK(cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int resident = 0;
  MADRL_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident, kfn, kWrThreads, smem));
  MADRL_REQUIRE(resident >= 1, "the writer-warp kernel does not fit an SM (%zu bytes of shared memory)", smem);
  const int per_sm = resident < kWrBlocksPerSm ? resident : kWrBlocksPerSm;
  const int groups = (p.E + kWrEnvs - 1) / kWrEnvs;
  const int grid = groups < h->sms * per_sm ? groups : h->sms * per_sm;
  MADRL_LAUNCH(kfn, grid, kWrThreads, smem, stream, p);
  g_launches.fetch_add(1);
  MADRL_CUDA_CHECK(cudaGetLastError());
  ww_log_launch<float, float, OPL, KCH, KC, false, 0, false, true>(grid);
  return MADRL_OK;
}

// The fused peer exchange is instantiated for native observations only (bf16 rollouts with peers are
// rejected in ww_launch): it adds nothing to the observation path.
template <typename real, typename O, int OPL, int KCH, int KC>
static int ww_launch_inst(madrl_ww* h, const WWParams<real, O>& p, cudaStream_t stream) {
  if (p.policy_obs0 != nullptr)
    return h->heuristic_norm == MADRL_HEURISTIC_NORM_ENV
               ? ww_launch_inst2<real, O, OPL, KCH, KC, false, kWwPolicyEnv>(h, p, 0, stream)
               : ww_launch_inst2<real, O, OPL, KCH, KC, false, kWwPolicyAgent>(h, p, 0, stream);
  if constexpr (sizeof(O) == sizeof(real))
    if (p.n_peers > 0) return ww_launch_inst2<real, O, OPL, KCH, KC, true, 0>(h, p, 0, stream);
  // only the plain open-loop rollout was measured with the default cap
  const int cap = p.mode == 0 ? ww_default_blocks_per_sm(h, p.T) : 0;
  if constexpr (sizeof(real) == 4)   // set_obs_cache refuses KEEP on fp64 handles
    if (p.mode == 0 && h->obs_cache == MADRL_OBS_CACHE_KEEP)
      return ww_launch_inst2<real, O, OPL, KCH, KC, false, 0, true>(h, p, cap, stream);
  // (with more than 32 objects, the writer instantiations spill registers at 2 blocks of 288 threads per SM)
  if constexpr (sizeof(real) == 4 && sizeof(O) == 4 && OPL == 1)
    if (ww_use_writer(h, p)) return ww_launch_writer<OPL, KCH, KC>(h, p, stream);
  return ww_launch_inst2<real, O, OPL, KCH, KC, false, 0>(h, p, cap, stream);
}

template <typename real, typename O>
static int ww_launch_t(madrl_ww* h, int mode, int T, const void* actions, void* obs, void* rew,
                       uint8_t* done, int32_t* info, const uint8_t* mask, int auto_reset,
                       cudaStream_t stream, const void* policy_obs0, void* actions_out) {
  const madrl_ww_config& c = h->cfg;
  WWParams<real, O> p;
  p.E = c.n_envs; p.env_id_base = c.env_id_base;
  p.Np = c.n_pursuers; p.Ne = c.n_evaders; p.Npo = c.n_poison; p.K = c.n_sensors;
  p.n_coop = c.n_coop; p.D = h->lay.obs_dim; p.Nall = h->lay.n_obj;
  p.reward_global = c.reward_global; p.addid = c.addid; p.speed_features = c.speed_features;
  p.random_obstacle = c.random_obstacle; p.timestep_limit = c.timestep_limit;
  p.max_path_length = c.max_path_length;
  p.T = T; p.mode = mode; p.auto_reset = auto_reset;
  p.obs_step = (size_t)p.E * p.Np * p.D; p.agent_step = (size_t)p.E * p.Np;
  // radii ww:108-118 (double arithmetic as in the reference, then narrowed once)
  const double r_p = c.radius, r_e = c.radius * 2, r_po = c.radius * 3 / 4;
  // the sensing thresholds rounded down, so that `x > thr` of a `real` x decides as the reference's double test
  p.r_p2 = round_down<real>(r_p * r_p);
  p.range = round_down<real>(c.sensor_range);
  p.range_up = std::nextafter(p.range, (real)INFINITY);
  // Exact conservative cull: sv <= range and d2 - sv^2 <= r^2 imply d2 <= range^2 + r^2.
  p.cull2 = (real)((c.sensor_range * c.sensor_range + r_p * r_p) * (1.0 + 1e-4) + 1e-12);
  p.coll2_e = exact_sq_threshold<real>(r_p + r_e);
  p.coll2_po = exact_sq_threshold<real>(r_p + r_po);
  p.obst2_p = exact_sq_threshold<real>(r_p + c.obstacle_radius);
  p.obst2_e = exact_sq_threshold<real>(r_e + c.obstacle_radius);
  p.obst2_po = exact_sq_threshold<real>(r_po + c.obstacle_radius);
  p.resp2_p = exact_sq_threshold<real>(r_p * 2 + c.obstacle_radius);
  p.resp2_e = exact_sq_threshold<real>(r_e * 2 + c.obstacle_radius);
  p.resp2_po = exact_sq_threshold<real>(r_po * 2 + c.obstacle_radius);
  p.obst_x = (real)c.obstacle_x; p.obst_y = (real)c.obstacle_y;
  p.ev_speed = (real)c.ev_speed; p.poison_speed = (real)c.poison_speed;
  p.action_scale = (real)c.action_scale;
  p.poison_reward = (real)c.poison_reward; p.food_reward = (real)c.food_reward;
  p.encounter_reward = (real)c.encounter_reward; p.control_penalty = (real)c.control_penalty;
  p.seed = c.seed;
  char* st = h->state;
  p.objs = (real*)(st + h->lay.objs);
  p.obst = (real*)(st + h->lay.obst);
  p.timestep = (int32_t*)(st + h->lay.timestep); p.path_len = (int32_t*)(st + h->lay.path_len);
  p.ctr = (uint64_t*)(st + h->lay.rng_counter);
  p.sensors = (const real*)(st + h->lay.sensors);
  p.actions = (const real*)actions; p.obs = (O*)obs; p.rew = (real*)rew;
  p.done = done; p.info = info; p.mask = mask;
  p.term_obs = (mode == 0) ? (O*)h->term_obs : nullptr;
  p.policy_obs0 = (const O*)policy_obs0; p.actions_out = (real*)actions_out;
  // the policy instantiation is single-GPU: its rows go through the copy-engine exchange, not peer stores
  p.n_peers = (mode == 0 && policy_obs0 == nullptr) ? h->n_peers : 0;
  p.peer_rank = h->peer_rank;
  MADRL_REQUIRE(p.n_peers == 0 || sizeof(O) == sizeof(real), "the fused peer exchange needs native observations (set_obs_format)");
  if (p.n_peers > 0) {
    MADRL_REQUIRE(T <= h->peer_tmax, "rollout of %d steps exceeds the peer buffers (t_max %d)", T, h->peer_tmax);
    p.peer_tmax = h->peer_tmax;
    for (int d = 0; d < 8; ++d) {
      p.peer_rew[d] = (real*)h->peer_rew[d % p.n_peers];
      p.peer_done[d] = (uint8_t*)h->peer_done[d % p.n_peers];
      p.peer_info[d] = (int32_t*)h->peer_info[d % p.n_peers];
    }
  }

  const int opl = (p.Nall + 31) / 32, kch = (p.K + 31) / 32;
  p.stage_step = ww_cand_bytes<real>(opl, p.Nall) + obs_stage_bytes(p.Np * p.D, sizeof(O)) <= kStepStageMaxBytes;
#define MADRL_WW_CASE(OP, KH, KC_) return ww_launch_inst<real, O, OP, KH, KC_>(h, p, stream)
  if (p.K == 30 && p.speed_features) {   // the reference's defaults (n_sensors = 30, speed features): compile-time K and layout
    if (opl == 1) MADRL_WW_CASE(1, 1, 30);
    if (opl == 2) MADRL_WW_CASE(2, 1, 30);
    if (opl <= 4) MADRL_WW_CASE(4, 1, 30);
    MADRL_WW_CASE(8, 1, 30);
  } else if (kch == 1) {
    if (opl == 1) MADRL_WW_CASE(1, 1, 0);
    if (opl == 2) MADRL_WW_CASE(2, 1, 0);
    if (opl <= 4) MADRL_WW_CASE(4, 1, 0);
    MADRL_WW_CASE(8, 1, 0);
  } else {
    if (opl == 1) MADRL_WW_CASE(1, 2, 0);
    if (opl == 2) MADRL_WW_CASE(2, 2, 0);
    if (opl <= 4) MADRL_WW_CASE(4, 2, 0);
    MADRL_WW_CASE(8, 2, 0);
  }
#undef MADRL_WW_CASE
}

// fp64 verification build, fp32 with fp32 observations, or fp32 with bfloat16 observations
static int ww_launch(madrl_ww* h, int mode, int T, const void* actions, void* obs, void* rew,
                     uint8_t* done, int32_t* info, const uint8_t* mask, int auto_reset,
                     cudaStream_t stream, const void* policy_obs0 = nullptr, void* actions_out = nullptr) {
  if (h->cfg.fp64)
    return ww_launch_t<double, double>(h, mode, T, actions, obs, rew, done, info, mask, auto_reset, stream, policy_obs0, actions_out);
  if (h->obs_format == MADRL_OBS_BF16)
    return ww_launch_t<float, uint16_t>(h, mode, T, actions, obs, rew, done, info, mask, auto_reset, stream, policy_obs0, actions_out);
  return ww_launch_t<float, float>(h, mode, T, actions, obs, rew, done, info, mask, auto_reset, stream, policy_obs0, actions_out);
}

extern "C" int madrl_ww_reset(madrl_ww* h, const uint8_t* mask_dev, void* obs_dev, void* stream) {
  MADRL_REQUIRE(h != nullptr && obs_dev != nullptr, "handle/obs is NULL");
  return ww_launch(h, 1, 1, nullptr, obs_dev, nullptr, nullptr, nullptr, mask_dev, 0, (cudaStream_t)stream);
}

extern "C" int madrl_ww_rollout(madrl_ww* h, int T, const void* actions_dev, void* obs_dev,
                                void* rew_dev, uint8_t* done_dev, int32_t* info_dev,
                                int auto_reset, void* stream) {
  MADRL_REQUIRE(h != nullptr, "handle is NULL");
  MADRL_REQUIRE(T >= 1, "T must be >= 1");
  MADRL_REQUIRE(actions_dev && obs_dev && rew_dev && done_dev && info_dev, "NULL trajectory buffer");
  MADRL_REQUIRE(((uintptr_t)info_dev & 7) == 0, "info_dev must be 8-byte aligned (rows are stored as one 8-byte word)");
  return ww_launch(h, 0, T, actions_dev, obs_dev, rew_dev, done_dev, info_dev, nullptr, auto_reset, (cudaStream_t)stream);
}

extern "C" int madrl_ww_rollout_heuristic(madrl_ww* h, int T, const void* obs0_dev, void* actions_out_dev,
                                          void* obs_dev, void* rew_dev, uint8_t* done_dev, int32_t* info_dev,
                                          int auto_reset, void* stream) {
  MADRL_REQUIRE(h != nullptr, "handle is NULL");
  MADRL_REQUIRE(T >= 1, "T must be >= 1");
  MADRL_REQUIRE(obs0_dev && obs_dev && rew_dev && done_dev && info_dev, "NULL trajectory buffer");
  MADRL_REQUIRE(((uintptr_t)info_dev & 7) == 0, "info_dev must be 8-byte aligned (rows are stored as one 8-byte word)");
  MADRL_REQUIRE(((uintptr_t)actions_out_dev & (h->cfg.fp64 ? 15 : 7)) == 0, "actions_out_dev must be aligned to one (x, y) pair");
  MADRL_REQUIRE(h->cfg.speed_features, "the heuristic policy reads the 7K feature layout (speed_features=True; "
                                       "heuristics/waterworld.py:12-22)");
  return ww_launch(h, 0, T, nullptr, obs_dev, rew_dev, done_dev, info_dev, nullptr, auto_reset, (cudaStream_t)stream,
                   obs0_dev, actions_out_dev);
}

extern "C" int madrl_ww_step(madrl_ww* h, const void* actions_dev, void* obs_dev, void* rew_dev,
                             uint8_t* done_dev, int32_t* info_dev, int auto_reset, void* stream) {
  return madrl_ww_rollout(h, 1, actions_dev, obs_dev, rew_dev, done_dev, info_dev, auto_reset, stream);
}

// ---- host-buffer entry points -------------------------------------------------------------------
extern "C" int madrl_ww_reset_host(madrl_ww* h, const uint8_t* mask_host, void* obs_host) {
  return engine_reset_host(h, mask_host, obs_host,
                           [h](uint8_t* mask, char* obs) { return madrl_ww_reset(h, mask, obs, nullptr); });
}

extern "C" int madrl_ww_rollout_host2(madrl_ww* h, int T, const void* actions_host, void* obs_host,
                                      void* rew_host, uint8_t* done_host, int32_t* info_host,
                                      int auto_reset, int flags) {
  // Each chunk is a launch of its own, and a launch writes its peer rows from step 0 of the gather buffers.
  // Refused whatever the chunk count, which depends on the buffer sizes (madrl_set_host_chunk_bytes).
  MADRL_REQUIRE(h == nullptr || h->n_peers == 0,
                "the host-buffer rollout runs in chunked launches, which the fused peer exchange does not support: "
                "clear set_peers first");
  return engine_rollout_host(h, T, actions_host, obs_host, rew_host, done_host, info_host, flags,
                             [&](int Tc, char* a, char* o, char* r, char* d, char* i, cudaStream_t st) {
                               return madrl_ww_rollout(h, Tc, a, o, r, (uint8_t*)d, (int32_t*)i, auto_reset, st);
                             });
}

extern "C" int madrl_ww_rollout_host(madrl_ww* h, int T, const void* actions_host, void* obs_host,
                                     void* rew_host, uint8_t* done_host, int32_t* info_host,
                                     int auto_reset) {
  return madrl_ww_rollout_host2(h, T, actions_host, obs_host, rew_host, done_host, info_host, auto_reset, 0);
}
