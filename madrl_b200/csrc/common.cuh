// Shared host/device helpers for the madrl_b200 C-ABI library.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>

#include "../../include/madrl_b200.h"

namespace madrl {

void set_error(const char* fmt, ...);
extern std::atomic<uint64_t> g_launches;
extern std::atomic<size_t> g_host_chunk_bytes;   // device->host bytes per chunk of the host-buffer rollouts
int sm_count(int device);

#define MADRL_CUDA_CHECK(expr)                                                          \
  do {                                                                                  \
    cudaError_t _e = (expr);                                                            \
    if (_e != cudaSuccess) {                                                            \
      madrl::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, \
                       __LINE__);                                                       \
      return MADRL_ECUDA;                                                               \
    }                                                                                   \
  } while (0)

#define MADRL_REQUIRE(cond, ...)      \
  do {                                \
    if (!(cond)) {                    \
      madrl::set_error(__VA_ARGS__);  \
      return MADRL_EINVAL;            \
    }                                 \
  } while (0)

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

constexpr unsigned FULL_MASK = 0xffffffffu;

template <typename real>
__device__ __forceinline__ real real_inf();
template <>
__device__ __forceinline__ float real_inf<float>() { return __int_as_float(0x7f800000); }
template <>
__device__ __forceinline__ double real_inf<double>() {
  return __longlong_as_double(0x7ff0000000000000ll);
}

// Streaming (evict-first) store for write-once trajectory tensors.
template <typename T>
__device__ __forceinline__ void store_stream(T* p, T v) {
  __stcs(p, v);
}

// Observation store of an env kernel: evict-first, or with KEEP (madrl_*_set_obs_cache(MADRL_OBS_CACHE_KEEP)) a
// plain store at normal L2 priority, for a policy that reads this step's rows right after the launch.
template <bool KEEP, typename T>
__device__ __forceinline__ void store_obs(T* p, T v) {
  if constexpr (KEEP) *p = v;
  else store_stream(p, v);
}

// Vector type of an (x, y) pair of `real`.
template <typename real> struct Vec2;
template <> struct Vec2<float> { typedef float2 type; };
template <> struct Vec2<double> { typedef double2 type; };

// Butterfly sum over the full warp: every lane gets the total.  (postproc.cu's `warp_sum` is a
// different reduction whose result lands in lane 0 only.)
template <typename real>
__device__ __forceinline__ real warp_allreduce_sum(real v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL_MASK, v, o);
  return v;
}

// The warp-per-env kernels are launched as 32-thread blocks (one env per block; see engine_launch in
// engine.cuh).  The env index then derives from blockIdx alone, so ptxas can prove the persistent loop
// and every branch on warp-uniform values uniform: the BRA.DIV guards in front of the warp collectives
// disappear, loop bookkeeping moves to the uniform datapath and the register count drops (Waterworld
// C2: 72 regs + spills -> 63, none: 32 resident one-warp blocks per SM, the hardware's block limit).

// Kernels are launched through one macro and the PTX-level helpers below sit behind one guard so
// that the test-only warp emulator (tests/emu: the kernels compiled by g++ against a fake
// <cuda_runtime.h>, lanes run as fibers) can substitute host versions.  Neither is ever defined in
// the product build.
#ifndef MADRL_LAUNCH
#define MADRL_LAUNCH(kfn, grid, block, smem, stream, ...) kfn<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)
#endif

#ifndef MADRL_EMU_PTX_HELPERS
// Explicit shared-window accesses on 32-bit shared addresses.  Keeping ONE 32-bit base address
// in a register (instead of a generic pointer the compiler re-derives from SR_CgaCtaId at every
// use) removes 3-4 instructions per shared-memory access in the hot loops.
__device__ __forceinline__ unsigned lanemask_lt() {
  unsigned m;
  asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
  return m;
}
__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ uint32_t lds_u32(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
  return v;
}
// Byte 0 of a 32-bit shared word.  Only that byte is consumed, so concurrent atomic updates of the
// upper bytes of the same word (Pursuit's packed cell word: building | pursuers << 8 | evaders << 16)
// by other lanes are harmless; the emulator's hazard checker relies on this being a separate helper.
__device__ __forceinline__ uint32_t lds_low_byte(uint32_t a) { return lds_u32(a) & 0xffu; }
__device__ __forceinline__ float lds_f32(uint32_t a) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t lds_u16(uint32_t a) {
  uint32_t v;
  asm volatile("{ .reg .u16 t; ld.shared.u16 t, [%1]; cvt.u32.u16 %0, t; }" : "=r"(v) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ void sts_u32(uint32_t a, uint32_t v) {
  asm volatile("st.shared.u32 [%0], %1;" ::"r"(a), "r"(v) : "memory");
}
__device__ __forceinline__ void sts_u16(uint32_t a, uint32_t v) {
  asm volatile("{ .reg .u16 t; cvt.u16.u32 t, %1; st.shared.u16 [%0], t; }" ::"r"(a), "r"(v) : "memory");
}
__device__ __forceinline__ void reds_add_u32(uint32_t a, uint32_t v) {
  asm volatile("red.shared.add.u32 [%0], %1;" ::"r"(a), "r"(v) : "memory");
}
__device__ __forceinline__ void reds_min_u32(uint32_t a, uint32_t v) {
  asm volatile("red.shared.min.u32 [%0], %1;" ::"r"(a), "r"(v) : "memory");
}
// Staged sensing candidate in shared memory (one slot per object that survives the range cull):
// {rx, ry, d2} = position relative to the sensing agent and its squared norm, {vx, vy} = velocity.
// 32-bit shared addresses, vector accesses: one broadcast load per candidate in the sensor loops.
template <typename real> struct CandSlot;
template <> struct CandSlot<float> {
  static constexpr uint32_t kStride = 32;   // +0 {rx, ry, d2, -}  +16 {vx, vy}
  __device__ static __forceinline__ void put(uint32_t a, float rx, float ry, float d2, float vx, float vy) {
    asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %3};" ::"r"(a), "f"(rx), "f"(ry), "f"(d2) : "memory");
    asm volatile("st.shared.v2.f32 [%0+16], {%1, %2};" ::"r"(a), "f"(vx), "f"(vy) : "memory");
  }
  __device__ static __forceinline__ void geom(uint32_t a, float& rx, float& ry, float& d2) {
    asm volatile("{ .reg .f32 pad; ld.shared.v4.f32 {%0, %1, %2, pad}, [%3]; }" : "=f"(rx), "=f"(ry), "=f"(d2) : "r"(a) : "memory");
  }
  __device__ static __forceinline__ void vel(uint32_t a, float& vx, float& vy) {
    asm volatile("ld.shared.v2.f32 {%0, %1}, [%2+16];" : "=f"(vx), "=f"(vy) : "r"(a) : "memory");
  }
};
template <> struct CandSlot<double> {
  static constexpr uint32_t kStride = 48;   // +0 {rx, ry}  +16 {d2, -}  +32 {vx, vy}
  __device__ static __forceinline__ void put(uint32_t a, double rx, double ry, double d2, double vx, double vy) {
    asm volatile("st.shared.v2.f64 [%0], {%1, %2};" ::"r"(a), "d"(rx), "d"(ry) : "memory");
    asm volatile("st.shared.f64 [%0+16], %1;" ::"r"(a), "d"(d2) : "memory");
    asm volatile("st.shared.v2.f64 [%0+32], {%1, %2};" ::"r"(a), "d"(vx), "d"(vy) : "memory");
  }
  __device__ static __forceinline__ void geom(uint32_t a, double& rx, double& ry, double& d2) {
    asm volatile("ld.shared.v2.f64 {%0, %1}, [%2];" : "=d"(rx), "=d"(ry) : "r"(a) : "memory");
    asm volatile("ld.shared.f64 %0, [%1+16];" : "=d"(d2) : "r"(a) : "memory");
  }
  __device__ static __forceinline__ void vel(uint32_t a, double& vx, double& vy) {
    asm volatile("ld.shared.v2.f64 {%0, %1}, [%2+32];" : "=d"(vx), "=d"(vy) : "r"(a) : "memory");
  }
};

// Pull a line towards L1/L2 without occupying a register (next step's action).
__device__ __forceinline__ void prefetch_l1(const void* p) { asm volatile("prefetch.global.L1 [%0];" ::"l"(p)); }

// Rows staged in shared memory leave through TMA bulk stores (cp.async.bulk, issued by one lane).
// The lanes that wrote the rows fence their shared stores into the async proxy and sync
// with the issuing lane; the issuer waits for the group to have READ its source before the buffer is
// refilled, and for full completion before anything rewrites or re-reads the same global bytes.
__device__ __forceinline__ void sts_real(uint32_t a, float v) { asm volatile("st.shared.f32 [%0], %1;" ::"r"(a), "f"(v) : "memory"); }
__device__ __forceinline__ void sts_real(uint32_t a, double v) { asm volatile("st.shared.f64 [%0], %1;" ::"r"(a), "d"(v) : "memory"); }
template <typename real> __device__ __forceinline__ real lds_real(uint32_t a);
template <> __device__ __forceinline__ float lds_real<float>(uint32_t a) { return lds_f32(a); }
template <> __device__ __forceinline__ double lds_real<double>(uint32_t a) {
  double v;
  asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ void fence_async_shared() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// `bytes` (a multiple of 16) from shared `src` to global `dst` (both 16-byte aligned) as one bulk group,
// L2 evict-first like store_stream.
__device__ __forceinline__ void bulk_store_stream(void* dst, uint32_t src, uint32_t bytes) {
  asm volatile("{ .reg .b64 pol;\n\t"
               "createpolicy.fractional.L2::evict_first.b64 pol, 1.0;\n\t"
               "cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, pol;\n\t"
               "cp.async.bulk.commit_group; }" ::"l"(dst), "r"(src), "r"(bytes) : "memory");
}
// The same without a cache hint: the rows stay in L2 at normal priority (store_obs<true>).
__device__ __forceinline__ void bulk_store_keep(void* dst, uint32_t src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;\n\t"
               "cp.async.bulk.commit_group;" ::"l"(dst), "r"(src), "r"(bytes) : "memory");
}
// Every bulk group / all but the most recent one have finished reading their shared source.
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read_all_but_1() { asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); }
// Every bulk group has completed, and its global writes are ordered before this thread's later
// generic-proxy accesses.
__device__ __forceinline__ void bulk_wait_all() {
  asm volatile("cp.async.bulk.wait_group 0;\n\tfence.proxy.async.global;" ::: "memory");
}
// mbarriers in shared memory (Waterworld's writer-warp ring): init with the number of arrivals that complete a
// phase; arrive (release, CTA scope) `count` of them; wait until the phase of parity `parity` has completed
// (acquire).  A barrier in its first phase counts the phase before it, parity 1, as completed.
__device__ __forceinline__ void mbar_init(uint32_t a, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(a), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t a, uint32_t count) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0], %1;" ::"r"(a), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t a, uint32_t parity) {
  asm volatile("{ .reg .pred p;\n\t"
               "WAIT:\n\t"
               "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
               "@!p bra WAIT; }" ::"r"(a), "r"(parity) : "memory");
}
// The writer warp's reads of Waterworld's writer-warp ring, which the ring's mbarriers order after the env warps'
// staging: 16 bytes, one float, or a 16-byte-aligned run as one evict-first bulk store (bulk_store_stream).  And
// 16 bytes to global memory evict-first (bits moved unchanged).
__device__ __forceinline__ float4 ring_lds_f32x4(uint32_t a) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ float ring_lds_f32(uint32_t a) { return lds_f32(a); }
__device__ __forceinline__ void ring_bulk_store(void* dst, uint32_t src, uint32_t bytes) { bulk_store_stream(dst, src, bytes); }
__device__ __forceinline__ void stcs_f32x4(void* p, float4 v) { __stcs(reinterpret_cast<float4*>(p), v); }
// bfloat16 bits of v, rounded to nearest even (cvt.rn), as a plain uint16_t: no cuda_bf16.h type enters the
// kernels.  The pair form packs `lo` into bits 0-15 (the lower address) and `hi` into bits 16-31.
__device__ __forceinline__ uint16_t bf16_rn(float v) {
  uint16_t r;
  asm("cvt.rn.bf16.f32 %0, %1;" : "=h"(r) : "f"(v));
  return r;
}
__device__ __forceinline__ uint32_t bf16x2_rn(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
#else   // MADRL_EMU_PTX_HELPERS
// Host versions of the bulk-store helpers above for the test emulator, built on the shared-memory
// primitives its <cuda_runtime.h> provides (emu_at, smem_access: the per-byte race checker).  The
// copy happens at issue, recorded as a shared read by the issuing lane, so refilling a staging buffer
// without a __syncwarp after the issue is reported as a race; the waits and fences are no-ops.  The
// alignment cp.async.bulk requires (16-byte addresses and size) is checked.
static inline void sts_real(uint32_t a, float v) { smem_access(a, 4, SMEM_WRITE); memcpy(emu_at(a), &v, 4); }
static inline void sts_real(uint32_t a, double v) { smem_access(a, 8, SMEM_WRITE); memcpy(emu_at(a), &v, 8); }
template <typename real> static inline real lds_real(uint32_t a) {
  smem_access(a, sizeof(real), SMEM_READ);
  real v;
  memcpy(&v, emu_at(a), sizeof v);
  return v;
}
static inline void fence_async_shared() {}
static inline void bulk_store_stream(void* dst, uint32_t src, uint32_t bytes) {
  if (((uintptr_t)dst | src | bytes) & 15u) {
    fprintf(stderr, "madrl_emu: misaligned bulk store dst=%p src=%u bytes=%u\n", dst, src, bytes);
    abort();
  }
  smem_access(src, bytes, SMEM_READ);
  memcpy(dst, emu_at(src), bytes);
}
static inline void bulk_store_keep(void* dst, uint32_t src, uint32_t bytes) { bulk_store_stream(dst, src, bytes); }
static inline void bulk_wait_read_all() {}
static inline void bulk_wait_read_all_but_1() {}
static inline void bulk_wait_all() {}
// mbarriers, on the emulator's warp rendezvous alone.  A barrier's state is its 8 bytes of shared memory: the
// arrivals still pending in the current phase, and the init count with the parity of the current phase in bit 31.
// Arrivals and waits are not plain accesses, so the hazard checker does not see them.  A wait is made by all
// lanes of a warp (as the kernels do): they poll together through warp_exchange, which hands the fiber schedule
// to the other warps, and leave together once every lane has seen the phase complete.  Polling long after the
// last arrival anywhere means a phase that never completes, i.e. a missing arrival: reported, then abort.
static long g_emu_mbar_arrivals = 0;
static inline void mbar_init(uint32_t a, uint32_t count) {
  const uint32_t st[2] = {count, count};
  memcpy(emu_at(a), st, 8);
}
static inline void mbar_arrive(uint32_t a, uint32_t count) {
  uint32_t st[2];
  memcpy(st, emu_at(a), 8);
  if (count == 0 || count > st[0]) {
    fprintf(stderr, "madrl_emu: mbarrier at offset %u: %u arrivals, %u pending in the phase\n", a, count, st[0]);
    abort();
  }
  st[0] -= count;
  if (st[0] == 0) { st[1] ^= 1u << 31; st[0] = st[1] & 0x7fffffffu; }   // phase complete: the next one starts
  memcpy(emu_at(a), st, 8);
  ++g_emu_mbar_arrivals;
}
static inline void mbar_wait(uint32_t a, uint32_t parity) {
  long seen = g_emu_mbar_arrivals, idle = 0;
  while (true) {
    uint32_t st[2];
    memcpy(st, emu_at(a), 8);
    const bool done = (st[1] >> 31) != (parity & 1u);   // the phase of that parity is no longer the current one
    const uint64_t* all = madrl_emu::warp_exchange(done ? 1u : 0u);
    bool every = true;
    for (int l = 0; l < 32; ++l) every = every && (all[l] & 1u);
    if (every) return;
    if (g_emu_mbar_arrivals != seen) { seen = g_emu_mbar_arrivals; idle = 0; }
    else if (++idle > (1L << 20)) {
      fprintf(stderr, "madrl_emu: mbarrier at offset %u never completes its phase of parity %u (block %u): a missing arrival\n",
              a, parity & 1u, blockIdx.x);
      abort();
    }
  }
}
// The writer warp's reads of the ring are ordered by the mbarriers, which the hazard checker (per-lane counts of
// __syncwarp / __syncthreads) cannot follow across warps, so they are not recorded; the env warps' accesses are.
static inline float4 ring_lds_f32x4(uint32_t a) { float4 v; memcpy(&v, emu_at(a), 16); return v; }
static inline float ring_lds_f32(uint32_t a) { float v; memcpy(&v, emu_at(a), 4); return v; }
static inline void ring_bulk_store(void* dst, uint32_t src, uint32_t bytes) {
  if (((uintptr_t)dst | src | bytes) & 15u) {
    fprintf(stderr, "madrl_emu: misaligned bulk store dst=%p src=%u bytes=%u\n", dst, src, bytes);
    abort();
  }
  memcpy(dst, emu_at(src), bytes);
}
static inline void stcs_f32x4(void* p, float4 v) {
  if ((uintptr_t)p & 15u) {
    fprintf(stderr, "madrl_emu: misaligned 16-byte store %p\n", p);
    abort();
  }
  memcpy(p, &v, 16);
}
// Round-to-nearest-even on the bit pattern, as cvt.rn.bf16.f32 rounds finite values and infinities.  A NaN
// maps to some NaN here; which one the hardware returns is not modelled (observations are never NaN).
static inline uint16_t bf16_rn(float v) {
  uint32_t u;
  memcpy(&u, &v, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x40u);
  return (uint16_t)((u + 0x7fffu + ((u >> 16) & 1u)) >> 16);
}
static inline uint32_t bf16x2_rn(float lo, float hi) { return (uint32_t)bf16_rn(lo) | ((uint32_t)bf16_rn(hi) << 16); }
#endif  // MADRL_EMU_PTX_HELPERS

template <bool KEEP>
__device__ __forceinline__ void bulk_store_obs(void* dst, uint32_t src, uint32_t bytes) {
  if constexpr (KEEP) bulk_store_keep(dst, src, bytes);
  else bulk_store_stream(dst, src, bytes);
}

// Observation element type O of an env kernel: its `real`, or uint16_t = bfloat16 bits (with real = float
// only; madrl_*_set_obs_format).  Features are computed in `real` either way and converted once, at the
// store, so a bf16 observation is exactly the rounded fp32 one.
template <typename O, typename real>
__device__ __forceinline__ O obs_cvt(real v) {
  if constexpr (sizeof(O) == 2) return bf16_rn(v);
  else return v;
}
// An observation element read back (the POLICY kernels' obs0) as `real`: bf16 widens exactly.
template <typename real, typename O>
__device__ __forceinline__ real obs_widen(O v) {
  if constexpr (sizeof(O) == 2) return __int_as_float((int)((uint32_t)v << 16));
  else return v;
}
// Shared-memory staging of observation elements (Waterworld's bulk-store rows).
__device__ __forceinline__ void sts_obs(uint32_t a, float v) { sts_real(a, v); }
__device__ __forceinline__ void sts_obs(uint32_t a, double v) { sts_real(a, v); }
__device__ __forceinline__ void sts_obs(uint32_t a, uint16_t v) { sts_u16(a, v); }
template <typename O> __device__ __forceinline__ O lds_obs(uint32_t a) {
  if constexpr (sizeof(O) == 2) return (O)lds_u16(a);
  else return lds_real<O>(a);
}
// Convert a `real` feature value to O and stage it.
template <typename O, typename real>
__device__ __forceinline__ void stage_obs(uint32_t a, real v) { sts_obs(a, obs_cvt<O>(v)); }

// The row of observations action r was taken in, for rollout row r = (t E + e) A + a of src [T][E][A][D], which holds
// the observation AFTER each step.  With `first` (the observations before the rollout, [E][A][D]) that is first[e][a]
// for t = 0 and src[t-1] afterwards (on a done step src already holds the reset observation, i.e. the next
// episode's first one); without it, src[t] as given.  t == 0 <=> r < E A, and then r = e A + a.  I: the index type
// of the caller's row arithmetic.
template <typename I, typename O>
__device__ __forceinline__ const O* action_obs_row(I r, I EA, int D, const O* src, const O* first) {
  return first ? (r < EA ? first + (size_t)r * D : src + (size_t)(r - EA) * D) : src + (size_t)r * D;
}

// Time index of the rows (t, e, .) with te = t E + e: the position in the path, plus t0[e] on env e's first path
// (seg_start from madrl_paths_plan).  The linear baselines' time features and the time-dependent baseline's bins.
template <typename I>
__device__ __forceinline__ int lfb_index(I te, int E, const int32_t* seg_start, const int32_t* t0) {
  const I t = te / (I)E, e = te - t * (I)E;
  const int s = seg_start[te];
  return (int)t - s + ((t0 != nullptr && s == 0) ? t0[e] : 0);
}

// StandardizedEnv sees the TERMINAL observation of an episode before the reset one
// (madrl_environments/__init__.py:283-291 step(), then reset()); under auto-reset the rollout's obs slot is
// overwritten by the reset observation, so -- when the caller asked for it -- the rows of a finished env
// are first copied to the same slot of a side tensor.  Executed by one warp on done steps only.
template <typename T>
__device__ __forceinline__ void keep_terminal_rows(const T* src, T* dst, int n, int lane) {
  __syncwarp();                                   // the rows were stored by other lanes of this warp
  for (int i = lane; i < n; i += 32) dst[i] = __ldcg(src + i);
  __syncwarp();                                   // ... and the reset pass overwrites them next
}
// The same from rows still staged in shared memory at `src` (the caller has synced the warp after staging them).
template <typename O>
__device__ __forceinline__ void keep_terminal_rows_staged(uint32_t src, O* dst, int n, int lane) {
  for (int i = lane; i < n; i += 32) dst[i] = lds_obs<O>(src + (uint32_t)(i * sizeof(O)));
  __syncwarp();                                   // the reset pass overwrites them next
}

template <typename real>
__device__ __forceinline__ real clip01(real x) {
  return x < (real)0 ? (real)0 : (x > (real)1 ? (real)1 : x);
}

// FP64 tensor-core MMA (baseline.cu's Gram kernel) and the float64 shared-memory tile accesses around it.
// mma.m16n8k16.f64: C[16x8] += A[16x16] B[16x8]; lane = 4 g + q (g = lane >> 2, q = lane & 3) holds
//   a[i] = A[g + 8 (i & 1)][q + 4 (i >> 1)],  b[i] = B[q + 4 i][g],  c[i] = C[g + 8 (i >> 1)][2 q + (i & 1)].
#ifndef MADRL_EMU_PTX_HELPERS
__device__ __forceinline__ double lds_f64(const double* p) { return *p; }
__device__ __forceinline__ void sts_f64(double* p, double v) { *p = v; }
__device__ __forceinline__ void mma_f64_16816(double (&c)[4], const double (&a)[8], const double (&b)[4]) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0, %1, %2, %3}, "
               "{%4, %5, %6, %7, %8, %9, %10, %11}, {%12, %13, %14, %15}, {%0, %1, %2, %3};"
               : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
               : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]),
                 "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
}
#else   // MADRL_EMU_PTX_HELPERS
// Host versions: the tile accesses are recorded by the race checker; the MMA gathers every lane's fragment
// registers through the emulator's warp exchange (one rendezvous per register, as the hardware's operand
// collection is warp-wide) and forms each of this lane's four outputs as c + sum_k A[m][k] B[k][n], k ascending.
static inline double lds_f64(const double* p) { smem_access(smem_addr(p), 8, SMEM_READ); return *p; }
static inline void sts_f64(double* p, double v) { smem_access(smem_addr(p), 8, SMEM_WRITE); *p = v; }
static inline void mma_f64_16816(double (&c)[4], const double (&a)[8], const double (&b)[4]) {
  double A[8][32], B[4][32];
  for (int r = 0; r < 8; ++r) {
    const uint64_t* s = madrl_emu::warp_exchange(madrl_emu::to_bits(a[r]));
    for (int l = 0; l < 32; ++l) A[r][l] = madrl_emu::from_bits<double>(s[l]);
  }
  for (int r = 0; r < 4; ++r) {
    const uint64_t* s = madrl_emu::warp_exchange(madrl_emu::to_bits(b[r]));
    for (int l = 0; l < 32; ++l) B[r][l] = madrl_emu::from_bits<double>(s[l]);
  }
  const int lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
  for (int i = 0; i < 4; ++i) {
    const int m = g + 8 * (i >> 1), n = 2 * q + (i & 1);
    double acc = c[i];
    for (int k = 0; k < 16; ++k)   // A[m][k]: lane 4 (m & 7) + (k & 3), register (m >> 3) + 2 (k >> 2);  B[k][n]: lane 4 n + (k & 3), register k >> 2
      acc += A[(m >> 3) + 2 * (k >> 2)][4 * (m & 7) + (k & 3)] * B[k >> 2][4 * n + (k & 3)];
    c[i] = acc;
  }
}
#endif  // MADRL_EMU_PTX_HELPERS

}  // namespace madrl
