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
// C2: 72 regs + spills -> 56, none).

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
#endif  // MADRL_EMU_PTX_HELPERS

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

template <typename real>
__device__ __forceinline__ real clip01(real x) {
  return x < (real)0 ? (real)0 : (x > (real)1 ? (real)1 : x);
}

}  // namespace madrl
