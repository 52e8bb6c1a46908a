// rllab's LinearFeatureBaseline (rllab/rllab/baselines/linear_feature_baseline.py) on the rollout tensors,
// decentralized mode: one baseline over the [T][E][A] rows of a rollout, pooled over envs and agents.
//
// Row r = (t, e, a) has the observation o the action of step t was taken in (obs_before[e][a] for t = 0 and
// obs[t-1] afterwards when obs_before is given, obs[t] otherwise) and the time index i = its 0-based position in
// its path (paths cut at `done`, seg_start from madrl_paths_plan), plus t0[e] on env e's first segment.  Its
// features (_features, :19-23), Df = 2 D + 4 of them, and the return y as column Df:
//     [clip(o, -10, 10), clip(o, -10, 10)^2, i/100, (i/100)^2, (i/100)^3, 1 | y]
// Observations are widened to float32 (bfloat16 exactly), clipped, then to float64, where the square is exact.
//
//   madrl_lfb_normal_eq_*  G = [F y]^T [F y] in float64 (the normal equations of fit(), :25-37, with F^T y as
//                          column Df) on the FP64 tensor cores, features generated per chunk of rows in shared
//                          memory: no [N][Df] matrix exists and the workspace does not depend on N.
//   madrl_lfb_predict_*    values[r] = features(r) . c in float64, stored as float32 (predict, :39-43).
//
// Concurrent mode (one baseline per agent, rllab/sandbox/rocky/tf/samplers/batch_ma_sampler.py:64-188): the
// *_agents entry points run the same kernels over A row groups, group a = the rows r = k A + a of agent a.  Each
// group's normal equations read that agent's rows only, so all A systems come from one launch with the same rows,
// tile pairs and MMAs as the pooled one; predict reads coefficient row a for agent a's rows.
//
// rltools' LinearFeatureBaseline (rltools/rltools/baselines/linear.py) is the same pair of kernels with another
// feature map (the kMap template parameter, kLfbRltools; entry points madrl_lfbr_*): Df = D + 3 features
//     [(o - mu) / s, i/100, (i/100)^2, 1 | y]
// where mu and s are the baseline's obsnorm (nn.Standardizer) per column, passed as float64 `norm` [2][D] (mean,
// stdev + eps; [A][2][D] per agent), o is widened to float64 and not clipped, and the quotient is a float64
// division, as NumPy takes it.  norm == NULL is the NoOpStandardizer: the columns are o itself.
#include "common.cuh"

namespace madrl {

// Gram kernel: the (Df+1)-column matrix is cut into 64-column tiles; a CTA owns one tile pair (I <= J) of one
// row slice and accumulates F_I^T F_J over the slice in registers (mma.m16n8k16.f64: M = columns of tile I,
// N = columns of tile J, K = rows).  kLfbSlices fixed row slices, independent of the SM count; the CTAs of one
// slice are adjacent in the grid, so they read the same rows while they sit in L2.  Partial tiles go to the
// workspace and lfb_reduce_kernel sums them over the slices in ascending order: same inputs, same bits.
// Per agent (kAgents): group g = rows k A + g, k in [0, T E), cut into lfb_agent_slices(A) slices; the grid is
// (group, slice, pair) with the pair fastest, so the CTAs of one (group, slice) stay adjacent.  The pooled
// launch is the one-group case with kLfbSlices slices.
constexpr int kLfbTile = 64;
constexpr int kLfbRows = 32;             // rows per shared-memory chunk: 2 MMA k-steps
constexpr int kLfbLd = kLfbTile + 4;     // row pitch (doubles): a half-warp's fragment loads hit 16 distinct bank pairs
constexpr int kLfbThreads = 128;         // 4 warps, each a 32 x 32 quarter of the 64 x 64 tile
#ifndef MADRL_LFB_SLICES
#define MADRL_LFB_SLICES 48              // (the CPU emulator of tests/emu builds with fewer)
#endif
constexpr int kLfbSlices = MADRL_LFB_SLICES;
// The register accumulators are added into the CTA's workspace tile every kLfbFlush chunks (2 048 rows), so no
// float64 sum chain is longer than that: a slice of a C2 launch is 109 000 rows.
constexpr int kLfbFlush = 64;

// The feature maps: rllab's (Df = 2 D + 4) and rltools' (Df = D + 3).  Columns = Df + 1 (the return).
enum LfbMap { kLfbRllab = 0, kLfbRltools = 1 };
template <int kMap>
__host__ __device__ __forceinline__ int lfb_cols(int D) { return kMap == kLfbRllab ? 2 * D + 5 : D + 4; }
template <int kMap>
static inline int lfb_tiles(int D) { return (lfb_cols<kMap>(D) + kLfbTile - 1) / kLfbTile; }
__host__ __device__ __forceinline__ int lfb_agent_slices(int A) { return (kLfbSlices + A - 1) / A; }

// Source row and time index of row r.
template <typename O>
__device__ __forceinline__ const O* lfb_row(size_t r, int E, int A, int D, const O* obs, const O* obs_before,
                                            const int32_t* seg_start, const int32_t* t0, int& idx) {
  idx = lfb_index(r / A, E, seg_start, t0);
  return action_obs_row(r, (size_t)E * A, D, obs, obs_before);
}

// a = i / 100 (correctly rounded, as NumPy's arange(l) / 100.0), a^2 = a * a, a^3 = (a^2 + its rounding error) * a
// rounded once: the correctly rounded cube of a (checked against exact rational arithmetic for every i < 200 000),
// the same on every device and host.  NumPy's al ** 3 (the reference's _features, and oracle/baseline_oracle.py)
// goes through a pow() that is within 1 ulp of it; which indices differ depends on the host's NumPy build and SIMD
// path.
__device__ __forceinline__ void lfb_time(int idx, double& a1, double& a2, double& a3) {
  a1 = (double)idx / 100.0;
  a2 = a1 * a1;
  const double lo = fma(a1, a1, -a2);
  a3 = fma(a2, a1, lo * a1);
}

__device__ __forceinline__ double lfb_clip(float v) { return (double)(v < -10.f ? -10.f : (v > 10.f ? 10.f : v)); }

// The value of observation column d (squared: rllab's second block) from the widened observation v.  rltools:
// (v - mu[d]) / s[d] with norm = [mu | s] ([2][D]), or v itself without an obsnorm.
template <int kMap>
__device__ __forceinline__ double lfb_obs(float v, bool sq, int d, int D, const double* norm) {
  if (kMap == kLfbRllab) {
    const double x = lfb_clip(v);
    return sq ? x * x : x;
  }
  const double x = (double)v;
  return norm ? (x - norm[d]) / norm[D + d] : x;
}

// A row past the slice fetches 0, which gives every rllab feature 0; rltools' standardised 0 is not, so its rows
// past the slice store 0 explicitly.
template <int kMap>
__device__ __forceinline__ double lfb_pad(bool valid, double v) {
  if constexpr (kMap == kLfbRllab) return v;
  else return valid ? v : 0.0;
}

// tile pair p -> (I, J), I <= J, enumerated row by row
__device__ __forceinline__ void lfb_pair(int p, int nb, int& I, int& J) {
  I = 0;
  while (p >= nb - I) { p -= nb - I; ++I; }
  J = I + p;
}

// What a thread's column of a tile holds: an observation value (linear or squared), a time feature, the
// constant, the return, or nothing (padding past Df + 1).
enum LfbKind { kLfbObs = 0, kLfbObsSq, kLfbA1, kLfbA2, kLfbA3, kLfbOne, kLfbY, kLfbPad };

// The 32-bit value a column needs from row r, fetched a chunk ahead: the observation (as float bits), the time
// index, the return (float bits), or 1 / 0 for the constant column (0 on rows past the slice: they add nothing).
template <typename O>
__device__ __forceinline__ uint32_t lfb_fetch(int kind, int d, uint32_t r, bool valid, int E, int A, int D,
                                              const O* obs, const O* obs_before, const int32_t* seg_start,
                                              const int32_t* t0, const float* ret) {
  if (!valid || kind == kLfbPad) return 0u;
  if (kind <= kLfbObsSq)            // row r's source row, no division
    return __float_as_uint(obs_widen<float>(action_obs_row(r, (uint32_t)E * A, D, obs, obs_before)[d]));
  if (kind == kLfbY) return __float_as_uint(ret[r]);
  if (kind == kLfbOne) return 1u;
  return (uint32_t)lfb_index(r / (uint32_t)A, E, seg_start, t0);
}

template <int kMap>
__device__ __forceinline__ double lfb_value(int kind, uint32_t v, int d, int D, const double* norm) {
  if (kind <= kLfbObsSq) return lfb_obs<kMap>(__int_as_float((int)v), kind != kLfbObs, d, D, norm);
  if (kind == kLfbY) return (double)__int_as_float((int)v);
  if (kind == kLfbOne) return (double)v;
  if (kind == kLfbPad) return 0.0;
  double a1, a2, a3;
  lfb_time((int)v, a1, a2, a3);
  return kind == kLfbA1 ? a1 : (kind == kLfbA2 ? a2 : a3);
}

// kAgents = false: one group (every row), kLfbSlices slices.  kAgents = true: A groups of T E rows each (row
// k A + g of group g), lfb_agent_slices(A) slices per group.  The loop runs over the group's row counter k.
// norm: rltools' obsnorm ([groups][2][D], or NULL); the rllab map never reads it.
template <typename O, bool kAgents, int kMap>
__global__ void __launch_bounds__(kLfbThreads, 2)
lfb_gram_kernel(int T, int E, int A, int D, const O* __restrict__ obs, const O* __restrict__ obs_before,
                const int32_t* __restrict__ seg_start, const int32_t* __restrict__ t0, const float* __restrict__ ret,
                double* __restrict__ ws, const double* __restrict__ norm) {
  __shared__ __align__(16) double sF[2][kLfbRows][kLfbLd];   // features of tiles I and J (J only if J != I)
  const int nb = (lfb_cols<kMap>(D) + kLfbTile - 1) / kLfbTile, P = nb * (nb + 1) / 2;
  const int pair = blockIdx.x % P, gs = blockIdx.x / P;      // gs = group * S + slice
  const int S = kAgents ? lfb_agent_slices(A) : kLfbSlices;
  const int group = kAgents ? gs / S : 0, slice = kAgents ? gs - group * S : gs;
  if (kMap == kLfbRltools && kAgents && norm) norm += (size_t)group * 2 * D;
  int I, J;
  lfb_pair(pair, nb, I, J);
  const uint32_t N = kAgents ? (uint32_t)T * E : (uint32_t)T * E * A;   // rows of the group
  const uint32_t r_begin = (uint32_t)((uint64_t)N * slice / S);
  const uint32_t r_end = (uint32_t)((uint64_t)N * (slice + 1) / S);
  // rollout row of the group's k-th row
  auto row_of = [&](uint32_t k) -> uint32_t { return kAgents ? k * (uint32_t)A + (uint32_t)group : k; };
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5, g = lane >> 2, q = lane & 3;
  const int wm = (w & 1) * 32, wn = (w >> 1) * 32;
  const int j = tid & (kLfbTile - 1), k0 = tid >> 6;     // feature fill: column j, rows k0, k0 + 2, ...
  const int nbuf = I == J ? 1 : 2;
  // Most tiles hold observation columns only (plain / squared): they take a fetch and a fill without the kind
  // dispatch (a CTA-uniform branch), which would otherwise cost every value the time-feature path.
  int kind[2], d[2];
  bool obs_only[2];
#pragma unroll
  for (int b = 0; b < 2; ++b) {
    const int tile = b == 0 ? I : J, c = tile * kLfbTile + j;
    if (kMap == kLfbRllab) {
      kind[b] = c < D ? kLfbObs : (c < 2 * D ? kLfbObsSq : (c < 2 * D + 5 ? kLfbA1 + (c - 2 * D) : kLfbPad));
      d[b] = c < D ? c : c - D;
      obs_only[b] = (tile + 1) * kLfbTile <= 2 * D;
    } else {                   // [obs | a1, a2 | 1 | y]
      kind[b] = c < D ? kLfbObs : (c < D + 2 ? kLfbA1 + (c - D) : (c < D + 4 ? kLfbOne + (c - D - 2) : kLfbPad));
      d[b] = c;
      obs_only[b] = (tile + 1) * kLfbTile <= D;
    }
  }
  const uint32_t EA = (uint32_t)E * A;
  double acc[2][4][4];
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[mt][nt][i] = 0.0;

  // every thread owns its 32 elements of the tile: the first flush stores, later ones add (fixed order)
  double* out = ws + ((size_t)gs * P + pair) * (kLfbTile * kLfbTile);
  bool first = true;
  int pending = 0;
  auto flush = [&]() {
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < 4; ++nt)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          double* o = out + (wm + mt * 16 + g + 8 * (i >> 1)) * kLfbTile + wn + nt * 8 + 2 * q + (i & 1);
          *o = first ? acc[mt][nt][i] : *o + acc[mt][nt][i];
          acc[mt][nt][i] = 0.0;
        }
    first = false;
    pending = 0;
  };

  // the values of the next chunk are fetched into registers before the MMAs of the current one
  uint32_t nxt[2][kLfbRows / 2];
  auto fetch = [&](uint32_t r0) {
#pragma unroll
    for (int b = 0; b < 2; ++b) {
      if (b == nbuf) break;
      if (obs_only[b]) {
#pragma unroll
        for (int i = 0; i < kLfbRows / 2; ++i) {
          const uint32_t k = r0 + k0 + 2 * i;
          const O* src = action_obs_row(row_of(k), EA, D, obs, obs_before);
          nxt[b][i] = k < r_end ? __float_as_uint(obs_widen<float>(src[d[b]])) : 0u;
        }
      } else {
#pragma unroll
        for (int i = 0; i < kLfbRows / 2; ++i) {
          const uint32_t k = r0 + k0 + 2 * i;
          nxt[b][i] = lfb_fetch(kind[b], d[b], row_of(k), k < r_end, E, A, D, obs, obs_before, seg_start, t0, ret);
        }
      }
    }
  };
  if (r_begin < r_end) fetch(r_begin);
  for (uint32_t r0 = r_begin; r0 < r_end; r0 += kLfbRows) {
#pragma unroll
    for (int b = 0; b < 2; ++b) {
      if (b == nbuf) break;
      if (obs_only[b]) {
        const bool sq = kind[b] == kLfbObsSq;
#pragma unroll
        for (int i = 0; i < kLfbRows / 2; ++i)
          sts_f64(&sF[b][k0 + 2 * i][j], lfb_pad<kMap>(r0 + k0 + 2 * i < r_end,
                                                       lfb_obs<kMap>(__int_as_float((int)nxt[b][i]), sq, d[b], D, norm)));
      } else {
#pragma unroll
        for (int i = 0; i < kLfbRows / 2; ++i)
          sts_f64(&sF[b][k0 + 2 * i][j], lfb_pad<kMap>(r0 + k0 + 2 * i < r_end,
                                                       lfb_value<kMap>(kind[b], nxt[b][i], d[b], D, norm)));
      }
    }
    __syncthreads();
    if (r0 + kLfbRows < r_end) fetch(r0 + kLfbRows);
    const double(*fB)[kLfbLd] = sF[nbuf - 1];
#pragma unroll
    for (int ks = 0; ks < kLfbRows; ks += 16) {
      double af[2][8];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int i = 0; i < 8; ++i) af[mt][i] = lds_f64(&sF[0][ks + q + 4 * (i >> 1)][wm + mt * 16 + g + 8 * (i & 1)]);
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        double bf[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) bf[i] = lds_f64(&fB[ks + q + 4 * i][wn + nt * 8 + g]);
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) mma_f64_16816(acc[mt][nt], af[mt], bf);
      }
    }
    if (++pending == kLfbFlush) flush();
    __syncthreads();
  }
  if (first || pending) flush();
}

// G[i][j] = G[j][i] = sum over the slices (ascending) of the partial tiles; the upper triangle of a diagonal tile
// is mirrored, so G is exactly symmetric.  One CTA per (group, tile pair), S slices per group;
// G: [groups][Df+1][Df+1].
template <int kMap>
__global__ void lfb_reduce_kernel(int D, int S, const double* __restrict__ ws, double* __restrict__ G) {
  const int Dc = lfb_cols<kMap>(D), nb = (Dc + kLfbTile - 1) / kLfbTile, P = nb * (nb + 1) / 2;
  const int pair = blockIdx.x % P, group = blockIdx.x / P;
  int I, J;
  lfb_pair(pair, nb, I, J);
  ws += (size_t)group * S * P * (kLfbTile * kLfbTile);
  G += (size_t)group * Dc * Dc;
  for (int x = threadIdx.x; x < kLfbTile * kLfbTile; x += blockDim.x) {
    const int m = x / kLfbTile, n = x % kLfbTile, i = I * kLfbTile + m, j = J * kLfbTile + n;
    if (i >= Dc || j >= Dc || (I == J && m > n)) continue;
    double s = 0.0;
    for (int sl = 0; sl < S; ++sl) s += ws[((size_t)sl * P + pair) * (kLfbTile * kLfbTile) + x];
    G[(size_t)i * Dc + j] = s;
    G[(size_t)j * Dc + i] = s;
  }
}

// One warp per row: lanes stride over the D observation values (coalesced), float64 FMAs, butterfly sum.
// kAgents: coef is [A][Df] and row (t, e, a) uses row a (and, rltools, norm block a).
template <typename O, bool kAgents, int kMap>
__global__ void lfb_predict_kernel(int T, int E, int A, int D, const O* __restrict__ obs,
                                   const O* __restrict__ obs_before, const int32_t* __restrict__ seg_start,
                                   const int32_t* __restrict__ t0, const double* __restrict__ coef,
                                   float* __restrict__ values, const double* __restrict__ norm) {
  const size_t r = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= (size_t)T * E * A) return;                  // warp-uniform
  if (kAgents) coef += (size_t)(r % (size_t)A) * (lfb_cols<kMap>(D) - 1);
  int idx;
  const O* src = lfb_row(r, E, A, D, obs, obs_before, seg_start, t0, idx);
  double acc = 0.0;
  if (kMap == kLfbRltools && kAgents && norm) norm += (size_t)(r % (size_t)A) * 2 * D;
  for (int d = lane; d < D; d += 32) {
    if constexpr (kMap == kLfbRllab) {
      const double x = lfb_clip(obs_widen<float>(__ldcs(src + d)));
      acc = fma(x, __ldg(coef + d), acc);
      acc = fma(x * x, __ldg(coef + D + d), acc);
    } else {
      acc = fma(lfb_obs<kMap>(obs_widen<float>(__ldcs(src + d)), false, d, D, norm), __ldg(coef + d), acc);
    }
  }
  acc = warp_allreduce_sum(acc);
  if (lane == 0) {
    double a1, a2, a3;
    lfb_time(idx, a1, a2, a3);
    const double* ct = coef + (kMap == kLfbRllab ? 2 * D : D);
    acc = fma(a1, ct[0], acc);
    acc = fma(a2, ct[1], acc);
    if constexpr (kMap == kLfbRllab) {
      acc = fma(a3, ct[2], acc);
      __stcs(values + r, (float)(acc + ct[3]));
    } else {
      __stcs(values + r, (float)(acc + ct[2]));
    }
  }
}

}  // namespace madrl

using namespace madrl;

static const int kLfbMaxD = 8192;

// Bytes of scratch for `groups` row groups of S slices each.
template <int kMap>
static size_t lfb_ws_bytes(int D, int groups, int S) {
  const size_t nb = (size_t)lfb_tiles<kMap>(D);
  return (size_t)groups * S * (nb * (nb + 1) / 2) * kLfbTile * kLfbTile * sizeof(double);
}

template <int kMap>
static int lfb_workspace_size(int D, int A, size_t* bytes) {
  MADRL_REQUIRE(D >= 1 && D <= kLfbMaxD, "obs_dim must be in [1, %d], got %d", kLfbMaxD, D);
  MADRL_REQUIRE(A >= 1 && A <= MADRL_AGENTS_MAX, "n_agents must be in [1, %d], got %d", MADRL_AGENTS_MAX, A);
  MADRL_REQUIRE(bytes, "NULL pointer");
  *bytes = lfb_ws_bytes<kMap>(D, A, A == 1 ? kLfbSlices : lfb_agent_slices(A));
  return MADRL_OK;
}

extern "C" int madrl_lfb_workspace_size(int D, size_t* bytes) { return lfb_workspace_size<kLfbRllab>(D, 1, bytes); }

extern "C" int madrl_lfb_agents_workspace_size(int D, int A, size_t* bytes) {
  return lfb_workspace_size<kLfbRllab>(D, A, bytes);
}

extern "C" int madrl_lfbr_workspace_size(int D, size_t* bytes) { return lfb_workspace_size<kLfbRltools>(D, 1, bytes); }

extern "C" int madrl_lfbr_agents_workspace_size(int D, int A, size_t* bytes) {
  return lfb_workspace_size<kLfbRltools>(D, A, bytes);
}

static int lfb_check(int T, int E, int A, int D) {
  MADRL_REQUIRE(T >= 1 && E >= 1 && A >= 1, "bad shape");
  MADRL_REQUIRE(D >= 1 && D <= kLfbMaxD, "obs_dim must be in [1, %d], got %d", kLfbMaxD, D);
  MADRL_REQUIRE((size_t)T * E * A < ((size_t)1 << 31), "T*E*A must be < 2^31");
  return MADRL_OK;
}

template <typename O, bool kAgents, int kMap>
static int lfb_normal_eq(int T, int E, int A, int D, const void* obs_dev, const void* obs_before_dev,
                         const int32_t* seg_start_dev, const int32_t* t0_dev, const float* ret_dev,
                         const double* norm_dev, double* G_dev, double* ws_dev, void* stream) {
  const int rc = lfb_check(T, E, A, D);
  if (rc) return rc;
  if (kAgents)
    MADRL_REQUIRE(A <= MADRL_AGENTS_MAX, "n_agents must be in [1, %d], got %d", MADRL_AGENTS_MAX, A);
  MADRL_REQUIRE(obs_dev && seg_start_dev && ret_dev && G_dev && ws_dev, "NULL buffer");
  const int nb = lfb_tiles<kMap>(D), P = nb * (nb + 1) / 2;
  const int groups = kAgents ? A : 1, S = kAgents ? lfb_agent_slices(A) : kLfbSlices;
  cudaStream_t s = (cudaStream_t)stream;
  MADRL_LAUNCH((lfb_gram_kernel<O, kAgents, kMap>), (unsigned)(P * S * groups), kLfbThreads, 0, s, T, E, A, D,
               (const O*)obs_dev, (const O*)obs_before_dev, seg_start_dev, t0_dev, ret_dev, ws_dev, norm_dev);
  MADRL_LAUNCH(lfb_reduce_kernel<kMap>, (unsigned)(P * groups), 128, 0, s, D, S, ws_dev, G_dev);
  g_launches.fetch_add(2);
  MADRL_CUDA_CHECK(cudaGetLastError());
  return MADRL_OK;
}

template <typename O, bool kAgents, int kMap>
static int lfb_predict(int T, int E, int A, int D, const void* obs_dev, const void* obs_before_dev,
                       const int32_t* seg_start_dev, const int32_t* t0_dev, const double* norm_dev,
                       const double* coef_dev, float* values_dev, void* stream) {
  const int rc = lfb_check(T, E, A, D);
  if (rc) return rc;
  if (kAgents)
    MADRL_REQUIRE(A <= MADRL_AGENTS_MAX, "n_agents must be in [1, %d], got %d", MADRL_AGENTS_MAX, A);
  MADRL_REQUIRE(obs_dev && seg_start_dev && coef_dev && values_dev, "NULL buffer");
  const size_t rows = (size_t)T * E * A;
  MADRL_LAUNCH((lfb_predict_kernel<O, kAgents, kMap>), (unsigned)((rows * 32 + 255) / 256), 256, 0,
               (cudaStream_t)stream, T, E, A, D, (const O*)obs_dev, (const O*)obs_before_dev, seg_start_dev, t0_dev,
               coef_dev, values_dev, norm_dev);
  g_launches.fetch_add(1);
  MADRL_CUDA_CHECK(cudaGetLastError());
  return MADRL_OK;
}

extern "C" int madrl_lfb_normal_eq_f32(int T, int E, int A, int D, const float* obs_dev, const float* obs_before_dev,
    const int32_t* seg_start_dev, const int32_t* t0_dev, const float* ret_dev, double* G_dev, double* ws_dev,
    void* stream) {
  return lfb_normal_eq<float, false, kLfbRllab>(T, E, A, D, obs_dev, obs_before_dev, seg_start_dev, t0_dev, ret_dev, nullptr,
      G_dev, ws_dev, stream);
}

extern "C" int madrl_lfb_predict_f32(int T, int E, int A, int D, const float* obs_dev, const float* obs_before_dev,
    const int32_t* seg_start_dev, const int32_t* t0_dev, const double* coef_dev, float* values_dev, void* stream) {
  return lfb_predict<float, false, kLfbRllab>(T, E, A, D, obs_dev, obs_before_dev, seg_start_dev, t0_dev, nullptr, coef_dev,
      values_dev, stream);
}

extern "C" int madrl_lfb_normal_eq_bf16(int T, int E, int A, int D, const void* obs_dev, const void* obs_before_dev,
    const int32_t* seg_start_dev, const int32_t* t0_dev, const float* ret_dev, double* G_dev, double* ws_dev,
    void* stream) {
  return lfb_normal_eq<uint16_t, false, kLfbRllab>(T, E, A, D, obs_dev, obs_before_dev, seg_start_dev, t0_dev, ret_dev, nullptr,
      G_dev, ws_dev, stream);
}

extern "C" int madrl_lfb_predict_bf16(int T, int E, int A, int D, const void* obs_dev, const void* obs_before_dev,
    const int32_t* seg_start_dev, const int32_t* t0_dev, const double* coef_dev, float* values_dev, void* stream) {
  return lfb_predict<uint16_t, false, kLfbRllab>(T, E, A, D, obs_dev, obs_before_dev, seg_start_dev, t0_dev, nullptr, coef_dev,
      values_dev, stream);
}

extern "C" int madrl_lfb_normal_eq_agents_f32(int T, int E, int A, int D, const float* obs_dev, const float* obs_before_dev,
    const int32_t* seg_start_dev, const int32_t* t0_dev, const float* ret_dev, double* G_dev, double* ws_dev,
    void* stream) {
  return lfb_normal_eq<float, true, kLfbRllab>(T, E, A, D, obs_dev, obs_before_dev, seg_start_dev, t0_dev, ret_dev, nullptr,
      G_dev, ws_dev, stream);
}

extern "C" int madrl_lfb_predict_agents_f32(int T, int E, int A, int D, const float* obs_dev, const float* obs_before_dev,
    const int32_t* seg_start_dev, const int32_t* t0_dev, const double* coef_dev, float* values_dev, void* stream) {
  return lfb_predict<float, true, kLfbRllab>(T, E, A, D, obs_dev, obs_before_dev, seg_start_dev, t0_dev, nullptr, coef_dev,
      values_dev, stream);
}

extern "C" int madrl_lfb_normal_eq_agents_bf16(int T, int E, int A, int D, const void* obs_dev, const void* obs_before_dev,
    const int32_t* seg_start_dev, const int32_t* t0_dev, const float* ret_dev, double* G_dev, double* ws_dev,
    void* stream) {
  return lfb_normal_eq<uint16_t, true, kLfbRllab>(T, E, A, D, obs_dev, obs_before_dev, seg_start_dev, t0_dev, ret_dev, nullptr,
      G_dev, ws_dev, stream);
}

extern "C" int madrl_lfb_predict_agents_bf16(int T, int E, int A, int D, const void* obs_dev, const void* obs_before_dev,
    const int32_t* seg_start_dev, const int32_t* t0_dev, const double* coef_dev, float* values_dev, void* stream) {
  return lfb_predict<uint16_t, true, kLfbRllab>(T, E, A, D, obs_dev, obs_before_dev, seg_start_dev, t0_dev, nullptr, coef_dev,
      values_dev, stream);
}

extern "C" int madrl_lfbr_normal_eq_f32(int T, int E, int A, int D, const float* obs_dev, const float* obs_before_dev,
    const int32_t* seg_start_dev, const int32_t* t0_dev, const float* ret_dev, const double* norm_dev, double* G_dev, double* ws_dev,
    void* stream) {
  return lfb_normal_eq<float, false, kLfbRltools>(T, E, A, D, obs_dev, obs_before_dev, seg_start_dev, t0_dev, ret_dev, norm_dev,
      G_dev, ws_dev, stream);
}

extern "C" int madrl_lfbr_predict_f32(int T, int E, int A, int D, const float* obs_dev, const float* obs_before_dev,
    const int32_t* seg_start_dev, const int32_t* t0_dev, const double* norm_dev, const double* coef_dev, float* values_dev, void* stream) {
  return lfb_predict<float, false, kLfbRltools>(T, E, A, D, obs_dev, obs_before_dev, seg_start_dev, t0_dev, norm_dev, coef_dev,
      values_dev, stream);
}

extern "C" int madrl_lfbr_normal_eq_bf16(int T, int E, int A, int D, const void* obs_dev, const void* obs_before_dev,
    const int32_t* seg_start_dev, const int32_t* t0_dev, const float* ret_dev, const double* norm_dev, double* G_dev, double* ws_dev,
    void* stream) {
  return lfb_normal_eq<uint16_t, false, kLfbRltools>(T, E, A, D, obs_dev, obs_before_dev, seg_start_dev, t0_dev, ret_dev, norm_dev,
      G_dev, ws_dev, stream);
}

extern "C" int madrl_lfbr_predict_bf16(int T, int E, int A, int D, const void* obs_dev, const void* obs_before_dev,
    const int32_t* seg_start_dev, const int32_t* t0_dev, const double* norm_dev, const double* coef_dev, float* values_dev, void* stream) {
  return lfb_predict<uint16_t, false, kLfbRltools>(T, E, A, D, obs_dev, obs_before_dev, seg_start_dev, t0_dev, norm_dev, coef_dev,
      values_dev, stream);
}

extern "C" int madrl_lfbr_normal_eq_agents_f32(int T, int E, int A, int D, const float* obs_dev, const float* obs_before_dev,
    const int32_t* seg_start_dev, const int32_t* t0_dev, const float* ret_dev, const double* norm_dev, double* G_dev, double* ws_dev,
    void* stream) {
  return lfb_normal_eq<float, true, kLfbRltools>(T, E, A, D, obs_dev, obs_before_dev, seg_start_dev, t0_dev, ret_dev, norm_dev,
      G_dev, ws_dev, stream);
}

extern "C" int madrl_lfbr_predict_agents_f32(int T, int E, int A, int D, const float* obs_dev, const float* obs_before_dev,
    const int32_t* seg_start_dev, const int32_t* t0_dev, const double* norm_dev, const double* coef_dev, float* values_dev, void* stream) {
  return lfb_predict<float, true, kLfbRltools>(T, E, A, D, obs_dev, obs_before_dev, seg_start_dev, t0_dev, norm_dev, coef_dev,
      values_dev, stream);
}

extern "C" int madrl_lfbr_normal_eq_agents_bf16(int T, int E, int A, int D, const void* obs_dev, const void* obs_before_dev,
    const int32_t* seg_start_dev, const int32_t* t0_dev, const float* ret_dev, const double* norm_dev, double* G_dev, double* ws_dev,
    void* stream) {
  return lfb_normal_eq<uint16_t, true, kLfbRltools>(T, E, A, D, obs_dev, obs_before_dev, seg_start_dev, t0_dev, ret_dev, norm_dev,
      G_dev, ws_dev, stream);
}

extern "C" int madrl_lfbr_predict_agents_bf16(int T, int E, int A, int D, const void* obs_dev, const void* obs_before_dev,
    const int32_t* seg_start_dev, const int32_t* t0_dev, const double* norm_dev, const double* coef_dev, float* values_dev, void* stream) {
  return lfb_predict<uint16_t, true, kLfbRltools>(T, E, A, D, obs_dev, obs_before_dev, seg_start_dev, t0_dev, norm_dev, coef_dev,
      values_dev, stream);
}
