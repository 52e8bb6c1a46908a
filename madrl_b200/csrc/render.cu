// Frames of chosen envs, drawn on the device from the state blob (DESIGN §4.10).
//
// Waterworld and Hostage: what the reference's render bodies draw (waterworld.py:438-479 ww:LINE,
// hostage.py:431-478 hr:LINE) with OpenCV's 8-connected primitives in place of the anti-aliased ones, the
// background blend of cv2.addWeighted(255, 0.4, img, 0.6, 0), RGB.  One block draws one 32 x 32 tile of one frame:
// it builds the env's primitives in painter's order 256 at a time, keeps those whose box meets the tile (in
// order, through a ballot compaction into shared memory), and every pixel walks them forward, so the last
// primitive that covers a pixel gives its colour.  Pursuit: the integer picture of pursuit_evade.py:274-295, one
// thread per pixel.
//
// The kernels only read the state: no env state, draw counter or launch setting changes.
#include <math.h>

#include "engine.cuh"

namespace madrl {

constexpr int RT = 32;         // tile edge (pixels)
constexpr int RTHREADS = 256;  // 8 warps; warp w draws rows w, w + 8, w + 16 and w + 24 of its tile
constexpr int R_ROWS = RT * RT / RTHREADS;
constexpr int RENDER_MAX_SIZE = 32768;   // largest frame edge: every clipped coordinate and Bresenham term fits int32
// Radii and sensor reaches (|sensor_range| S) stay below 2^29 pixels, so a coordinate the 2^30 clamp moves belongs to
// a primitive that misses the frame both before and after the clamp (a NaN coordinate clamps to -2^30 and misses).
constexpr double RENDER_MAX_REACH = (double)(1ll << 29);
constexpr long long RENDER_COORD_LIMIT = 1ll << 30;
constexpr size_t RENDER_MAX_GRID = 1u << 20;   // blocks per launch; larger batches loop over work items
constexpr unsigned KIND_CIRCLE = 1u << 24, KIND_LINE = 2u << 24, RGB_MASK = 0xffffffu;

// One primitive: a filled circle (a, b) radius c, or a line from (a, b) to (c, d) clipped to the frame with
// a <= c; m = kind | colour (0xRRGGBB).  m == 0: nothing to draw.
struct Prim {
  int a, b, c, d;
  unsigned m;
};

// int(float64(x) * S), truncated toward zero as NumPy's astype(int) does
__device__ __forceinline__ long long to_px(double x, int S) {
  const double v = __dmul_rn(x, (double)S);
  return (long long)fmin(fmax(v, (double)-RENDER_COORD_LIMIT), (double)RENDER_COORD_LIMIT);
}

__device__ __forceinline__ long long isqrt64(long long n) {
  long long s = (long long)sqrt((double)n);
  while (s * s > n) --s;
  while ((s + 1) * (s + 1) <= n) ++s;
  return s;
}

__device__ __forceinline__ Prim circle_prim(long long cx, long long cy, int r, unsigned rgb) {
  return Prim{(int)cx, (int)cy, r, 0, KIND_CIRCLE | rgb};
}

// OpenCV's clipLine on [0, W-1] x [0, H-1] (y edges first, each move a truncated float64 quotient), then the end
// points ordered left to right as the 8-connected walk takes them.
__device__ Prim line_prim(long long x1, long long y1, long long x2, long long y2, int W, int H, unsigned rgb) {
  const long long right = W - 1, bottom = H - 1;
  int c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8;
  int c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8;
  if ((c1 & c2) == 0 && (c1 | c2) != 0) {
    long long a;
    if (c1 & 12) {
      a = c1 < 8 ? 0 : bottom;
      x1 += (long long)(__dmul_rn((double)(a - y1), (double)(x2 - x1)) / (double)(y2 - y1));
      y1 = a;
      c1 = (x1 < 0) + (x1 > right) * 2;
    }
    if (c2 & 12) {
      a = c2 < 8 ? 0 : bottom;
      x2 += (long long)(__dmul_rn((double)(a - y2), (double)(x2 - x1)) / (double)(y2 - y1));
      y2 = a;
      c2 = (x2 < 0) + (x2 > right) * 2;
    }
    if ((c1 & c2) == 0 && (c1 | c2) != 0) {
      if (c1) {
        a = c1 == 1 ? 0 : right;
        y1 += (long long)(__dmul_rn((double)(a - x1), (double)(y2 - y1)) / (double)(x2 - x1));
        x1 = a;
        c1 = 0;
      }
      if (c2) {
        a = c2 == 1 ? 0 : right;
        y2 += (long long)(__dmul_rn((double)(a - x2), (double)(y2 - y1)) / (double)(x2 - x1));
        x2 = a;
        c2 = 0;
      }
    }
  }
  if (c1 | c2) return Prim{0, 0, 0, 0, 0u};
  if (x2 < x1) return Prim{(int)x2, (int)y2, (int)x1, (int)y1, KIND_LINE | rgb};
  return Prim{(int)x1, (int)y1, (int)x2, (int)y2, KIND_LINE | rgb};
}

// Does the primitive's box meet the tile [x0, x0 + RT) x [y0, y0 + RT)?
__device__ __forceinline__ bool meets(const Prim& q, int x0, int y0) {
  if (q.m == 0u) return false;
  long long lx, hx, ly, hy;
  if ((q.m & ~RGB_MASK) == KIND_CIRCLE) {
    lx = (long long)q.a - q.c; hx = (long long)q.a + q.c; ly = (long long)q.b - q.c; hy = (long long)q.b + q.c;
  } else {
    lx = q.a; hx = q.c; ly = min(q.b, q.d); hy = max(q.b, q.d);
  }
  return hx >= x0 && lx < x0 + RT && hy >= y0 && ly < y0 + RT;
}

// Pixel (x, y) of the primitive?  Circle: OpenCV's filled LINE_8 circle, whose row offset oy spans |x - cx| <= m,
// m = isqrt(r^2 - oy^2), for the rows its first-octant walk reaches (2 oy^2 <= r^2, or m^2 + (oy + 1)^2 > r^2).
// Line: step k of the walk along the major axis moves the minor coordinate (2 minor k + major - 1) div (2 major).
__device__ __forceinline__ bool covers(const Prim& q, int x, int y) {
  if ((q.m & ~RGB_MASK) == KIND_CIRCLE) {
    const long long ox = llabs((long long)x - q.a), oy = llabs((long long)y - q.b), r = q.c;
    if (ox > r || oy > r) return false;
    const long long r2 = r * r, oy2 = oy * oy;
    if (ox * ox + oy2 > r2) return false;
    if (2 * oy2 <= r2) return true;
    const long long m = isqrt64(r2 - oy2);
    return ox <= m && m * m + (oy + 1) * (oy + 1) > r2;
  }
  const int dx = q.c - q.a, ady = abs(q.d - q.b), sy = q.d < q.b ? -1 : 1;
  if (ady > dx) {
    const int k = (y - q.b) * sy;
    if (k < 0 || k > ady) return false;
    return x == q.a + (2 * dx * k + ady - 1) / (2 * ady);
  }
  const int k = x - q.a;
  if (k < 0 || k > dx) return false;
  return y == q.b + sy * (dx > 0 ? (2 * ady * k + dx - 1) / (2 * dx) : 0);
}

// cv2.addWeighted(255, 0.4, v, 0.6, 0) on uint8: round(102 + 0.6 v).  0.6 v has a fractional part of 0, .2, .4, .6
// or .8, far from the ties where float32's rounding of the products and sum could tip it, so the integer form is
// exact (tests/test_render_cpu.py pins the oracle's float32 table, which equals it, against cv2 on all 256 values).
__device__ __forceinline__ unsigned char blend_bg(unsigned v) { return (unsigned char)(102u + (6u * v + 5u) / 10u); }

// A pursuer's or rescuer's group: sensor line j (< K) from its centre, then its body (j == K).  The reference
// redraws the body after every line; the last redraw leaves what one body drawn after all K lines leaves.
template <typename real>
__device__ __forceinline__ Prim sensor_prim(real px, real py, int j, int K, double range, const double* dirs, int S,
                                            int r_body, unsigned body_rgb) {
  const long long cx = to_px((double)px, S), cy = to_px((double)py, S);
  if (j == K) return circle_prim(cx, cy, r_body, body_rgb);
  const double ex = __dadd_rn((double)px, __dmul_rn(range, dirs[j]));       // ww:455 position + range * sensor
  const double ey = __dadd_rn((double)py, __dmul_rn(range, dirs[K + j]));
  return line_prim(cx, cy, to_px(ex, S), to_px(ey, S), S, S, 0x000000u);
}

struct WWScene {
  const char* state;
  size_t objs, obst;
  int n_obj, Np, Ne, K;
  int r_obst, r_pur, r_ev, r_po;
  double range;
  const double* dirs;   // float64 [2][K]: cos row, sin row

  __device__ int count() const { return 1 + Np * (K + 1) + Ne + (n_obj - Np - Ne); }

  // ww:442-472: obstacle; per pursuer its sensor lines and body; evaders; poison
  template <typename real>
  __device__ Prim prim(int e, int p, int S) const {
    const real* o = (const real*)(state + objs) + (size_t)e * 4 * n_obj;
    if (p == 0) {
      const real* c = (const real*)(state + obst) + 2 * (size_t)e;
      return circle_prim(to_px((double)c[0], S), to_px((double)c[1], S), r_obst, 0x008080u);
    }
    p -= 1;
    if (p < Np * (K + 1)) {
      const int i = p / (K + 1);
      return sensor_prim<real>(o[i], o[n_obj + i], p - i * (K + 1), K, range, dirs, S, r_pur, 0x0000ffu);
    }
    const int i = p - Np * (K + 1) + Np;
    return circle_prim(to_px((double)o[i], S), to_px((double)o[n_obj + i], S), i < Np + Ne ? r_ev : r_po,
                       i < Np + Ne ? 0x00ff00u : 0xff0000u);
  }
};

struct HWScene {
  const char* state;
  size_t objs, fixed, saved, flags;
  int n_obj, Ng, Nb, Nh, K;
  int r_body, r_hostage, r_bomb;
  double range;
  const double* dirs;

  __device__ int count() const { return 3 + Nh + Nb + Ng * (K + 1); }

  // hr:436-472: gate line and key while the gate is closed; bomb; hostages not saved; criminals; rescuers with
  // their sensor lines
  template <typename real>
  __device__ Prim prim(int e, int p, int S) const {
    const real* o = (const real*)(state + objs) + (size_t)e * 4 * n_obj;
    const real* f = (const real*)(state + fixed) + 4 * (size_t)e;
    if (p < 2) {
      if (((const int32_t*)(state + flags))[e] & 1) return Prim{0, 0, 0, 0, 0u};
      if (p == 0) {
        const long long gy = (long long)(0.5 * (double)S);
        return line_prim(0, gy, S, gy, S, S, 0xc88080u);
      }
      return circle_prim(to_px((double)f[0], S), to_px((double)f[1], S), r_body, 0xff0000u);
    }
    if (p == 2) return circle_prim(to_px((double)f[2], S), to_px((double)f[3], S), r_bomb, 0xff0000u);
    p -= 3;
    if (p < Nh) {
      if (((const uint8_t*)(state + saved))[(size_t)e * Nh + p]) return Prim{0, 0, 0, 0, 0u};
      const int i = Ng + Nb + p;
      return circle_prim(to_px((double)o[i], S), to_px((double)o[n_obj + i], S), r_hostage, 0x0078ffu);
    }
    p -= Nh;
    if (p < Nb) return circle_prim(to_px((double)o[Ng + p], S), to_px((double)o[n_obj + Ng + p], S), r_body, 0xc83232u);
    p -= Nb;
    const int i = p / (K + 1);
    return sensor_prim<real>(o[i], o[n_obj + i], p - i * (K + 1), K, range, dirs, S, r_body, 0x0000ffu);
  }
};

// Block-wide work items w = f * tiles + t (frame f, tile t), grid-stride.  Shared memory (dynamic, through the
// 32-bit shared-address helpers): the chunk's kept primitives, 5 words each, then one count per warp.  An id outside
// [0, E) gets an all-zero frame, which no drawn frame equals (the background blend lifts every channel to >= 102).
constexpr size_t RENDER_SMEM = (size_t)RTHREADS * 5 * 4 + RTHREADS / 32 * 4;

template <typename real, class Scene>
__global__ void __launch_bounds__(RTHREADS) render_tiles_kernel(Scene sc, int E, int n, const int32_t* __restrict__ ids,
                                                                int S, unsigned char* __restrict__ out) {
  extern __shared__ __align__(16) uint32_t smem_u32[];
  const uint32_t prim_a = smem_addr(smem_u32), cnt_a = prim_a + RTHREADS * 5 * 4;
  const int tiles_x = (S + RT - 1) / RT;
  const size_t tiles = (size_t)tiles_x * tiles_x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int P = sc.count();
  for (size_t w = blockIdx.x; w < (size_t)n * tiles; w += gridDim.x) {
    const int f = (int)(w / tiles), t = (int)(w - (size_t)f * tiles);
    const int x0 = (t % tiles_x) * RT, y0 = (t / tiles_x) * RT, x = x0 + lane;
    const int e = ids[f];
    const bool valid = e >= 0 && e < E;
    unsigned col[R_ROWS];
#pragma unroll
    for (int r = 0; r < R_ROWS; ++r) col[r] = 0xffffffu;
    for (int base = 0; valid && base < P; base += RTHREADS) {
      const int p = base + threadIdx.x;
      Prim q{0, 0, 0, 0, 0u};
      if (p < P) q = sc.template prim<real>(e, p, S);
      const bool keep = meets(q, x0, y0);
      const unsigned bal = __ballot_sync(FULL_MASK, keep);
      if (lane == 0) sts_u32(cnt_a + 4 * warp, __popc(bal));
      __syncthreads();
      int off = 0, total = 0;
#pragma unroll
      for (int v = 0; v < RTHREADS / 32; ++v) {
        const int c = (int)lds_u32(cnt_a + 4 * v);
        off += v < warp ? c : 0;
        total += c;
      }
      if (keep) {
        const uint32_t a = prim_a + 20u * (uint32_t)(off + __popc(bal & lanemask_lt()));
        sts_u32(a, (uint32_t)q.a); sts_u32(a + 4, (uint32_t)q.b); sts_u32(a + 8, (uint32_t)q.c);
        sts_u32(a + 12, (uint32_t)q.d); sts_u32(a + 16, q.m);
      }
      __syncthreads();
      for (int i = 0; i < total; ++i) {
        const uint32_t a = prim_a + 20u * (uint32_t)i;
        const Prim t = {(int)lds_u32(a), (int)lds_u32(a + 4), (int)lds_u32(a + 8), (int)lds_u32(a + 12), lds_u32(a + 16)};
#pragma unroll
        for (int r = 0; r < R_ROWS; ++r)
          if (covers(t, x, y0 + warp + 8 * r)) col[r] = t.m & RGB_MASK;
      }
      __syncthreads();   // the next chunk rewrites the primitives and the counts
    }
    if (x < S) {
#pragma unroll
      for (int r = 0; r < R_ROWS; ++r) {
        const int y = y0 + warp + 8 * r;
        if (y >= S) break;
        unsigned char* px = out + (((size_t)f * S + y) * S + x) * 3;
        px[0] = valid ? blend_bg(col[r] >> 16) : 0;
        px[1] = valid ? blend_bg((col[r] >> 8) & 255u) : 0;
        px[2] = valid ? blend_bg(col[r] & 255u) : 0;
      }
    }
  }
}

// Pursuit (DESIGN §4.10): pixel (row, col) shows cell (col / c, row / c): white, or (64, 64, 64) for a building;
// blended (v + o + 1) >> 1 with o = #FF9848 once per pursuer whose observation window holds the cell; then the
// marker square [c/4, c - c/4)^2 of a pursuer (255, 0, 0) and over it of a live evader (0, 0, 255).
struct PEScene {
  const uint8_t* pos;       // [E][2][Nag]
  const uint64_t* gone;     // [E]
  const int32_t* map_id;    // [E]
  const uint32_t* maps;     // [n_maps][ncellP], cell (x, y) at (x + pad) ysP + (y + pad), bit 0 building
  int Np, Ne, R, off, pad, ysP, ncellP;
};

// Work items w = f * blocks + b (frame f, 256-pixel block b), grid-stride; shared memory: the env's agent cells, one
// word per coordinate (x row, then y row, as the state keeps them).
constexpr int PE_THREADS = 256;

__global__ void __launch_bounds__(PE_THREADS) render_pursuit_kernel(PEScene sc, int E, int n,
                                                                    const int32_t* __restrict__ ids, int cell, int W,
                                                                    int H, unsigned char* __restrict__ out) {
  extern __shared__ __align__(16) uint32_t smem_u32[];
  const uint32_t pos_a = smem_addr(smem_u32);
  const int Nag = sc.Np + sc.Ne;
  const size_t npx = (size_t)W * H, blocks = (npx + PE_THREADS - 1) / PE_THREADS;
  const int lo = cell / 4, hi = cell - cell / 4;
  for (size_t w = blockIdx.x; w < (size_t)n * blocks; w += gridDim.x) {
    const int f = (int)(w / blocks);
    const size_t idx = (w - (size_t)f * blocks) * PE_THREADS + threadIdx.x;
    const int e = ids[f];
    const bool valid = e >= 0 && e < E;
    __syncthreads();   // the previous item's cells are read
    if (valid)
      for (int i = threadIdx.x; i < 2 * Nag; i += PE_THREADS) sts_u32(pos_a + 4 * i, sc.pos[(size_t)e * 2 * Nag + i]);
    __syncthreads();
    if (idx >= npx) continue;
    unsigned char* px = out + ((size_t)f * npx + idx) * 3;
    if (!valid) {
      px[0] = px[1] = px[2] = 0;
      continue;
    }
    const int row = (int)(idx / W), colp = (int)(idx % W);
    const int x = colp / cell, y = row / cell, ox = colp - x * cell, oy = row - y * cell;
    const uint32_t word = sc.maps[(size_t)sc.map_id[e] * sc.ncellP + (size_t)(x + sc.pad) * sc.ysP + (y + sc.pad)];
    unsigned r = (word & 1u) ? 64u : 255u, g = r, b = r;
    bool pur = false, ev = false;
    for (int i = 0; i < sc.Np; ++i) {
      const int px_ = (int)lds_u32(pos_a + 4 * i), py_ = (int)lds_u32(pos_a + 4 * (Nag + i));
      const int wx = x - px_ + sc.off, wy = y - py_ + sc.off;
      if (wx >= 0 && wx < sc.R && wy >= 0 && wy < sc.R) {   // pe window: cells [p - off, p - off + R)
        r = (r + 255u + 1u) >> 1;
        g = (g + 152u + 1u) >> 1;
        b = (b + 72u + 1u) >> 1;
      }
      pur |= px_ == x && py_ == y;
    }
    const uint64_t gone = sc.gone[e];
    for (int j = 0; j < sc.Ne; ++j)
      ev |= !((gone >> j) & 1u) && (int)lds_u32(pos_a + 4 * (sc.Np + j)) == x &&
            (int)lds_u32(pos_a + 4 * (Nag + sc.Np + j)) == y;
    if (ox >= lo && ox < hi && oy >= lo && oy < hi) {
      if (ev) { r = 0; g = 0; b = 255; }
      else if (pur) { r = 255; g = 0; b = 0; }
    }
    px[0] = (unsigned char)r;
    px[1] = (unsigned char)g;
    px[2] = (unsigned char)b;
  }
}

// A radius in pixels, int(radius * S) as the reference computes it; MADRL_EINVAL from RENDER_MAX_REACH up
static int radius_px(double radius, int S, int* out) {
  const double v = radius * (double)S;
  MADRL_REQUIRE(v >= 0.0 && v < RENDER_MAX_REACH, "a radius of %g at screen_size %d is out of range", radius, S);
  *out = (int)v;
  return MADRL_OK;
}

// MADRL_EINVAL unless |sensor_range| S < RENDER_MAX_REACH (a NaN or infinite range fails it)
static int check_sensor_reach(double range, int S) {
  MADRL_REQUIRE(fabs(range) * (double)S < RENDER_MAX_REACH,
                "a sensor_range of %g at screen_size %d reaches 2^29 pixels or more", range, S);
  return MADRL_OK;
}

template <class Scene>
static int launch_tiles(bool fp64, const Scene& sc, int E, int n, const int32_t* ids, int S, void* out, void* stream) {
  const size_t items = (size_t)n * ((S + RT - 1) / RT) * ((S + RT - 1) / RT);
  const unsigned grid = (unsigned)(items < RENDER_MAX_GRID ? items : RENDER_MAX_GRID);
  void (*kfn)(Scene, int, int, const int32_t*, int, unsigned char*) =
      fp64 ? render_tiles_kernel<double, Scene> : render_tiles_kernel<float, Scene>;
  MADRL_LAUNCH(kfn, grid, RTHREADS, RENDER_SMEM, (cudaStream_t)stream, sc, E, n, ids, S, (unsigned char*)out);
  g_launches.fetch_add(1);
  MADRL_CUDA_CHECK(cudaGetLastError());
  return MADRL_OK;
}

static int check_render_args(const void* h, int n, const int32_t* ids, int size, const void* out, const char* what) {
  MADRL_REQUIRE(h != nullptr, "handle is NULL");
  MADRL_REQUIRE(n >= 1, "n must be >= 1, got %d", n);
  MADRL_REQUIRE(ids != nullptr && out != nullptr, "NULL env_ids or out");
  MADRL_REQUIRE(size >= 1 && size <= RENDER_MAX_SIZE, "%s must be in [1, %d], got %d", what, RENDER_MAX_SIZE, size);
  return MADRL_OK;
}

}  // namespace madrl

using namespace madrl;

extern "C" int madrl_ww_render(madrl_ww* h, int n, const int32_t* env_ids_dev, int screen_size,
                               const double* sensor_dirs_dev, uint8_t* out_dev, void* stream) {
  int rc = check_render_args(h, n, env_ids_dev, screen_size, out_dev, "screen_size");
  if (rc) return rc;
  MADRL_REQUIRE(sensor_dirs_dev != nullptr, "NULL sensor_dirs");
  const auto v = handle_view(h);
  const madrl_ww_config& c = *v.cfg;
  const int S = screen_size;
  WWScene sc{v.state, v.lay->objs, v.lay->obst, v.lay->n_obj, c.n_pursuers, c.n_evaders, c.n_sensors,
             0, 0, 0, 0, c.sensor_range, sensor_dirs_dev};
  if ((rc = check_sensor_reach(c.sensor_range, S)) || (rc = radius_px(c.obstacle_radius, S, &sc.r_obst)) ||
      (rc = radius_px(c.radius, S, &sc.r_pur)) ||
      (rc = radius_px(c.radius * 2, S, &sc.r_ev)) || (rc = radius_px(c.radius * 3 / 4, S, &sc.r_po)))
    return rc;   // ww:109-117: evaders radius * 2, poison radius * 3 / 4
  return launch_tiles(c.fp64 != 0, sc, c.n_envs, n, env_ids_dev, S, out_dev, stream);
}

extern "C" int madrl_hostage_render(madrl_hostage* h, int n, const int32_t* env_ids_dev, int screen_size,
                                    const double* sensor_dirs_dev, uint8_t* out_dev, void* stream) {
  int rc = check_render_args(h, n, env_ids_dev, screen_size, out_dev, "screen_size");
  if (rc) return rc;
  MADRL_REQUIRE(sensor_dirs_dev != nullptr, "NULL sensor_dirs");
  const auto v = handle_view(h);
  const madrl_hostage_config& c = *v.cfg;
  const int S = screen_size;
  HWScene sc{v.state, v.lay->objs, v.lay->fixed, v.lay->saved, v.lay->flags, v.lay->n_obj, c.n_good, c.n_bad,
             c.n_hostages, c.n_sensors, 0, 0, 0, c.sensor_range, sensor_dirs_dev};
  if ((rc = check_sensor_reach(c.sensor_range, S)) || (rc = radius_px(c.radius, S, &sc.r_body)) ||
      (rc = radius_px(c.radius * 2, S, &sc.r_hostage)) ||
      (rc = radius_px(c.bomb_radius, S, &sc.r_bomb)))
    return rc;   // hostage.py:122-129: hostages radius * 2; the key is drawn with `radius` (hr:447)
  return launch_tiles(c.fp64 != 0, sc, c.n_envs, n, env_ids_dev, S, out_dev, stream);
}

extern "C" int madrl_pursuit_render(madrl_pursuit* h, int n, const int32_t* env_ids_dev, int cell, uint8_t* out_dev,
                                    void* stream) {
  int rc = check_render_args(h, n, env_ids_dev, cell, out_dev, "cell");
  if (rc) return rc;
  const auto v = handle_view(h);
  const madrl_pursuit_config& c = *v.cfg;
  MADRL_REQUIRE((long long)c.xs * cell <= RENDER_MAX_SIZE && (long long)c.ys * cell <= RENDER_MAX_SIZE,
                "a %d x %d map at cell %d is larger than %d pixels a side", c.xs, c.ys, cell, RENDER_MAX_SIZE);
  const int pad = (c.obs_range - 1) / 2 + 1, ysP = c.ys + 2 * pad;
  PEScene sc{(const uint8_t*)(v.state + v.lay->pos), (const uint64_t*)(v.state + v.lay->gone),
             (const int32_t*)(v.state + v.lay->map_id), (const uint32_t*)(v.state + v.lay->maps), c.n_pursuers,
             c.n_evaders, c.obs_range, (c.obs_range - 1) / 2, pad, ysP, (c.xs + 2 * pad) * ysP};
  const int W = c.xs * cell, H = c.ys * cell;
  const size_t items = (size_t)n * (((size_t)W * H + PE_THREADS - 1) / PE_THREADS);
  const unsigned grid = (unsigned)(items < RENDER_MAX_GRID ? items : RENDER_MAX_GRID);
  MADRL_LAUNCH(render_pursuit_kernel, grid, PE_THREADS, (size_t)2 * (c.n_pursuers + c.n_evaders) * 4,
               (cudaStream_t)stream, sc, c.n_envs, n, env_ids_dev, cell, W, H, out_dev);
  g_launches.fetch_add(1);
  MADRL_CUDA_CHECK(cudaGetLastError());
  return MADRL_OK;
}
