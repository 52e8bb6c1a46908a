// Trajectory post-processing kernels on the rollout tensors (SURVEY.md 8f rows 2 and 3): the
// consumers that sit right after the env hot path in the reference's sampler loop.  All three are
// pure HBM-bound streaming passes over [T][E][A][...] tensors, one thread per (env, agent[, dim])
// column walking the time axis, so every load / store is coalesced across the warp.
//
//   madrl_gae_f32            rllab/rllab/sampler/base.py:48-68 (deltas, GAE advantages, discounted
//                            returns via special.discount_cumsum, rllab/rllab/misc/special.py:107-111),
//                            paths segmented by `done`
//   madrl_frame_stack_f32    madrl_environments/__init__.py:143-196  ObservationBuffer
//   madrl_standardize_f32    madrl_environments/__init__.py:204-291  StandardizedEnv
// The observation passes (frame stack, standardize, path packing) also take bfloat16 observations
// (madrl_*_set_obs_format): element type O = uint16_t holding bfloat16 bits.  Values are widened to the
// same float / double arithmetic as the float32 pass and rounded once, at the store, so a bf16 result is
// the f32 pass's result on the widened input, rounded to nearest even.
#include "common.cuh"

namespace madrl {

// y[t] = x[t] + g * y[t+1] inside a path; a path ends where done[t] != 0 (bootstrap value 0, as
// base.py:57 appends 0) or at the end of the rollout (bootstrap = last_value or 0).
__global__ void gae_kernel(int T, int E, int A, const float* __restrict__ rew,
                           const float* __restrict__ val, const uint8_t* __restrict__ done,
                           const float* __restrict__ last_value, double discount, double gae_lambda,
                           float* __restrict__ adv, float* __restrict__ ret) {
  const size_t n = (size_t)E * A;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const size_t e = i / A;
  double next_v = last_value ? (double)last_value[i] : 0.0;
  double run_adv = 0.0, run_ret = last_value ? (double)last_value[i] : 0.0;
  const double gl = discount * gae_lambda;
  for (int t = T - 1; t >= 0; --t) {
    const size_t k = (size_t)t * n + i;
    if (done[(size_t)t * E + e]) { next_v = 0.0; run_adv = 0.0; run_ret = 0.0; }
    const double r = (double)rew[k], v = (double)val[k];
    const double delta = r + discount * next_v - v;                // base.py:58-60
    run_adv = delta + gl * run_adv;                                // base.py:61-62
    run_ret = r + discount * run_ret;                              // base.py:63
    __stcs(adv + k, (float)run_adv);
    __stcs(ret + k, (float)run_ret);
    next_v = v;
  }
}

// ObservationBuffer: out[t][..][d][b] = the observation b steps before the newest one; on a step
// whose `done` flag is set the obs slot holds the reset observation and reset() fills every slot
// of the buffer with it (__init__.py:186-196).  `carry` [E][A][D][B] holds the buffer between calls.
// Values are only moved, so the bf16 variant (O = uint16_t: obs, carry and out in bfloat16) is exact.
template <int B, typename O>
__global__ void frame_stack_kernel(int T, size_t n /* E*A*D */, int AD, const O* __restrict__ obs,
                                   const uint8_t* __restrict__ done, int E, O* __restrict__ carry,
                                   O* __restrict__ out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const size_t e = i / AD;
  O buf[B];
#pragma unroll
  for (int b = 0; b < B; ++b) buf[b] = carry[i * B + b];
  for (int t = 0; t < T; ++t) {
    const O x = obs[(size_t)t * n + i];
    if (done[(size_t)t * E + e]) {
#pragma unroll
      for (int b = 0; b < B; ++b) buf[b] = x;
    } else {
#pragma unroll
      for (int b = 0; b < B - 1; ++b) buf[b] = buf[b + 1];          // __init__.py:178-180
      buf[B - 1] = x;
    }
    O* o = out + ((size_t)t * n + i) * B;
#pragma unroll
    for (int b = 0; b < B; ++b) __stcs(o + b, buf[b]);
  }
#pragma unroll
  for (int b = 0; b < B; ++b) carry[i * B + b] = buf[b];
}

// StandardizedEnv running estimates (__init__.py:241-270), in place over the time axis.
//   mean <- (1-a) mean + a x ;  var <- (1-a) var + a (x - mean)^2 ;  out = (x - mean) / (sqrt(var) + eps)
// center = 1 for observations; rewards are only divided (and scaled), never centred.
// 1 / (sqrt(v) + eps) in float64 WITHOUT the DSQRT / DDIV sequences (each some two dozen FP64 instructions, which made
// these streaming passes FP64-bound at 29 % of the HBM roofline): float32 seeds (MUFU.RSQ / MUFU.RCP, ~1e-7) refined by
// one Newton step each in float64 (-> ~1e-14 relative; the result is rounded to float32 afterwards).  The running
// mean / variance recurrences themselves stay exact float64.  v == 0 (or denormal) takes the exact path.
__device__ __forceinline__ double inv_std(double v, double eps) {
  const float vf = (float)v;
  if (!(vf > 1e-30f) || !(vf < 1e30f)) return 1.0 / (sqrt(v) + eps);
  double y = (double)rsqrtf(vf);
  y = y * (1.5 - 0.5 * v * y * y);          // 1 / sqrt(v)
  const double den = v * y + eps;           // sqrt(v) + eps
  double r = (double)(1.0f / (float)den);
  r = r * (2.0 - den * r);
  return r;
}

// One element's running-estimate update (__init__.py:258-262), shared by every standardiser kernel so that the
// whole-rollout passes and the closed loop's per-step pass give the same bits.  The fused multiply-adds are
// spelled out: left to contraction, nvcc fused `(1-a) m + a x` as fma(m, 1-a, a x) in one kernel and as
// fma(x, a, (1-a) m) in another, so the running estimates drifted apart in their last bits.  These are the forms
// the whole-rollout kernels were compiled to before.
__device__ __forceinline__ void running_update(double x, double& m, double& v, double alpha) {
  m = fma(m, 1.0 - alpha, alpha * x);
  const double d = x - m;
  v = fma(v, 1.0 - alpha, alpha * d * d);
}

// The update, then x standardised by the updated estimate (observations: centred).
__device__ __forceinline__ double standardize_obs_one(double x, double& m, double& v, double alpha, double eps) {
  running_update(x, m, v, alpha);
  return (x - m) * inv_std(v, eps);
}

template <typename O>
__global__ void standardize_kernel(int T, size_t n, O* __restrict__ x, double* __restrict__ mean,
                                   double* __restrict__ var, double alpha, double eps, int center,
                                   double scale, int enable) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double m = mean[i], v = var[i];
  for (int t = 0; t < T; ++t) {
    const size_t k = (size_t)t * n + i;
    const double xv = (double)obs_widen<float>(x[k]);
    double o = xv;
    if (enable) {
      running_update(xv, m, v, alpha);
      o = (center ? (xv - m) : xv) * inv_std(v, eps);
    }
    x[k] = obs_cvt<O>((float)(scale * o));
  }
  mean[i] = m;
  var[i] = v;
}

// Observation standardiser for auto-reset rollouts with the terminal observations on the side.
template <typename O>
__global__ void standardize_terminal_kernel(int T, int E, size_t per_env, O* __restrict__ x,
                                            O* __restrict__ term, const uint8_t* __restrict__ done,
                                            double* __restrict__ mean, double* __restrict__ var, double alpha,
                                            double eps) {
  const size_t n = (size_t)E * per_env;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const size_t e = i / per_env;
  double m = mean[i], v = var[i];
  for (int t = 0; t < T; ++t) {
    const size_t k = (size_t)t * n + i;
    if (done[(size_t)t * E + e])                   // step(): the terminal observation comes first
      term[k] = obs_cvt<O>((float)standardize_obs_one((double)obs_widen<float>(term[k]), m, v, alpha, eps));
    x[k] = obs_cvt<O>((float)standardize_obs_one((double)obs_widen<float>(x[k]), m, v, alpha, eps));
  }
  mean[i] = m;
  var[i] = v;
}

// One closed-loop step of StandardizedEnv inside ObservationBuffer (PolicyRollout with a Standardizer and / or
// frame_stack > 1), right after the engine's one-step launch: the same values as standardize_terminal_kernel then
// frame_stack_kernel at T = 1, in one pass.  With mean / var (obsnorm): where done[e] is set the estimate is first
// updated with term (written back standardised), then with obs (written back standardised, in place).  Then the
// stack: out = the new value in every slot where done is set, else prev shifted left by one with the new value in
// slot B-1.  B = 1 needs no prev; out may be NULL there.  mean / var and prev are read once per step (evict-first);
// obs was just written by the launch and out is read by the policy next, so both keep normal L2 priority.
template <int B, typename O>
__global__ void obs_wrap_step_kernel(size_t n /* E*A*D */, size_t per_env, O* __restrict__ obs,
                                     O* __restrict__ term, const uint8_t* __restrict__ done,
                                     const O* __restrict__ prev, O* __restrict__ out, double* __restrict__ mean,
                                     double* __restrict__ var, double alpha, double eps) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const bool reset = done[i / per_env] != 0;
  O x = obs[i];
  if (mean) {
    double m = __ldcs(mean + i), v = __ldcs(var + i);
    if (reset)
      term[i] = obs_cvt<O>((float)standardize_obs_one((double)obs_widen<float>(term[i]), m, v, alpha, eps));
    x = obs_cvt<O>((float)standardize_obs_one((double)obs_widen<float>(x), m, v, alpha, eps));
    obs[i] = x;
    __stcs(mean + i, m);
    __stcs(var + i, v);
  }
  if (!out) return;
  O buf[B];
#pragma unroll
  for (int b = 0; b < B - 1; ++b) buf[b] = reset ? x : __ldcs(prev + i * B + b + 1);
  buf[B - 1] = x;
#pragma unroll
  for (int b = 0; b < B; ++b) out[i * B + b] = buf[b];
}

// DiagnosticsWrapper episode statistics (madrl_environments/__init__.py:314-369): per env, walk the
// time axis accumulating the per-agent episode reward, the episode length and the discounted return
// of the agent-mean reward; an episode closes where done[t] is set or its length reaches
// max_traj_len (the wrapper then restarts its counters even though the env goes on).
// carry [E][A+3] doubles: episode reward per agent, length, discounted return, discount power.
__global__ void episode_stats_kernel(int T, int E, int A, const float* __restrict__ rew,
                                     const uint8_t* __restrict__ done, double discount, int max_traj_len,
                                     double* __restrict__ carry, float* __restrict__ ep_reward,
                                     float* __restrict__ ep_disc, int32_t* __restrict__ ep_len,
                                     uint8_t* __restrict__ ep_end) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  double* c = carry + (size_t)e * (A + 3);
  double len = c[A], disc = c[A + 1], pw = c[A + 2];
  if (len == 0.0) pw = 1.0;
  for (int t = 0; t < T; ++t) {
    const size_t k = ((size_t)t * E + e);
    double mean = 0.0;
    for (int a = 0; a < A; ++a) {
      const double r = (double)rew[k * A + a];
      c[a] += r;                                              // _episode_reward += rewardlist
      mean += r;
    }
    mean /= (double)A;
    disc += mean * pw;                                        // _discount_sum of the agent-mean reward
    pw *= discount;
    len += 1.0;
    const bool end = done[k] != 0 || len >= (double)max_traj_len;   // __init__.py:352
    ep_end[k] = end ? 1 : 0;
    ep_len[k] = end ? (int32_t)len : 0;
    ep_disc[k] = end ? (float)disc : 0.0f;
    for (int a = 0; a < A; ++a) ep_reward[k * A + a] = end ? (float)c[a] : 0.0f;
    if (end) {
      for (int a = 0; a < A; ++a) c[a] = 0.0;
      len = 0.0; disc = 0.0; pw = 1.0;
    }
  }
  c[A] = len; c[A + 1] = disc; c[A + 2] = pw;
}

// Whole-episode records of an evaluation (rltools/rltools/util.py:141-231): one thread per (env, agent) column walks
// the time axis.  carry [E][A][MADRL_EVAL_CARRY_WORDS] 8-byte words: ret, qsum, G, discount^len (doubles), len,
// episodes completed, the C info sums (int64; only agent 0's column sums the env's info); zeroed = a fresh start.
// G_s = sum_{j<=s} discount^j is carried forward, so sum_t q_t = sum_s r_s G_s needs no future reward.  Every
// float64 operation is rounded on its own (__dadd_rn / __dmul_rn): a contraction into fma would change the bits
// between builds and against the NumPy oracle.
template <typename R>
__global__ void eval_episodes_kernel(int T, int E, int A, int C, const R* __restrict__ rew,
                                     const uint8_t* __restrict__ done, const int32_t* __restrict__ info,
                                     double discount, int K, void* __restrict__ carry, double* __restrict__ ret_out,
                                     double* __restrict__ qsum_out, int32_t* __restrict__ len_out,
                                     int64_t* __restrict__ info_out) {
  const size_t n = (size_t)E * A;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int e = (int)(i / A), a = (int)(i - (size_t)e * A);
  double* cd = (double*)carry + i * MADRL_EVAL_CARRY_WORDS;
  int64_t* ci = (int64_t*)carry + i * MADRL_EVAL_CARRY_WORDS;
  double ret = cd[0], qsum = cd[1], G = cd[2];
  int64_t len = ci[4], k = ci[5];
  double pw = len == 0 ? 1.0 : cd[3];
  int64_t isum[MADRL_EVAL_INFO_MAX];
#pragma unroll
  for (int j = 0; j < MADRL_EVAL_INFO_MAX; ++j) isum[j] = ci[6 + j];
  for (int t = 0; t < T; ++t) {
    const size_t te = (size_t)t * E + e;
    const double r = (double)rew[te * A + a];
    ret = __dadd_rn(ret, r);
    G = __dadd_rn(G, pw);
    qsum = __dadd_rn(qsum, __dmul_rn(r, G));
    pw = __dmul_rn(pw, discount);
    ++len;
    if (a == 0) {
#pragma unroll
      for (int j = 0; j < MADRL_EVAL_INFO_MAX; ++j)
        if (j < C) isum[j] += info[te * C + j];
    }
    if (done[te]) {
      if (k < K) {
        const size_t rec = (size_t)k * E + e;
        ret_out[rec * A + a] = ret;
        qsum_out[rec * A + a] = qsum;
        if (a == 0) {
          len_out[rec] = (int32_t)len;
#pragma unroll
          for (int j = 0; j < MADRL_EVAL_INFO_MAX; ++j)
            if (j < C) info_out[rec * C + j] = isum[j];
        }
      }
      ++k;
      ret = qsum = G = 0.0;
      pw = 1.0;
      len = 0;
#pragma unroll
      for (int j = 0; j < MADRL_EVAL_INFO_MAX; ++j) isum[j] = 0;
    }
  }
  cd[0] = ret; cd[1] = qsum; cd[2] = G; cd[3] = pw;
  ci[4] = len; ci[5] = k;
#pragma unroll
  for (int j = 0; j < MADRL_EVAL_INFO_MAX; ++j) ci[6 + j] = isum[j];
}


// ---------------------------------------------------------------------------------------------
// Whole-batch moments for advantage centring (rllab/rllab/algos/util.py:7-12, applied at
// rllab/rllab/sampler/base.py:82-86) and explained variance (rllab/rllab/misc/special.py:51-59).
// NumPy semantics: mean, then the population variance as the mean of squared deviations (two
// passes), float64 accumulation.  Deterministic: fixed grid, per-block partials combined in a fixed
// order by one warp (no atomics), so a given input always yields the same bits.
//
// Three series are derived per element from (a, b):  s0 = a,  s1 = b,  s2 = b - a  (b optional).
// The statistics are taken per column of a [rows][A] tensor (one agent's samples, concurrent mode), one group of
// kMomBlocks CTAs per column; the whole-batch passes are the one-column case.
#ifndef MADRL_MOM_BLOCKS
#define MADRL_MOM_BLOCKS 528           // 4 CTAs x 132 SMs (H100 SXM) (the CPU emulator of tests/emu builds with fewer)
#endif
constexpr int kMomBlocks = MADRL_MOM_BLOCKS;
constexpr int kMomThreads = 256;
constexpr int kMomSeries = 3;
static_assert(kMomBlocks * 2 * kMomSeries <= MADRL_MOMENTS_WS, "workspace too small");

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_min(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_down_sync(0xffffffffu, v, o));
  return v;
}

// pass 0 (means == nullptr): partial sums and minima; pass 1: partial sums of squared deviations.
// a, b are [n][A]; CTA blockIdx.x covers column blockIdx.x / kMomBlocks (an agent) as block blockIdx.x % kMomBlocks of
// a whole-batch pass over that column, whose means and part [kMomBlocks][2*kMomSeries] are that column's
// [MADRL_MOMENTS_STATS] and [MADRL_MOMENTS_WS] blocks.  The whole batch is the one-column case.
__global__ void __launch_bounds__(kMomThreads) moments_partial_kernel(size_t n, int A, const float* __restrict__ a,
                                                                      const float* __restrict__ b,
                                                                      const double* __restrict__ means,
                                                                      double* __restrict__ part) {
  const int col = (int)(blockIdx.x / kMomBlocks);
  const unsigned blk = blockIdx.x - col * kMomBlocks;
  if (means) means += (size_t)col * MADRL_MOMENTS_STATS;
  part += (size_t)col * MADRL_MOMENTS_WS;
  double acc[kMomSeries] = {0.0, 0.0, 0.0};
  double mn[kMomSeries] = {INFINITY, INFINITY, INFINITY};
  double mu[kMomSeries] = {0.0, 0.0, 0.0};
  if (means) {
#pragma unroll
    for (int s = 0; s < kMomSeries; ++s) mu[s] = means[s];
  }
  // element i of the column sits at k = i A + col; the loop runs over k, so that no 64-bit multiply or second
  // induction variable sits on the path to each load
  const size_t end = n * A, step = (size_t)kMomBlocks * blockDim.x * A;
  for (size_t k = ((size_t)blk * blockDim.x + threadIdx.x) * A + col; k < end; k += step) {
    const double va = (double)__ldcs(a + k);
    const double vb = b ? (double)__ldcs(b + k) : 0.0;
    const double v[kMomSeries] = {va, vb, vb - va};
#pragma unroll
    for (int s = 0; s < kMomSeries; ++s) {
      if (means) {
        const double d = v[s] - mu[s];
        acc[s] += d * d;
      } else {
        acc[s] += v[s];
        mn[s] = fmin(mn[s], v[s]);
      }
    }
  }
  __shared__ double sh[kMomThreads / 32][2 * kMomSeries];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int s = 0; s < kMomSeries; ++s) {
    const double t = warp_sum(acc[s]);
    const double m = warp_min(mn[s]);
    if (lane == 0) { sh[w][2 * s] = t; sh[w][2 * s + 1] = m; }
  }
  __syncthreads();
  if (threadIdx.x < 2 * kMomSeries) {
    double r = sh[0][threadIdx.x];
    for (int k = 1; k < kMomThreads / 32; ++k)
      r = (threadIdx.x & 1) ? fmin(r, sh[k][threadIdx.x]) : r + sh[k][threadIdx.x];
    part[(size_t)blk * 2 * kMomSeries + threadIdx.x] = r;
  }
}

// One warp folds the block partials in a fixed order.  pass 0: stats[s] = mean_s, stats[6+s] = min_s;
// pass 1: stats[3+s] = var_s (population).
// One warp per column (agent): CTA c folds the partials at part + c * MADRL_MOMENTS_WS into stats + c * 9.
__global__ void moments_finalize_kernel(size_t n, const double* __restrict__ part, int pass,
                                        double* __restrict__ stats) {
  const int lane = threadIdx.x;
  part += (size_t)blockIdx.x * MADRL_MOMENTS_WS;
  stats += (size_t)blockIdx.x * MADRL_MOMENTS_STATS;
#pragma unroll
  for (int s = 0; s < kMomSeries; ++s) {
    double t = 0.0, m = INFINITY;
    for (int k = lane; k < kMomBlocks; k += 32) {
      t += part[(size_t)k * 2 * kMomSeries + 2 * s];
      m = fmin(m, part[(size_t)k * 2 * kMomSeries + 2 * s + 1]);
    }
    t = warp_sum(t);
    m = warp_min(m);
    if (lane == 0) {
      if (pass == 0) { stats[s] = t / (double)n; stats[6 + s] = m; }
      else stats[3 + s] = t / (double)n;
    }
  }
}

// center_advantages: (x - mean) / (std + 1e-8); shift_advantages_to_positive: (x - min) + 1e-8 on the
// (possibly centred) values, util.py:7-12.
__global__ void center_apply_kernel(size_t n, float* __restrict__ x, const double* __restrict__ stats,
                                    int center, int positive) {
  const double mean = stats[0], sd = sqrt(stats[3]) + 1e-8, mn = stats[6];
  const double cmin = center ? (mn - mean) / sd : mn;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    double v = (double)x[i];
    if (center) v = (v - mean) / sd;
    if (positive) v = (v - cmin) + 1e-8;
    __stcs(x + i, (float)v);
  }
}

// The same per column of x [n][A], with column a's statistics (stats [A][MADRL_MOMENTS_STATS]); the per-agent
// constants are formed once per CTA by the expressions above.
__global__ void center_apply_agents_kernel(size_t n, int A, float* __restrict__ x, const double* __restrict__ stats,
                                           int center, int positive) {
  __shared__ double sc[MADRL_AGENTS_MAX][3];
  for (int c = threadIdx.x; c < A; c += blockDim.x) {
    const double* st = stats + (size_t)c * MADRL_MOMENTS_STATS;
    const double mean = st[0], sd = sqrt(st[3]) + 1e-8, mn = st[6];
    sc[c][0] = mean;
    sc[c][1] = sd;
    sc[c][2] = center ? (mn - mean) / sd : mn;
  }
  __syncthreads();
  const size_t total = n * (size_t)A, stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int c = (int)(i % (size_t)A);
    double v = (double)x[i];
    if (center) v = (v - sc[c][0]) / sc[c][1];
    if (positive) v = (v - sc[c][2]) + 1e-8;
    __stcs(x + i, (float)v);
  }
}


// ---- path packing: time-major rollout tensors -> rllab's per-(env, episode, agent) paths --------
// (rllab/rllab/sampler/ma_sampler.py:52-100 dec_rollout returns one path dict per agent with
// `observations / actions / rewards / env_infos` arrays; VecEnvExecutor cuts episodes at `done`,
// rllab/sandbox/rocky/tf/envs/vec_env_executor.py:16-28.)  Every (t, env, agent) row of a rollout
// belongs to exactly one path, so packing is a permutation of rows: paths are ordered (env, episode,
// agent) like the host `to_paths`, the rows of a path are consecutive, and row (t, e, a) lands at
//     e*T*A + s*A + a*L + (t - s)        s, L = start and length of the episode containing t.
// paths_plan_kernel: one thread per env walks `done` once (T bytes) and writes s / L per (t, env),
// the per-episode records and the episode count; paths_pack_kernel: one warp per source row, coalesced
// reads and writes of D 4-byte words -- a pure HBM-bound permutation (2 x the tensor's bytes).
__global__ void paths_plan_kernel(int T, int E, int A, const uint8_t* __restrict__ done,
                                  int32_t* __restrict__ seg_start, int32_t* __restrict__ seg_len,
                                  int32_t* __restrict__ n_episodes, int32_t* __restrict__ ep_rec) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  int s = 0, n = 0;
  for (int t = 0; t < T; ++t) {
    const bool end = done[(size_t)t * E + e] != 0;
    if (end || t == T - 1) {
      const int L = t + 1 - s;
      for (int u = s; u <= t; ++u) { seg_start[(size_t)u * E + e] = s; seg_len[(size_t)u * E + e] = L; }
      // episode record n of this env (at most T episodes): start step, length, terminated
      int32_t* r = ep_rec + 3 * ((size_t)e * T + n);
      r[0] = s; r[1] = L; r[2] = end ? 1 : 0;
      ++n;
      s = t + 1;
    }
  }
  n_episodes[e] = n;
}

// The D words of one row, moved by kLanes threads: a warp (32, lanes stride over the words: coalesced, streaming
// accesses) or one thread (1: rows of at most 4 words -- rewards, returns, advantages, actions, infos -- with plain
// accesses: pad_paths at the C2 shape ran about 3 % faster with them than with streaming ones on an H100 80GB HBM3 at
// 700 W).  in == NULL writes zeros.
template <int kLanes, typename W>
__device__ __forceinline__ void copy_row(W* __restrict__ out, const W* __restrict__ in, int D) {
  if (kLanes == 1) {
    if (in)
      for (int d = 0; d < D; ++d) out[d] = in[d];
    else
      for (int d = 0; d < D; ++d) out[d] = (W)0;
    return;
  }
  const int lane = threadIdx.x % kLanes;
  if (in)
    for (int d = lane; d < D; d += kLanes) __stcs(out + d, __ldcs(in + d));
  else
    for (int d = lane; d < D; d += kLanes) __stcs(out + d, (W)0);
}

// W = the row element: uint32_t (4-byte words) or uint16_t (bfloat16 observations; rows of odd length).
// `first` != NULL: observations are shifted by one step (action_obs_row).
template <int kLanes, typename W>
__global__ void paths_pack_kernel(int T, int E, int A, int D, const W* __restrict__ src,
                                  const W* __restrict__ first, const int32_t* __restrict__ seg_start,
                                  const int32_t* __restrict__ seg_len, W* __restrict__ dst) {
  const size_t row = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) / kLanes;   // source row (t, e, a)
  const size_t rows = (size_t)T * E * A;
  if (row >= rows) return;
  const int a = (int)(row % A);
  const size_t te = row / A;
  const int e = (int)(te % E), t = (int)(te / E);
  const int s = seg_start[te], L = seg_len[te];
  W* out = dst + ((size_t)e * T * A + (size_t)s * A + (size_t)a * L + (t - s)) * D;
  copy_row<kLanes>(out, action_obs_row(row, (size_t)E * A, D, src, first), D);
}

// ---- padded paths: rllab's recurrent sample batch (rllab/rllab/sampler/base.py:105-161) ----------
// Every path of a record table rec [P][4] = (env, agent, start, length) becomes Lmax rows of dst [P][Lmax][D]: its
// steps, then zeros (tensor_utils.pad_tensor_n).  Organised by DESTINATION row (p, i), so each output word is
// written once -- the padding by the same store stream as the data, no clearing pass -- and each source row is read
// once.  A = 1 (per-env tensors): the record's agent is ignored.  `first`: the one-step shift of paths_pack_kernel.
template <int kLanes, typename W>
__global__ void paths_pad_kernel(int E, int A, int D, size_t rows, int Lmax, const W* __restrict__ src,
                                 const W* __restrict__ first, const int32_t* __restrict__ rec, W* __restrict__ dst) {
  const size_t row = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) / kLanes;   // padded row (p, i)
  if (row >= rows) return;
  const size_t p = row / Lmax;
  const int i = (int)(row - p * Lmax);
  const int32_t* r = rec + 4 * p;
  const W* in = nullptr;
  if (i < __ldg(r + 3)) {
    const int e = __ldg(r), a = A == 1 ? 0 : __ldg(r + 1), t = __ldg(r + 2) + i;
    in = action_obs_row(((size_t)t * E + e) * A + a, (size_t)E * A, D, src, first);
  }
  copy_row<kLanes>(dst + row * D, in, D);
}

// Per path: the float64 sum of its rewards in time order (Python's sum() over the reference's float64 rewards) and
// its first return, the two per-path inputs of process_samples' tabular statistics (base.py:144-147, :170-180).
__global__ void path_sums_kernel(int E, int A, int P, const float* __restrict__ rew, const float* __restrict__ ret,
                                 const int32_t* __restrict__ rec, double* __restrict__ sums,
                                 double* __restrict__ first_ret) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const int32_t* r = rec + 4 * (size_t)p;
  const int e = r[0], a = A == 1 ? 0 : r[1], s = r[2], L = r[3];
  const size_t stride = (size_t)E * A, k0 = ((size_t)s * E + e) * A + a;
  double acc = 0.0;
  for (int i = 0; i < L; ++i) acc += (double)rew[k0 + (size_t)i * stride];
  sums[p] = acc;
  first_ret[p] = (double)ret[k0];
}


// ---- rltools' sample processing (rltools/rltools/samplers/__init__.py:35-88) -----------------------------------
// Running standardiser (nn.Standardizer, rltools/rltools/nn.py:533-592): the float64 column sums of x and x^2 over
// the rows of a batch, from which the caller forms the batch means of update().  Rows r = k G + g of group g
// (G = 1: every row; G = A: agent g's rows of a [..][A][D] tensor), read through action_obs_row (shift = the rows
// before the first step).  Fixed grid: each group's rows are cut into rm_slices(G) slices, a CTA owns 32 columns
// of one slice (8 warps over its rows, lane = column), and the slice partials are summed in ascending order by a
// second pass: same inputs, same bits, on any SM count.  Squares of widened float32 values are exact in float64.
#ifndef MADRL_RM_SLICES
#define MADRL_RM_SLICES 64             // (the CPU emulator tests of tests/test_emulated_rltools.py build with fewer)
#endif
constexpr int kRmSlices = MADRL_RM_SLICES;
constexpr int kRmWarps = 8;
__host__ __device__ __forceinline__ int rm_slices(int G) { return (kRmSlices + G - 1) / G; }

template <typename O>
__global__ void __launch_bounds__(kRmWarps * 32) running_moments_partial_kernel(size_t R, int G, int D, size_t shift,
                                                                                const O* __restrict__ x,
                                                                                const O* __restrict__ first,
                                                                                double* __restrict__ ws) {
  const int CB = (D + 31) / 32, S = rm_slices(G);
  const int cb = (int)(blockIdx.x % CB), gs = (int)(blockIdx.x / CB), g = gs / S, sl = gs - g * S;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, d = cb * 32 + lane;
  const size_t k1 = R * (sl + 1) / S;
  double s1 = 0.0, s2 = 0.0;
  if (d < D)
    for (size_t k = R * sl / S + w; k < k1; k += kRmWarps) {
      const double v = (double)obs_widen<float>(action_obs_row(k * G + g, shift, D, x, first)[d]);
      s1 += v;
      s2 += v * v;
    }
  __shared__ double sh[kRmWarps][2][32];
  sh[w][0][lane] = s1;
  sh[w][1][lane] = s2;
  __syncthreads();
  if (w < 2 && d < D) {
    double t = 0.0;
    for (int i = 0; i < kRmWarps; ++i) t += sh[i][w][lane];
    ws[((size_t)gs * 2 + w) * D + d] = t;
  }
}

// sums[g][j][d] (j = 0: x, 1: x^2) = the slices' partials in ascending order.
__global__ void running_moments_finalize_kernel(int G, int D, const double* __restrict__ ws, double* __restrict__ sums) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)G * 2 * D) return;
  const int S = rm_slices(G);
  const size_t g = i / (2 * (size_t)D), jd = i - g * 2 * D;
  double t = 0.0;
  for (int sl = 0; sl < S; ++sl) t += ws[((size_t)g * S + sl) * 2 * D + jd];
  sums[i] = t;
}

// Time-dependent baseline (samplers/__init__.py:46-52): bin i of group g holds the float64 sum of q and the count
// of the rows with time index i (lfb_index: the baseline's own rule), i.e. of the paths that reach i; G = 1 pools
// every agent's rows, G = A keeps one set of bins per agent.  The envs are cut into tb_slices(G) fixed slices; a
// thread owns one (group, slice, bin) and walks its slice's envs and their paths in order (madrl_paths_plan's
// records), so each partial has one fixed order; the second pass sums them over the slices in ascending order and
// the third writes mean = sum / count back to every row.  No atomics: same inputs, same bits.  Each thread scans
// every path record of its slice for its one bin, so the work is O(L x paths), not O(rows): cheap while paths are
// few per env, more when one env runs the whole horizon (L = T) while the others end often.
#ifndef MADRL_TB_SLICES
#define MADRL_TB_SLICES 32             // (the CPU emulator tests of tests/test_emulated_rltools.py build with fewer)
#endif
constexpr int kTbSlices = MADRL_TB_SLICES;
constexpr int kTbThreads = 128;
__host__ __device__ __forceinline__ int tb_slices(int G) { return (kTbSlices + G - 1) / G; }

__global__ void time_baseline_partial_kernel(int T, int E, int A, int G, int L, const float* __restrict__ q,
                                             const int32_t* __restrict__ n_ep, const int32_t* __restrict__ ep_rec,
                                             const int32_t* __restrict__ t0, double* __restrict__ ws_sum,
                                             int32_t* __restrict__ ws_cnt) {
  const int LB = (L + kTbThreads - 1) / kTbThreads, S = tb_slices(G);
  const int lb = (int)(blockIdx.x % LB), gs = (int)(blockIdx.x / LB), g = gs / S, sl = gs - g * S;
  const int i = lb * kTbThreads + threadIdx.x;
  if (i >= L) return;
  const int e1 = (int)((int64_t)E * (sl + 1) / S);
  double sum = 0.0;
  int32_t cnt = 0;
  for (int e = (int)((int64_t)E * sl / S); e < e1; ++e) {
    const int n = n_ep[e];
    for (int j = 0; j < n; ++j) {
      const int32_t* rec = ep_rec + 3 * ((size_t)e * T + j);
      const int pos = i - ((j == 0 && t0 != nullptr) ? t0[e] : 0);
      if (pos < 0 || pos >= rec[1]) continue;
      const float* qr = q + ((size_t)(rec[0] + pos) * E + e) * A;
      if (G == 1) {
        for (int a = 0; a < A; ++a) sum += (double)qr[a];
        cnt += A;
      } else {
        sum += (double)qr[g];
        cnt += 1;
      }
    }
  }
  ws_sum[(size_t)gs * L + i] = sum;
  ws_cnt[(size_t)gs * L + i] = cnt;
}

__global__ void time_baseline_bins_kernel(int G, int L, const double* __restrict__ ws_sum,
                                          const int32_t* __restrict__ ws_cnt, double* __restrict__ bin_sum,
                                          int32_t* __restrict__ bin_cnt) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)G * L) return;
  const int S = tb_slices(G);
  const size_t g = i / L, b = i - g * L;
  double sum = 0.0;
  int32_t cnt = 0;
  for (int sl = 0; sl < S; ++sl) {
    sum += ws_sum[((size_t)g * S + sl) * L + b];
    cnt += ws_cnt[((size_t)g * S + sl) * L + b];
  }
  bin_sum[i] = sum;
  bin_cnt[i] = cnt;
}

// simplev[t][e][a] = the mean of its bin (nanmean's sum / count), float32.  A row whose index is past the L bins
// (an L too small for the rollout) gets NaN rather than another bin's value.
__global__ void time_baseline_apply_kernel(int T, int E, int A, int G, int L, const int32_t* __restrict__ seg_start,
                                           const int32_t* __restrict__ t0, const double* __restrict__ bin_sum,
                                           const int32_t* __restrict__ bin_cnt, float* __restrict__ simplev) {
  const size_t r = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= (size_t)T * E * A) return;
  const size_t te = r / A;
  const int idx = lfb_index(te, E, seg_start, t0);
  const size_t b = (G == 1 ? 0 : (r - te * A) * (size_t)L) + idx;
  simplev[r] = (idx >= 0 && idx < L) ? (float)(bin_sum[b] / (double)bin_cnt[b]) : __int_as_float(0x7fc00000);
}

}  // namespace madrl

using namespace madrl;

extern "C" int madrl_episode_stats_f32(int T, int E, int A, const float* rew_dev, const uint8_t* done_dev,
                                       double discount, int max_traj_len, double* carry_dev,
                                       float* ep_reward_dev, float* ep_disc_dev, int32_t* ep_len_dev,
                                       uint8_t* ep_end_dev, void* stream) {
  MADRL_REQUIRE(T >= 1 && E >= 1 && A >= 1 && max_traj_len >= 1, "bad sizes");
  MADRL_REQUIRE(rew_dev && done_dev && carry_dev && ep_reward_dev && ep_disc_dev && ep_len_dev && ep_end_dev,
                "NULL buffer");
  MADRL_LAUNCH(episode_stats_kernel, (unsigned)((E + 127) / 128), 128, 0, (cudaStream_t)stream, 
      T, E, A, rew_dev, done_dev, discount, max_traj_len, carry_dev, ep_reward_dev, ep_disc_dev, ep_len_dev,
      ep_end_dev);
  g_launches.fetch_add(1);
  MADRL_CUDA_CHECK(cudaGetLastError());
  return MADRL_OK;
}

template <typename R>
static int eval_episodes(int T, int E, int A, int C, const R* rew_dev, const uint8_t* done_dev, const int32_t* info_dev,
                         double discount, int K, void* carry_dev, double* ret_dev, double* qsum_dev, int32_t* len_dev,
                         int64_t* info_sum_dev, void* stream) {
  MADRL_REQUIRE(T >= 1 && E >= 1 && A >= 1 && K >= 1, "bad sizes");
  MADRL_REQUIRE(C >= 0 && C <= MADRL_EVAL_INFO_MAX, "info columns must be in [0, %d], got %d", MADRL_EVAL_INFO_MAX, C);
  MADRL_REQUIRE((size_t)K * E * A < ((size_t)1 << 31), "K*E*A must be < 2^31");
  MADRL_REQUIRE(discount >= 0.0 && discount <= 1.0, "discount must be in [0, 1], got %g", discount);
  MADRL_REQUIRE(rew_dev && done_dev && carry_dev && ret_dev && qsum_dev && len_dev, "NULL buffer");
  MADRL_REQUIRE(C == 0 || (info_dev && info_sum_dev), "NULL info buffer with %d info columns", C);
  const size_t n = (size_t)E * A;
  MADRL_LAUNCH(eval_episodes_kernel<R>, (unsigned)((n + 127) / 128), 128, 0, (cudaStream_t)stream, T, E, A, C, rew_dev,
               done_dev, info_dev, discount, K, carry_dev, ret_dev, qsum_dev, len_dev, info_sum_dev);
  g_launches.fetch_add(1);
  MADRL_CUDA_CHECK(cudaGetLastError());
  return MADRL_OK;
}

extern "C" int madrl_eval_episodes_f32(int T, int E, int A, int C, const float* rew_dev, const uint8_t* done_dev,
                                       const int32_t* info_dev, double discount, int K, void* carry_dev,
                                       double* ret_dev, double* qsum_dev, int32_t* len_dev, int64_t* info_sum_dev,
                                       void* stream) {
  return eval_episodes(T, E, A, C, rew_dev, done_dev, info_dev, discount, K, carry_dev, ret_dev, qsum_dev, len_dev,
                       info_sum_dev, stream);
}

extern "C" int madrl_eval_episodes_f64(int T, int E, int A, int C, const double* rew_dev, const uint8_t* done_dev,
                                       const int32_t* info_dev, double discount, int K, void* carry_dev,
                                       double* ret_dev, double* qsum_dev, int32_t* len_dev, int64_t* info_sum_dev,
                                       void* stream) {
  return eval_episodes(T, E, A, C, rew_dev, done_dev, info_dev, discount, K, carry_dev, ret_dev, qsum_dev, len_dev,
                       info_sum_dev, stream);
}

extern "C" int madrl_gae_f32(int T, int E, int A, const float* rew_dev, const float* value_dev,
                             const uint8_t* done_dev, const float* last_value_dev, double discount,
                             double gae_lambda, float* adv_dev, float* ret_dev, void* stream) {
  MADRL_REQUIRE(T >= 1 && E >= 1 && A >= 1, "bad sizes");
  MADRL_REQUIRE(rew_dev && value_dev && done_dev && adv_dev && ret_dev, "NULL buffer");
  const size_t n = (size_t)E * A;
  MADRL_LAUNCH(gae_kernel, (unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream, 
      T, E, A, rew_dev, value_dev, done_dev, last_value_dev, discount, gae_lambda, adv_dev, ret_dev);
  g_launches.fetch_add(1);
  MADRL_CUDA_CHECK(cudaGetLastError());
  return MADRL_OK;
}

template <typename O>
static int frame_stack(int T, int E, int A, int D, int B, const O* obs_dev, const uint8_t* done_dev, O* carry_dev,
                       O* out_dev, void* stream) {
  MADRL_REQUIRE(T >= 1 && E >= 1 && A >= 1 && D >= 1, "bad sizes");
  MADRL_REQUIRE(B >= 1 && B <= 8, "buffer_size must be in [1,8], got %d", B);
  MADRL_REQUIRE(obs_dev && done_dev && carry_dev && out_dev, "NULL buffer");
  const size_t n = (size_t)E * A * D;
  const unsigned grid = (unsigned)((n + 255) / 256);
  cudaStream_t s = (cudaStream_t)stream;
#define MADRL_FS(BB) case BB: MADRL_LAUNCH((frame_stack_kernel<BB, O>), grid, 256, 0, s, T, n, A * D, obs_dev, done_dev, E, carry_dev, out_dev); break
  switch (B) { MADRL_FS(1); MADRL_FS(2); MADRL_FS(3); MADRL_FS(4); MADRL_FS(5); MADRL_FS(6); MADRL_FS(7); MADRL_FS(8); }
#undef MADRL_FS
  g_launches.fetch_add(1);
  MADRL_CUDA_CHECK(cudaGetLastError());
  return MADRL_OK;
}

extern "C" int madrl_frame_stack_f32(int T, int E, int A, int D, int B, const float* obs_dev,
                                     const uint8_t* done_dev, float* carry_dev, float* out_dev,
                                     void* stream) {
  return frame_stack(T, E, A, D, B, obs_dev, done_dev, carry_dev, out_dev, stream);
}

extern "C" int madrl_frame_stack_bf16(int T, int E, int A, int D, int B, const void* obs_dev,
                                      const uint8_t* done_dev, void* carry_dev, void* out_dev, void* stream) {
  return frame_stack(T, E, A, D, B, (const uint16_t*)obs_dev, done_dev, (uint16_t*)carry_dev, (uint16_t*)out_dev, stream);
}

template <typename O>
static int standardize(int T, size_t n, O* x_dev, double* mean_dev, double* var_dev, double alpha, double eps,
                       int center, double scale, int enable, void* stream) {
  MADRL_REQUIRE(T >= 1 && n >= 1, "bad sizes");
  MADRL_REQUIRE(x_dev && mean_dev && var_dev, "NULL buffer");
  MADRL_LAUNCH(standardize_kernel<O>, (unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream,
      T, n, x_dev, mean_dev, var_dev, alpha, eps, center, scale, enable);
  g_launches.fetch_add(1);
  MADRL_CUDA_CHECK(cudaGetLastError());
  return MADRL_OK;
}

extern "C" int madrl_standardize_f32(int T, size_t n, float* x_dev, double* mean_dev, double* var_dev,
                                     double alpha, double eps, int center, double scale, int enable,
                                     void* stream) {
  return standardize(T, n, x_dev, mean_dev, var_dev, alpha, eps, center, scale, enable, stream);
}

extern "C" int madrl_standardize_bf16(int T, size_t n, void* x_dev, double* mean_dev, double* var_dev,
                                      double alpha, double eps, int center, double scale, int enable,
                                      void* stream) {
  return standardize(T, n, (uint16_t*)x_dev, mean_dev, var_dev, alpha, eps, center, scale, enable, stream);
}

// The A columns of [n][A]; the whole batch of n elements is A = 1.
static int run_moments(size_t n, int A, const float* a, const float* b, double* stats, double* ws, cudaStream_t s) {
  const unsigned grid = (unsigned)(kMomBlocks * A);
  MADRL_LAUNCH(moments_partial_kernel, grid, kMomThreads, 0, s, n, A, a, b, nullptr, ws);
  MADRL_LAUNCH(moments_finalize_kernel, (unsigned)A, 32, 0, s, n, ws, 0, stats);
  MADRL_LAUNCH(moments_partial_kernel, grid, kMomThreads, 0, s, n, A, a, b, stats, ws);
  MADRL_LAUNCH(moments_finalize_kernel, (unsigned)A, 32, 0, s, n, ws, 1, stats);
  g_launches.fetch_add(4);
  MADRL_CUDA_CHECK(cudaGetLastError());
  return MADRL_OK;
}

extern "C" int madrl_center_advantages_f32(size_t n, float* adv_dev, int center, int positive,
                                           double* stats_dev, double* workspace_dev, void* stream) {
  MADRL_REQUIRE(n >= 1, "bad sizes");
  MADRL_REQUIRE(adv_dev && stats_dev && workspace_dev, "NULL buffer");
  cudaStream_t s = (cudaStream_t)stream;
  const int rc = run_moments(n, 1, adv_dev, nullptr, stats_dev, workspace_dev, s);
  if (rc) return rc;
  if (center || positive) {
    MADRL_LAUNCH(center_apply_kernel, kMomBlocks, kMomThreads, 0, s, n, adv_dev, stats_dev, center, positive);
    g_launches.fetch_add(1);
    MADRL_CUDA_CHECK(cudaGetLastError());
  }
  return MADRL_OK;
}

extern "C" int madrl_moments_f32(size_t n, const float* a_dev, const float* b_dev, double* stats_dev,
                                 double* workspace_dev, void* stream) {
  MADRL_REQUIRE(n >= 1, "bad sizes");
  MADRL_REQUIRE(a_dev && stats_dev && workspace_dev, "NULL buffer");
  return run_moments(n, 1, a_dev, b_dev, stats_dev, workspace_dev, (cudaStream_t)stream);
}

extern "C" int madrl_center_advantages_agents_f32(size_t rows, int A, float* adv_dev, int center, int positive,
                                                  double* stats_dev, double* workspace_dev, void* stream) {
  MADRL_REQUIRE(rows >= 1, "bad sizes");
  MADRL_REQUIRE(A >= 1 && A <= MADRL_AGENTS_MAX, "n_agents must be in [1, %d], got %d", MADRL_AGENTS_MAX, A);
  MADRL_REQUIRE(adv_dev && stats_dev && workspace_dev, "NULL buffer");
  cudaStream_t s = (cudaStream_t)stream;
  const int rc = run_moments(rows, A, adv_dev, nullptr, stats_dev, workspace_dev, s);
  if (rc) return rc;
  if (center || positive) {
    MADRL_LAUNCH(center_apply_agents_kernel, kMomBlocks, kMomThreads, 0, s, rows, A, adv_dev, stats_dev, center,
                 positive);
    g_launches.fetch_add(1);
    MADRL_CUDA_CHECK(cudaGetLastError());
  }
  return MADRL_OK;
}

extern "C" int madrl_moments_agents_f32(size_t rows, int A, const float* a_dev, const float* b_dev,
                                        double* stats_dev, double* workspace_dev, void* stream) {
  MADRL_REQUIRE(rows >= 1, "bad sizes");
  MADRL_REQUIRE(A >= 1 && A <= MADRL_AGENTS_MAX, "n_agents must be in [1, %d], got %d", MADRL_AGENTS_MAX, A);
  MADRL_REQUIRE(a_dev && stats_dev && workspace_dev, "NULL buffer");
  return run_moments(rows, A, a_dev, b_dev, stats_dev, workspace_dev, (cudaStream_t)stream);
}

extern "C" int madrl_paths_plan(int T, int E, int A, const uint8_t* done_dev, int32_t* seg_start_dev,
                                int32_t* seg_len_dev, int32_t* n_episodes_dev, int32_t* ep_rec_dev, void* stream) {
  MADRL_REQUIRE(T >= 1 && E >= 1 && A >= 1, "bad shape");
  MADRL_REQUIRE((size_t)T * E * A < ((size_t)1 << 31), "T*E*A must be < 2^31 (row offsets are int32)");
  MADRL_REQUIRE(done_dev && seg_start_dev && seg_len_dev && n_episodes_dev && ep_rec_dev, "NULL pointer");
  MADRL_LAUNCH(paths_plan_kernel, (E + 127) / 128, 128, 0, (cudaStream_t)stream, T, E, A, done_dev, seg_start_dev,
               seg_len_dev, n_episodes_dev, ep_rec_dev);
  g_launches.fetch_add(1);
  MADRL_CUDA_CHECK(cudaGetLastError());
  return MADRL_OK;
}

// The grid of the row-copy kernels: one thread per row of at most 4 words, one warp per wider row.
template <typename... P, typename... Args>
static int launch_rows(void (*one_thread)(P...), void (*one_warp)(P...), size_t rows, int D, void* stream,
                       Args... args) {
  const bool narrow = D <= 4;
  const size_t blocks = ((narrow ? rows : rows * 32) + 255) / 256;
  MADRL_REQUIRE(blocks < ((size_t)1 << 31), "too many rows for one launch");
  if (narrow)
    MADRL_LAUNCH(one_thread, (unsigned)blocks, 256, 0, (cudaStream_t)stream, args...);
  else
    MADRL_LAUNCH(one_warp, (unsigned)blocks, 256, 0, (cudaStream_t)stream, args...);
  g_launches.fetch_add(1);
  MADRL_CUDA_CHECK(cudaGetLastError());
  return MADRL_OK;
}

template <typename W>
static int paths_pack(int T, int E, int A, int D, const void* src_dev, const void* first_dev,
                      const int32_t* seg_start_dev, const int32_t* seg_len_dev, void* dst_dev, void* stream) {
  MADRL_REQUIRE(T >= 1 && E >= 1 && A >= 1 && D >= 1, "bad shape");
  MADRL_REQUIRE(src_dev && seg_start_dev && seg_len_dev && dst_dev, "NULL pointer");
  return launch_rows(paths_pack_kernel<1, W>, paths_pack_kernel<32, W>, (size_t)T * E * A, D, stream, T, E, A, D,
                     (const W*)src_dev, (const W*)first_dev, seg_start_dev, seg_len_dev, (W*)dst_dev);
}

extern "C" int madrl_paths_pack_u32(int T, int E, int A, int D, const void* src_dev, const void* first_dev,
                                    const int32_t* seg_start_dev, const int32_t* seg_len_dev, void* dst_dev,
                                    void* stream) {
  return paths_pack<uint32_t>(T, E, A, D, src_dev, first_dev, seg_start_dev, seg_len_dev, dst_dev, stream);
}

extern "C" int madrl_paths_pack_u16(int T, int E, int A, int D, const void* src_dev, const void* first_dev,
                                    const int32_t* seg_start_dev, const int32_t* seg_len_dev, void* dst_dev,
                                    void* stream) {
  return paths_pack<uint16_t>(T, E, A, D, src_dev, first_dev, seg_start_dev, seg_len_dev, dst_dev, stream);
}

template <typename W>
static int paths_pad(int T, int E, int A, int D, int P, int Lmax, const void* src_dev, const void* first_dev,
                     const int32_t* rec_dev, void* dst_dev, void* stream) {
  MADRL_REQUIRE(T >= 1 && E >= 1 && A >= 1 && D >= 1 && P >= 1 && Lmax >= 1, "bad shape");
  MADRL_REQUIRE(src_dev && rec_dev && dst_dev, "NULL pointer");
  const size_t rows = (size_t)P * Lmax;
  return launch_rows(paths_pad_kernel<1, W>, paths_pad_kernel<32, W>, rows, D, stream, E, A, D, rows, Lmax,
                     (const W*)src_dev, (const W*)first_dev, rec_dev, (W*)dst_dev);
}

extern "C" int madrl_paths_pad_u32(int T, int E, int A, int D, int P, int Lmax, const void* src_dev,
                                   const void* first_dev, const int32_t* rec_dev, void* dst_dev, void* stream) {
  return paths_pad<uint32_t>(T, E, A, D, P, Lmax, src_dev, first_dev, rec_dev, dst_dev, stream);
}

extern "C" int madrl_paths_pad_u16(int T, int E, int A, int D, int P, int Lmax, const void* src_dev,
                                   const void* first_dev, const int32_t* rec_dev, void* dst_dev, void* stream) {
  return paths_pad<uint16_t>(T, E, A, D, P, Lmax, src_dev, first_dev, rec_dev, dst_dev, stream);
}

extern "C" int madrl_path_sums_f32(int T, int E, int A, int P, const float* rew_dev, const float* ret_dev,
                                   const int32_t* rec_dev, double* sums_dev, double* first_ret_dev, void* stream) {
  MADRL_REQUIRE(T >= 1 && E >= 1 && A >= 1 && P >= 1, "bad shape");
  MADRL_REQUIRE(rew_dev && ret_dev && rec_dev && sums_dev && first_ret_dev, "NULL pointer");
  MADRL_LAUNCH(path_sums_kernel, (unsigned)((P + 127) / 128), 128, 0, (cudaStream_t)stream, E, A, P, rew_dev, ret_dev,
               rec_dev, sums_dev, first_ret_dev);
  g_launches.fetch_add(1);
  MADRL_CUDA_CHECK(cudaGetLastError());
  return MADRL_OK;
}

template <typename O>
static int standardize_obs_terminal(int T, int E, size_t per_env, O* x_dev, O* term_dev, const uint8_t* done_dev,
                                    double* mean_dev, double* var_dev, double alpha, double eps, void* stream) {
  MADRL_REQUIRE(T >= 1 && E >= 1 && per_env >= 1, "bad sizes");
  MADRL_REQUIRE(x_dev && term_dev && done_dev && mean_dev && var_dev, "NULL buffer");
  const size_t n = (size_t)E * per_env;
  MADRL_LAUNCH(standardize_terminal_kernel<O>, (unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream, T, E, per_env,
               x_dev, term_dev, done_dev, mean_dev, var_dev, alpha, eps);
  g_launches.fetch_add(1);
  MADRL_CUDA_CHECK(cudaGetLastError());
  return MADRL_OK;
}

extern "C" int madrl_standardize_obs_terminal_f32(int T, int E, size_t per_env, float* x_dev, float* term_dev,
                                                  const uint8_t* done_dev, double* mean_dev, double* var_dev,
                                                  double alpha, double eps, void* stream) {
  return standardize_obs_terminal(T, E, per_env, x_dev, term_dev, done_dev, mean_dev, var_dev, alpha, eps, stream);
}

extern "C" int madrl_standardize_obs_terminal_bf16(int T, int E, size_t per_env, void* x_dev, void* term_dev,
                                                   const uint8_t* done_dev, double* mean_dev, double* var_dev,
                                                   double alpha, double eps, void* stream) {
  return standardize_obs_terminal(T, E, per_env, (uint16_t*)x_dev, (uint16_t*)term_dev, done_dev, mean_dev, var_dev,
                                  alpha, eps, stream);
}

template <typename O>
static int obs_wrap_step(int E, int A, int D, int B, O* obs_dev, O* term_dev, const uint8_t* done_dev,
                         const O* prev_dev, O* out_dev, double* mean_dev, double* var_dev, double alpha, double eps,
                         void* stream) {
  MADRL_REQUIRE(E >= 1 && A >= 1 && D >= 1, "bad sizes");
  MADRL_REQUIRE(B >= 1 && B <= 8, "buffer_size must be in [1,8], got %d", B);
  MADRL_REQUIRE(obs_dev && done_dev, "NULL buffer");
  MADRL_REQUIRE(!mean_dev == !var_dev, "mean and var must both be given (obsnorm) or both be NULL");
  MADRL_REQUIRE(!mean_dev || term_dev, "obsnorm needs the terminal observations");
  MADRL_REQUIRE(B == 1 || (prev_dev && out_dev), "buffer_size > 1 needs prev and out");
  const size_t per_env = (size_t)A * D, n = (size_t)E * per_env;
  const unsigned grid = (unsigned)((n + 255) / 256);
  cudaStream_t s = (cudaStream_t)stream;
#define MADRL_WS(BB) case BB: MADRL_LAUNCH((obs_wrap_step_kernel<BB, O>), grid, 256, 0, s, n, per_env, obs_dev, term_dev, done_dev, prev_dev, out_dev, mean_dev, var_dev, alpha, eps); break
  switch (B) { MADRL_WS(1); MADRL_WS(2); MADRL_WS(3); MADRL_WS(4); MADRL_WS(5); MADRL_WS(6); MADRL_WS(7); MADRL_WS(8); }
#undef MADRL_WS
  g_launches.fetch_add(1);
  MADRL_CUDA_CHECK(cudaGetLastError());
  return MADRL_OK;
}

extern "C" int madrl_obs_wrap_step_f32(int E, int A, int D, int B, float* obs_dev, float* term_dev,
                                       const uint8_t* done_dev, const float* prev_dev, float* out_dev,
                                       double* mean_dev, double* var_dev, double alpha, double eps, void* stream) {
  return obs_wrap_step(E, A, D, B, obs_dev, term_dev, done_dev, prev_dev, out_dev, mean_dev, var_dev, alpha, eps,
                       stream);
}

extern "C" int madrl_obs_wrap_step_bf16(int E, int A, int D, int B, void* obs_dev, void* term_dev,
                                        const uint8_t* done_dev, const void* prev_dev, void* out_dev,
                                        double* mean_dev, double* var_dev, double alpha, double eps, void* stream) {
  return obs_wrap_step(E, A, D, B, (uint16_t*)obs_dev, (uint16_t*)term_dev, done_dev, (const uint16_t*)prev_dev,
                       (uint16_t*)out_dev, mean_dev, var_dev, alpha, eps, stream);
}

template <typename O>
static int running_moments(size_t R, int G, int D, size_t shift, const void* x_dev, const void* first_dev,
                           double* sums_dev, double* ws_dev, void* stream) {
  MADRL_REQUIRE(R >= 1 && D >= 1, "bad sizes");
  MADRL_REQUIRE(G >= 1 && G <= MADRL_AGENTS_MAX, "groups must be in [1, %d], got %d", MADRL_AGENTS_MAX, G);
  MADRL_REQUIRE(!first_dev || (shift >= 1 && shift <= R * G), "shift must be in [1, rows] with a first row block");
  MADRL_REQUIRE(x_dev && sums_dev && ws_dev, "NULL buffer");
  const size_t blocks = (size_t)((D + 31) / 32) * rm_slices(G) * G;
  MADRL_REQUIRE(blocks < ((size_t)1 << 31), "too many columns for one launch");
  cudaStream_t s = (cudaStream_t)stream;
  MADRL_LAUNCH(running_moments_partial_kernel<O>, (unsigned)blocks, kRmWarps * 32, 0, s, R, G, D, shift,
               (const O*)x_dev, (const O*)first_dev, ws_dev);
  const size_t n = (size_t)G * 2 * D;
  MADRL_LAUNCH(running_moments_finalize_kernel, (unsigned)((n + 255) / 256), 256, 0, s, G, D, ws_dev, sums_dev);
  g_launches.fetch_add(2);
  MADRL_CUDA_CHECK(cudaGetLastError());
  return MADRL_OK;
}

extern "C" int madrl_running_moments_workspace_size(int G, int D, size_t* bytes) {
  MADRL_REQUIRE(G >= 1 && G <= MADRL_AGENTS_MAX && D >= 1, "bad sizes");
  MADRL_REQUIRE(bytes, "NULL pointer");
  *bytes = (size_t)rm_slices(G) * G * 2 * D * sizeof(double);
  return MADRL_OK;
}

extern "C" int madrl_running_moments_f32(size_t R, int G, int D, size_t shift, const float* x_dev,
                                         const float* first_dev, double* sums_dev, double* ws_dev, void* stream) {
  return running_moments<float>(R, G, D, shift, x_dev, first_dev, sums_dev, ws_dev, stream);
}

extern "C" int madrl_running_moments_bf16(size_t R, int G, int D, size_t shift, const void* x_dev,
                                          const void* first_dev, double* sums_dev, double* ws_dev, void* stream) {
  return running_moments<uint16_t>(R, G, D, shift, x_dev, first_dev, sums_dev, ws_dev, stream);
}

extern "C" int madrl_time_baseline_workspace_size(int G, int L, size_t* bytes) {
  MADRL_REQUIRE(G >= 1 && G <= MADRL_AGENTS_MAX && L >= 1, "bad sizes");
  MADRL_REQUIRE(bytes, "NULL pointer");
  *bytes = (size_t)tb_slices(G) * G * L * (sizeof(double) + sizeof(int32_t));
  return MADRL_OK;
}

extern "C" int madrl_time_baseline_f32(int T, int E, int A, int per_agent, int L, const float* q_dev,
                                       const int32_t* seg_start_dev, const int32_t* n_ep_dev,
                                       const int32_t* ep_rec_dev, const int32_t* t0_dev, double* bin_sum_dev,
                                       int32_t* bin_count_dev, float* simplev_dev, void* ws_dev, void* stream) {
  MADRL_REQUIRE(T >= 1 && E >= 1 && A >= 1 && L >= 1, "bad sizes");
  MADRL_REQUIRE((size_t)T * E * A < ((size_t)1 << 31), "T*E*A must be < 2^31");
  MADRL_REQUIRE(!per_agent || A <= MADRL_AGENTS_MAX, "n_agents must be in [1, %d], got %d", MADRL_AGENTS_MAX, A);
  MADRL_REQUIRE(q_dev && seg_start_dev && n_ep_dev && ep_rec_dev && bin_sum_dev && bin_count_dev && simplev_dev &&
                ws_dev, "NULL buffer");
  const int G = per_agent ? A : 1, S = tb_slices(G);
  const size_t part = (size_t)S * G * L;
  double* ws_sum = (double*)ws_dev;
  int32_t* ws_cnt = (int32_t*)(ws_sum + part);
  cudaStream_t s = (cudaStream_t)stream;
  const size_t blocks = (size_t)((L + kTbThreads - 1) / kTbThreads) * S * G;
  MADRL_REQUIRE(blocks < ((size_t)1 << 31), "too many bins for one launch");
  MADRL_LAUNCH(time_baseline_partial_kernel, (unsigned)blocks, kTbThreads, 0, s, T, E, A, G, L, q_dev, n_ep_dev,
               ep_rec_dev, t0_dev, ws_sum, ws_cnt);
  const size_t nb = (size_t)G * L, rows = (size_t)T * E * A;
  MADRL_LAUNCH(time_baseline_bins_kernel, (unsigned)((nb + 255) / 256), 256, 0, s, G, L, ws_sum, ws_cnt, bin_sum_dev,
               bin_count_dev);
  MADRL_LAUNCH(time_baseline_apply_kernel, (unsigned)((rows + 255) / 256), 256, 0, s, T, E, A, G, L, seg_start_dev,
               t0_dev, bin_sum_dev, bin_count_dev, simplev_dev);
  g_launches.fetch_add(3);
  MADRL_CUDA_CHECK(cudaGetLastError());
  return MADRL_OK;
}
