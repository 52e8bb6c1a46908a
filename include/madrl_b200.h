/* madrl_b200 -- C ABI of the H100 batched multi-agent environment engine.
 *
 * One handle = E independent environment instances of one family, resident in HBM (one
 * struct-of-arrays record per env) and stepped in lockstep by sm_90a CUDA kernels.  Every entry
 * point replaces, for a whole batch, one method of the reference's Python environment interface
 * (`madrl_environments/__init__.py:27-119`, AbstractMAEnv):
 *
 *   madrl_ww_*      <-> MAWaterWorld            madrl_environments/pursuit/waterworld.py
 *        _reset     <-> reset()                 :144-172
 *        _step      <-> step(action)            :220-436   (T = 1)
 *        _rollout   <-> T x step() under rllab's VecEnvExecutor.step auto-reset contract
 *                       rllab/sandbox/rocky/tf/envs/vec_env_executor.py:16-28
 *        _seed      <-> seed(seed)              :135-137
 *   madrl_pursuit_* <-> PursuitEvade            madrl_environments/pursuit/pursuit_evade.py
 *        _reset :173-207, _step :209-262, _seed :166-168
 *   madrl_hostage_* <-> ContinuousHostageWorld  madrl_environments/hostage.py
 *        _reset :142-179, _step :228-429, _seed :134-136
 *
 * Conventions
 *   - plain C types only; every function returns 0 on success or a negative MADRL_E* code and
 *     never throws; `madrl_last_error()` returns a thread-local message for the last failure.
 *   - `*_dev` pointers are device pointers owned by the caller (e.g. torch tensors); the
 *     `_host` variants take host pointers and perform the host<->device copies themselves.
 *   - the per-env state lives in one device blob.  The caller may provide it
 *     (`state_dev`, size from `*_state_layout`) or pass NULL to let the library cudaMalloc it.
 *     The layout (byte offsets of the per-env records and constant tables) is reported by
 *     `*_state_layout` so that parity harnesses and `set_param_values`-style callers can read
 *     and write state directly.
 *   - `stream` is a cudaStream_t passed as void* (NULL = default stream).  One handle is used
 *     from one host thread / stream at a time.
 *   - randomness: counter-based Philox4x32-10 streams keyed by (seed, global env id); the
 *     per-env draw counter is part of the state (csrc/philox.cuh).
 *   - `real` below means float when cfg.fp64 == 0 (production) and double when cfg.fp64 == 1
 *     (verification build used by the parity tests).
 */
#ifndef MADRL_B200_H
#define MADRL_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MADRL_OK 0
#define MADRL_EINVAL (-1)   /* bad argument / unsupported configuration */
#define MADRL_ECUDA (-2)    /* CUDA runtime error (see madrl_last_error) */
#define MADRL_ENOMEM (-3)

const char* madrl_last_error(void);
int madrl_version(void);
/* sizeof(madrl_{ww,pursuit,hostage}_{config,layout}) as this library was compiled: a foreign-language
 * binding compares them with its own struct definitions before the first call. */
void madrl_abi_sizes(int32_t* out6);
/* Number of kernels launched by this library since load (bench.py's gpu_launches).  A launch recorded into a CUDA
 * graph during stream capture counts once, at capture; replays of the graph do not count. */
uint64_t madrl_launch_count(void);
/* Device->host bytes per pipeline chunk of the `*_rollout_host` entry points (0 = default 32 MB). */
void madrl_set_host_chunk_bytes(size_t bytes);

/* CUDA-IPC buffers for the fused multi-GPU exchange (see madrl_ww_set_peers): allocate + export on
 * the owning rank, open on every other rank with ITS device current (peer access over NVLink is
 * enabled lazily), close / free at teardown.  handle64 is the 64-byte cudaIpcMemHandle_t. */
int madrl_ipc_alloc(size_t bytes, void** ptr, unsigned char* handle64);
int madrl_ipc_open(const unsigned char* handle64, void** ptr);
int madrl_ipc_close(void* ptr);
int madrl_ipc_free(void* ptr);

/* Stream-ordered primitives of the per-rollout multi-GPU exchange (madrl_b200/dist.py
 * AsyncRootGather): executed by the copy engines / the stream front end, no SM involved, so the
 * persistent rollout kernel of the next rollout is not disturbed.  The reference's counterpart is
 * the workers' pickled path return to the master (rllab/rllab/sampler/stateful_pool.py:102-157).
 *   madrl_copy_async          device->device copy; either side may be a CUDA-IPC peer mapping (NVLink)
 *   madrl_stream_write32      *addr = value when the stream reaches this point (LOCAL device memory)
 *   madrl_stream_wait_geq32   the stream waits until (int32)(*addr - value) >= 0 (LOCAL device memory)
 *   madrl_stream_memops_available   1 if the driver exports the two stream memory operations */
int madrl_stream_memops_available(void);
int madrl_copy_async(void* dst_dev, const void* src_dev, size_t bytes, void* stream);
int madrl_stream_write32(void* stream, void* addr_dev, uint32_t value);
int madrl_stream_wait_geq32(void* stream, void* addr_dev, uint32_t value);

/* Observation formats (madrl_{ww,pursuit,hostage}_set_obs_format).  NATIVE: observations have the handle's
 * `real` type (float, or double when fp64).  BF16: bfloat16 (2 bytes), fp32 handles only.  Features are computed
 * in float either way and rounded to nearest even once, at the store: a BF16 observation is bit-identical to the
 * NATIVE one converted to bfloat16, and state, rewards, dones and infos are the same.  The format applies to
 * every observation buffer of the calls that follow it: reset, rollout, step, rollout_heuristic (obs0 and obs),
 * the _host variants and the set_terminal_obs buffer.  It returns MADRL_EINVAL for an unknown format or BF16 on
 * an fp64 handle.  Waterworld's fused peer exchange (madrl_ww_set_peers) needs NATIVE observations. */
#define MADRL_OBS_NATIVE 0
#define MADRL_OBS_BF16 1

/* L2 cache policy of the observation stores (madrl_{ww,pursuit,hostage}_set_obs_cache).  STREAM (the default):
 * evict-first stores, right for long open-loop trajectories that nothing reads back soon.  KEEP: normal-priority
 * stores, for a closed loop whose policy reads each step's observations right after the launch.  The mode applies
 * to the observation rows of the `*_rollout` / `*_step` entry points (and the _host variants, which call them);
 * resets, the heuristic-policy and peer-exchange rollouts and the set_terminal_obs copies always stream.  Every
 * value written is the same in both modes.  MADRL_EINVAL for an unknown mode, a NULL handle or KEEP on an fp64
 * handle.
 * CUDA-graph capture: between their argument checks and the launch, `*_rollout` and `*_step` make no host
 * synchronisation, allocation or host copy, so they may be captured into a graph on a capturing stream; the graph
 * then holds the pointers, T and the handle's settings of the capture. */
#define MADRL_OBS_CACHE_STREAM 0
#define MADRL_OBS_CACHE_KEEP 1

/* ------------------------------------------------------------------ MAWaterWorld ------------ */
typedef struct madrl_ww_config {
  int32_t n_envs;          /* envs in THIS handle (the local shard)                              */
  int32_t env_id_base;     /* global id of local env 0: RNG key is (seed, env_id_base + e)       */
  int32_t n_pursuers, n_evaders, n_poison, n_sensors, n_coop;   /* waterworld.py:77-79          */
  int32_t reward_global;   /* reward_mech == 'global'                                            */
  int32_t addid, speed_features;
  int32_t random_obstacle; /* obstacle_loc is None -> drawn at reset (waterworld.py:147-148)     */
  int32_t timestep_limit;  /* 1000 (waterworld.py:124-126)                                       */
  int32_t max_path_length; /* VecEnvExecutor horizon, 0 = none                                   */
  int32_t fp64;            /* 0: fp32 arithmetic and buffers; 1: fp64 verification build         */
  double radius, obstacle_radius, obstacle_x, obstacle_y, ev_speed, poison_speed, sensor_range,
      action_scale, poison_reward, food_reward, encounter_reward, control_penalty;
  uint64_t seed;
} madrl_ww_config;

/* Byte offsets into the state blob.  The dynamic state is one record per env:
 * objs real [E][4][n_obj] = rows x, y, vx, vy; objects ordered pursuers, evaders, poisons
 * (one warp owns one env, so a record is one coalesced read per launch). */
typedef struct madrl_ww_layout {
  size_t total_bytes;
  size_t objs;                         /* real [E][4][n_obj]                                   */
  size_t obst;                         /* real [E][2] obstacle centre                          */
  size_t timestep;                     /* int32 [E]  env._timesteps                            */
  size_t path_len;                     /* int32 [E]  VecEnvExecutor.ts                         */
  size_t rng_counter;                  /* uint64 [E] draws consumed                            */
  size_t sensors;                      /* real [2][n_sensors] unit vectors (cos row, sin row)  */
  int32_t n_obj, obs_dim, real_bytes, _pad;
} madrl_ww_layout;

typedef struct madrl_ww madrl_ww;

int madrl_ww_state_layout(const madrl_ww_config* cfg, madrl_ww_layout* out);
int madrl_ww_create(const madrl_ww_config* cfg, void* state_dev, madrl_ww** out);
int madrl_ww_destroy(madrl_ww* h);
void* madrl_ww_state_ptr(madrl_ww* h);
/* seed(): new key, draw counters reset to 0 (waterworld.py:135-137 creates a fresh generator). */
int madrl_ww_seed(madrl_ww* h, uint64_t seed, void* stream);
/* Launch geometry override (0 = library default, see below): resident blocks per SM.  Blocks are one warp
 * (= one env); `warps_per_block` is range-checked ([0,4]) for ABI stability and otherwise ignored.  The same
 * holds for madrl_pursuit_set_launch and madrl_hostage_set_launch, whose default is as many as fit. */
int madrl_ww_set_launch(madrl_ww* h, int warps_per_block, int blocks_per_sm);
/* The library default's cap on resident env warps per SM for an open-loop rollout of T steps of this handle
 * (madrl_ww_rollout / _step / _rollout_host*): 16 for some float32-observation batches (DESIGN §4.3), else 0
 * = as many as fit.  Where it caps, the writer-warp kernel runs if it can (madrl_ww_set_obs_writer), else
 * one-warp blocks.  Resets, heuristic-policy and peer-exchange rollouts always use as many as fit.
 * Negative on error. */
int madrl_ww_default_blocks_per_sm(madrl_ww* h, int T);
/* Which kernel each Waterworld launch ran, for tests of the launch paths.  Returns the number of ww_kernel launches
 * (of any handle) since the previous call, copies the first min(that, max_records, 4096) records into `records`
 * (10 int32 each: sizeof(real), sizeof(observation element), OPL, KCH, KC, PEER, POLICY, KEEP, WRITER and the
 * launch's grid), clears the log and turns logging on (enable != 0) or off (the default).  A launch is logged when
 * it is enqueued, or when it is recorded under stream capture.  MADRL_EINVAL if max_records > 0 and records is NULL. */
int madrl_ww_launch_log(int enable, int32_t* records, int max_records);
/* Observation write path of Waterworld's float32 open-loop rollouts (madrl_ww_rollout / _step / _rollout_host*).
 * The writer-warp kernel runs blocks of 8 warps that step 8 adjacent envs and stage each step's rows in shared
 * memory, plus one warp that copies those rows to the observation tensor (DESIGN §4.1).  It needs at most 32
 * objects, the env-step's rows to be staged whole (as for C2) and a 16-byte-aligned obs pointer and step stride (n_envs * n_pursuers *
 * obs_dim a multiple of 4).  AUTO (the default): it replaces the launches madrl_ww_default_blocks_per_sm caps,
 * whose cap then counts env warps per SM, unless madrl_ww_set_launch set a geometry.  ON: wherever it can run.
 * OFF: never.  Every value written is the same on either path.  MADRL_EINVAL for an unknown mode. */
#define MADRL_WW_OBS_WRITER_AUTO 0
#define MADRL_WW_OBS_WRITER_OFF 1
#define MADRL_WW_OBS_WRITER_ON 2
int madrl_ww_set_obs_writer(madrl_ww* h, int mode);
/* Norm of madrl_ww_rollout_heuristic's actions.  AGENT (the default): each pursuer's action is divided by its own
 * norm, as the reference's Visualizer calls the policy (one agent per call).  ENV: all Np actions of an env are
 * divided by one Frobenius norm, as rltools' decrollout calls it (heuristics/waterworld.py:47-51 on the env's
 * Np x 2 batch; all zero when that norm is 0).  MADRL_EINVAL for an unknown value. */
#define MADRL_HEURISTIC_NORM_AGENT 0
#define MADRL_HEURISTIC_NORM_ENV 1
int madrl_ww_set_heuristic_norm(madrl_ww* h, int norm);
/* Terminal observations: with auto_reset the obs slot of a done step holds the RESET observation
 * (VecEnvExecutor semantics); StandardizedEnv (madrl_environments/__init__.py:283-291) also sees the
 * terminal one.  After this call every `*_rollout` (device pointers) with auto_reset first copies the rows
 * of a finished env to the same [t][e] slot of term_obs_dev (same shape as that rollout's obs tensor;
 * other slots are left untouched).  NULL switches it off. */
int madrl_ww_set_terminal_obs(madrl_ww* h, void* term_obs_dev);
int madrl_ww_set_obs_format(madrl_ww* h, int format);
int madrl_ww_set_obs_cache(madrl_ww* h, int mode);
/* Fused per-rollout exchange for env-sharded multi-GPU runs: after this call every rollout also
 * stores its reward / done / info rows into slot `slot` of each of the `n_dest` listed gather
 * buffers (peer-mapped device pointers: CUDA-IPC mappings of other ranks' buffers over NVLink; one
 * destination = gather-to-root, world destinations = all-gather).  Env-major layout per buffer:
 *   rew  real  [n_slots][E][t_max][Np]    done uint8 [n_slots][E][t_max]
 *   info int32 [n_slots][E][t_max][2]
 * Rows are staged in registers and written as coalesced runs.  A stream-ordered barrier between the
 * ranks after the rollout completes the gather.  n_dest = 0 disables.
 * Every launch writes steps [0, T) of the buffers, so a rollout must be one launch: the device rollout or
 * step.  madrl_ww_rollout_host2 (and _host), which cut a rollout into chunked launches, return MADRL_EINVAL
 * while peers are set.  madrl_ww_rollout_heuristic writes no peer rows. */
int madrl_ww_set_peers(madrl_ww* h, int n_dest, int slot, int t_max, void* const* rew_dest,
                       void* const* done_dest, void* const* info_dest);

/* reset(): envs with mask_dev[e] != 0 (all if NULL) are re-initialised and advanced by the
 * reference's internal step(zeros); obs_dev real [E][Np][obs_dim], rows of unmasked envs untouched. */
int madrl_ww_reset(madrl_ww* h, const uint8_t* mask_dev, void* obs_dev, void* stream);
/* T lockstep steps in ONE launch.  actions_dev real [T][E][Np][2]; obs_dev real [T][E][Np][obs_dim];
 * rew_dev real [T][E][Np]; done_dev uint8 [T][E]; info_dev int32 [T][E][2] = (evcatches, pocatches),
 * 8-byte aligned (a row is one 8-byte store).
 * auto_reset != 0: VecEnvExecutor.step semantics -- a done env is reset in place and the obs
 * slot of that step holds the reset observation. */
int madrl_ww_rollout(madrl_ww* h, int T, const void* actions_dev, void* obs_dev, void* rew_dev,
                     uint8_t* done_dev, int32_t* info_dev, int auto_reset, void* stream);
/* Closed-loop rollout: the actions come from the reference's hand-written policy
 * (heuristics/waterworld.py:11-53 WaterworldHeuristicPolicy.sample_actions: flee the obstacle and poison,
 * chase evaders, close in on allies; unit vector or zero), evaluated INSIDE the rollout kernel on the
 * features each warp has just computed -- no action tensor is read, no per-step launch.
 * obs0_dev real [E][Np][obs_dim]: the observation the first action is computed from (the reset
 * observation, or the last observation of the previous rollout); actions_out_dev real [T][E][Np][2]
 * receives the actions taken (NULL = not recorded).  Needs speed_features (the 7K layout the policy
 * indexes).  Each agent row is normalised by its own norm (the reference is called per agent, B = 1), or, after
 * madrl_ww_set_heuristic_norm(h, MADRL_HEURISTIC_NORM_ENV), all of an env's rows by one norm.
 * Other arguments as madrl_ww_rollout. */
int madrl_ww_rollout_heuristic(madrl_ww* h, int T, const void* obs0_dev, void* actions_out_dev,
                               void* obs_dev, void* rew_dev, uint8_t* done_dev, int32_t* info_dev,
                               int auto_reset, void* stream);
/* step() == rollout with T = 1. */
int madrl_ww_step(madrl_ww* h, const void* actions_dev, void* obs_dev, void* rew_dev,
                  uint8_t* done_dev, int32_t* info_dev, int auto_reset, void* stream);
/* Host-buffer variants (what a non-torch FFI caller binds): copies are part of the call and the
 * call returns after the results are in the host buffers (pinned memory for full PCIe speed).  The
 * rollout is chunked: the copy engines drain chunk c while chunk c+1 is computed.  They run on two
 * internal streams that are ordered after earlier work on the legacy default stream; work the caller
 * queued on other streams must be synchronised by the caller.
 * `_host2` takes flags: MADRL_HOST_OBS_LAST = only the LAST step's observations come back (obs_host is
 * then [E][Np][D]) -- the policy-on-device mode: rewards / dones / infos of every step + the
 * observation needed to continue; the call then runs at the kernel's rate instead of PCIe's.
 * Waterworld's host variants return MADRL_EINVAL while madrl_ww_set_peers is set. */
#define MADRL_HOST_OBS_LAST 1
int madrl_ww_reset_host(madrl_ww* h, const uint8_t* mask_host, void* obs_host);
int madrl_ww_rollout_host(madrl_ww* h, int T, const void* actions_host, void* obs_host,
                          void* rew_host, uint8_t* done_host, int32_t* info_host, int auto_reset);
int madrl_ww_rollout_host2(madrl_ww* h, int T, const void* actions_host, void* obs_host,
                           void* rew_host, uint8_t* done_host, int32_t* info_host, int auto_reset,
                           int flags);

/* ------------------------------------------------------------------ PursuitEvade ------------ */
typedef struct madrl_pursuit_config {
  int32_t n_envs, env_id_base;
  int32_t n_pursuers, n_evaders;      /* pursuit_evade.py:60-61 (<= 32 / <= 64)                 */
  int32_t xs, ys, n_maps;             /* map_pool shape (n_maps, xs, ys); -1 = building         */
  int32_t obs_range;                  /* pursuit_evade.py:63                                     */
  int32_t flatten;                    /* pursuit_evade.py:67; 0 = conv layout (R, R, 4)          */
  int32_t n_catch, surround;          /* pursuit_evade.py:79,142                                 */
  int32_t reward_global, include_id, sample_maps;
  int32_t max_path_length;            /* VecEnvExecutor horizon, 0 = none                        */
  int32_t max_opponents;              /* random_opponents (pursuit_evade.py:81-82,177-181): > 0 = every reset
                                         draws randint(1, max_opponents) live evaders (<= n_evaders); 0 = off */
  double layer_norm, catchr, term_pursuit, urgency_reward, constraint_window;
  uint64_t seed;
} madrl_pursuit_config;

/* Byte offsets into the state blob (one record per env). */
typedef struct madrl_pursuit_layout {
  size_t total_bytes;
  size_t pos;          /* uint8  [E][2][n_agents]  x row, y row; pursuers first, then evaders     */
  size_t gone;         /* uint64 [E]  bit j: evader j has been removed (evaders_gone)             */
  size_t map_id;       /* int32  [E]  index into the map pool                                     */
  size_t path_len;     /* int32  [E]  VecEnvExecutor.ts                                           */
  size_t rng_counter;  /* uint64 [E]                                                              */
  size_t stale;        /* uint16 [E][Np][R*R]  the never-cleared channels 1-2 of local_obs
                          (pursuit_evade.py:119,438): pursuer count | evader count << 8           */
  size_t maps;         /* uint32 [n_maps][(xs+2p)(ys+2p)], p = (obs_range-1)/2+1: per map the empty cell grid
                          with its border of p marker cells, as the kernel keeps it in shared memory:
                          bit 0 building, bits 24-26 need_to_surround (pursuit_evade.py:523-540), border
                          cells 0x80000001 (constant)                                             */
  size_t lut, idv;     /* float tables (constant)                                                 */
  int32_t n_agents, obs_dim;
} madrl_pursuit_layout;

typedef struct madrl_pursuit madrl_pursuit;

int madrl_pursuit_state_layout(const madrl_pursuit_config* cfg, madrl_pursuit_layout* out);
/* map_pool_host: int32 [n_maps][xs][ys] (the .npy the reference loads, maps/map_pool16.npy). */
int madrl_pursuit_create(const madrl_pursuit_config* cfg, const int32_t* map_pool_host,
                         void* state_dev, madrl_pursuit** out);
int madrl_pursuit_destroy(madrl_pursuit* h);
void* madrl_pursuit_state_ptr(madrl_pursuit* h);
int madrl_pursuit_seed(madrl_pursuit* h, uint64_t seed, void* stream);
int madrl_pursuit_set_launch(madrl_pursuit* h, int warps_per_block, int blocks_per_sm);
/* Which kernel each Pursuit launch ran: madrl_ww_launch_log's contract for pe_kernel launches, with records of 8
 * int32: sizeof(observation element), EPL, CPL, RC, POLICY, FLAT, KEEP and the launch's grid.  POLICY's bit 0 is the
 * in-kernel heuristic, bit 1 the evader-control instantiation (madrl_pursuit_set_evader_control). */
int madrl_pursuit_launch_log(int enable, int32_t* records, int max_records);
/* Terminal observations: with auto_reset the obs slot of a done step holds the RESET observation
 * (VecEnvExecutor semantics); StandardizedEnv (madrl_environments/__init__.py:283-291) also sees the
 * terminal one.  After this call every `*_rollout` (device pointers) with auto_reset first copies the rows
 * of a finished env to the same [t][e] slot of term_obs_dev (same shape as that rollout's obs tensor;
 * other slots are left untouched).  NULL switches it off. */
int madrl_pursuit_set_terminal_obs(madrl_pursuit* h, void* term_obs_dev);
/* obs buffers below are float, or bfloat16 after set_obs_format(MADRL_OBS_BF16). */
int madrl_pursuit_set_obs_format(madrl_pursuit* h, int format);
int madrl_pursuit_set_obs_cache(madrl_pursuit* h, int mode);
/* Curriculum knobs that survive pickling in the reference (pursuit_evade.py:264-272,397-411). */
int madrl_pursuit_set_params(madrl_pursuit* h, double catchr, double constraint_window);
/* reset(): obs_dev float [E][Np][obs_dim]. */
int madrl_pursuit_reset(madrl_pursuit* h, const uint8_t* mask_dev, void* obs_dev, void* stream);
/* actions_dev int32 [T][E][Np] in {0 left,1 right,2 up,3 down,4 stay} (DiscreteAgent.py:28-38);
 * obs_dev float [T][E][Np][obs_dim] (obs_dim = 3R^2+id if flatten else 4R^2 laid out [x][y][ch]);
 * rew_dev float [T][E][Np] (computed in float64, narrowed once);
 * done_dev uint8 [T][E]; info_dev int32 [T][E] = removed. */
int madrl_pursuit_rollout(madrl_pursuit* h, int T, const int32_t* actions_dev, void* obs_dev,
                          float* rew_dev, uint8_t* done_dev, int32_t* info_dev, int auto_reset,
                          void* stream);
/* Closed-loop rollout: the pursuers' actions come from the reference's hand-written policy
 * (heuristics/pursuit.py:18-50 PursuitHeuristicPolicy.sample_actions: walk towards the nearest evader of the
 * observation window, a random move when none is visible), evaluated INSIDE the rollout kernel on the window
 * each warp has just assembled.  obs0_dev float [E][Np][obs_dim]: the observation the first action is
 * computed from; actions_out_dev int32 [T][E][Np] receives the actions taken (NULL = not recorded).
 * floor_centre != 0: the window centre is (R//2, R//2) -- what `xs / 2` (heuristics/pursuit.py:23) gives under
 * Python 2, the reference's language; 0: (R/2, R/2) true division, what the same line gives under Python 3.
 * The policy's own draws (`action_space.sample()`, :48,50) are an injected counter-based stream: pursuer q
 * deciding on an observation produced when the env's draw counter stood at c takes word 32 c + q of the
 * (seed, env id, tag 2) Philox stream, mapped to {0..4} like every other range draw.  Other arguments as
 * madrl_pursuit_rollout. */
int madrl_pursuit_rollout_heuristic(madrl_pursuit* h, int T, const void* obs0_dev, int32_t* actions_out_dev,
                                    void* obs_dev, float* rew_dev, uint8_t* done_dev, int32_t* info_dev,
                                    int auto_reset, int floor_centre, void* stream);
int madrl_pursuit_step(madrl_pursuit* h, const int32_t* actions_dev, void* obs_dev, float* rew_dev,
                       uint8_t* done_dev, int32_t* info_dev, int auto_reset, void* stream);
/* The evaders' controller (pursuit_evade.py:87 evader_controller, called once per live evader per step, :237-241).
 * set_evader_control sets the handle's default, used by every launch that is given no evader actions:
 * MADRL_PURSUIT_EVADERS_RANDOM (the default) moves each live evader by one draw of the env's stream (RandomPolicy);
 * MADRL_PURSUIT_EVADERS_FIXED moves every evader by `action` (SingleActionPolicy(action)).
 * The *_evaders entries take the evaders' actions of this launch instead: evader j of env e at step t moves by
 * ev_act_dev[t * ev_st + e * ev_se + j] (int32, j its ORIGINAL index; strides 0 and 0 make one int a fixed
 * controller); entries of removed evaders and of evaders that do not exist this episode are not read.
 * A caller's action outside 0..3 means stay.  Whatever the controller, the env's draw counter advances by the live
 * evader count each step, so the reset draws and the heuristic policy's fallback draws use the words they would
 * under the random controller.  Other arguments as madrl_pursuit_rollout / madrl_pursuit_rollout_heuristic. */
#define MADRL_PURSUIT_EVADERS_RANDOM 0
#define MADRL_PURSUIT_EVADERS_FIXED 1
int madrl_pursuit_set_evader_control(madrl_pursuit* h, int mode, int action);
int madrl_pursuit_rollout_evaders(madrl_pursuit* h, int T, const int32_t* actions_dev, const int32_t* ev_act_dev,
                                  size_t ev_st, size_t ev_se, void* obs_dev, float* rew_dev, uint8_t* done_dev,
                                  int32_t* info_dev, int auto_reset, void* stream);
int madrl_pursuit_rollout_heuristic_evaders(madrl_pursuit* h, int T, const void* obs0_dev, int32_t* actions_out_dev,
                                            const int32_t* ev_act_dev, size_t ev_st, size_t ev_se, void* obs_dev,
                                            float* rew_dev, uint8_t* done_dev, int32_t* info_dev, int auto_reset,
                                            int floor_centre, void* stream);
/* model_state (pursuit_evade.py:152): after this call reset() and every rollout (device pointers) write
 * model_state_dev float [E][4][xs][ys] of the envs they touch, as the env stands after the launch's last step:
 * channel 0 the map (-1 building, 0 free: what the map pool holds for pools of 0 / -1), 1 the pursuer count,
 * 2 the evader count, 3 zero.  Like the reference (pursuit_evade.py:244-249) it is the occupancy before that
 * step's removals, so an evader caught at the last step is still counted; after an auto-reset it is the reset's.
 * The launch log marks such launches (and those with caller-controlled evaders) with bit 1 of its POLICY field.
 * NULL switches it off. */
int madrl_pursuit_set_model_state(madrl_pursuit* h, float* model_state_dev);
int madrl_pursuit_reset_host(madrl_pursuit* h, const uint8_t* mask_host, void* obs_host);
int madrl_pursuit_rollout_host(madrl_pursuit* h, int T, const int32_t* actions_host, void* obs_host,
                               float* rew_host, uint8_t* done_host, int32_t* info_host,
                               int auto_reset);
int madrl_pursuit_rollout_host2(madrl_pursuit* h, int T, const int32_t* actions_host, void* obs_host,
                                float* rew_host, uint8_t* done_host, int32_t* info_host,
                                int auto_reset, int flags);

/* ------------------------------------------------------------------ ContinuousHostageWorld -- */
typedef struct madrl_hostage_config {
  int32_t n_envs, env_id_base;
  int32_t n_good, n_hostages, n_bad, n_coop_save, n_coop_avoid, n_sensors;   /* hostage.py:75-76 */
  int32_t reward_global, addid;
  int32_t random_key;       /* key_loc is None: drawn at the first reset, then kept (hostage.py:148) */
  int32_t timestep_limit, max_path_length, fp64;
  double radius, key_x, key_y, bad_speed, sensor_range, action_scale, save_reward, hit_reward,
      encounter_reward, not_saved_reward, bomb_reward, bomb_radius, key_radius, control_penalty;
  uint64_t seed;
} madrl_hostage_config;

typedef struct madrl_hostage_layout {
  size_t total_bytes;
  size_t objs;         /* real  [E][4][n_obj] rows x, y, vx, vy; rescuers, criminals, hostages   */
  size_t fixed;        /* real  [E][4] key x, key y, bomb x, bomb y                              */
  size_t saved;        /* uint8 [E][n_hostages] curr_host_saved_mask                             */
  size_t flags;        /* int32 [E] bit0 gate open, bit1 bombed, bit2 key location drawn         */
  size_t timestep, path_len;   /* int32 [E]                                                      */
  size_t rng_counter;  /* uint64 [E]                                                             */
  size_t sensors;      /* real [2][n_sensors]                                                    */
  int32_t n_obj, obs_dim, real_bytes, _pad;
} madrl_hostage_layout;

typedef struct madrl_hostage madrl_hostage;

int madrl_hostage_state_layout(const madrl_hostage_config* cfg, madrl_hostage_layout* out);
int madrl_hostage_create(const madrl_hostage_config* cfg, void* state_dev, madrl_hostage** out);
int madrl_hostage_destroy(madrl_hostage* h);
void* madrl_hostage_state_ptr(madrl_hostage* h);
int madrl_hostage_seed(madrl_hostage* h, uint64_t seed, void* stream);
int madrl_hostage_set_launch(madrl_hostage* h, int warps_per_block, int blocks_per_sm);
/* Which kernel each Hostage launch ran: madrl_ww_launch_log's contract for hw_kernel launches, with records of 7
 * int32: sizeof(real), sizeof(observation element), OPL, KCH, KC, KEEP and the launch's grid. */
int madrl_hostage_launch_log(int enable, int32_t* records, int max_records);
/* Terminal observations: with auto_reset the obs slot of a done step holds the RESET observation
 * (VecEnvExecutor semantics); StandardizedEnv (madrl_environments/__init__.py:283-291) also sees the
 * terminal one.  After this call every `*_rollout` (device pointers) with auto_reset first copies the rows
 * of a finished env to the same [t][e] slot of term_obs_dev (same shape as that rollout's obs tensor;
 * other slots are left untouched).  NULL switches it off. */
int madrl_hostage_set_terminal_obs(madrl_hostage* h, void* term_obs_dev);
int madrl_hostage_set_obs_format(madrl_hostage* h, int format);
int madrl_hostage_set_obs_cache(madrl_hostage* h, int mode);
/* obs_dev real [E][n_good][obs_dim] */
int madrl_hostage_reset(madrl_hostage* h, const uint8_t* mask_dev, void* obs_dev, void* stream);
/* actions_dev real [T][E][n_good][2]; obs_dev real [T][E][n_good][obs_dim]; rew_dev real
 * [T][E][n_good]; done_dev uint8 [T][E]; info_dev int32 [T][E][2] = (ho_saved, cr_encs), 8-byte
 * aligned (a row is one 8-byte store). */
int madrl_hostage_rollout(madrl_hostage* h, int T, const void* actions_dev, void* obs_dev,
                          void* rew_dev, uint8_t* done_dev, int32_t* info_dev, int auto_reset,
                          void* stream);
int madrl_hostage_step(madrl_hostage* h, const void* actions_dev, void* obs_dev, void* rew_dev,
                       uint8_t* done_dev, int32_t* info_dev, int auto_reset, void* stream);
int madrl_hostage_reset_host(madrl_hostage* h, const uint8_t* mask_host, void* obs_host);
int madrl_hostage_rollout_host(madrl_hostage* h, int T, const void* actions_host, void* obs_host,
                               void* rew_host, uint8_t* done_host, int32_t* info_host,
                               int auto_reset);
int madrl_hostage_rollout_host2(madrl_hostage* h, int T, const void* actions_host, void* obs_host,
                                void* rew_host, uint8_t* done_host, int32_t* info_host,
                                int auto_reset, int flags);

/* ------------------------------------------------------------------ frames ---------------------
 * Frames of n chosen envs drawn on the device from the state blob (csrc/render.cu, DESIGN §4.10), RGB uint8.
 * env_ids_dev int32 [n] (repeats allowed).  The kernels only read the state, and make no host synchronisation or
 * allocation, so a render may be captured into a CUDA graph.  The ids are not read on the host: the frame of an id
 * outside [0, n_envs) is written all zero, which no drawn frame is.  An object with a non-finite coordinate draws
 * nothing.
 *   madrl_ww_render       out [n][S][S][3]: the reference's MAWaterWorld.render (waterworld.py:438-479) drawn with
 *                         8-connected lines and circles (LINE_8) and its background blend; S = screen_size.
 *                         sensor_dirs_dev float64 [2][n_sensors]: the cos and sin rows of the sensor angles
 *                         linspace(0, 2 pi, K + 1)[:-1], built once by the caller (end points are computed in
 *                         float64 from it, never from a device cos / sin).
 *   madrl_hostage_render  the same for ContinuousHostageWorld.render (hostage.py:431-478).
 *   madrl_pursuit_render  out [n][ys * cell][xs * cell][3]: the integer Pursuit picture of DESIGN §4.10.
 * MADRL_EINVAL for a NULL handle or buffer, n < 1, screen_size or cell outside [1, 32768], a Pursuit frame more
 * than 32768 pixels a side, a radius of 2^29 pixels or more, or a sensor_range that is not finite or reaches
 * |sensor_range| * screen_size >= 2^29 pixels. */
int madrl_ww_render(madrl_ww* h, int n, const int32_t* env_ids_dev, int screen_size, const double* sensor_dirs_dev,
                    uint8_t* out_dev, void* stream);
int madrl_hostage_render(madrl_hostage* h, int n, const int32_t* env_ids_dev, int screen_size,
                         const double* sensor_dirs_dev, uint8_t* out_dev, void* stream);
int madrl_pursuit_render(madrl_pursuit* h, int n, const int32_t* env_ids_dev, int cell, uint8_t* out_dev,
                         void* stream);

/* ------------------------------------------------------------------ hand-written policies -----
 * The reference's heuristic policies as stand-alone action generators over n_rows observation rows (one
 * row = one agent's observation), for callers that step an env one batch at a time; the
 * `*_rollout_heuristic` entry points above evaluate the same policies inside the rollout kernels.
 * madrl_ww_heuristic_actions       heuristics/waterworld.py:11-53: obs real [n_rows][obs_dim] in the 7K+2(+1)
 *                                  layout (:12-22) -> actions real [n_rows][2]; each row normalised by its own
 *                                  norm (the reference is called per agent).
 * madrl_pursuit_heuristic_actions  heuristics/pursuit.py:18-50: obs float [n_rows][obs_dim], flatten != 0: the
 *                                  (3R^2 [+1]) layout, else (R, R, 4); fallback int32 [n_rows] = the action taken
 *                                  when no evader is visible (`action_space.sample()`, drawn by the caller);
 *                                  floor_centre as in madrl_pursuit_rollout_heuristic; lut_dev: R*R bytes of
 *                                  device scratch (the per-cell action table, filled by the call). */
int madrl_ww_heuristic_actions(int fp64, size_t n_rows, int n_sensors, int obs_dim, const void* obs_dev,
                               void* actions_dev, void* stream);
int madrl_pursuit_heuristic_actions(size_t n_rows, int obs_range, int flatten, int obs_dim, int floor_centre,
                                    const float* obs_dev, const int32_t* fallback_dev, uint8_t* lut_dev,
                                    int32_t* actions_dev, void* stream);

/* ------------------------------------------------------------------ trajectory post-processing
 * (SURVEY.md 8f rows 2-3).  All tensors are device pointers, float32 unless noted, time-major. */
/* GAE advantages + discounted returns over paths segmented by `done`
 * (rllab/rllab/sampler/base.py:48-68).  rew, value, adv, ret: [T][E][A]; done: uint8 [T][E];
 * last_value [E][A] bootstraps the unfinished tail (NULL = 0, rllab's truncated-path convention). */
int madrl_gae_f32(int T, int E, int A, const float* rew_dev, const float* value_dev,
                  const uint8_t* done_dev, const float* last_value_dev, double discount,
                  double gae_lambda, float* adv_dev, float* ret_dev, void* stream);
/* ObservationBuffer frame stack (madrl_environments/__init__.py:143-196): obs [T][E][A][D] ->
 * out [T][E][A][D][B]; carry [E][A][D][B] is the buffer kept between calls; B <= 8. */
int madrl_frame_stack_f32(int T, int E, int A, int D, int B, const float* obs_dev,
                          const uint8_t* done_dev, float* carry_dev, float* out_dev, void* stream);
/* bfloat16 observations (madrl_*_set_obs_format): obs, carry and out hold bfloat16. */
int madrl_frame_stack_bf16(int T, int E, int A, int D, int B, const void* obs_dev,
                           const uint8_t* done_dev, void* carry_dev, void* out_dev, void* stream);
/* StandardizedEnv running mean / variance normalisation (madrl_environments/__init__.py:241-291),
 * in place over x [T][n] with float64 state mean/var [n]; center=1 for observations, 0 for rewards
 * (which are divided by the running std and multiplied by `scale`); enable=0 only applies `scale`. */
int madrl_standardize_f32(int T, size_t n, float* x_dev, double* mean_dev, double* var_dev,
                          double alpha, double eps, int center, double scale, int enable,
                          void* stream);
/* Same over bfloat16 x: each value is widened, takes the float32 pass's float64 arithmetic and float32
 * result, and is rounded to bfloat16 once, at the store (bit-identical to the f32 pass on the widened
 * input, rounded to nearest even). */
int madrl_standardize_bf16(int T, size_t n, void* x_dev, double* mean_dev, double* var_dev,
                           double alpha, double eps, int center, double scale, int enable,
                           void* stream);
/* Same, for observations of an auto-reset rollout with the terminal observations kept on the side
 * (madrl_*_set_terminal_obs): at a step with done[t][e] set, the running estimate of env e's columns is
 * first updated with term[t] (which is standardised in place too) and then with x[t] -- the reference
 * order: step() standardises the terminal observation, reset() the first one of the next episode.
 * x, term [T][E][per_env]; done uint8 [T][E]; mean, var float64 [E][per_env]. */
int madrl_standardize_obs_terminal_f32(int T, int E, size_t per_env, float* x_dev, float* term_dev,
                                       const uint8_t* done_dev, double* mean_dev, double* var_dev,
                                       double alpha, double eps, void* stream);
/* Same over bfloat16 x and term, rounded as madrl_standardize_bf16. */
int madrl_standardize_obs_terminal_bf16(int T, int E, size_t per_env, void* x_dev, void* term_dev,
                                        const uint8_t* done_dev, double* mean_dev, double* var_dev,
                                        double alpha, double eps, void* stream);
/* One closed-loop step of StandardizedEnv inside ObservationBuffer (madrl_b200.closed_loop.PolicyRollout), run
 * after a one-step rollout launch: the values of madrl_standardize_obs_terminal_* then madrl_frame_stack_* at
 * T = 1, bit for bit, in one pass.  obs, term [E][A][D] (the step's observations and terminal observations);
 * done uint8 [E]; prev, out [E][A][D][B] (the stack the policy read at this step, and the next one); mean, var
 * float64 [E][A][D] (the running estimates) or both NULL.
 *   obsnorm (mean, var given): where done[e] is set the estimate is updated with term, which is written back
 *                              standardised; then with obs, which is written back standardised, in place.
 *   stack:                     out = the (standardised) obs in every slot where done[e] is set, otherwise prev
 *                              shifted left by one slot with it in slot B-1.  With B = 1, prev is not read and
 *                              out may be NULL (obsnorm only).
 * MADRL_EINVAL for E, A or D < 1, B outside [1, 8], NULL obs or done, only one of mean / var, mean without term,
 * or B > 1 without prev and out. */
int madrl_obs_wrap_step_f32(int E, int A, int D, int B, float* obs_dev, float* term_dev, const uint8_t* done_dev,
                            const float* prev_dev, float* out_dev, double* mean_dev, double* var_dev, double alpha,
                            double eps, void* stream);
/* Same over bfloat16 obs, term, prev and out, rounded as madrl_standardize_bf16. */
int madrl_obs_wrap_step_bf16(int E, int A, int D, int B, void* obs_dev, void* term_dev, const uint8_t* done_dev,
                             const void* prev_dev, void* out_dev, double* mean_dev, double* var_dev, double alpha,
                             double eps, void* stream);
/* DiagnosticsWrapper episode statistics (madrl_environments/__init__.py:314-369): rew [T][E][A],
 * done uint8 [T][E]; carry float64 [E][A+3] (zero-initialised by the caller, kept between calls);
 * outputs at the steps where an episode closes (ep_end[t][e] = 1; zeros elsewhere):
 * ep_reward [T][E][A], ep_disc [T][E] (discounted return of the agent-mean reward), ep_len [T][E]. */
int madrl_episode_stats_f32(int T, int E, int A, const float* rew_dev, const uint8_t* done_dev,
                            double discount, int max_traj_len, double* carry_dev, float* ep_reward_dev,
                            float* ep_disc_dev, int32_t* ep_len_dev, uint8_t* ep_end_dev, void* stream);
/* Whole-episode records of an evaluation (rltools/rltools/util.py:141-231 evaluate_policy), over a rollout cut into
 * launches of any length: rew real [T][E][A] (float32 or float64), done uint8 [T][E], info int32 [T][E][C]
 * (0 <= C <= MADRL_EVAL_INFO_MAX; NULL with C = 0).  carry: MADRL_EVAL_CARRY_WORDS 8-byte words per (e, a), zeroed by
 * the caller when the evaluation starts and kept between calls, so any cut gives the same bits.  The k-th episode
 * env e completes (k < K) goes to record k * E + e; later ones are not recorded:
 *   ret  float64 [K*E][A]  sum of the episode's rewards in time order;
 *   qsum float64 [K*E][A]  sum over its steps t of the discounted reward-to-go q_t, accumulated forward as
 *                          sum_s r_s * G_s with G_s = sum_{j<=s} discount^j (no fused multiply-adds);
 *   len  int32 [K*E]       its length;
 *   info_sum int64 [K*E][C] its info sums (rltools/rltools/trajutil.py:105-108).
 * One thread per (e, a), no atomics, no host synchronisation. */
#define MADRL_EVAL_CARRY_WORDS 8
#define MADRL_EVAL_INFO_MAX 2
int madrl_eval_episodes_f32(int T, int E, int A, int C, const float* rew_dev, const uint8_t* done_dev,
                            const int32_t* info_dev, double discount, int K, void* carry_dev, double* ret_dev,
                            double* qsum_dev, int32_t* len_dev, int64_t* info_sum_dev, void* stream);
int madrl_eval_episodes_f64(int T, int E, int A, int C, const double* rew_dev, const uint8_t* done_dev,
                            const int32_t* info_dev, double discount, int K, void* carry_dev, double* ret_dev,
                            double* qsum_dev, int32_t* len_dev, int64_t* info_sum_dev, void* stream);

/* Per-column moments, deterministic (fixed grid, fixed combination order), float64 accumulation, NumPy's two-pass
 * population variance.  a, b are [rows][A] (A = the innermost axis, e.g. a [T][E][A] tensor with rows = T*E; the
 * whole batch is A = 1) and every statistic is taken over one column, i.e. one agent's samples.  Series s0 = a,
 * s1 = b, s2 = b - a (b may be NULL).  stats [A][MADRL_MOMENTS_STATS]: column c's block holds the means at [0..2],
 * the population variances at [3..5] and the minima at [6..8]; workspace: MADRL_MOMENTS_WS * A doubles of device
 * scratch.  With a = baseline prediction and b = returns the block gives explained_variance_1d's terms
 * (rllab/rllab/misc/special.py:51-59): var(y) = [4], var(y - ypred) = [5], var(ypred) = [3].
 *
 * madrl_moments_pass_f32 runs one of the two passes and leaves the division by the rows to the caller, so that
 * the statistics of the shards of a batch can be pooled between the passes: pass 0 writes the SUMS of the three
 * series to stats[.][0..2] and their minima to stats[.][6..8]; pass 1 reads the means from stats[.][0..2] and
 * writes the SUMS of squared deviations about them to stats[.][3..5].  Dividing pass 0's sums by the rows before
 * pass 1, and pass 1's sums by the rows after it, gives the block above.
 *
 * madrl_center_apply_f32: center_advantages / shift_advantages_to_positive (rllab/rllab/algos/util.py:7-12,
 * applied to the concatenated advantages at rllab/rllab/sampler/base.py:82-86), in place over adv [rows][A] with
 * column a's statistics from stats [A][MADRL_MOMENTS_STATS] (mean [0], variance [3], minimum [6]):
 * center: (x - mean) / (std + 1e-8); positive: (x - min) + 1e-8 (after centring when both).
 *
 * MADRL_EINVAL for A outside [1, MADRL_AGENTS_MAX] (declared below), rows == 0, a pass other than 0 and 1, or a
 * NULL required buffer. */
#define MADRL_MOMENTS_STATS 9
#define MADRL_MOMENTS_WS 4096
int madrl_moments_pass_f32(size_t rows, int A, const float* a_dev, const float* b_dev, int pass, double* stats_dev,
                           double* workspace_dev, void* stream);
int madrl_center_apply_f32(size_t rows, int A, float* adv_dev, const double* stats_dev, int center, int positive,
                           void* stream);

/* Path packing: time-major rollout tensors -> rllab's per-(env, episode, agent) paths
 * (rllab/rllab/sampler/ma_sampler.py:52-100 `dec_rollout`, episodes cut at `done` as
 * rllab/sandbox/rocky/tf/envs/vec_env_executor.py:16-28 does).  Paths are ordered (env, episode, agent);
 * the rows of a path are consecutive in the packed arrays.
 *   madrl_paths_plan      done uint8 [T][E] -> seg_start / seg_len int32 [T][E] (start and length of the
 *                         episode containing step t), n_episodes int32 [E], ep_rec int32 [E][T][3] =
 *                         (start step, length, terminated) of the first n_episodes[e] episodes of env e;
 *                         path (e, episode j, agent a) occupies rows [e*T*A + s_j*A + a*L_j, +L_j)
 *   madrl_paths_pack_u32  src [T][E][A][D] of 4-byte words -> dst [E*T*A][D] in path order.  first != NULL:
 *                         rows are shifted by one step (row t = first[e][a] for t = 0, src[t-1] afterwards):
 *                         the observation each action was taken in, with first = the observations before
 *                         the rollout.  Per-env tensors (infos, dones) are packed with A = 1. */
int madrl_paths_plan(int T, int E, int A, const uint8_t* done_dev, int32_t* seg_start_dev, int32_t* seg_len_dev,
                     int32_t* n_episodes_dev, int32_t* ep_rec_dev, void* stream);
int madrl_paths_pack_u32(int T, int E, int A, int D, const void* src_dev, const void* first_dev,
                         const int32_t* seg_start_dev, const int32_t* seg_len_dev, void* dst_dev, void* stream);
/* madrl_paths_pack_u32 for rows of D 2-byte elements (bfloat16 observations; D may be odd). */
int madrl_paths_pack_u16(int T, int E, int A, int D, const void* src_dev, const void* first_dev,
                         const int32_t* seg_start_dev, const int32_t* seg_len_dev, void* dst_dev, void* stream);

/* Padded paths: rllab's recurrent sample batch (rllab/rllab/sampler/base.py:105-161, tensor_utils.pad_tensor_n),
 * every path zero-padded to Lmax steps.  rec int32 [P][4] = (env, agent, start step, length) of each path, in the
 * output's path order (any order: one kernel serves every control mode); 0 <= env < E, 0 <= start,
 * start + length <= T, 1 <= length <= Lmax, and 0 <= agent < A unless A = 1.
 *   madrl_paths_pad_u32  src [T][E][A][D] of 4-byte words -> dst [P][Lmax][D]: row (p, i) is src row
 *                        (start + i, env, agent) for i < length, zeros otherwise; every dst word is written
 *                        exactly once (no separate clearing pass).  first != NULL: rows are shifted by one step
 *                        as in madrl_paths_pack_u32.  A = 1: per-env tensors [T][E][D] (infos); the agent field is
 *                        ignored, so every agent's path reads its env's row.
 *   madrl_paths_pad_u16  the same for rows of D 2-byte elements (bfloat16 observations; D may be odd).
 *   madrl_path_sums_f32  rew, ret float32 [T][E][A] -> per path: sums[p] = the float64 sum of its rewards in time
 *                        order (Python's sum(path["rewards"])), first_ret[p] = ret at its first step (the path's
 *                        returns[0]).  Same table conventions; A = 1 reads column 0 of [T][E][1].
 * MADRL_EINVAL for T, E, A, D, P or Lmax < 1, more padded rows than one launch's grid covers (P * Lmax >= 2^34
 * for D > 4 words) or a NULL required buffer. */
int madrl_paths_pad_u32(int T, int E, int A, int D, int P, int Lmax, const void* src_dev, const void* first_dev,
                        const int32_t* rec_dev, void* dst_dev, void* stream);
int madrl_paths_pad_u16(int T, int E, int A, int D, int P, int Lmax, const void* src_dev, const void* first_dev,
                        const int32_t* rec_dev, void* dst_dev, void* stream);
int madrl_path_sums_f32(int T, int E, int A, int P, const float* rew_dev, const float* ret_dev,
                        const int32_t* rec_dev, double* sums_dev, double* first_ret_dev, void* stream);

/* Whole-path sampling (rllab's BatchMASampler with whole_paths=True; DESIGN §4.9).  E lockstep envs, all reset at
 * step 0, run in launches of T steps; global step g = t_base + t.  Per env, carry int32 [3][E] = (last done step,
 * end step of the kept paths, paths kept), initialised to (-1, -1, 0); acc int64 [5] = (env-steps in finished
 * paths, t*, finished flag, N rows kept, P paths kept), initialised to (0, -1, 0, 0, 0).
 *   madrl_whole_paths_fold    folds one launch's done uint8 [T][E]: t* = the first step at which the env-steps of
 *                             the paths finished so far reach batch_size; env e keeps steps [0, end_e], end_e = its
 *                             first done at or after t*.  One CTA, no atomics.  finished = t* found and every end_e
 *                             set; then N = sum (end_e + 1) and P = the done steps in the kept rows.
 *   madrl_whole_paths_finish  after the fold has finished: env_off int32 [2][E] (first output row and first path of
 *                             env e, env-major), path_start int32 [P+1] (first row of each path, then N) and done_flat uint8 [N] from
 *                             the done columns of every launch, done_stage uint8 [S][E] (S >= max end_e + 1).
 *   madrl_whole_paths_gather  one launch's per-(step, env) slabs src [T][E][slab_bytes] -> dst [N][slab_bytes],
 *                             row env_off[e] + g for g <= end_e.  first != NULL: src is shifted by one step (step t
 *                             reads src[t-1], step 0 first [E][slab_bytes]), as the policy reads its observations.
 *                             16-byte vector copies when slab_bytes and the pointers allow them.
 * Over the ranks of a sharded batch (each rank holding its own envs' carry and acc) the fold runs in two calls around
 * a sum of the ranks' increments, so that t* is the whole batch's:
 *   madrl_whole_paths_steps   inc int64 [T]: this rank's increment of the count at step t_base + t, the env-steps of
 *                             its paths that end there (from carry's last done and the launch's own dones).  It
 *                             does not write carry.  One CTA, no atomics.
 *   madrl_whole_paths_fold_pooled  madrl_whole_paths_fold with the count advanced by inc[t], the increments summed
 *                             over the ranks; the finished flag, N and P are this rank's.
 * MADRL_EINVAL for sizes < 1, batch_size < 1 or >= 2^62, or a NULL required buffer. */
int madrl_whole_paths_fold(int T, int E, int t_base, size_t batch_size, const uint8_t* done_dev, int32_t* carry_dev,
                           int64_t* acc_dev, void* stream);
int madrl_whole_paths_steps(int T, int E, int t_base, const uint8_t* done_dev, const int32_t* carry_dev,
                            int64_t* inc_dev, void* stream);
int madrl_whole_paths_fold_pooled(int T, int E, int t_base, size_t batch_size, const uint8_t* done_dev,
                                  const int64_t* inc_dev, int32_t* carry_dev, int64_t* acc_dev, void* stream);
int madrl_whole_paths_finish(int E, int S, const uint8_t* done_stage_dev, const int32_t* carry_dev,
                             int32_t* env_off_dev, int32_t* path_start_dev, uint8_t* done_flat_dev, void* stream);
int madrl_whole_paths_gather(int T, int E, size_t slab_bytes, int t_base, const void* src_dev, const void* first_dev,
                             const int32_t* carry_dev, const int32_t* env_off_dev, void* dst_dev, void* stream);
/* The path plan of a flat batch of N rows cut at path_start int32 [P+1] (the rollout view T = N, E = 1):
 * madrl_paths_plan's seg_start / seg_len [N], n_episodes [1] = P and ep_rec [N][3] (rows >= P untouched), one thread
 * per row / path.  madrl_gae_paths_f32: madrl_gae_f32 over the same view ([N][A] tensors, every path terminated),
 * one thread per (path, agent), bit for bit the serial walk's arithmetic. */
int madrl_paths_plan_flat(int N, int P, const int32_t* path_start_dev, int32_t* seg_start_dev, int32_t* seg_len_dev,
                          int32_t* n_episodes_dev, int32_t* ep_rec_dev, void* stream);
int madrl_gae_paths_f32(int P, int A, const int32_t* path_start_dev, const float* rew_dev, const float* value_dev,
                        double discount, double gae_lambda, float* adv_dev, float* ret_dev, void* stream);

/* rllab's LinearFeatureBaseline (rllab/rllab/baselines/linear_feature_baseline.py), decentralized mode: one
 * baseline over every (t, e, a) row of a rollout.  Row (t, e, a) uses the observation the action of step t was
 * taken in (obs_before != NULL: obs_before [E][A][D] for t = 0, obs[t-1] afterwards; NULL: obs[t]) and the time
 * index i = t - seg_start[t][e] (seg_start from madrl_paths_plan), plus t0[e] when seg_start[t][e] == 0
 * (t0 int32 [E] or NULL).  Features, Df = 2D + 4: [clip(o,-10,10), clip(o,-10,10)^2, i/100, (i/100)^2,
 * (i/100)^3, 1], in float64 (observations widened exactly, bfloat16 ones first to float32).
 *   madrl_lfb_normal_eq_*  ret float32 [T][E][A] -> G float64 [Df+1][Df+1] = [F y]^T [F y]: F^T F, with F^T y as
 *                          row / column Df and y^T y at [Df][Df]; exactly symmetric, deterministic (fixed row
 *                          partition and combination order).  ws: madrl_lfb_workspace_size bytes of device scratch,
 *                          which depends on D only:  48 * P * 32768 bytes, P = nb (nb + 1) / 2, nb = ceil((2D+5)/64).
 *   madrl_lfb_predict_*    coef float64 [Df] -> values float32 [T][E][A] = features . coef, evaluated in float64.
 * MADRL_EINVAL for D outside [1, 8192], T*E*A >= 2^31 or a NULL required buffer. */
int madrl_lfb_workspace_size(int D, size_t* bytes);
int madrl_lfb_normal_eq_f32(int T, int E, int A, int D, const float* obs_dev, const float* obs_before_dev,
                            const int32_t* seg_start_dev, const int32_t* t0_dev, const float* ret_dev, double* G_dev,
                            double* ws_dev, void* stream);
int madrl_lfb_normal_eq_bf16(int T, int E, int A, int D, const void* obs_dev, const void* obs_before_dev,
                             const int32_t* seg_start_dev, const int32_t* t0_dev, const float* ret_dev, double* G_dev,
                             double* ws_dev, void* stream);
int madrl_lfb_predict_f32(int T, int E, int A, int D, const float* obs_dev, const float* obs_before_dev,
                          const int32_t* seg_start_dev, const int32_t* t0_dev, const double* coef_dev,
                          float* values_dev, void* stream);
int madrl_lfb_predict_bf16(int T, int E, int A, int D, const void* obs_dev, const void* obs_before_dev,
                           const int32_t* seg_start_dev, const int32_t* t0_dev, const double* coef_dev,
                           float* values_dev, void* stream);

/* Concurrent mode: one LinearFeatureBaseline per agent (rllab/sandbox/rocky/tf/samplers/batch_ma_sampler.py:64-188).
 * Agent a's rows are (t, e, a) for every t, e; rows, features and time indices as above.
 *   madrl_lfb_normal_eq_agents_*  G float64 [A][Df+1][Df+1]: agent a's [F y]^T [F y] over its own rows only, each
 *                                 exactly symmetric and deterministic, all A from one launch.  Agent a's rows are
 *                                 cut into S = ceil(48 / A) fixed slices.  ws: madrl_lfb_agents_workspace_size bytes,
 *                                 A * S * P * 32768 (D = 213: 45.9 MB at A = 5, 55.1 MB at A = 20).  With A = 1 the
 *                                 result equals madrl_lfb_normal_eq_* bit for bit.
 *   madrl_lfb_predict_agents_*    coef float64 [A][Df]: row (t, e, a) is evaluated with coef[a].
 * MADRL_EINVAL as above, and for A outside [1, MADRL_AGENTS_MAX]. */
#define MADRL_AGENTS_MAX 1024
int madrl_lfb_agents_workspace_size(int D, int A, size_t* bytes);
int madrl_lfb_normal_eq_agents_f32(int T, int E, int A, int D, const float* obs_dev, const float* obs_before_dev,
                                   const int32_t* seg_start_dev, const int32_t* t0_dev, const float* ret_dev,
                                   double* G_dev, double* ws_dev, void* stream);
int madrl_lfb_normal_eq_agents_bf16(int T, int E, int A, int D, const void* obs_dev, const void* obs_before_dev,
                                    const int32_t* seg_start_dev, const int32_t* t0_dev, const float* ret_dev,
                                    double* G_dev, double* ws_dev, void* stream);
int madrl_lfb_predict_agents_f32(int T, int E, int A, int D, const float* obs_dev, const float* obs_before_dev,
                                 const int32_t* seg_start_dev, const int32_t* t0_dev, const double* coef_dev,
                                 float* values_dev, void* stream);
int madrl_lfb_predict_agents_bf16(int T, int E, int A, int D, const void* obs_dev, const void* obs_before_dev,
                                  const int32_t* seg_start_dev, const int32_t* t0_dev, const double* coef_dev,
                                  float* values_dev, void* stream);

/* rltools' sample processing (rltools/rltools/samplers/__init__.py:35-88).
 *   madrl_running_moments_*  nn.Standardizer's batch statistics: sums float64 [G][2][D] = the column sums of x and
 *                            of x^2 over the rows k G + g (k < R) of group g of x [R*G][D] (float32, or bfloat16
 *                            widened), deterministic (fixed row slices, ascending combination).  first != NULL:
 *                            row r is read from first [shift][D] for r < shift and from x[r - shift] afterwards
 *                            (the observation an action was taken in; shift = E*A).  ws:
 *                            madrl_running_moments_workspace_size bytes.  MADRL_EINVAL for R, D < 1, G outside
 *                            [1, MADRL_AGENTS_MAX], a shift outside [1, R*G] with first, or a NULL required buffer.
 *   madrl_time_baseline_bins_f32   q float32 [T][E][A] -> bin_sum float64 [G][L], bin_count int32 [G][L] (G = A
 *                            with per_agent, else 1 over every agent's rows): the sum of q and the number of rows
 *                            whose time index (as madrl_lfb_*: t - seg_start, plus t0[e] on env e's first path) is
 *                            i.  n_ep, ep_rec: madrl_paths_plan's outputs.  ws:
 *                            madrl_time_baseline_workspace_size(G, L) bytes.
 *   madrl_time_baseline_apply_f32  simplev float32 [T][E][A] = sum / count of the row's bin in the bins it is given
 *                            (NaN for an index >= L); seg_start: madrl_paths_plan's.  The bins of the shards of a
 *                            batch may be summed between the two calls.
 *                            Both deterministic, no atomics.  MADRL_EINVAL for sizes below 1, T*E*A >= 2^31,
 *                            per_agent with A > MADRL_AGENTS_MAX or a NULL required buffer. */
int madrl_running_moments_workspace_size(int G, int D, size_t* bytes);
int madrl_running_moments_f32(size_t R, int G, int D, size_t shift, const float* x_dev, const float* first_dev,
                              double* sums_dev, double* ws_dev, void* stream);
int madrl_running_moments_bf16(size_t R, int G, int D, size_t shift, const void* x_dev, const void* first_dev,
                               double* sums_dev, double* ws_dev, void* stream);
int madrl_time_baseline_workspace_size(int G, int L, size_t* bytes);
int madrl_time_baseline_bins_f32(int T, int E, int A, int per_agent, int L, const float* q_dev,
                                 const int32_t* n_ep_dev, const int32_t* ep_rec_dev, const int32_t* t0_dev,
                                 double* bin_sum_dev, int32_t* bin_count_dev, void* ws_dev, void* stream);
int madrl_time_baseline_apply_f32(int T, int E, int A, int per_agent, int L, const int32_t* seg_start_dev,
                                  const int32_t* t0_dev, const double* bin_sum_dev, const int32_t* bin_count_dev,
                                  float* simplev_dev, void* stream);

/* rltools' LinearFeatureBaseline (rltools/rltools/baselines/linear.py): the madrl_lfb_* kernels with rltools'
 * feature map, Df = D + 3: [(o - mu) / s, i/100, (i/100)^2, 1] with o widened to float64 and not clipped.
 * norm float64 [2][D] ([A][2][D] for the _agents entry points) = the obsnorm's mean and stdev + eps per column
 * (the quotient is a float64 division), or NULL for no obsnorm (the columns are o).  Rows, time indices,
 * determinism, argument checks and the _agents grouping as for madrl_lfb_*; ws: madrl_lfbr_workspace_size /
 * madrl_lfbr_agents_workspace_size bytes (nb = ceil((D+4)/64)). */
int madrl_lfbr_workspace_size(int D, size_t* bytes);
int madrl_lfbr_agents_workspace_size(int D, int A, size_t* bytes);
int madrl_lfbr_normal_eq_f32(int T, int E, int A, int D, const float* obs_dev, const float* obs_before_dev,
    const int32_t* seg_start_dev, const int32_t* t0_dev, const float* ret_dev, const double* norm_dev, double* G_dev,
    double* ws_dev, void* stream);
int madrl_lfbr_predict_f32(int T, int E, int A, int D, const float* obs_dev, const float* obs_before_dev,
    const int32_t* seg_start_dev, const int32_t* t0_dev, const double* norm_dev, const double* coef_dev,
    float* values_dev, void* stream);
int madrl_lfbr_normal_eq_bf16(int T, int E, int A, int D, const void* obs_dev, const void* obs_before_dev,
    const int32_t* seg_start_dev, const int32_t* t0_dev, const float* ret_dev, const double* norm_dev, double* G_dev,
    double* ws_dev, void* stream);
int madrl_lfbr_predict_bf16(int T, int E, int A, int D, const void* obs_dev, const void* obs_before_dev,
    const int32_t* seg_start_dev, const int32_t* t0_dev, const double* norm_dev, const double* coef_dev,
    float* values_dev, void* stream);
int madrl_lfbr_normal_eq_agents_f32(int T, int E, int A, int D, const float* obs_dev, const float* obs_before_dev,
    const int32_t* seg_start_dev, const int32_t* t0_dev, const float* ret_dev, const double* norm_dev, double* G_dev,
    double* ws_dev, void* stream);
int madrl_lfbr_predict_agents_f32(int T, int E, int A, int D, const float* obs_dev, const float* obs_before_dev,
    const int32_t* seg_start_dev, const int32_t* t0_dev, const double* norm_dev, const double* coef_dev,
    float* values_dev, void* stream);
int madrl_lfbr_normal_eq_agents_bf16(int T, int E, int A, int D, const void* obs_dev, const void* obs_before_dev,
    const int32_t* seg_start_dev, const int32_t* t0_dev, const float* ret_dev, const double* norm_dev, double* G_dev,
    double* ws_dev, void* stream);
int madrl_lfbr_predict_agents_bf16(int T, int E, int A, int D, const void* obs_dev, const void* obs_before_dev,
    const int32_t* seg_start_dev, const int32_t* t0_dev, const double* norm_dev, const double* coef_dev,
    float* values_dev, void* stream);

/* rllab's DDPG replay pool (rllab/rllab/algos/ddpg.py:85-145 MAReplayPool), decentralized mode, in device memory
 * (csrc/replay.cu).  The pool of M = max_pool_size slots: pool_obs / pool_next [M][D] (float32 or bfloat16 bits),
 * pool_act float32 [M][Ad], pool_rew float32 [M], pool_term uint8 [M]; ctl int64 [4] = top, bottom, size and the
 * sampler's draw counter, all read and written on the device only.
 *   madrl_replay_add_*     inserts the transitions of one rollout as DDPG.train adds them (:285-353): (t, e, a) order;
 *                          observation obs[t-1] (obs_before [E][A][D] at t = 0), action act[t] (float32 [T][E][A][Ad]),
 *                          reward float32(double(rew[t]) * scale_reward), next observation term[t] where done[t]
 *                          else obs[t], terminal done[t].  Paths continue from path_len0 / timestep0 (int32 [E], the
 *                          engine's counters before the launch); a done step with path length >= max_path_length
 *                          (> 0) and timestep < timestep_limit is a horizon cut, dropped unless include_horizon.
 *                          When K kept transitions exceed M only the last M land; ctl moves as K add_sample calls.
 *                          ws: madrl_replay_workspace_size(T, E) bytes, 16-byte aligned.  Three launches.
 *   madrl_replay_sample_*  n x B draws with replacement, uniform over slots [0, size - 1) (the set random_batch's
 *                          rejection loop accepts): slot of draw c = mulhi64(Philox4x32-10 words 1:0 of counter
 *                          (c, 0, 0, 2) under key seed, max(size - 1, 1)), c = ctl[3] + row; ctl[3] += n * B.
 *                          Writes idx int64 [n*B] and the rows of obs / next observations / actions / rewards /
 *                          terminals.  Two launches. */
int madrl_replay_workspace_size(int T, int E, size_t* bytes);
int madrl_replay_add_f32(int T, int E, int A, int D, int Ad, size_t M, const float* obs_dev, const float* act_dev,
    const float* rew_dev, const uint8_t* done_dev, const float* obs_before_dev, const float* term_dev,
    const int32_t* path_len0_dev, const int32_t* timestep0_dev, int max_path_length, int timestep_limit,
    int include_horizon, double scale_reward, float* pool_obs_dev, float* pool_next_dev, float* pool_act_dev,
    float* pool_rew_dev, uint8_t* pool_term_dev, int64_t* ctl_dev, void* ws_dev, void* stream);
int madrl_replay_add_bf16(int T, int E, int A, int D, int Ad, size_t M, const void* obs_dev, const float* act_dev,
    const float* rew_dev, const uint8_t* done_dev, const void* obs_before_dev, const void* term_dev,
    const int32_t* path_len0_dev, const int32_t* timestep0_dev, int max_path_length, int timestep_limit,
    int include_horizon, double scale_reward, void* pool_obs_dev, void* pool_next_dev, float* pool_act_dev,
    float* pool_rew_dev, uint8_t* pool_term_dev, int64_t* ctl_dev, void* ws_dev, void* stream);
int madrl_replay_sample_f32(int n, int B, int D, int Ad, size_t M, uint64_t seed, const float* pool_obs_dev,
    const float* pool_next_dev, const float* pool_act_dev, const float* pool_rew_dev, const uint8_t* pool_term_dev,
    int64_t* ctl_dev, int64_t* idx_dev, float* obs_out_dev, float* next_out_dev, float* act_out_dev,
    float* rew_out_dev, uint8_t* term_out_dev, void* stream);
int madrl_replay_sample_bf16(int n, int B, int D, int Ad, size_t M, uint64_t seed, const void* pool_obs_dev,
    const void* pool_next_dev, const float* pool_act_dev, const float* pool_rew_dev, const uint8_t* pool_term_dev,
    int64_t* ctl_dev, int64_t* idx_dev, void* obs_out_dev, void* next_out_dev, float* act_out_dev,
    float* rew_out_dev, uint8_t* term_out_dev, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MADRL_B200_H */
