"""ctypes binding of the C ABI declared in ``include/madrl_b200.h``.

The CUDA library is the product: if it cannot be loaded there is NO fallback -- importing an
engine class raises.  PyTorch is used only to own device memory and streams.
"""
import ctypes as C
import os

import torch

from . import build as _build

_lib = None


class EngineError(RuntimeError):
    pass


# observation formats (madrl_*_set_obs_format)
OBS_NATIVE, OBS_BF16 = 0, 1
# L2 policy of the rollouts' observation stores (madrl_*_set_obs_cache)
OBS_CACHE_STREAM, OBS_CACHE_KEEP = 0, 1
# Waterworld's observation write path (madrl_ww_set_obs_writer)
WW_OBS_WRITER_AUTO, WW_OBS_WRITER_OFF, WW_OBS_WRITER_ON = 0, 1, 2
# norm of Waterworld's in-kernel heuristic actions (madrl_ww_set_heuristic_norm)
HEURISTIC_NORM_AGENT, HEURISTIC_NORM_ENV = 0, 1
# evaluation records (madrl_eval_episodes_*): 8-byte carry words per (env, agent), most info columns
EVAL_CARRY_WORDS, EVAL_INFO_MAX = 8, 2


class WWConfig(C.Structure):
    _fields_ = [
        ("n_envs", C.c_int32), ("env_id_base", C.c_int32),
        ("n_pursuers", C.c_int32), ("n_evaders", C.c_int32), ("n_poison", C.c_int32),
        ("n_sensors", C.c_int32), ("n_coop", C.c_int32),
        ("reward_global", C.c_int32), ("addid", C.c_int32), ("speed_features", C.c_int32),
        ("random_obstacle", C.c_int32), ("timestep_limit", C.c_int32),
        ("max_path_length", C.c_int32), ("fp64", C.c_int32),
        ("radius", C.c_double), ("obstacle_radius", C.c_double), ("obstacle_x", C.c_double),
        ("obstacle_y", C.c_double), ("ev_speed", C.c_double), ("poison_speed", C.c_double),
        ("sensor_range", C.c_double), ("action_scale", C.c_double), ("poison_reward", C.c_double),
        ("food_reward", C.c_double), ("encounter_reward", C.c_double),
        ("control_penalty", C.c_double), ("seed", C.c_uint64),
    ]


class WWLayout(C.Structure):
    _fields_ = [
        ("total_bytes", C.c_size_t), ("objs", C.c_size_t), ("obst", C.c_size_t),
        ("timestep", C.c_size_t), ("path_len", C.c_size_t), ("rng_counter", C.c_size_t),
        ("sensors", C.c_size_t),
        ("n_obj", C.c_int32), ("obs_dim", C.c_int32), ("real_bytes", C.c_int32), ("_pad", C.c_int32),
    ]


class PEConfig(C.Structure):
    _fields_ = [
        ("n_envs", C.c_int32), ("env_id_base", C.c_int32), ("n_pursuers", C.c_int32),
        ("n_evaders", C.c_int32), ("xs", C.c_int32), ("ys", C.c_int32), ("n_maps", C.c_int32),
        ("obs_range", C.c_int32), ("flatten", C.c_int32), ("n_catch", C.c_int32),
        ("surround", C.c_int32), ("reward_global", C.c_int32), ("include_id", C.c_int32),
        ("sample_maps", C.c_int32), ("max_path_length", C.c_int32), ("max_opponents", C.c_int32),
        ("layer_norm", C.c_double), ("catchr", C.c_double), ("term_pursuit", C.c_double),
        ("urgency_reward", C.c_double), ("constraint_window", C.c_double), ("seed", C.c_uint64),
    ]


class PELayout(C.Structure):
    _fields_ = [
        ("total_bytes", C.c_size_t), ("pos", C.c_size_t), ("gone", C.c_size_t),
        ("map_id", C.c_size_t), ("path_len", C.c_size_t), ("rng_counter", C.c_size_t),
        ("stale", C.c_size_t), ("maps", C.c_size_t), ("lut", C.c_size_t), ("idv", C.c_size_t),
        ("n_agents", C.c_int32), ("obs_dim", C.c_int32),
    ]


class HWConfig(C.Structure):
    _fields_ = [
        ("n_envs", C.c_int32), ("env_id_base", C.c_int32), ("n_good", C.c_int32),
        ("n_hostages", C.c_int32), ("n_bad", C.c_int32), ("n_coop_save", C.c_int32),
        ("n_coop_avoid", C.c_int32), ("n_sensors", C.c_int32), ("reward_global", C.c_int32),
        ("addid", C.c_int32), ("random_key", C.c_int32), ("timestep_limit", C.c_int32),
        ("max_path_length", C.c_int32), ("fp64", C.c_int32),
        ("radius", C.c_double), ("key_x", C.c_double), ("key_y", C.c_double),
        ("bad_speed", C.c_double), ("sensor_range", C.c_double), ("action_scale", C.c_double),
        ("save_reward", C.c_double), ("hit_reward", C.c_double), ("encounter_reward", C.c_double),
        ("not_saved_reward", C.c_double), ("bomb_reward", C.c_double), ("bomb_radius", C.c_double),
        ("key_radius", C.c_double), ("control_penalty", C.c_double), ("seed", C.c_uint64),
    ]


class HWLayout(C.Structure):
    _fields_ = [
        ("total_bytes", C.c_size_t), ("objs", C.c_size_t), ("fixed", C.c_size_t),
        ("saved", C.c_size_t), ("flags", C.c_size_t), ("timestep", C.c_size_t),
        ("path_len", C.c_size_t), ("rng_counter", C.c_size_t), ("sensors", C.c_size_t),
        ("n_obj", C.c_int32), ("obs_dim", C.c_int32), ("real_bytes", C.c_int32), ("_pad", C.c_int32),
    ]


def _ptr(t):
    """A tensor's data pointer for the C ABI (None -> NULL)."""
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _signatures():
    """(restype, argtypes) of every function of include/madrl_b200.h, grouped as the header groups them.
    Every pointer is a c_void_p except the config / layout structs, the out-parameters callers pass with
    byref (handles, sizes, device pointers), madrl_abi_sizes' array, and the error message and IPC handles
    (bytes).  tests/test_abi_signatures_cpu.py checks the table against the header."""
    vp, i32, sz, f64, u32, u64, P = C.c_void_p, C.c_int, C.c_size_t, C.c_double, C.c_uint32, C.c_uint64, C.POINTER
    sig = {
        "madrl_last_error": (C.c_char_p, []),
        "madrl_version": (i32, []),
        "madrl_abi_sizes": (None, [P(C.c_int32)]),
        "madrl_launch_count": (u64, []),
        "madrl_set_host_chunk_bytes": (None, [sz]),
        # CUDA-IPC buffers
        "madrl_ipc_alloc": (i32, [sz, P(vp), C.c_char_p]),
        "madrl_ipc_open": (i32, [C.c_char_p, P(vp)]),
        "madrl_ipc_close": (i32, [vp]),
        "madrl_ipc_free": (i32, [vp]),
        # stream-ordered primitives of the multi-GPU exchange
        "madrl_stream_memops_available": (i32, []),
        "madrl_copy_async": (i32, [vp, vp, sz, vp]),
        "madrl_stream_write32": (i32, [vp, vp, u32]),
        "madrl_stream_wait_geq32": (i32, [vp, vp, u32]),
    }
    # the env families: the same entry points apart from their structs, Pursuit's map pool and a few extras
    for fam, cfg, lay in (("ww", WWConfig, WWLayout), ("pursuit", PEConfig, PELayout),
                          ("hostage", HWConfig, HWLayout)):
        pool = [vp] if fam == "pursuit" else []
        sig.update(("madrl_%s_%s" % (fam, name), s) for name, s in (
            ("state_layout", (i32, [P(cfg), P(lay)])),
            ("create", (i32, [P(cfg)] + pool + [vp, P(vp)])),
            ("destroy", (i32, [vp])),
            ("state_ptr", (vp, [vp])),
            ("seed", (i32, [vp, u64, vp])),
            ("set_launch", (i32, [vp, i32, i32])),
            ("set_terminal_obs", (i32, [vp, vp])),
            ("set_obs_format", (i32, [vp, i32])),
            ("set_obs_cache", (i32, [vp, i32])),
            ("reset", (i32, [vp, vp, vp, vp])),
            ("rollout", (i32, [vp, i32, vp, vp, vp, vp, vp, i32, vp])),
            ("step", (i32, [vp, vp, vp, vp, vp, vp, i32, vp])),
            ("reset_host", (i32, [vp, vp, vp])),
            ("rollout_host", (i32, [vp, i32, vp, vp, vp, vp, vp, i32])),
            ("rollout_host2", (i32, [vp, i32, vp, vp, vp, vp, vp, i32, i32]))))
    sig.update({
        "madrl_ww_default_blocks_per_sm": (i32, [vp, i32]),
        "madrl_ww_launch_log": (i32, [i32, vp, i32]),
        "madrl_ww_set_obs_writer": (i32, [vp, i32]),
        "madrl_ww_set_heuristic_norm": (i32, [vp, i32]),
        "madrl_ww_set_peers": (i32, [vp, i32, i32, i32, P(vp), P(vp), P(vp)]),
        "madrl_ww_rollout_heuristic": (i32, [vp, i32, vp, vp, vp, vp, vp, vp, i32, vp]),
        "madrl_pursuit_set_params": (i32, [vp, f64, f64]),
        "madrl_pursuit_rollout_heuristic": (i32, [vp, i32, vp, vp, vp, vp, vp, vp, i32, i32, vp]),
        # hand-written policies
        "madrl_ww_heuristic_actions": (i32, [i32, sz, i32, i32, vp, vp, vp]),
        "madrl_pursuit_heuristic_actions": (i32, [sz, i32, i32, i32, i32, vp, vp, vp, vp, vp]),
        # trajectory post-processing
        "madrl_gae_f32": (i32, [i32, i32, i32, vp, vp, vp, vp, f64, f64, vp, vp, vp]),
        "madrl_frame_stack_f32": (i32, [i32] * 5 + [vp] * 5),
        "madrl_frame_stack_bf16": (i32, [i32] * 5 + [vp] * 5),
        "madrl_standardize_f32": (i32, [i32, sz, vp, vp, vp, f64, f64, i32, f64, i32, vp]),
        "madrl_standardize_bf16": (i32, [i32, sz, vp, vp, vp, f64, f64, i32, f64, i32, vp]),
        "madrl_standardize_obs_terminal_f32": (i32, [i32, i32, sz] + [vp] * 5 + [f64, f64, vp]),
        "madrl_standardize_obs_terminal_bf16": (i32, [i32, i32, sz] + [vp] * 5 + [f64, f64, vp]),
        "madrl_obs_wrap_step_f32": (i32, [i32] * 4 + [vp] * 7 + [f64, f64, vp]),
        "madrl_obs_wrap_step_bf16": (i32, [i32] * 4 + [vp] * 7 + [f64, f64, vp]),
        "madrl_episode_stats_f32": (i32, [i32, i32, i32, vp, vp, f64, i32, vp, vp, vp, vp, vp, vp]),
        "madrl_eval_episodes_f32": (i32, [i32] * 4 + [vp] * 3 + [f64, i32] + [vp] * 6),
        "madrl_eval_episodes_f64": (i32, [i32] * 4 + [vp] * 3 + [f64, i32] + [vp] * 6),
        # moments and advantage centring
        "madrl_moments_pass_f32": (i32, [sz, i32, vp, vp, i32, vp, vp, vp]),
        "madrl_center_apply_f32": (i32, [sz, i32, vp, vp, i32, i32, vp]),
        # path packing and padding
        "madrl_paths_plan": (i32, [i32, i32, i32] + [vp] * 6),
        "madrl_paths_pack_u32": (i32, [i32] * 4 + [vp] * 6),
        "madrl_paths_pack_u16": (i32, [i32] * 4 + [vp] * 6),
        "madrl_paths_pad_u32": (i32, [i32] * 6 + [vp] * 5),
        "madrl_paths_pad_u16": (i32, [i32] * 6 + [vp] * 5),
        "madrl_path_sums_f32": (i32, [i32] * 4 + [vp] * 6),
        # whole-path sampling and the flat batch's path-parallel passes
        "madrl_whole_paths_fold": (i32, [i32] * 3 + [sz] + [vp] * 4),
        "madrl_whole_paths_finish": (i32, [i32] * 2 + [vp] * 6),
        "madrl_whole_paths_gather": (i32, [i32, i32, sz, i32] + [vp] * 6),
        "madrl_paths_plan_flat": (i32, [i32] * 2 + [vp] * 6),
        "madrl_gae_paths_f32": (i32, [i32] * 2 + [vp] * 3 + [f64, f64] + [vp] * 3),
        # rllab's linear feature baseline, pooled and per agent
        "madrl_lfb_workspace_size": (i32, [i32, P(sz)]),
        "madrl_lfb_normal_eq_f32": (i32, [i32] * 4 + [vp] * 8),
        "madrl_lfb_normal_eq_bf16": (i32, [i32] * 4 + [vp] * 8),
        "madrl_lfb_predict_f32": (i32, [i32] * 4 + [vp] * 7),
        "madrl_lfb_predict_bf16": (i32, [i32] * 4 + [vp] * 7),
        "madrl_lfb_agents_workspace_size": (i32, [i32, i32, P(sz)]),
        "madrl_lfb_normal_eq_agents_f32": (i32, [i32] * 4 + [vp] * 8),
        "madrl_lfb_normal_eq_agents_bf16": (i32, [i32] * 4 + [vp] * 8),
        "madrl_lfb_predict_agents_f32": (i32, [i32] * 4 + [vp] * 7),
        "madrl_lfb_predict_agents_bf16": (i32, [i32] * 4 + [vp] * 7),
        # rltools' sample processing
        "madrl_running_moments_workspace_size": (i32, [i32, i32, P(sz)]),
        "madrl_running_moments_f32": (i32, [sz, i32, i32, sz] + [vp] * 5),
        "madrl_running_moments_bf16": (i32, [sz, i32, i32, sz] + [vp] * 5),
        "madrl_time_baseline_workspace_size": (i32, [i32, i32, P(sz)]),
        "madrl_time_baseline_bins_f32": (i32, [i32] * 5 + [vp] * 8),
        "madrl_time_baseline_apply_f32": (i32, [i32] * 5 + [vp] * 6),
        # rltools' linear feature baseline
        "madrl_lfbr_workspace_size": (i32, [i32, P(sz)]),
        "madrl_lfbr_agents_workspace_size": (i32, [i32, i32, P(sz)]),
        # rllab's DDPG replay pool
        "madrl_replay_workspace_size": (i32, [i32, i32, P(sz)]),
        "madrl_replay_add_f32": (i32, [i32] * 5 + [sz] + [vp] * 8 + [i32] * 3 + [f64] + [vp] * 8),
        "madrl_replay_add_bf16": (i32, [i32] * 5 + [sz] + [vp] * 8 + [i32] * 3 + [f64] + [vp] * 8),
        "madrl_replay_sample_f32": (i32, [i32] * 4 + [sz, u64] + [vp] * 13),
        "madrl_replay_sample_bf16": (i32, [i32] * 4 + [sz, u64] + [vp] * 13),
    })
    for ag in ("", "_agents"):
        for dt in ("f32", "bf16"):
            sig["madrl_lfbr_normal_eq%s_%s" % (ag, dt)] = (i32, [i32] * 4 + [vp] * 9)
            sig["madrl_lfbr_predict%s_%s" % (ag, dt)] = (i32, [i32] * 4 + [vp] * 8)
    return sig


SIGNATURES = _signatures()


def declare(lib):
    """Set restype and argtypes of every SIGNATURES function `lib` exports.  Absent ones are skipped, so that
    MADRL_B200_LIB can load libraries built before an entry point existed (timed side by side by scripts/)."""
    for name, (restype, argtypes) in SIGNATURES.items():
        f = getattr(lib, name, None)
        if f is not None:
            f.restype, f.argtypes = restype, argtypes


# The env families' entry points are part of the full table now; test drivers written against the former
# engine-only declaration call it under this name.
_declare_engines = declare


def check_struct_sizes(lib, path):
    """Raise EngineError unless `lib` was compiled with the config / layout structs this binding declares."""
    sizes = (C.c_int32 * 6)()
    lib.madrl_abi_sizes(sizes)
    want = [C.sizeof(t) for t in (WWConfig, WWLayout, PEConfig, PELayout, HWConfig, HWLayout)]
    if list(sizes) != want:
        raise EngineError("%s was built against another include/madrl_b200.h: struct sizes %s, this "
                          "binding expects %s" % (path, list(sizes), want))


def lib():
    """Load (building if needed) the CUDA library.  Raises EngineError on failure."""
    global _lib
    if _lib is None:
        path = os.environ.get("MADRL_B200_LIB")            # override: kernel-variant experiments
        if path is None:
            # build() is a no-op when the library was built from exactly the sources in the tree
            # (content hash); a stale git-ignored .so left over from other sources is rebuilt, not loaded
            try:
                path = _build.build(force=bool(os.environ.get("MADRL_B200_REBUILD")))
            except Exception as e:  # no nvcc / compile error: there is no CPU fallback
                raise EngineError("madrl_b200 CUDA library is missing or stale and could not be built: %s" % e)
        try:
            lib_ = C.CDLL(path)
        except OSError as e:
            raise EngineError("cannot load %s: %s" % (path, e))
        declare(lib_)
        check_struct_sizes(lib_, path)
        _lib = lib_
    return _lib


def require_tensor(t, name, dtype, shape, device, contiguous=True, optional=False):
    """Validate a caller-supplied tensor before its data_ptr() crosses the C ABI.  The kernels trust the
    sizes they are given: a wrong dtype, a short buffer, a host or foreign-device pointer or a strided view
    would otherwise be silent garbage or an out-of-bounds device access.

    `dtype`: a dtype or a tuple of them.  `shape`: a tuple of sizes; None matches any size, and a trailing
    ``...`` any number of further dimensions (``(...,)``: any shape).  `device`: a torch.device; 'cuda' for
    any CUDA device; 'cpu' for host buffers; None to leave it to a later call, once the shapes of every
    tensor of the call are checked.  `contiguous=False`: a read-only input the caller copies with
    .contiguous().  `optional=True`: None passes through.  Raises TypeError (not a tensor, wrong dtype),
    then ValueError (shape, device, contiguity), naming `name`; returns `t`."""
    if t is None and optional:
        return None
    if not isinstance(t, torch.Tensor):
        raise TypeError("%s must be a torch.Tensor, got %r" % (name, type(t)))
    dtypes = dtype if isinstance(dtype, tuple) else (dtype,)
    if t.dtype not in dtypes:
        raise TypeError("%s must be %s, got %s" % (name, " or ".join(map(str, dtypes)), t.dtype))
    got = tuple(t.shape)
    if got != shape:
        tail = shape[-1:] == (...,)
        fixed = shape[:-1] if tail else shape
        if (len(got) < len(fixed) if tail else len(got) != len(fixed)) or \
                any(s is not None and s != n for s, n in zip(fixed, got)):
            raise ValueError("%s must have shape [%s], got [%s]" % (
                name, ", ".join("*" if s is None else "..." if s is ... else str(s) for s in shape),
                ", ".join(map(str, got))))
    if device is not None and (t.device.type != device if isinstance(device, str) else t.device != device):
        raise ValueError("%s must live on %s, got %s" % (name, device, t.device))
    if contiguous and not t.is_contiguous():
        raise ValueError("%s must be contiguous" % name)
    return t


def stream(device):
    """The current torch stream of `device`, as the cudaStream_t argument of the C ABI."""
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def check(rc):
    if rc != 0:
        raise EngineError("madrl_b200 error %d: %s" % (rc, lib().madrl_last_error().decode()))


def launch_count():
    return int(lib().madrl_launch_count())
