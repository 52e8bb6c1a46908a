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


def _declare_engines(lib):
    """argtypes of the env families' entry points (madrl_{ww,pursuit,hostage}_*)."""
    vp, i32, u64 = C.c_void_p, C.c_int, C.c_uint64
    for fam, cfg, lay in (("ww", WWConfig, WWLayout), ("hostage", HWConfig, HWLayout),
                          ("pursuit", PEConfig, PELayout)):
        f = lambda name: getattr(lib, "madrl_%s_%s" % (fam, name))   # noqa: E731
        f("state_layout").argtypes = [C.POINTER(cfg), C.POINTER(lay)]
        # pursuit: the map pool comes before the state blob
        f("create").argtypes = [C.POINTER(cfg)] + ([vp] if fam == "pursuit" else []) + [vp, C.POINTER(vp)]
        f("destroy").argtypes = [vp]
        f("state_ptr").argtypes = [vp]
        f("state_ptr").restype = vp
        f("seed").argtypes = [vp, u64, vp]
        f("set_launch").argtypes = [vp, i32, i32]
        f("set_terminal_obs").argtypes = [vp, vp]
        f("reset").argtypes = [vp, vp, vp, vp]
        f("rollout").argtypes = [vp, i32, vp, vp, vp, vp, vp, i32, vp]
        f("step").argtypes = [vp, vp, vp, vp, vp, vp, i32, vp]
        f("reset_host").argtypes = [vp, vp, vp]
        f("rollout_host").argtypes = [vp, i32, vp, vp, vp, vp, vp, i32]
        f("rollout_host2").argtypes = [vp, i32, vp, vp, vp, vp, vp, i32, i32]
        # absent from libraries built before the bfloat16 observation format (timed side by side by scripts/)
        if hasattr(lib, "madrl_%s_set_obs_format" % fam):
            f("set_obs_format").argtypes = [vp, i32]
    if hasattr(lib, "madrl_ww_default_blocks_per_sm"):   # absent from older builds timed by scripts/
        lib.madrl_ww_default_blocks_per_sm.argtypes = [vp, i32]
    lib.madrl_ww_set_peers.argtypes = [vp, i32, i32, i32, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp)]
    lib.madrl_ww_rollout_heuristic.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp, i32, vp]
    lib.madrl_pursuit_set_params.argtypes = [vp, C.c_double, C.c_double]
    lib.madrl_pursuit_rollout_heuristic.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp, i32, i32, vp]


def _declare(lib):
    vp, i32 = C.c_void_p, C.c_int
    _declare_engines(lib)
    lib.madrl_last_error.restype = C.c_char_p
    lib.madrl_version.restype = C.c_int
    lib.madrl_abi_sizes.argtypes = [C.POINTER(C.c_int32)]
    lib.madrl_abi_sizes.restype = None
    lib.madrl_launch_count.restype = C.c_uint64
    lib.madrl_set_host_chunk_bytes.argtypes = [C.c_size_t]
    lib.madrl_set_host_chunk_bytes.restype = None
    lib.madrl_ipc_alloc.argtypes = [C.c_size_t, C.POINTER(vp), C.c_char_p]
    lib.madrl_ipc_open.argtypes = [C.c_char_p, C.POINTER(vp)]
    lib.madrl_ipc_close.argtypes = [vp]
    lib.madrl_ipc_free.argtypes = [vp]
    lib.madrl_stream_memops_available.restype = C.c_int
    lib.madrl_copy_async.argtypes = [vp, vp, C.c_size_t, vp]
    lib.madrl_stream_write32.argtypes = [vp, vp, C.c_uint32]
    lib.madrl_stream_wait_geq32.argtypes = [vp, vp, C.c_uint32]
    lib.madrl_ww_heuristic_actions.argtypes = [i32, C.c_size_t, i32, i32, vp, vp, vp]
    lib.madrl_pursuit_heuristic_actions.argtypes = [C.c_size_t, i32, i32, i32, i32, vp, vp, vp, vp, vp]
    lib.madrl_gae_f32.argtypes = [i32, i32, i32, vp, vp, vp, vp, C.c_double, C.c_double, vp, vp, vp]
    lib.madrl_frame_stack_f32.argtypes = [i32, i32, i32, i32, i32, vp, vp, vp, vp, vp]
    lib.madrl_standardize_f32.argtypes = [i32, C.c_size_t, vp, vp, vp, C.c_double, C.c_double, i32,
                                          C.c_double, i32, vp]
    lib.madrl_episode_stats_f32.argtypes = [i32, i32, i32, vp, vp, C.c_double, i32, vp, vp, vp, vp, vp, vp]
    lib.madrl_standardize_obs_terminal_f32.argtypes = [i32, i32, C.c_size_t, vp, vp, vp, vp, vp, C.c_double, C.c_double, vp]
    lib.madrl_paths_plan.argtypes = [i32, i32, i32, vp, vp, vp, vp, vp, vp]
    lib.madrl_paths_pack_u32.argtypes = [i32, i32, i32, i32, vp, vp, vp, vp, vp, vp]
    lib.madrl_moments_f32.argtypes = [C.c_size_t, vp, vp, vp, vp, vp]
    lib.madrl_center_advantages_f32.argtypes = [C.c_size_t, vp, i32, i32, vp, vp, vp]
    if hasattr(lib, "madrl_frame_stack_bf16"):   # bfloat16 observation passes (absent from older builds)
        lib.madrl_frame_stack_bf16.argtypes = lib.madrl_frame_stack_f32.argtypes
        lib.madrl_standardize_bf16.argtypes = lib.madrl_standardize_f32.argtypes
        lib.madrl_standardize_obs_terminal_bf16.argtypes = lib.madrl_standardize_obs_terminal_f32.argtypes
        lib.madrl_paths_pack_u16.argtypes = lib.madrl_paths_pack_u32.argtypes
    if hasattr(lib, "madrl_lfb_normal_eq_f32"):  # linear feature baseline (absent from older builds)
        lib.madrl_lfb_workspace_size.argtypes = [i32, C.POINTER(C.c_size_t)]
        for dt in ("f32", "bf16"):
            getattr(lib, "madrl_lfb_normal_eq_" + dt).argtypes = [i32, i32, i32, i32] + [vp] * 8
            getattr(lib, "madrl_lfb_predict_" + dt).argtypes = [i32, i32, i32, i32] + [vp] * 7
    if hasattr(lib, "madrl_lfb_normal_eq_agents_f32"):  # per-agent baselines (absent from older builds)
        lib.madrl_lfb_agents_workspace_size.argtypes = [i32, i32, C.POINTER(C.c_size_t)]
        for dt in ("f32", "bf16"):
            getattr(lib, "madrl_lfb_normal_eq_agents_" + dt).argtypes = [i32, i32, i32, i32] + [vp] * 8
            getattr(lib, "madrl_lfb_predict_agents_" + dt).argtypes = [i32, i32, i32, i32] + [vp] * 7
        lib.madrl_moments_agents_f32.argtypes = [C.c_size_t, i32, vp, vp, vp, vp, vp]
        lib.madrl_center_advantages_agents_f32.argtypes = [C.c_size_t, i32, vp, i32, i32, vp, vp, vp]
    if hasattr(lib, "madrl_paths_pad_u32"):    # padded paths of the recurrent sample batch (absent from older builds)
        lib.madrl_paths_pad_u32.argtypes = [i32] * 6 + [vp] * 5
        lib.madrl_paths_pad_u16.argtypes = lib.madrl_paths_pad_u32.argtypes
        lib.madrl_path_sums_f32.argtypes = [i32] * 4 + [vp] * 6


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
        _declare(lib_)
        sizes = (C.c_int32 * 6)()
        lib_.madrl_abi_sizes(sizes)
        want = [C.sizeof(t) for t in (WWConfig, WWLayout, PEConfig, PELayout, HWConfig, HWLayout)]
        if list(sizes) != want:
            raise EngineError("%s was built against another include/madrl_b200.h: struct sizes %s, this "
                              "binding expects %s" % (path, list(sizes), want))
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
