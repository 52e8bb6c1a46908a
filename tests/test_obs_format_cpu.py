"""The observation-format setters of the C ABI and the `obs_dtype` argument, without a GPU (the emulated
kernels are in test_emulated_obs_bf16.py, the device runs in test_obs_bf16_gpu.py)."""
import ctypes as C

import pytest
import torch


def test_library_exports_the_obs_format_setters():
    from madrl_b200 import _lib
    lib = _lib.lib()
    for fam in ("ww", "pursuit", "hostage"):
        f = getattr(lib, "madrl_%s_set_obs_format" % fam)
        assert f.argtypes == [C.c_void_p, C.c_int]
        assert f(None, _lib.OBS_BF16) == -1                # MADRL_EINVAL
        assert b"NULL" in lib.madrl_last_error()


@pytest.mark.parametrize("cls", ["BatchedMAWaterWorld", "BatchedHostageWorld", "BatchedPursuitEvade"])
def test_unsupported_obs_dtype_raises_before_the_abi(cls):
    import numpy as np

    import madrl_b200
    args = {"BatchedMAWaterWorld": (4, 5, 5), "BatchedHostageWorld": (4, 10, 16, 16, 4, 2),
            "BatchedPursuitEvade": (4, np.zeros((1, 5, 5), np.int32))}[cls]
    for bad in (torch.float16, torch.float64, torch.int32):
        with pytest.raises(ValueError, match="obs_dtype"):
            getattr(madrl_b200, cls)(*args, obs_dtype=bad)
    if cls != "BatchedPursuitEvade":   # bfloat16 observations need float32 rewards
        with pytest.raises(ValueError, match="obs_dtype"):
            getattr(madrl_b200, cls)(*args, dtype=torch.float64, obs_dtype=torch.bfloat16)


def test_packed_trajectory_obs_section_takes_obs_dtype():
    from madrl_b200.dist import PackedTrajectory
    a = PackedTrajectory(3, 4, 5, 2, "cpu", obs_dim=7)
    b = PackedTrajectory(3, 4, 5, 2, "cpu", obs_dim=7, obs_dtype=torch.bfloat16)
    assert a.obs.dtype == torch.float32 and b.obs.dtype == torch.bfloat16
    assert a.obs.shape == b.obs.shape == (3, 4, 5, 7) and b.nbytes < a.nbytes


def test_library_exports_the_bf16_postproc_passes():
    from madrl_b200 import _lib
    lib = _lib.lib()
    for name in ("frame_stack_bf16", "standardize_bf16", "standardize_obs_terminal_bf16", "paths_pack_u16"):
        assert hasattr(lib, "madrl_" + name), name
    assert lib.madrl_frame_stack_bf16(1, 1, 1, 1, 9, None, None, None, None, None) == -1   # buffer_size > 8
    assert lib.madrl_standardize_bf16(1, 1, None, None, None, 0.1, 1e-8, 1, 1.0, 1, None) == -1
    assert lib.madrl_paths_pack_u16(1, 1, 1, 1, None, None, None, None, None, None) == -1


def test_postproc_wrappers_reject_unsupported_dtypes():
    """A wrong dtype never reaches a raw-buffer pass (a 2-byte buffer read as 4-byte floats would run off
    its end): every wrapper checks before the ABI is called."""
    from madrl_b200 import postproc as P
    T, E, A, D = 2, 3, 2, 5
    done = torch.zeros((T, E), dtype=torch.uint8)
    fs = P.FrameStack(E, A, D, 3, "cpu")
    for bad in (torch.bfloat16, torch.float16, torch.float64):
        with pytest.raises(TypeError):
            fs.rollout(torch.zeros((T, E, A, D), dtype=bad), done)
        with pytest.raises(TypeError):
            fs.reset(torch.zeros((E, A, D), dtype=bad))
    fsb = P.FrameStack(E, A, D, 3, "cpu", dtype=torch.bfloat16)
    with pytest.raises(TypeError):
        fsb.rollout(torch.zeros((T, E, A, D)), done)
    st = P.Standardizer(E, A, D, "cpu", enable_obsnorm=True)
    for bad in (torch.float16, torch.float64):
        with pytest.raises(TypeError):
            st.obs(torch.zeros((T, E, A, D), dtype=bad))
    with pytest.raises(TypeError):   # terminal observations must have the observations' dtype
        st.obs(torch.zeros((T, E, A, D), dtype=torch.bfloat16), done, torch.zeros((T, E, A, D)))
    with pytest.raises(TypeError):
        st.rew(torch.zeros((T, E, A), dtype=torch.bfloat16))
    with pytest.raises(TypeError):
        P.pack_paths(torch.zeros((T, E, A, D), dtype=torch.float16), torch.zeros((T, E, A, 2)),
                     torch.zeros((T, E, A)), done)
    for fn, args in ((P.gae, (torch.zeros((T, E, A), dtype=torch.bfloat16), torch.zeros((T, E, A)), done, 0.99, 0.95)),
                     (P.center_advantages, (torch.zeros(8, dtype=torch.bfloat16),)),
                     (P.moments, (torch.zeros(8, dtype=torch.float64),))):
        with pytest.raises(TypeError):
            fn(*args)
    with pytest.raises(TypeError):
        P.EpisodeStats(E, A, "cpu").rollout(torch.zeros((T, E, A), dtype=torch.bfloat16), done)
