"""Per-env episode control without a GPU: mv_reset_envs and mv_step_device_ends refuse a null handle, and the Python surfaces exist."""
import ctypes as C
import inspect


def test_episode_control_calls_refuse_a_null_handle(built):
    from megaverse_b200 import capi

    L = capi.lib()
    envs, seeds = (C.c_int32 * 1)(0), (C.c_int32 * 1)(7)
    assert L.mv_reset_envs(None, envs, seeds, 1) == capi.MV_ERR_ARG
    assert L.mv_reset_envs(None, envs, None, 1) == capi.MV_ERR_ARG
    assert L.mv_reset_envs(None, None, None, 0) == capi.MV_ERR_ARG
    assert L.mv_step_device_ends(None, None, None) == capi.MV_ERR_ARG


def test_episode_control_signatures(built):
    from megaverse_b200 import capi
    from megaverse_b200.extension.megaverse import MegaverseGym
    from megaverse_b200.megaverse_env import MegaverseEnv

    assert {"mv_reset_envs", "mv_step_device_ends"} <= set(capi.EXPORTS)
    assert list(inspect.signature(capi.Engine.reset_envs).parameters) == ["self", "envs", "seeds"]
    assert inspect.signature(capi.Engine.reset_envs).parameters["seeds"].default is None
    params = inspect.signature(capi.Engine.step_device).parameters
    assert list(params) == ["self", "d_masks_ptr", "d_ends_ptr"] and params["d_ends_ptr"].default is None
    assert "envs" in MegaverseGym.reset_envs.__doc__ and "seeds" in MegaverseGym.reset_envs.__doc__
    assert list(inspect.signature(MegaverseEnv.reset_envs).parameters) == ["self", "envs", "seeds"]
