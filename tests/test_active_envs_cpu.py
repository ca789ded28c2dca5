"""Steps with an active set without a GPU: mv_step_envs and mv_step_device_active refuse a null handle, and the Python surfaces exist."""
import ctypes as C
import inspect


def test_active_set_calls_refuse_a_null_handle(built):
    from megaverse_b200 import capi

    L = capi.lib()
    envs = (C.c_int32 * 2)(0, 1)
    assert L.mv_step_envs(None, envs, 2) == capi.MV_ERR_ARG
    assert L.mv_step_envs(None, None, 0) == capi.MV_ERR_ARG
    assert L.mv_step_device_active(None, None, None, None) == capi.MV_ERR_ARG


def test_active_set_signatures(built):
    from megaverse_b200 import capi
    from megaverse_b200.extension.megaverse import MegaverseGym
    from megaverse_b200.megaverse_env import MegaverseEnv

    assert {"mv_step_envs", "mv_step_device_active"} <= set(capi.EXPORTS)
    assert list(inspect.signature(capi.Engine.step_envs).parameters) == ["self", "masks", "envs"]
    assert list(inspect.signature(capi.Engine.step_device_active).parameters) == ["self", "d_masks_ptr", "d_ends_ptr", "d_active_ptr"]
    assert "envs" in MegaverseGym.step_envs.__doc__
    assert list(inspect.signature(MegaverseEnv.step_envs).parameters) == ["self", "envs", "actions"]
    # the full calls keep their parameters
    assert list(inspect.signature(capi.Engine.step_device).parameters) == ["self", "d_masks_ptr", "d_ends_ptr"]
    assert list(inspect.signature(MegaverseEnv.step).parameters) == ["self", "actions"]
