"""Autoreset modes without a GPU: the new exports and their ctypes signatures, the null-handle refusals, and MegaverseEnv's argument checks
(which run before any engine is created)."""
import ctypes as C

import pytest


def test_exports_and_signatures(built):
    from megaverse_b200 import capi

    new = ["mv_awaiting_reset_host", "mv_awaiting_reset_device"]
    assert set(new) <= set(capi.EXPORTS)
    for name in new:
        fn = getattr(capi.lib(), name)
        assert fn.argtypes == [C.c_void_p, C.POINTER(C.c_void_p)]
    assert callable(capi.Engine.awaiting_reset)
    assert (capi.AUTORESET_SAME_STEP, capi.AUTORESET_NEXT_STEP, capi.AUTORESET_DISABLED) == (0, 1, 2)
    from megaverse_b200.extension import megaverse

    assert hasattr(megaverse.MegaverseGym, "get_awaiting_reset")


def test_null_handle(built):
    from megaverse_b200 import capi

    L = capi.lib()
    p = C.c_void_p()
    assert L.mv_awaiting_reset_host(None, C.byref(p)) == capi.MV_ERR_ARG
    assert L.mv_awaiting_reset_device(None, C.byref(p)) == capi.MV_ERR_ARG
    assert L.mv_awaiting_reset_host(None, None) == capi.MV_ERR_ARG
    assert L.mv_awaiting_reset_device(None, None) == capi.MV_ERR_ARG


def test_env_argument_checks(built):
    from megaverse_b200.megaverse_env import MegaverseEnv

    assert MegaverseEnv.AUTORESET_MODES == ("same_step", "next_step", "disabled")
    for bad in ("next", "NEXT_STEP", 1, None, ""):
        with pytest.raises(ValueError, match="autoreset_mode"):
            MegaverseEnv("TowerBuilding", 2, 1, 1, autoreset_mode=bad)
    for mode in ("next_step", "disabled"):
        with pytest.raises(ValueError, match="final_observation"):
            MegaverseEnv("TowerBuilding", 2, 1, 1, final_observation=True, autoreset_mode=mode)
