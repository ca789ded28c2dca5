"""The agent warp test hook without a GPU: mv_debug_warp_agent refuses a null handle whatever else it is given, and the Python surface
exists.  Its refusals on a live engine (bad env or agent, null pointers, non-finite values, call order) are in test_events_gpu.py."""
import ctypes as C
import inspect


def test_warp_hook_refuses_a_null_handle(built):
    from megaverse_b200 import capi

    L = capi.lib()
    pos, basis = (C.c_float * 3)(1, 2, 3), (C.c_float * 9)(1, 0, 0, 0, 1, 0, 0, 0, 1)
    for env, agent in ((0, 0), (-1, 0), (0, -1), (1 << 20, 0), (0, 8)):
        assert L.mv_debug_warp_agent(None, env, agent, pos, basis) == capi.MV_ERR_ARG
    assert L.mv_debug_warp_agent(None, 0, 0, None, None) == capi.MV_ERR_ARG


def test_warp_hook_is_exported(built):
    from megaverse_b200 import capi

    assert "mv_debug_warp_agent" in capi.EXPORTS
    assert hasattr(C.CDLL(capi.LIB_PATH), "mv_debug_warp_agent")
    assert list(inspect.signature(capi.Engine.warp_agent).parameters) == ["self", "env", "agent", "pos", "basis"]
