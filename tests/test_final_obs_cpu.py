"""Terminal frames and end reasons without a GPU: every new entry point refuses a null handle, and the Python surfaces exist with the reference's
positional signature of MegaverseEnv unchanged."""
import ctypes as C
import inspect

NEW = ["mv_done_reasons", "mv_done_reasons_device", "mv_true_objectives_device", "mv_final_obs_host", "mv_final_depth_host", "mv_final_obs_device",
       "mv_final_depth_device", "mv_last_final_ms"]


def test_final_obs_calls_refuse_a_null_handle(built):
    from megaverse_b200 import capi

    L = capi.lib()
    p = C.c_void_p()
    for name in NEW:
        if name == "mv_last_final_ms":
            assert L.mv_last_final_ms(None, C.byref(C.c_float())) == capi.MV_ERR_ARG
        else:
            assert getattr(L, name)(None, C.byref(p)) == capi.MV_ERR_ARG, name
    assert L.mv_set_option(None, b"final_obs", 1) == capi.MV_ERR_ARG


def test_final_obs_exports_and_signatures(built):
    from megaverse_b200 import capi
    from megaverse_b200.extension.megaverse import MegaverseGym
    from megaverse_b200.megaverse_env import MegaverseEnv

    assert set(NEW) <= set(capi.EXPORTS)
    assert (capi.MV_END_NONE, capi.MV_END_TIME, capi.MV_END_SOLVED, capi.MV_END_REQUESTED) == (0, 1, 2, 3)
    for name in ("done_reasons", "final_obs", "final_depth", "last_final_ms"):
        assert list(inspect.signature(getattr(capi.Engine, name)).parameters) == ["self"], name
    assert "final_obs" in capi.Engine.device_array.__doc__ and "done_reasons" in capi.Engine.device_array.__doc__
    assert "true_objectives" in capi.Engine.device_array.__doc__
    assert "solved" in MegaverseGym.get_done_reasons.__doc__ and "final_obs" in MegaverseGym.get_final_observations.__doc__
    params = inspect.signature(MegaverseEnv.__init__).parameters
    positional = [n for n, p in params.items() if p.kind == p.POSITIONAL_OR_KEYWORD]
    assert positional == ["self", "scenario_name", "num_envs", "num_agents_per_env", "num_simulation_threads", "use_vulkan", "params"]
    assert params["final_observation"].kind == inspect.Parameter.KEYWORD_ONLY and params["final_observation"].default is False

