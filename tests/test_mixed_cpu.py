"""Mixed-scenario engine (mv_create_mixed) without a GPU: argument errors are reported before any CUDA call, with the env they concern,
and a valid list fails loudly when there is no device."""
import ctypes as C

import pytest


def _create_mixed(names, E=None, A=1, w=128, h=72, params=None):
    """raw call: names may hold None (a null entry) or be None itself (a null list); returns (code, message)"""
    from megaverse_b200 import capi

    L = capi.lib()
    params = params or {}
    keys = (C.c_char_p * max(1, len(params)))(*[k.encode() for k in params])
    vals = (C.c_float * max(1, len(params)))(*[float(v) for v in params.values()])
    arr = None if names is None else (C.c_char_p * max(1, len(names)))(*[None if n is None else n.encode() for n in names])
    E = len(names) if E is None else E
    out = C.c_void_p()
    rc = L.mv_create_mixed(arr, w, h, E, A, 1, 0, keys, vals, len(params), C.byref(out))
    assert not out.value
    return rc, (L.mv_last_error(None) or b"").decode()


def test_mixed_argument_errors(built):
    from megaverse_b200 import capi

    good = ["TowerBuilding", "Collect", "ObstaclesHard"]
    for names, kwargs, needle in (
        (None, {"E": 3}, "null scenario list"),
        (["Collect", "Sokoban", "NoSuchScenario", "Empty"], {}, "unknown scenario NoSuchScenario for env 2"),
        (["Collect", None], {}, "unknown scenario (null) for env 1"),
        (good, {"E": 0}, "num_envs"),
        (good, {"A": 0}, "num_agents_per_env"),
        (good, {"A": 99}, "num_agents_per_env"),
        (good, {"w": 100}, "render size"),
        (good, {"h": 70}, "render size"),
        (good, {"params": {"useUIRewardIndicators": 1.0}}, "useUIRewardIndicators"),
    ):
        rc, msg = _create_mixed(names, **kwargs)
        assert rc == capi.MV_ERR_ARG, (names, kwargs, rc, msg)
        assert needle in msg, (names, kwargs, msg)


def test_engine_accepts_a_list_and_needs_a_device(built):
    import torch
    from megaverse_b200 import capi

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    with pytest.raises(capi.MegaverseError) as ei:
        capi.Engine(["TowerBuilding", "Collect", "obstacleshard", "Test"], 4, 1)
    assert ei.value.code == capi.MV_ERR_CUDA
    with pytest.raises(capi.MegaverseError) as ei:
        capi.Engine(["TowerBuilding", "Collect"], 3, 1)  # one name per env
    assert ei.value.code == capi.MV_ERR_ARG
    with pytest.raises(capi.MegaverseError) as ei:
        capi.Engine(["TowerBuilding", "Nope"], 2, 1)
    assert ei.value.code == capi.MV_ERR_ARG and "for env 1" in str(ei.value)
