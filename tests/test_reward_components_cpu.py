"""Reward components without a GPU: the key table (mv_reward_component_keys against the restated one), the masked-weight oracle twins
that give the per-slot reference columns, the surfaces and the refusals that need no device."""
import ctypes as C

import numpy as np
import pytest

import helpers
import reward_components as rc


def test_surfaces(built):
    from megaverse_b200 import capi

    new = ["mv_reward_components_host", "mv_reward_components_device", "mv_reward_component_keys"]
    assert set(new) <= set(capi.EXPORTS)
    for name in new:
        assert hasattr(capi.lib(), name)
    assert callable(capi.reward_component_keys) and callable(capi.Engine.reward_components)
    from megaverse_b200.extension import megaverse

    assert hasattr(megaverse.MegaverseGym, "get_reward_components") and hasattr(megaverse.MegaverseGym, "get_episode_reward_components")
    assert callable(megaverse.reward_component_keys)


@pytest.mark.parametrize("scenario", rc.NAMES)
def test_key_table_matches_the_engine(built, scenario):
    from megaverse_b200 import capi
    from megaverse_b200.extension import megaverse

    want = rc.keys8(scenario)
    assert capi.reward_component_keys(scenario) == want
    assert capi.reward_component_keys(scenario.upper()) == want
    assert megaverse.reward_component_keys(scenario) == want
    # every key of the scenario's default shaping has a column, and nothing else does
    shaping_keys = set()
    defaults = (C.c_char * 4096)()
    n = capi.lib().mv_debug_defaults(scenario.encode(), defaults, 4096)
    assert n > 0
    for line in defaults.value.decode().splitlines():
        if line.startswith("R "):
            shaping_keys.add(line[2:].split("=")[0])
    assert set(k for k in want if k) == shaping_keys - {"teamSpirit"}


def test_key_refusals(built):
    from megaverse_b200 import capi

    L = capi.lib()
    out = (C.c_char_p * 8)()
    assert L.mv_reward_component_keys(b"NoSuchScenario", out) == capi.MV_ERR_ARG
    assert L.mv_reward_component_keys(None, out) == capi.MV_ERR_ARG
    assert L.mv_reward_component_keys(b"Collect", None) == capi.MV_ERR_ARG
    with pytest.raises(capi.MegaverseError):
        capi.reward_component_keys("NoSuchScenario")


def test_getters_refuse_a_null_handle(built):
    from megaverse_b200 import capi

    L = capi.lib()
    p, q = C.c_void_p(), C.c_void_p()
    assert L.mv_reward_components_host(None, C.byref(p), C.byref(q)) == capi.MV_ERR_ARG
    assert L.mv_reward_components_device(None, C.byref(p), C.byref(q)) == capi.MV_ERR_ARG


def _run_twins(scenario, A, E, steps, seed, shaping_kind):
    rng = np.random.default_rng(seed)
    params = {"episodeLengthSec": 4.0} if rc.family(scenario) != "sokoban" else {"episodeLengthSec": 6.0}
    shaping = None
    if shaping_kind == "random":
        shaping = [d for _ in range(E) for d in rc.random_shaping(rng, scenario, A)]
    ref = rc.SlotOracles(scenario, E, A, params=params, shaping=shaping)
    try:
        for e in range(E):
            ref.seed_env(e, seed + 31 * e)
        ref.reset()
        paid = 0
        for t in range(steps):
            acts = helpers.purposeful_actions(rng, E * A, t)
            ref.step(acts)
            cols, r = ref.columns(), ref.rewards()
            assert not cols[:, 0].any(), "column 0 paid"
            s = cols.astype(np.float64).sum(axis=1)
            tol = 1e-5 + 1e-6 * np.abs(r.astype(np.float64))
            assert np.all(np.abs(s - r) <= tol), "%s t=%d: columns sum %s, reward %s" % (scenario, t, s, r)
            paid += int(np.count_nonzero(cols))
        return paid
    finally:
        ref.close()


@pytest.mark.parametrize("scenario", ["TowerBuilding", "Collect", "ObstaclesHard", "Sokoban", "Rearrange", "HexExplore", "HexMemory", "Empty"])
@pytest.mark.parametrize("A", [1, 2, 4])
@pytest.mark.parametrize("shaping_kind", ["default", "random"])
def test_columns_sum_to_the_oracle_reward(built, scenario, A, shaping_kind):
    _run_twins(scenario, A, 3, 90, 11 + A, shaping_kind)


def test_twins_see_payments(built):
    """the check above is not vacuous: purposeful walks in Collect and TowerBuilding get paid"""
    assert _run_twins("Collect", 2, 4, 120, 5, "random") > 0
    assert _run_twins("TowerBuilding", 2, 4, 120, 6, "random") > 0


def test_totals_follow_call_order():
    t = rc.Totals(4, 2)
    a = np.full((4, 8), 0.1, dtype=np.float32)
    t.add(a, [0, 0])
    t.add(a, [1, 0])
    want = (np.float32(0.0) + np.float32(0.1)) + np.float32(0.1)
    assert t.episode[0, 0] == want and t.episode[2, 0] == 0.0
    assert not t.run[:2].any() and t.run[2, 0] == want
    t.restart([1])
    assert not t.run.any()
