"""State tensors (option "state_tensors") without a GPU: every new entry point refuses a null handle, the Python surfaces exist with the
reference's positional signature of MegaverseEnv unchanged, and the helper that builds expected rows from the oracle's dumps holds its
invariants on the oracle alone, for every scenario name, through carried objects and collected rewards."""
import ctypes as C
import inspect

import numpy as np
import pytest

import helpers
import state_rows

NEW = ["mv_state_tensors_host", "mv_state_tensors_device", "mv_final_state_tensors_host", "mv_final_state_tensors_device"]
SCENARIOS = ["TowerBuilding", "Collect", "Rearrange", "Sokoban", "HexExplore", "HexMemory", "Empty", "ObstaclesEasy", "ObstaclesMedium",
             "ObstaclesHard", "ObstaclesWalls", "ObstaclesSteps", "ObstaclesLava"]


def test_state_tensor_calls_refuse_a_null_handle(built):
    from megaverse_b200 import capi

    L = capi.lib()
    p = [C.c_void_p() for _ in range(4)]
    for name in NEW:
        assert getattr(L, name)(None, *[C.byref(x) for x in p]) == capi.MV_ERR_ARG, name
        assert getattr(L, name)(None, None, None, None, None) == capi.MV_ERR_ARG, name
    assert L.mv_set_option(None, b"state_tensors", 1) == capi.MV_ERR_ARG


def test_state_tensor_exports_and_signatures(built):
    from megaverse_b200 import capi
    from megaverse_b200.extension.megaverse import MegaverseGym
    from megaverse_b200.megaverse_env import MegaverseEnv

    assert set(NEW) <= set(capi.EXPORTS)
    for name in NEW:
        assert hasattr(capi.lib(), name)
    assert capi.STATE_TENSORS == ("agents", "envs", "objects", "rewards")
    for name in ("state_tensors", "final_state_tensors"):
        assert list(inspect.signature(getattr(capi.Engine, name)).parameters) == ["self"], name
    assert "state_agents" in capi.Engine.device_array.__doc__ and "final_state_agents" in capi.Engine.device_array.__doc__
    assert "state_tensors" in MegaverseGym.get_state_tensors.__doc__ and "final_obs" in MegaverseGym.get_final_state_tensors.__doc__
    params = inspect.signature(MegaverseEnv.__init__).parameters
    positional = [n for n, p in params.items() if p.kind == p.POSITIONAL_OR_KEYWORD]
    assert positional == ["self", "scenario_name", "num_envs", "num_agents_per_env", "num_simulation_threads", "use_vulkan", "params"]
    assert params["state_tensors"].kind == inspect.Parameter.KEYWORD_ONLY and params["state_tensors"].default is False
    assert list(inspect.signature(MegaverseEnv.state_tensors).parameters) == ["self"]


def _check_invariants(tag, name, A, rows, known, sign_only):
    ag, en, ob, rw = rows["agents"], rows["envs"], rows["objects"], rows["rewards"]
    n_obj = int(en[4])
    assert (ob[n_obj:] == 0).all(), tag
    for a in range(A):
        c = int(ag[a, 14])
        if c >= 0:
            assert c < n_obj and int(ob[c, 3]) == a, "%s: agent %d carries %d, whose carrier is %d" % (tag, a, c, int(ob[c, 3]))
    for i in range(n_obj):
        if ob[i, 3] >= 0:
            assert int(ag[int(ob[i, 3]), 14]) == i, "%s: object %d names carrier %d, which does not carry it" % (tag, i, int(ob[i, 3]))
    if known["envs"][5]:
        nr = int(en[5])
        assert (rw[nr:] == 0).all() and known["rewards"][nr:].all(), tag
    assert set(np.unique(rw[:, 3][known["rewards"][:, 3]])) <= {-1.0, 0.0, 1.0}, tag
    assert int(en[3]) == state_rows.scenario_code(name)
    for k in rows:
        assert rows[k].dtype == np.float32 and not np.isnan(rows[k]).any()
        assert not (sign_only[k] & ~known[k]).any()


@pytest.mark.parametrize("name", SCENARIOS)
def test_expected_rows_on_the_oracle(built, name):
    import orc

    A = 2
    E, steps = (4, 300) if name == "Rearrange" else (2, 160)  # the scripted solver needs a while to reach its first object
    o = orc.Oracle(name, E, A, render=False, params={"episodeLengthSec": 4.0} if name not in ("Collect", "Rearrange") else None)
    try:
        o.seed(11)
        o.reset()
        rng = np.random.default_rng(5)
        carried = taken = 0
        for t in range(steps):
            if name == "Rearrange":
                acts = np.concatenate([helpers.rearrange_controller(o, e, A) for e in range(E)])
            else:
                acts = helpers.purposeful_actions(rng, E * A, t)
            o.step(acts)
            for e in range(E):
                rows, known, sign_only = state_rows.expected_rows(name, A, o.state(e), o.level(e))
                tag = "%s step %d env %d" % (name, t, e)
                _check_invariants(tag, name, A, rows, known, sign_only)
                carried += int((rows["agents"][:, 14] >= 0).any())
                n_reward = int(rows["envs"][5]) if known["envs"][5] else 0
                taken += int((rows["rewards"][:n_reward, 3] == 0).any())
        if name == "Rearrange":
            assert carried > 0, "the scripted solver never carried an object"
        if name == "Collect":
            assert taken > 0, "no reward object was collected"
    finally:
        o.close()
