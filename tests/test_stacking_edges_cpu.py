"""The stacking scenes on the oracle alone: every script reaches the branch it is built for, and the invariant that lets the step kernel
find an object outside its dense voxel grid holds for every level the generator makes.

The scripts assert their reach clauses as they go (landing voxels, refusals, stack heights; stacking_scenes.py); here each scene must
also have met every clause it is named for.  The step kernel looks up a voxel outside the grid by scanning the env's resting objects
for the one whose translation floors to it, so every object must rest at its voxel + 0.5: a put-down places it there, and the levels
start it there, which the second test checks over many levels per scenario."""
import numpy as np
import pytest

import stacking_scenes as ss

# the reach clauses each scene must meet
REACHED = {
    "void_columns_obstacles": {"void_outside", "column_inside"},
    "void_columns_obstacles_a2": {"void_outside", "column_inside"},
    "void_columns_collect": {"void_outside", "column_inside"},
    "void_stack_obstacles": {"void_stack"},
    "void_stack_collect": {"void_stack"},
    "void_pickup_collect": {"void_stack", "void_pickup", "void_pickup_blocked"},
    "above_top_tower": {"from_above", "top_row_pickup", "past_headroom", "past_headroom_pickup"},
    "above_top_collect": {"from_above"},
    "above_top_obstacles": {"from_above"},
    "above_top_rearrange": {"from_above"},
    "zone_edges_and_pickup_height_tower": {"zone_accepted", "zone_refused", "zone_pickup", "pickup_height_1", "pickup_height_2", "pickup_height_3"},
    "pedestal_edges_rearrange": {"pedestal_accepted", "pedestal_refused"},
    "pickup_height_collect": {"pickup_height_1", "pickup_height_2", "pickup_height_3"},
    "agent_in_target_collect": {"agent_refused", "agent_beside_accepted"},
    "agent_in_target_obstacles": {"agent_refused", "agent_beside_accepted"},
}


def test_every_scene_is_listed():
    assert set(REACHED) == set(ss.SCENES)


@pytest.mark.parametrize("name", sorted(ss.SCENES))
def test_scene_reaches_its_branches(built, name):
    ctxs, ticks = ss.run_scene(name, ss.OracleRun)
    reached = {w for c in ctxs for w, _ in c.log}
    assert REACHED[name] <= reached, "%s: never reached %s" % (name, REACHED[name] - reached)
    log = [x for c in ctxs for x in c.log]
    if name.startswith("void_columns"):
        fam = ss.family(ss.SCENES[name][0])
        outside = [v for w, v in log if w == "void_outside"]
        assert len(outside) == 4 * 2, "two distances past the grid on each of the four faces: %s" % outside  # margin + 1 and 30
        assert len([v for w, v in log if w == "column_inside"]) == 4 * len({0, 1, ss.MARGIN[fam]})
    if name.startswith("void_stack"):
        k = 10 if "collect" in name else 4
        for w, hs in log:
            assert hs == list(range(ss.VOID_Y, ss.VOID_Y + k)) + [ss.VOID_Y]
    if name == "zone_edges_and_pickup_height_tower":
        refused = [v for w, v in log if w == "zone_refused"]
        assert len(refused) == 4 * 2 and len([v for w, v in log if w == "zone_accepted"]) == 4 * 2
    if name == "pedestal_edges_rearrange":
        acc = {v for w, v in log if w == "pedestal_accepted"}
        ref = {v for w, v in log if w == "pedestal_refused"}
        assert {(2, 0), (-2, 0), (0, 2), (0, -2), (2, 2)} <= acc and {(3, 0), (-3, 0), (0, 3), (0, -3), (-2, 3)} <= ref


def test_above_top_scene_says_where_a_column_past_the_headroom_is_built():
    """only TowerBuilding levels hold enough objects for a column from the floor past its 18 cells of head-room (about 24 objects);
    Collect's, Obstacles' and Rearrange's scenes put down from above the top face only"""
    assert ss.SCENES["above_top_tower"][5] >= 24
    assert all(ss.SCENES["above_top_%s" % f][5] == 1 for f in ("collect", "obstacles", "rearrange"))


@pytest.mark.parametrize("scenario", ["TowerBuilding", "ObstaclesEasy", "ObstaclesHard", "ObstaclesWalls", "Collect", "Rearrange"])
def test_initial_objects_rest_in_the_voxel_they_are_recorded_under(built, scenario):
    """over 1 024 levels: every object's starting translation floors to the voxel the level lists it under, so that a scan of the
    resting objects by translation finds exactly what the reference's voxel map holds"""
    import orc

    E, rounds = 256, 4
    o = orc.Oracle(scenario, E, 1, render=False, threads=4)
    n = 0
    try:
        for r in range(rounds):
            for e in range(E):
                o.seed_env(e, 1000 + r * E + e)
            o.reset()
            for e in range(E):
                L, st = o.level(e), o.state(e)
                k = int(L[2])
                at = 9 + 8 * int(L[0]) + 7 * int(L[1])
                voxels = L[at: at + 3 * k].reshape(k, 3)
                objs = st[8 + ss.AG: 8 + ss.AG + 9 * k].reshape(k, 9)
                assert np.array_equal(np.floor(objs[:, :3]).astype(np.int32), voxels), "%s level %d" % (scenario, r * E + e)
                assert np.all(objs[:, :3] - voxels == 0.5) and np.all(objs[:, 6] < 0)
                n += k
    finally:
        o.close()
    assert n > 0
