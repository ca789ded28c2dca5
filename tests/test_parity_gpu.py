"""GPU parity: the CUDA path (through the C ABI) against the CPU oracle on identical seeds and action streams.
Bar (BASELINE.json north_star): rewards / dones / voxel occupancy / kinematic state bit-exact; RGB within +-1 LSB with the fast
fragment stage (fast_shading=1), byte-exact frames and bit-exact depth with fast_shading=0."""
import numpy as np
import pytest

import helpers

pytestmark = pytest.mark.gpu


def _pair(scenario, E, A, seed, w=128, h=72, params=None, depth=False, fast_shading=False):
    import orc
    from megaverse_b200 import capi

    o = orc.Oracle(scenario, E, A, w, h, params=params, depth=depth)
    g = capi.Engine(scenario, E, A, w, h, num_threads=2, params=params, depth=depth)
    # the bit-exact fragment stage for the byte-exact checks; fast_shading=True is the default production mode (+-1 LSB)
    g.set_option("fast_shading", 1 if fast_shading else 0)
    o.seed(seed)
    g.seed(seed)
    o.reset()
    g.reset()
    return o, g


def _assert_same_frame(o, g, tag, fast=False):
    """engines built with fast_shading=0 draw byte-exact frames; the +-1 LSB / 99.9 % rule is for the fast fragment stage only"""
    a, b = o.obs(), np.array(g.obs())
    diff = np.abs(a.astype(np.int16) - b.astype(np.int16))
    if not fast:
        assert np.array_equal(a, b), "%s: frames differ in %d bytes (max diff %d)" % (tag, int((diff > 0).sum()), diff.max())
        return 1.0
    assert diff.max() <= 1, "%s: max RGB diff %d (mismatching pixels %d)" % (tag, diff.max(), int((diff > 1).sum()))
    exact = float((diff == 0).mean())
    assert exact > 0.999, "%s: only %.5f of the bytes exact" % (tag, exact)
    return exact


def _assert_same_depth(o, g, tag):
    a, b = o.depth(), np.array(g.depth())
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), "%s: depth differs in %d pixels" % (tag, int((a != b).sum()))


def _assert_same_state(o, g, E, tag):
    for e in range(E):
        so, sg = o.state(e), g.state(e)
        assert so.shape == sg.shape, tag
        if not np.array_equal(so.view(np.uint32), sg.view(np.uint32)):
            bad = np.nonzero(so.view(np.uint32) != sg.view(np.uint32))[0]
            raise AssertionError("%s env %d: state words differ at %s: oracle %s device %s" % (tag, e, bad[:8], so[bad[:8]], sg[bad[:8]]))


@pytest.mark.parametrize("seed", [42, 7])
def test_tower_reset_parity(built, seed):
    E = 8
    o, g = _pair("TowerBuilding", E, 1, seed)
    for e in range(E):
        assert np.array_equal(o.level(e), g.level(e)), "level %d" % e
        assert np.array_equal(o.voxels(e), g.voxels(e)), "voxels %d" % e
        assert np.array_equal(o.instances(e).view(np.uint32), g.instances(e).view(np.uint32)), "instances %d" % e
        assert np.array_equal(o.view(e, 0).view(np.uint32), g.view(e, 0).view(np.uint32)), "view %d" % e
    _assert_same_state(o, g, E, "reset")
    exact = _assert_same_frame(o, g, "reset")
    assert exact == 1.0, "first frame not byte-exact: %.6f" % exact
    assert g.faults() == 0
    o.close(); g.close()


@pytest.mark.parametrize("policy", ["bits", "heads", "purposeful"])
def test_tower_trajectory_parity(built, policy):
    E, steps = 16, 600
    o, g = _pair("TowerBuilding", E, 1, 1234, depth=True)
    rng = np.random.default_rng(99)
    total_reward = 0.0
    for t in range(steps):
        if policy == "bits":
            acts = helpers.random_bit_actions(rng, E)
        elif policy == "heads":
            acts = helpers.random_head_actions(rng, E)
        else:
            acts = helpers.purposeful_actions(rng, E, t)
        o.step(acts)
        g.step(acts)
        ro, rg = o.rewards(), np.array(g.rewards())
        assert np.array_equal(ro.view(np.uint32), rg.view(np.uint32)), "step %d rewards %s vs %s" % (t, ro, rg)
        assert np.array_equal(o.dones(), np.array(g.dones())), "step %d dones" % t
        total_reward += float(np.abs(ro).sum())
        if t % 25 == 0 or t == steps - 1:
            _assert_same_state(o, g, E, "step %d" % t)
            for e in range(0, E, 5):
                assert np.array_equal(o.voxels(e), g.voxels(e)), "step %d voxels %d" % (t, e)
            _assert_same_frame(o, g, "step %d" % t)
            _assert_same_depth(o, g, "step %d" % t)
    if policy == "purposeful":
        assert total_reward > 0.0, "the purposeful policy should have earned shaping rewards"
    assert g.faults() == 0
    o.close(); g.close()


def test_tower_episode_turnover(built):
    """short episodes: done flags, terminal-reward zeroing, true objective capture, in-kernel reset to the next level"""
    # episodeLengthSec() = base + 4 * #boxes (scenario_tower_building.cpp:263-266) with 4..73 boxes: a negative base makes
    # small levels end on their first step (reset every step) and larger ones after a few hundred steps
    E = 24
    params = {"episodeLengthSec": -41.5}
    o, g = _pair("TowerBuilding", E, 1, 5, params=params)
    rng = np.random.default_rng(3)
    ndone = 0
    for t in range(500):
        acts = helpers.purposeful_actions(rng, E, t)
        o.step(acts)
        g.step(acts)
        d = o.dones()
        assert np.array_equal(d, np.array(g.dones())), "step %d" % t
        assert np.array_equal(o.rewards().view(np.uint32), np.array(g.rewards()).view(np.uint32)), "step %d" % t
        assert np.array_equal(o.true_objectives(), np.array(g.true_objectives())), "step %d" % t
        if d.any():
            ndone += int(d.sum())
            for e in np.nonzero(d)[0]:
                assert np.array_equal(o.level(e), g.level(e)), "step %d level of env %d after reset" % (t, e)
            _assert_same_state(o, g, E, "step %d" % t)
            _assert_same_frame(o, g, "step %d" % t)
    assert ndone >= 3
    assert g.faults() == 0
    o.close(); g.close()


def test_multi_agent_parity(built):
    E, A = 6, 4
    o, g = _pair("TowerBuilding", E, A, 77)
    rng = np.random.default_rng(11)
    _assert_same_state(o, g, E, "reset")
    _assert_same_frame(o, g, "reset")
    for t in range(300):
        acts = helpers.purposeful_actions(rng, E * A, t)
        o.step(acts)
        g.step(acts)
        assert np.array_equal(o.rewards().view(np.uint32), np.array(g.rewards()).view(np.uint32)), "step %d" % t
        if t % 20 == 0:
            _assert_same_state(o, g, E, "step %d" % t)
            _assert_same_frame(o, g, "step %d" % t)
    assert g.faults() == 0
    o.close(); g.close()


def test_config1_64x64(built):
    """BASELINE config 1: TowerBuilding 1 env x 1 agent at 64x64"""
    o, g = _pair("TowerBuilding", 1, 1, 42, w=64, h=64)
    rng = np.random.default_rng(0)
    assert _assert_same_frame(o, g, "reset") == 1.0
    for t in range(100):
        acts = helpers.random_head_actions(rng, 1)
        o.step(acts)
        g.step(acts)
    _assert_same_state(o, g, 1, "end")
    _assert_same_frame(o, g, "end")
    o.close(); g.close()


def test_depth_output(built):
    o, g = _pair("TowerBuilding", 4, 1, 9, depth=True)
    a, b = o.depth(), np.array(g.depth())
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    assert (a > 0).any()
    o.close(); g.close()


def test_seed_determinism(built):
    """megaverse/tests/test_env.py:42-53: two envs seeded alike give identical first observations"""
    from megaverse_b200 import capi

    g1 = capi.Engine("TowerBuilding", 2, 2)
    g2 = capi.Engine("TowerBuilding", 2, 2)
    g1.seed(42); g2.seed(42)
    g1.reset(); g2.reset()
    assert np.array_equal(np.array(g1.obs()), np.array(g2.obs()))
    g1.close(); g2.close()


@pytest.mark.parametrize("scenario,A", [("TowerBuilding", 1), ("ObstaclesHard", 2), ("Collect", 4), ("Rearrange", 2), ("Sokoban", 2), ("HexExplore", 2), ("HexMemory", 2), ("Empty", 3)])
def test_fast_shading_within_one_lsb(built, scenario, A):
    """the production fragment stage (rsqrt.approx + FMA, per-triangle unit normals on flat faces, highlight cut-off) against the oracle
    on every scenario family -- boxes, capsules (other agents), spheres / cones / cylinders (interpolated normals, the pow-300 highlight):
    every channel within +-1 LSB (north-star tolerance for RGB) and at least 99.9 % of the bytes identical; physics / rewards stay
    bit-exact because only the fragment colour arithmetic changes"""
    E = 12
    o, g = _pair(scenario, E, A, 4321, fast_shading=True)
    rng = np.random.default_rng(17)
    worst_exact = 1.0
    for t in range(120):
        acts = helpers.purposeful_actions(rng, E * A, t)
        o.step(acts)
        g.step(acts)
        assert np.array_equal(o.rewards().view(np.uint32), np.array(g.rewards()).view(np.uint32)), "step %d" % t
        if t % 10 == 0:
            a, b = o.obs(), np.array(g.obs())
            diff = np.abs(a.astype(np.int16) - b.astype(np.int16))
            assert diff.max() <= 1, "step %d: max RGB diff %d" % (t, diff.max())
            assert np.array_equal(a[..., 3], b[..., 3])
            worst_exact = min(worst_exact, float((diff == 0).mean()))
    _assert_same_state(o, g, E, "end")
    assert worst_exact > 0.999, worst_exact
    print("fast shading %s: worst exact-byte fraction %.6f" % (scenario, worst_exact))
    o.close(); g.close()


# ------------------------------------------------------------------------------------------------ Obstacles family
@pytest.mark.parametrize("scenario,A", [("ObstaclesHard", 1), ("ObstaclesEasy", 2), ("ObstaclesLava", 1)])
def test_obstacles_reset_parity(built, scenario, A):
    E = 8
    o, g = _pair(scenario, E, A, 11)
    for e in range(E):
        assert np.array_equal(o.level(e), g.level(e)), "level %d" % e
        assert np.array_equal(o.voxels(e), g.voxels(e)), "voxels %d" % e
        assert np.array_equal(o.instances(e).view(np.uint32), g.instances(e).view(np.uint32)), "instances %d" % e
    _assert_same_state(o, g, E, "reset")
    assert _assert_same_frame(o, g, "reset") == 1.0
    assert g.faults() == 0
    o.close(); g.close()


@pytest.mark.parametrize("scenario,A,policy", [("ObstaclesHard", 1, "purposeful"), ("ObstaclesHard", 1, "bits"), ("ObstaclesMedium", 2, "purposeful"), ("Test", 2, "forward")])
def test_obstacles_trajectory_parity(built, scenario, A, policy):
    """BASELINE config 3 scenario (with the float32 depth output): physics incl. steps / gaps / lava teleports, exit + extra
    rewards, doneWithTimer; the Test variant (start + exit platform only) makes agents reach the exit quickly"""
    E, steps = 12, 500
    o, g = _pair(scenario, E, A, 2024, depth=True)
    rng = np.random.default_rng(5)
    total = 0.0
    ndone = 0
    for t in range(steps):
        if policy == "bits":
            acts = helpers.random_bit_actions(rng, E * A)
        elif policy == "forward":
            acts = np.where(rng.random(E * A) < 0.85, 1 << 3, 1 << 5).astype(np.int32)
        else:
            acts = helpers.purposeful_actions(rng, E * A, t)
        o.step(acts)
        g.step(acts)
        ro, rg = o.rewards(), np.array(g.rewards())
        assert np.array_equal(ro.view(np.uint32), rg.view(np.uint32)), "step %d rewards %s vs %s" % (t, ro, rg)
        assert np.array_equal(o.dones(), np.array(g.dones())), "step %d dones" % t
        assert np.array_equal(o.true_objectives(), np.array(g.true_objectives())), "step %d" % t
        total += float(np.abs(ro).sum())
        ndone += int(o.dones().sum())
        if t % 25 == 0 or t == steps - 1 or o.dones().any():
            _assert_same_state(o, g, E, "step %d" % t)
            _assert_same_frame(o, g, "step %d" % t)
            assert np.array_equal(o.depth().view(np.uint32), np.array(g.depth()).view(np.uint32)), "step %d depth" % t
    if policy == "forward":
        assert total > 0 and ndone > 0, "the Test variant should be solved by walking forward (reward %.2f, dones %d)" % (total, ndone)
    assert g.faults() == 0
    o.close(); g.close()


# ------------------------------------------------------------------------------------------------ Collect (BASELINE config 4: 4 agents / env)
def test_collect_reset_parity(built):
    E, A = 6, 4
    o, g = _pair("Collect", E, A, 21)
    for e in range(E):
        assert np.array_equal(o.level(e), g.level(e)), "level %d" % e
        assert np.array_equal(o.voxels(e), g.voxels(e)), "voxels %d" % e
        assert np.array_equal(o.instances(e).view(np.uint32), g.instances(e).view(np.uint32)), "instances %d" % e
    _assert_same_state(o, g, E, "reset")
    assert _assert_same_frame(o, g, "reset") == 1.0
    assert g.faults() == 0
    o.close(); g.close()


@pytest.mark.parametrize("policy", ["purposeful", "heads"])
def test_collect_trajectory_parity(built, policy):
    """multi-agent Perlin landscapes: agent-agent capsule collisions, reward diamonds (+1/-1), falling off the edge
    (teleport + penalty), collectAll + doneWithTimer"""
    E, A, steps = 8, 4, 700
    o, g = _pair("Collect", E, A, 99, depth=True)
    rng = np.random.default_rng(8)
    total, ndone = 0.0, 0
    for t in range(steps):
        acts = helpers.purposeful_actions(rng, E * A, t) if policy == "purposeful" else helpers.random_head_actions(rng, E * A)
        o.step(acts)
        g.step(acts)
        ro, rg = o.rewards(), np.array(g.rewards())
        assert np.array_equal(ro.view(np.uint32), rg.view(np.uint32)), "step %d rewards %s vs %s" % (t, ro, rg)
        assert np.array_equal(o.dones(), np.array(g.dones())), "step %d dones" % t
        assert np.array_equal(o.true_objectives(), np.array(g.true_objectives())), "step %d" % t
        total += float(np.abs(ro).sum()); ndone += int(o.dones().sum())
        if t % 50 == 0 or t == steps - 1 or o.dones().any():
            _assert_same_state(o, g, E, "step %d" % t)
            _assert_same_frame(o, g, "step %d" % t)
            _assert_same_depth(o, g, "step %d" % t)
    if policy == "purposeful":
        assert total > 0.0
    assert g.faults() == 0
    o.close(); g.close()


def test_async_device_loop_matches_oracle(built):
    """mv_step_device (asynchronous, action masks resident in HBM, obs left in HBM, host bookkeeping two steps late):
    after mv_sync the state, the last step's rewards/dones and the device obs tensor equal the oracle's, across episode
    turnovers (in-kernel flip to the pre-staged level while the host regenerates in the background)"""
    import torch

    E, A, steps = 32, 1, 420
    params = {"episodeLengthSec": -33.0}  # base + 4 * #boxes: episodes of a few dozen to a few hundred steps (>= 4 steps each)
    o, g = _pair("TowerBuilding", E, A, 21, params=params)
    rng = np.random.default_rng(5)
    acts = np.stack([helpers.purposeful_actions(rng, E * A, t) for t in range(steps)]).astype(np.int32)
    dacts = torch.from_numpy(acts).cuda()
    torch.cuda.synchronize()
    ndone = 0
    for t in range(steps):
        o.step(acts[t])
        ndone += int(o.dones().sum())
        g.step_device(dacts.data_ptr() + t * E * A * 4)
        if t % 97 == 96:  # mid-run synchronisation points must not disturb the pipeline
            g.sync()
            assert np.array_equal(o.rewards().view(np.uint32), np.array(g.rewards()).view(np.uint32)), "step %d" % t
            assert np.array_equal(o.dones(), np.array(g.dones())), "step %d" % t
    g.sync()
    assert ndone >= 3
    assert g.faults() == 0
    assert np.array_equal(o.rewards().view(np.uint32), np.array(g.rewards()).view(np.uint32))
    assert np.array_equal(o.dones(), np.array(g.dones()))
    assert np.array_equal(o.true_objectives(), np.array(g.true_objectives()))
    _assert_same_state(o, g, E, "after %d async steps" % steps)
    g.fetch_obs()  # device obs tensor -> host buffer on demand
    assert _assert_same_frame(o, g, "after %d async steps" % steps) == 1.0
    g.step(acts[0])  # the synchronous call drains the pipeline and carries on from the same state
    o.step(acts[0])
    _assert_same_state(o, g, E, "sync step after async")
    assert _assert_same_frame(o, g, "sync step after async") == 1.0
    o.close(); g.close()


@pytest.mark.parametrize("zero_copy", [1, 0])
def test_split_host_step_matches_oracle(built, zero_copy):
    """mv_step_begin / mv_step_end (the double-buffered consumer's call pair): two engines holding the two halves of the env range
    step alternately -- begin on one while the other's result is read -- and every delivered frame / reward / done equals the
    oracle's, across episode turnovers; the protocol errors are MV_ERR_STATE"""
    import orc
    from megaverse_b200 import capi

    E, A, steps = 16, 2, 200
    params = {"episodeLengthSec": -2.0}  # Collect: base + 2 * #rewards -> staggered turnovers from tick 29 on
    half = E // 2
    gs = []
    for k in range(2):
        e = capi.Engine("Collect", half, A, 128, 72, num_threads=2, params=params)
        e.set_option("fast_shading", 0)
        e.set_option("zero_copy", zero_copy)
        gs.append(e)
    o = orc.Oracle("Collect", E, A, params=params)
    for e in range(E):  # Env::seed per env, the same value on both sides
        o.seed_env(e, 1000 + e)
        gs[e // half].seed_env(e % half, 1000 + e)
    o.reset()
    for e in gs:
        e.reset()
    rng = np.random.default_rng(9)
    with pytest.raises(capi.MegaverseError):
        gs[0].step_end()  # nothing outstanding
    ndone = 0
    acts = helpers.purposeful_actions(rng, E * A, 0)
    for k in range(2):
        gs[k].step_begin(acts[k * half * A:(k + 1) * half * A])
    with pytest.raises(capi.MegaverseError):
        gs[0].step_begin(acts[:half * A])  # already begun
    for t in range(steps):
        o.step(acts)
        ndone += int(o.dones().sum())
        nxt = helpers.purposeful_actions(rng, E * A, t + 1)
        for k in range(2):
            gs[k].step_end()
            sl = slice(k * half * A, (k + 1) * half * A)
            assert np.array_equal(o.rewards()[sl].view(np.uint32), np.array(gs[k].rewards()).view(np.uint32)), "step %d group %d" % (t, k)
            assert np.array_equal(o.dones()[k * half:(k + 1) * half], np.array(gs[k].dones())), "step %d group %d" % (t, k)
            assert np.array_equal(o.obs()[sl], np.array(gs[k].obs())), "frames, step %d group %d" % (t, k)
            if t + 1 < steps:
                gs[k].step_begin(nxt[sl])
        acts = nxt
    assert ndone >= 4
    for e in gs:
        assert e.faults() == 0
        e.close()
    o.close()


@pytest.mark.parametrize("A", [1, 3])
def test_rearrange_reset_parity(built, A):
    """Rearrange: target arrangement (static colliders + sphere / capsule / cylinder / box drawables), its interactive copy,
    pedestals; draw order = the reference's insertion order per mesh type"""
    E = 8
    o, g = _pair("Rearrange", E, A, 5)
    for e in range(E):
        assert np.array_equal(o.level(e), g.level(e)), "level %d" % e
        assert np.array_equal(o.voxels(e), g.voxels(e)), "voxels %d" % e
        assert np.array_equal(o.instances(e).view(np.uint32), g.instances(e).view(np.uint32)), "instances %d" % e
    _assert_same_state(o, g, E, "reset")
    assert _assert_same_frame(o, g, "reset") == 1.0
    assert g.faults() == 0
    o.close(); g.close()


@pytest.mark.parametrize("policy", ["purposeful", "heads"])
def test_rearrange_trajectory_parity(built, policy):
    """pick up / put down arrangement objects (placement only on the work pedestal), matching-count rewards, solved + timer"""
    E, A, steps = 12, 2, 900
    o, g = _pair("Rearrange", E, A, 31, depth=True)
    rng = np.random.default_rng(12)
    total, interactions = 0.0, 0
    for t in range(steps):
        acts = helpers.purposeful_actions(rng, E * A, t) if policy == "purposeful" else helpers.random_head_actions(rng, E * A)
        o.step(acts)
        g.step(acts)
        ro, rg = o.rewards(), np.array(g.rewards())
        assert np.array_equal(ro.view(np.uint32), rg.view(np.uint32)), "step %d rewards %s vs %s" % (t, ro, rg)
        assert np.array_equal(o.dones(), np.array(g.dones())), "step %d dones" % t
        assert np.array_equal(o.true_objectives(), np.array(g.true_objectives())), "step %d" % t
        total += float(np.abs(ro).sum())
        if t % 60 == 0 or t == steps - 1 or o.dones().any():
            _assert_same_state(o, g, E, "step %d" % t)
            for e in range(0, E, 5):
                assert np.array_equal(o.instances(e).view(np.uint32), g.instances(e).view(np.uint32)), "step %d instances %d" % (t, e)
                assert np.array_equal(o.voxels(e), g.voxels(e)), "step %d voxels %d" % (t, e)
            _assert_same_frame(o, g, "step %d" % t)
            _assert_same_depth(o, g, "step %d" % t)
    assert g.faults() == 0
    o.close(); g.close()


def test_rearrange_solved_by_script(built):
    """a scripted agent (driven from the oracle's state) fetches misplaced objects and puts them on their target cells:
    exercises canPlaceObject, the matching count, rearrangeOneMoreObjectCorrectPosition / rearrangeAllObjectsCorrectPosition
    with the team-spirit split, doneWithTimer and the true objective -- identical on both sides"""
    E, A, steps = 8, 2, 420
    o, g = _pair("Rearrange", E, A, 3)
    total, solved = 0.0, 0
    for t in range(steps):
        acts = np.concatenate([helpers.rearrange_controller(o, e, A) for e in range(E)])
        o.step(acts)
        g.step(acts)
        ro, rg = o.rewards(), np.array(g.rewards())
        assert np.array_equal(ro.view(np.uint32), rg.view(np.uint32)), "step %d rewards %s vs %s" % (t, ro, rg)
        assert np.array_equal(o.dones(), np.array(g.dones())), "step %d dones" % t
        assert np.array_equal(o.true_objectives(), np.array(g.true_objectives())), "step %d" % t
        total += float(np.abs(ro).sum())
        if o.dones().any():
            solved += int((o.true_objectives().reshape(E, A)[:, 0] * o.dones()).sum())
        if float(np.abs(ro).sum()) > 0 or o.dones().any() or t % 50 == 0:
            _assert_same_state(o, g, E, "step %d" % t)
            _assert_same_frame(o, g, "step %d" % t)
    assert total >= 5.0 and solved >= 1, (total, solved)
    assert g.faults() == 0
    o.close(); g.close()


@pytest.mark.parametrize("A", [1, 4])
def test_sokoban_reset_parity(built, A):
    """Sokoban (synthetic Boxoban-format rooms): voxel size 2, invisible wall colliders + low wall / goal markers, pushable boxes"""
    E = 8
    o, g = _pair("Sokoban", E, A, 9)
    for e in range(E):
        assert np.array_equal(o.level(e), g.level(e)), "level %d" % e
        assert np.array_equal(o.voxels(e), g.voxels(e)), "voxels %d" % e
        assert np.array_equal(o.instances(e).view(np.uint32), g.instances(e).view(np.uint32)), "instances %d" % e
    _assert_same_state(o, g, E, "reset")
    assert _assert_same_frame(o, g, "reset") == 1.0
    assert g.faults() == 0
    o.close(); g.close()


def test_sokoban_trajectory_parity(built):
    """boxes pushed around (and occasionally onto / off goals: +1 / -1 team rewards), episode turnover at 80 s with the next
    room taken from the env's shuffled level list"""
    E, A, steps = 48, 2, 1260
    o, g = _pair("Sokoban", E, A, 5, depth=True)
    rng = np.random.default_rng(3)
    events, ndone = 0, 0
    for t in range(steps):
        acts = helpers.purposeful_actions(rng, E * A, t)
        o.step(acts)
        g.step(acts)
        ro, rg = o.rewards(), np.array(g.rewards())
        assert np.array_equal(ro.view(np.uint32), rg.view(np.uint32)), "step %d rewards %s vs %s" % (t, ro, rg)
        assert np.array_equal(o.dones(), np.array(g.dones())), "step %d dones" % t
        assert np.array_equal(o.true_objectives(), np.array(g.true_objectives())), "step %d" % t
        events += int(np.abs(ro).sum() > 0); ndone += int(o.dones().sum())
        if t % 100 == 0 or t == steps - 1 or o.dones().any() or np.abs(ro).sum() > 0:
            _assert_same_state(o, g, E, "step %d" % t)
            for e in range(0, E, 7):
                assert np.array_equal(o.voxels(e), g.voxels(e)), "step %d voxels %d" % (t, e)
                assert np.array_equal(o.instances(e).view(np.uint32), g.instances(e).view(np.uint32)), "step %d instances %d" % (t, e)
            _assert_same_frame(o, g, "step %d" % t)
            _assert_same_depth(o, g, "step %d" % t)
    assert events >= 1 and ndone == E
    assert g.faults() == 0
    o.close(); g.close()


@pytest.mark.parametrize("A", [1, 3])
def test_hex_explore_reset_parity(built, A):
    """HexExplore: honeycomb maze (Kruskal), walls as boxes rotated about Y (colliders + drawables), landmark and edging boxes,
    the diamond; hundreds of instances per view"""
    E = 6
    o, g = _pair("HexExplore", E, A, 17)
    for e in range(E):
        assert np.array_equal(o.level(e), g.level(e)), "level %d" % e
        assert np.array_equal(o.instances(e).view(np.uint32), g.instances(e).view(np.uint32)), "instances %d" % e
    _assert_same_state(o, g, E, "reset")
    assert _assert_same_frame(o, g, "reset") == 1.0
    assert g.faults() == 0
    o.close(); g.close()


@pytest.mark.parametrize("policy", ["purposeful", "bits"])
def test_hex_explore_trajectory_parity(built, policy):
    """agents sliding along rotated walls (capsule vs oriented box sweeps / recoveries), finding the diamond: exploreSolved,
    timer, the diamond moved away"""
    E, A, steps = 24, 2, 930
    o, g = _pair("HexExplore", E, A, 23, depth=True)
    rng = np.random.default_rng(4)
    total, ndone = 0.0, 0
    for t in range(steps):
        acts = helpers.purposeful_actions(rng, E * A, t) if policy == "purposeful" else helpers.random_bit_actions(rng, E * A)
        o.step(acts)
        g.step(acts)
        ro, rg = o.rewards(), np.array(g.rewards())
        assert np.array_equal(ro.view(np.uint32), rg.view(np.uint32)), "step %d rewards %s vs %s" % (t, ro, rg)
        assert np.array_equal(o.dones(), np.array(g.dones())), "step %d dones" % t
        assert np.array_equal(o.true_objectives(), np.array(g.true_objectives())), "step %d" % t
        total += float(np.abs(ro).sum()); ndone += int(o.dones().sum())
        if t % 40 == 0 or t == steps - 1 or o.dones().any() or np.abs(ro).sum() > 0:
            _assert_same_state(o, g, E, "step %d" % t)
            _assert_same_frame(o, g, "step %d" % t)
            _assert_same_depth(o, g, "step %d" % t)
    if policy == "purposeful":
        assert total > 0.0
    assert ndone >= E
    assert g.faults() == 0
    o.close(); g.close()


@pytest.mark.parametrize("A", [1, 4])
def test_hex_memory_reset_parity(built, A):
    """HexMemory: landmark object in the central cell, good / bad collectables (pillars = cylinder + two re-parented caps,
    diamonds = two cones, spheres), agents on a circle with evenly spaced headings"""
    E = 6
    o, g = _pair("HexMemory", E, A, 29)
    for e in range(E):
        assert np.array_equal(o.level(e), g.level(e)), "level %d" % e
        assert np.array_equal(o.instances(e).view(np.uint32), g.instances(e).view(np.uint32)), "instances %d" % e
    _assert_same_state(o, g, E, "reset")
    assert _assert_same_frame(o, g, "reset") == 1.0
    assert g.faults() == 0
    o.close(); g.close()


@pytest.mark.parametrize("policy", ["purposeful", "bits"])
def test_hex_memory_trajectory_parity(built, policy):
    """collecting good (+1) and bad (-1) objects within the collect radius, all-good-collected -> solved + timer, objects moved
    away; episode length grows with the number of good objects"""
    E, A, steps = 16, 2, 1000
    o, g = _pair("HexMemory", E, A, 41, depth=True)
    rng = np.random.default_rng(6)
    total, ndone = 0.0, 0
    for t in range(steps):
        acts = helpers.purposeful_actions(rng, E * A, t) if policy == "purposeful" else helpers.random_bit_actions(rng, E * A)
        o.step(acts)
        g.step(acts)
        ro, rg = o.rewards(), np.array(g.rewards())
        assert np.array_equal(ro.view(np.uint32), rg.view(np.uint32)), "step %d rewards %s vs %s" % (t, ro, rg)
        assert np.array_equal(o.dones(), np.array(g.dones())), "step %d dones" % t
        assert np.array_equal(o.true_objectives(), np.array(g.true_objectives())), "step %d" % t
        total += float(np.abs(ro).sum()); ndone += int(o.dones().sum())
        if t % 50 == 0 or t == steps - 1 or o.dones().any() or np.abs(ro).sum() > 0:
            _assert_same_state(o, g, E, "step %d" % t)
            for e in range(0, E, 5):
                assert np.array_equal(o.instances(e).view(np.uint32), g.instances(e).view(np.uint32)), "step %d instances %d" % (t, e)
            _assert_same_frame(o, g, "step %d" % t)
            _assert_same_depth(o, g, "step %d" % t)
    assert total > 0.0
    assert g.faults() == 0
    o.close(); g.close()


def test_hires_render_matches_oracle(built):
    """draw_hires (megaverse.cpp:154-177): the same state rendered at 768x432 equals an oracle that renders at 768x432"""
    import orc
    from megaverse_b200 import capi

    E, A = 3, 2
    o = orc.Oracle("ObstaclesHard", E, A, 768, 432)
    g = capi.Engine("ObstaclesHard", E, A, 128, 72, num_threads=2)
    g.set_option("fast_shading", 0)
    o.seed(11); g.seed(11); o.reset(); g.reset()
    rng = np.random.default_rng(2)
    for t in range(40):
        acts = helpers.purposeful_actions(rng, E * A, t)
        o.step(acts); g.step(acts)
    hi = np.array(g.draw_hires(768, 432))
    assert hi.shape == (E * A, 432, 768, 4)
    assert np.array_equal(hi, o.obs()), "hi-res frame differs: %d pixels" % int((hi != o.obs()).any(axis=-1).sum())
    lo = np.array(g.obs())  # the training-resolution pass is undisturbed
    g.step(np.zeros(E * A, dtype=np.int32)); o.step(np.zeros(E * A, dtype=np.int32))
    assert np.array(g.obs()).shape == lo.shape and g.faults() == 0
    _assert_same_state(o, g, E, "after hires")
    o.close(); g.close()


def test_device_tensor_interface(built):
    """the obs tensor through the CUDA array interface (what a GPU learner consumes, SURVEY.md 8f rank 1): zero-copy, equals the
    host copy of the same step"""
    import torch
    from megaverse_b200 import capi

    g = capi.Engine("Collect", 4, 2, 128, 72, num_threads=2)
    g.seed(3); g.reset()
    g.step(np.full(8, 1 << 3, dtype=np.int32))
    # the default delivery is zero-copy stores into the host buffer: the HBM tensor is stale and the engine says so
    with pytest.raises(capi.MegaverseError):
        g.device_array("obs")
    host = np.array(g.obs()).copy()
    g.fetch_obs()  # must not overwrite the (newer) host copy with the stale HBM tensor
    assert np.array_equal(host, np.array(g.obs()))
    g.set_option("zero_copy", 0)  # make the kernel write HBM and copy down, so both copies exist
    g.step(np.full(8, 1 << 3, dtype=np.int32))
    t = torch.as_tensor(g.device_array("obs"), device="cuda")
    assert t.shape == (8, 72, 128, 4) and t.dtype == torch.uint8 and t.data_ptr() == g.device_ptr("obs")
    torch.cuda.synchronize()
    assert np.array_equal(t.cpu().numpy(), np.array(g.obs()))
    r = torch.as_tensor(g.device_array("rewards"), device="cuda")
    assert np.array_equal(r.cpu().numpy(), np.array(g.rewards()))
    g.close()


@pytest.mark.parametrize("scenario,A,w,h", [("Collect", 8, 64, 64), ("Rearrange", 8, 160, 96), ("HexMemory", 8, 64, 64), ("Sokoban", 8, 128, 72)])
def test_many_agents_other_resolutions(built, scenario, A, w, h):
    """eight agents per env (the engine's maximum) and non-default render sizes: agent-agent capsule contacts, eight views per env"""
    E, steps = 3, 160
    o, g = _pair(scenario, E, A, 13, w=w, h=h)
    rng = np.random.default_rng(9)
    _assert_same_state(o, g, E, "reset")
    assert _assert_same_frame(o, g, "reset") == 1.0
    for t in range(steps):
        acts = helpers.purposeful_actions(rng, E * A, t)
        o.step(acts)
        g.step(acts)
        assert np.array_equal(o.rewards().view(np.uint32), np.array(g.rewards()).view(np.uint32)), "step %d" % t
        assert np.array_equal(o.dones(), np.array(g.dones())), "step %d" % t
    _assert_same_state(o, g, E, "end")
    assert _assert_same_frame(o, g, "end") == 1.0
    assert g.faults() == 0
    o.close(); g.close()


@pytest.mark.parametrize("scenario,A", [("TowerBuilding", 2), ("HexExplore", 2), ("HexMemory", 1), ("Collect", 4), ("ObstaclesHard", 1), ("Rearrange", 2)])
def test_raster_partitioning_keeps_frames_identical(built, scenario, A):
    """how the rasteriser splits its work must not change a single byte: a triangle list of 32 entries per CTA (every view is drawn in many
    batches through the spill slab, repainting pixels that later batches win), the default list, views cut into 1, 2 or 3 row bands, the
    cost-ordered work queue, a raster grid of three or five CTAs -- engines on the same seeds and actions, frames and depth compared every step; each against the oracle at the end"""
    import orc
    from megaverse_b200 import capi

    E, steps = 6, 90
    gs = []
    for tri_cap, bands, sched, grid in ((32, 1, 0, 0), (0, 3, 2, 0), (200, 2, 2, 5), (0, 1, 0, 0), (0, 1, 2, 3)):
        g = capi.Engine(scenario, E, A, 128, 72, num_threads=2, depth=True)
        g.set_option("fast_shading", 0)
        if tri_cap:
            g.set_option("tri_cap", tri_cap)
        g.set_option("raster_bands", bands)
        g.set_option("raster_sched", sched)  # 2: the cost-ordered work queue even at this small size
        g.set_option("raster_grid", grid)    # a handful of CTAs: every CTA draws many work items
        g.seed(77)
        g.reset()
        gs.append(g)
    o = orc.Oracle(scenario, E, A, 128, 72, depth=True)
    o.seed(77)
    o.reset()
    rng = np.random.default_rng(2)
    for g in gs[1:]:
        assert np.array_equal(np.array(gs[0].obs()), np.array(g.obs())), "first frame"
    for t in range(steps):
        acts = helpers.purposeful_actions(rng, E * A, t)
        for g in gs:
            g.step(acts)
        o.step(acts)
        for i, g in enumerate(gs[1:]):
            assert np.array_equal(np.array(gs[0].obs()), np.array(g.obs())), "frames of configuration %d differ at step %d" % (i + 1, t)
            assert np.array_equal(np.array(gs[0].depth()), np.array(g.depth())), "depth of configuration %d differs at step %d" % (i + 1, t)
    for i, g in enumerate(gs):
        assert np.array_equal(o.obs(), np.array(g.obs())), "configuration %d vs oracle" % i
        assert np.array_equal(o.depth().view(np.uint32), np.array(g.depth()).view(np.uint32)), "configuration %d vs oracle (depth)" % i
        assert g.faults() == 0
        g.close()
    o.close()


def test_cost_ordered_work_queue_keeps_frames_identical(built):
    """the persistent raster grid draws the envs in the order of what their views cost in the previous step, most expensive first (option
    raster_sched, default for launches with several views per CTA; the step kernel steps the envs in the same order).  The order in which
    views are drawn must not change a byte: 700 Collect envs x 2 agents (1400 views on 296 CTAs), cost-ordered vs natural order, frames
    compared every few steps; no view is drawn twice or skipped (a sentinel written into the obs tensor before each step must be gone
    everywhere)"""
    from megaverse_b200 import capi

    E, A, steps = 700, 2, 24
    gs = []
    for sched in (1, 0):
        g = capi.Engine("Collect", E, A, 128, 72, num_threads=8)
        g.set_option("raster_sched", sched)
        for e in range(E):
            g.seed_env(e, 300 + e)
        g.reset()
        gs.append(g)
    rng = np.random.default_rng(5)
    for t in range(steps):
        acts = helpers.random_bit_actions(rng, E * A).astype(np.int32)
        for g in gs:
            g.step(acts)
        if t % 4 == 3 or t < 3:
            a, b = np.array(gs[0].obs()), np.array(gs[1].obs())
            assert np.array_equal(a, b), "cost-ordered and natural-order frames differ at step %d" % t
            assert (a[..., 3] == 255).all(), "a view was not drawn at step %d" % t
            gs[0].obs()[...] = 0  # sentinel: alpha 0 must be overwritten by the next step's frames
    assert np.array_equal(np.array(gs[0].rewards()), np.array(gs[1].rewards()))
    for g in gs:
        assert g.faults() == 0
        g.close()


@pytest.mark.timeout(180)
@pytest.mark.parametrize("scenario,E,A,depth,slices", [("Collect", 300, 2, False, 8), ("ObstaclesHard", 100, 1, True, 16), ("TowerBuilding", 7, 3, False, 4)])
def test_sliced_host_delivery_matches_zero_copy(built, scenario, E, A, depth, slices):
    """host delivery into HBM in one raster launch per slice of envs, each slice downloaded by the copy engine while the next is drawn
    (zero_copy 0, host_slices), against the default zero-copy stores: frames, depth, rewards and dones identical every step, also when
    the number of envs is not a multiple of the slice count and when bands and the cost order are on"""
    from megaverse_b200 import capi

    gs = []
    for sliced in (False, True):
        g = capi.Engine(scenario, E, A, 128, 72, num_threads=4, depth=depth)
        if sliced:
            g.set_option("zero_copy", 0)
            g.set_option("host_slices", slices)
        g.set_option("raster_sched", 2 if sliced else 1)
        for e in range(E):
            g.seed_env(e, 900 + e)
        g.reset()
        gs.append(g)
    with pytest.raises(capi.MegaverseError):
        gs[1].set_option("host_progressive", 4)  # not an option: host delivery is zero-copy, one copy or sliced
    assert np.array_equal(np.array(gs[0].obs()), np.array(gs[1].obs())), "first frame"
    rng = np.random.default_rng(8)
    for t in range(30):
        acts = helpers.random_bit_actions(rng, E * A).astype(np.int32)
        for g in gs:
            g.step(acts)
        a, b = np.array(gs[0].obs()), np.array(gs[1].obs())
        assert np.array_equal(a, b), "frames differ at step %d (%d bytes)" % (t, int((a != b).sum()))
        if depth:
            assert np.array_equal(np.array(gs[0].depth()).view(np.uint32), np.array(gs[1].depth()).view(np.uint32)), "depth differs at step %d" % t
        assert np.array_equal(np.array(gs[0].rewards()), np.array(gs[1].rewards())) and np.array_equal(np.array(gs[0].dones()), np.array(gs[1].dones()))
        gs[1].obs()[...] = 0  # whatever the next step does not deliver stays black
    for g in gs:
        assert g.faults() == 0
        g.close()


@pytest.mark.parametrize("mode", ["host", "device"])
def test_static_box_arrays_grow_on_demand(built, mode):
    """the number of static boxes of a level has no bound (component_voxel_grid.hpp:108-187): the engine's per-level arrays and the instance
    lists that depend on them are re-pitched whenever a generated level needs more.  HexExplore mazes of random size with short episodes,
    arrays started at 16 boxes: growth at reset and again at later turnovers, while the device holds live instance lists, on the host-facing
    and on the asynchronous path.  State, rewards, dones and frames equal the oracle's throughout."""
    import torch

    import orc
    from megaverse_b200 import capi

    E, A, steps = 2, 2, 180  # (master seed 48: the first two mazes of both envs have < 100 walls, the third has ~280)
    params = {"episodeLengthSec": 0.6}
    o = orc.Oracle("HexExplore", E, A, 128, 72, params=params)
    g = capi.Engine("HexExplore", E, A, 128, 72, num_threads=3, params=params)
    g.set_option("fast_shading", 0)
    g.set_option("static_cap", 16)
    o.seed(48); g.seed(48)
    o.reset(); g.reset()
    cap0 = g.static_cap()
    assert cap0 > 16
    assert _assert_same_frame(o, g, "reset") == 1.0
    rng = np.random.default_rng(8)
    acts = np.stack([helpers.purposeful_actions(rng, E * A, t) for t in range(steps)]).astype(np.int32)
    dacts = torch.from_numpy(acts).cuda()
    torch.cuda.synchronize()
    ndone = 0
    for t in range(steps):
        o.step(acts[t])
        ndone += int(o.dones().sum())
        if mode == "host":
            g.step(acts[t])
            assert np.array_equal(o.rewards().view(np.uint32), np.array(g.rewards()).view(np.uint32)), "step %d" % t
            assert np.array_equal(o.dones(), np.array(g.dones())), "step %d" % t
            if o.dones().any():
                assert _assert_same_frame(o, g, "step %d" % t) == 1.0
        else:
            g.step_device(dacts.data_ptr() + t * E * A * 4)
    if mode == "device":
        g.sync()
        g.fetch_obs()
    assert ndone >= 10 * E
    assert g.static_cap() > cap0, "the case is meant to grow the arrays during the rollout (%d -> %d)" % (cap0, g.static_cap())
    _assert_same_state(o, g, E, "end")
    assert _assert_same_frame(o, g, "end") == 1.0
    assert g.faults() == 0
    o.close(); g.close()


def test_level_beyond_the_former_static_capacity(built):
    """a Collect landscape of more than 768 static boxes (round 1 refused it): level, instances, frames and a short rollout equal the oracle's"""
    import orc
    from megaverse_b200 import capi

    E, A = 3, 2
    o = orc.Oracle("Collect", E, A, 128, 72)
    g = capi.Engine("Collect", E, A, 128, 72, num_threads=2)
    g.set_option("fast_shading", 0)
    for e in range(E):
        seed = 889027061 if e == 1 else 300 + e
        o.seed_env(e, seed); g.seed_env(e, seed)
    o.reset(); g.reset()
    assert o.level(1)[0] > 768 and g.static_cap() >= o.level(1)[0]
    for e in range(E):
        assert np.array_equal(o.level(e), g.level(e)), "level %d" % e
        assert np.array_equal(o.instances(e).view(np.uint32), g.instances(e).view(np.uint32)), "instances %d" % e
    assert _assert_same_frame(o, g, "reset") == 1.0
    rng = np.random.default_rng(8)
    for t in range(40):
        acts = helpers.purposeful_actions(rng, E * A, t)
        o.step(acts); g.step(acts)
        assert np.array_equal(o.rewards().view(np.uint32), np.array(g.rewards()).view(np.uint32)), "step %d" % t
    _assert_same_state(o, g, E, "end")
    assert _assert_same_frame(o, g, "end") == 1.0
    assert g.faults() == 0
    o.close(); g.close()


def test_async_call_refuses_episodes_shorter_than_its_pipeline(built):
    """mv_step_device delivers an env's next level three calls after its episode ended; an episode of fewer than three steps is outside that
    contract and must be refused loudly (MV_ERR_STATE, fault bit latched), never answered with a stale level"""
    import torch
    from megaverse_b200 import capi

    E = 8
    g = capi.Engine("TowerBuilding", E, 1, 128, 72, num_threads=2, params={"episodeLengthSec": -400.0})  # every episode ends on its first step
    g.seed(1); g.reset()
    acts = torch.zeros((E,), dtype=torch.int32, device="cuda")
    with pytest.raises(capi.MegaverseError) as ei:
        for t in range(8):
            g.step_device(acts.data_ptr())
        g.sync()
    assert ei.value.code == capi.MV_ERR_STATE
    torch.cuda.synchronize()
    assert g.fault_word() & 1  # MV_FAULT_LEVEL_NOT_READY
    g.close()


@pytest.mark.parametrize("A", [1, 3])
def test_empty_scenario_parity(built, A):
    """the reference's debugging scenario (scenario_empty.cpp: one static box, all agents spawned on the same spot, no rules) -- the
    workload of the one throughput figure the reference publishes (README.md:243-245)"""
    E, steps = 5, 200
    o, g = _pair("Empty", E, A, 9, params={"episodeLengthSec": 6.0}, depth=True)
    for e in range(E):
        assert np.array_equal(o.level(e), g.level(e)), "level %d" % e
        assert np.array_equal(o.instances(e).view(np.uint32), g.instances(e).view(np.uint32)), "instances %d" % e
    assert _assert_same_frame(o, g, "reset") == 1.0
    rng = np.random.default_rng(4)
    ndone = 0
    for t in range(steps):
        acts = helpers.purposeful_actions(rng, E * A, t)
        o.step(acts); g.step(acts)
        assert np.array_equal(o.rewards().view(np.uint32), np.array(g.rewards()).view(np.uint32)), "step %d" % t
        assert np.array_equal(o.dones(), np.array(g.dones())), "step %d" % t
        assert np.array_equal(o.true_objectives(), np.array(g.true_objectives())), "step %d" % t
        ndone += int(o.dones().sum())
        if t % 40 == 0 or o.dones().any():
            _assert_same_state(o, g, E, "step %d" % t)
            assert _assert_same_frame(o, g, "step %d" % t) == 1.0
            _assert_same_depth(o, g, "step %d" % t)
    assert ndone >= E
    assert g.faults() == 0
    o.close(); g.close()
