"""Spectator cameras (mv_draw_cameras, mv_draw_cameras_device): the step's rasteriser drawing chosen envs from caller-placed viewpoints.

An agent's own view matrix as a camera gives the step's frame byte for byte (and mv_draw_hires' at 768 x 432); overview and chase cameras
equal the oracle's rasteriser on the oracle's instance list of the same state; the device call between asynchronous steps equals the host
call of a twin engine that synchronises, and leaves every output of the engine and its cost-ordered queue as they would be without it."""
import ctypes as C

import numpy as np
import pytest

import helpers

pytestmark = pytest.mark.gpu

SCENARIOS = ["TowerBuilding", "Collect", "Rearrange", "Sokoban", "HexExplore", "HexMemory", "Empty", "ObstaclesEasy", "ObstaclesMedium",
             "ObstaclesHard", "ObstaclesWalls", "ObstaclesSteps", "ObstaclesLava"]


def _params(name):
    """short episodes, so that 50 steps cross natural ends (the level adds time per object in TowerBuilding, Collect and HexMemory, and
    35 s per platform in the Obstacles family)"""
    if name.startswith("Obstacles"):
        return {"episodeLengthSec": 1.0, "obstaclesMinNumPlatforms": 0, "obstaclesMaxNumPlatforms": 0}
    return {"episodeLengthSec": {"TowerBuilding": -180.0, "Collect": -1.5, "HexMemory": -5.0}.get(name, 1.5)}


def _engine(name, E, A, w=128, h=72, fast=False, seed=1000, params=None, **opts):
    from megaverse_b200 import capi

    g = capi.Engine(name, E, A, w, h, num_threads=4, params=params, depth=True, segmentation=True)
    g.set_option("fast_shading", int(fast))
    for k, v in opts.items():
        g.set_option(k, v)
    for e in range(E):
        g.seed_env(e, seed + 7919 * e)
    g.reset()
    return g


def _agent_views(g):
    return np.stack([g.view(e, a) for e in range(g.E) for a in range(g.A)])


def _agent_envs(g):
    return np.repeat(np.arange(g.E, dtype=np.int32), g.A)


def _same_frames(tag, got, want_obs, want_depth=None, want_seg=None):
    assert np.array_equal(got.obs, want_obs), "%s: colour differs in %d pixels" % (tag, int((got.obs != want_obs).any(-1).sum()))
    if want_depth is not None:
        assert np.array_equal(got.depth.view(np.uint32), np.asarray(want_depth).view(np.uint32)), "%s: depth differs" % tag
    if want_seg is not None:
        assert np.array_equal(got.seg, want_seg), "%s: segmentation differs" % tag


# ---------------------------------------------------------------------------------------------------- 1. identity with the step
@pytest.mark.parametrize("fast", [False, True])
@pytest.mark.parametrize("name", SCENARIOS)
def test_agent_views_as_cameras_equal_the_step(name, fast):
    E, A = 4, 2
    g = _engine(name, E, A, fast=fast, params=_params(name))
    try:
        rng = np.random.default_rng(11)
        ends = 0
        for t in range(50):
            g.step(helpers.purposeful_actions(rng, E * A, t))
            ends += int(g.dones().sum())
        assert ends > 0, "no natural end in 50 steps"
        views, envs = _agent_views(g), _agent_envs(g)
        got = g.draw_cameras(envs, views, 128, 72, depth=True, seg=True)
        assert got.out_of_range == 0
        _same_frames(name, got, g.obs(), g.depth(), g.segmentation())
        hires = g.draw_hires(768, 432).copy()
        big = g.draw_cameras(envs, views, 768, 432)
        assert big.depth is None and big.seg is None and big.out_of_range == 0
        _same_frames(name + " 768x432", big, hires)
    finally:
        g.close()


# ---------------------------------------------------------------------------------------------------- 2. against the oracle
@pytest.mark.parametrize("name", SCENARIOS)
def test_overview_and_chase_against_the_oracle(name):
    import orc
    import orc_seg_view
    from megaverse_b200 import cameras

    E, A, W, H, seed = 2, 2, 256, 144, 300
    o = orc.Oracle(name, E, A, render=False, params=_params(name))
    g = _engine(name, E, A, seed=seed, params=_params(name))
    try:
        for e in range(E):
            o.seed_env(e, seed + 7919 * e)
        o.reset()
        rng = np.random.default_rng(12)
        for t in range(30):
            acts = helpers.purposeful_actions(rng, E * A, t)
            o.step(acts)
            g.step(acts)
        bounds = g.level_bounds()
        agent = np.stack([o.view(e, a) for e in range(E) for a in range(A)])
        assert np.array_equal(agent, _agent_views(g)), "engine and oracle are not in lockstep"
        views = np.concatenate([cameras.overview_views(bounds, W, H), cameras.chase_views(agent)])
        envs = np.concatenate([np.arange(E), _agent_envs(g)]).astype(np.int32)
        got = g.draw_cameras(envs, views, W, H, depth=True, seg=True)
        assert got.out_of_range == 0, "a camera pose left the exact range"
        for c, (e, v) in enumerate(zip(envs, views)):
            rgba, depth = orc.render_instances(v, o.instances(int(e)), W, H, want_depth=True)
            seg, sdepth = orc_seg_view.segmentation_view(o, int(e), v, W, H)
            tag = "%s camera %d" % (name, c)
            assert np.array_equal(sdepth.view(np.uint32), depth.view(np.uint32)), tag
            assert (got.obs[c, :, :, :3] != 0).any(), "%s shows nothing" % tag
            assert np.array_equal(got.obs[c], rgba), "%s: colour differs in %d pixels" % (tag, int((got.obs[c] != rgba).any(-1).sum()))
            assert np.array_equal(got.depth[c].view(np.uint32), depth.view(np.uint32)), "%s: depth differs" % tag
            assert np.array_equal(got.seg[c], seg), "%s: segmentation differs in %d pixels" % (tag, int((got.seg[c] != seg).sum()))
    finally:
        o.close()
        g.close()


# ---------------------------------------------------------------------------------------------------- 3. the device path
def _torch():
    return pytest.importorskip("torch")


@pytest.mark.parametrize("opts", [{"level_slots": 4}, {"level_set": 8, "level_set_seed": 5}])
def test_device_cameras_between_asynchronous_steps(opts):
    torch = _torch()
    from megaverse_b200 import cameras

    name, E, A, W, H, steps = "TowerBuilding", 6, 2, 128, 72, 40
    params = {"episodeLengthSec": 1.0}
    common = dict(params=params, raster_sched=2, **opts)
    ga, gb, gc = (_engine(name, E, A, **common) for _ in range(3))
    try:
        rng = np.random.default_rng(13)
        # cameras: a chase camera per agent (from the agents' first views) and one overview per env, the same table for the three engines
        views = np.concatenate([cameras.chase_views(_agent_views(gb)), cameras.overview_views(gb.level_bounds(), W, H)])
        envs = np.concatenate([_agent_envs(gb), np.arange(E, dtype=np.int32)])
        n = envs.size
        d_envs, d_views = torch.from_numpy(envs).cuda(), torch.from_numpy(views).cuda()
        d_obs = torch.zeros((n, H, W, 4), dtype=torch.uint8, device="cuda")
        d_depth = torch.zeros((n, H, W), dtype=torch.float32, device="cuda")
        d_seg = torch.zeros((n, H, W), dtype=torch.int16, device="cuda")
        ended = requested = 0
        for t in range(steps):
            acts = torch.from_numpy(helpers.purposeful_actions(rng, E * A, t)).cuda()
            ends = torch.from_numpy((rng.random(E) < 0.08).astype(np.uint8)).cuda()
            requested += int(ends.sum())
            torch.cuda.synchronize()
            for g in (ga, gb, gc):
                g.step_device(acts.data_ptr(), ends.data_ptr())
            before = ga.view_order()
            ctr = ga.draw_cameras_device(d_envs.data_ptr(), d_views.data_ptr(), n, W, H, d_obs.data_ptr(), d_depth.data_ptr(), d_seg.data_ptr())
            after = ga.view_order()
            assert np.array_equal(before, after), "step %d: the camera launch wrote the cost-ordered queue" % t
            gb.sync()
            want = gb.draw_cameras(envs, views, W, H, depth=True, seg=True)
            torch.cuda.synchronize()
            tag = "step %d" % t
            assert want.out_of_range == 0 and _read_u32(torch, ctr) == 0, tag
            assert np.array_equal(d_obs.cpu().numpy(), want.obs), tag
            assert np.array_equal(d_depth.cpu().numpy().view(np.uint32), want.depth.view(np.uint32)), tag
            assert np.array_equal(d_seg.cpu().numpy().view(np.uint16), want.seg), tag
            outs = ["obs", "rewards", "dones", "done_reasons", "true_objectives"] + (["level_ids"] if "level_set" in opts else [])
            for what in outs:
                a = torch.as_tensor(ga.device_array(what), device="cuda").cpu().numpy()
                c = torch.as_tensor(gc.device_array(what), device="cuda").cpu().numpy()
                assert np.array_equal(a.view(np.uint8), c.view(np.uint8)), "%s: %s differs from the engine that drew no cameras" % (tag, what)
            ended += int(torch.as_tensor(ga.device_array("dones"), device="cuda").sum())
        assert ended > 0 and requested > 0
        for g in (ga, gc):
            g.sync()
        assert np.array_equal(ga.rewards(), gc.rewards()) and np.array_equal(ga.dones(), gc.dones())
    finally:
        for g in (ga, gb, gc):
            g.close()


def _read_u32(torch, ptr):
    """one uint32 of device memory, through a tensor view of it"""
    class _A:
        __cuda_array_interface__ = {"shape": (1,), "typestr": "<u4", "data": (ptr, False), "version": 3}
    return int(torch.as_tensor(_A(), device="cuda").to(torch.int64).cpu()[0])


def test_views_device_holds_the_agent_views():
    torch = _torch()
    g = _engine("Collect", 3, 2)
    try:
        g.step(np.full(6, 1 << 3, dtype=np.int32))
        d = torch.as_tensor(g.device_array("views"), device="cuda").cpu().numpy()
        assert np.array_equal(d, _agent_views(g))
    finally:
        g.close()


# ---------------------------------------------------------------------------------------------------- 4. coverage
def test_mixed_engine_cameras_in_one_call():
    g = _engine(["Collect", "TowerBuilding", "HexMemory", "ObstaclesEasy", "Sokoban", "Rearrange"], 6, 2)
    try:
        rng = np.random.default_rng(14)
        for t in range(10):
            g.step(helpers.purposeful_actions(rng, 12, t))
        got = g.draw_cameras(_agent_envs(g), _agent_views(g), 128, 72, depth=True, seg=True)
        _same_frames("mixed", got, g.obs(), g.depth(), g.segmentation())
    finally:
        g.close()


def test_active_sets_restarts_and_state_loads():
    E, A = 5, 2
    g = _engine("ObstaclesHard", E, A)
    try:
        rng = np.random.default_rng(15)
        for t in range(5):
            g.step(helpers.purposeful_actions(rng, E * A, t))
        views, envs = _agent_views(g), _agent_envs(g)
        before = g.draw_cameras(envs, views, 128, 72, depth=True, seg=True)
        g.step_envs(helpers.purposeful_actions(rng, E * A, 5), [1, 3])
        after = g.draw_cameras(envs, _agent_views(g), 128, 72, depth=True, seg=True)
        _same_frames("active set", after, g.obs(), g.depth(), g.segmentation())
        for e in (0, 2, 4):  # inactive: the unchanged scene
            rows = slice(e * A, e * A + A)
            assert np.array_equal(after.obs[rows], before.obs[rows]) and np.array_equal(after.seg[rows], before.seg[rows]), e
        store = g.states_create(2)
        g.states_save(store, [0, 2], [0, 1])
        for t in range(4):
            g.step(helpers.purposeful_actions(rng, E * A, 6 + t))
        g.reset_envs([1, 4], seeds=[77, 78])
        _same_frames("reset_envs", g.draw_cameras(envs, _agent_views(g), 128, 72, depth=True, seg=True), g.obs(), g.depth(), g.segmentation())
        g.states_load(store, [0, 1], [3, 2])
        _same_frames("states_load", g.draw_cameras(envs, _agent_views(g), 128, 72, depth=True, seg=True), g.obs(), g.depth(), g.segmentation())
        rows = slice(3 * A, 3 * A + A)
        assert np.array_equal(g.draw_cameras(envs, _agent_views(g), 128, 72).obs[rows], before.obs[0:A]), "the loaded env shows another scene"
        g.states_destroy(store)
    finally:
        g.close()


def test_out_of_range_envs_give_all_zero_frames():
    torch = _torch()
    E, A, W, H = 3, 2, 128, 72
    g = _engine("Sokoban", E, A)
    try:
        g.step(np.full(E * A, 1 << 5, dtype=np.int32))
        views = _agent_views(g)[[0, 1, 2, 3, 4]]
        envs = np.array([0, -1, 1, E, 1 << 30], dtype=np.int32)
        n = envs.size
        d_obs = torch.full((n, H, W, 4), 7, dtype=torch.uint8, device="cuda")
        d_depth = torch.full((n, H, W), 7.0, dtype=torch.float32, device="cuda")
        d_seg = torch.full((n, H, W), 7, dtype=torch.int16, device="cuda")
        de, dv = torch.from_numpy(envs).cuda(), torch.from_numpy(views).cuda()
        torch.cuda.synchronize()
        g.draw_cameras_device(de.data_ptr(), dv.data_ptr(), n, W, H, d_obs.data_ptr(), d_depth.data_ptr(), d_seg.data_ptr())
        g.sync()
        obs, depth, seg = d_obs.cpu().numpy(), d_depth.cpu().numpy(), d_seg.cpu().numpy()
        for c in (1, 3, 4):
            assert not obs[c].any() and not depth[c].any() and not seg[c].any(), c
        good = [0, 2]
        want = g.draw_cameras(envs[good], views[good], W, H, depth=True, seg=True)
        assert np.array_equal(obs[good], want.obs) and np.array_equal(depth[good], want.depth) and np.array_equal(seg[good].view(np.uint16), want.seg)
    finally:
        g.close()


def test_range_counter_flags_a_stretched_view():
    """a constructed view that stretches camera-space x by 500: the floor slab crossing the camera plane then projects far beyond the range
    the integer set-up is exact in.  A wrong-pixel signal, not a fault: drawn once"""
    from megaverse_b200 import cameras

    g = _engine("ObstaclesEasy", 1, 1)
    try:
        bounds = g.level_bounds()[0]
        centre = 0.5 * (bounds[:3] + bounds[3:])
        eye = np.array([centre[0], bounds[1] + 0.6, centre[2]])
        v = cameras.look_at(eye, eye + np.array([1.0, -0.05, 0.3]))
        m = v.reshape(4, 4).T.astype(np.float64)
        m[0] *= 500.0
        stretched = np.ascontiguousarray(m.T.reshape(16), dtype=np.float32)
        assert g.draw_cameras([0], v[None], 128, 72).out_of_range == 0
        assert g.draw_cameras([0], stretched[None], 128, 72).out_of_range > 0
    finally:
        g.close()


def test_camera_call_errors():
    from megaverse_b200 import capi

    g = capi.Engine("Collect", 2, 1, 128, 72)
    try:
        v = np.zeros((1, 16), dtype=np.float32)
        for call in (lambda: g.draw_cameras([0], v, 128, 72), lambda: g.level_bounds()):
            with pytest.raises(capi.MegaverseError) as ex:
                call()
            assert ex.value.code == capi.MV_ERR_STATE and "before mv_reset" in str(ex.value)
        g.reset()
        obs = g.obs().copy()
        for envs, views, w, h, msg in (([2], v, 128, 72, "out of range"), ([-1], v, 128, 72, "out of range"), ([0], v, 100, 72, "multiple of 32"),
                                       ([0], v, 800, 72, "multiple of 32"), ([0], v, 128, 4100, "multiple of 32")):
            with pytest.raises(capi.MegaverseError) as ex:
                g.draw_cameras(envs, views, w, h)
            assert ex.value.code == capi.MV_ERR_ARG and msg in str(ex.value), msg
        L, h = capi.lib(), g._h
        assert L.mv_draw_cameras(h, None, None, -1, 128, 72, 0, 0, None, None, None, None) == capi.MV_ERR_ARG
        assert L.mv_draw_cameras(h, None, None, 1, 128, 72, 0, 0, None, None, None, None) == capi.MV_ERR_ARG
        assert "bad env / view tables" in L.mv_last_error(h).decode()
        assert L.mv_draw_cameras_device(h, None, None, 2, 128, 72, None, None, None, None) == capi.MV_ERR_ARG
        ok = C.c_void_p(1)
        assert L.mv_draw_cameras_device(h, ok, ok, 2, 128, 72, None, None, None, None) == capi.MV_ERR_ARG
        assert "null obs buffer" in L.mv_last_error(h).decode()
        assert L.mv_draw_cameras_device(h, ok, ok, 2, 96, 70, ok, None, None, None) == capi.MV_ERR_ARG
        assert np.array_equal(g.obs(), obs), "a rejected call changed the observations"
        g.step_begin(np.zeros(2, dtype=np.int32))
        with pytest.raises(capi.MegaverseError) as ex:
            g.draw_cameras([0], v, 128, 72)
        assert ex.value.code == capi.MV_ERR_STATE and "mv_step_begin" in str(ex.value)
        assert L.mv_draw_cameras_device(h, ok, ok, 1, 128, 72, ok, None, None, None) == capi.MV_ERR_STATE
        g.step_end()
        empty = g.draw_cameras([], np.zeros((0, 16), dtype=np.float32), 128, 72)
        assert empty.obs.shape == (0, 72, 128, 4) and empty.out_of_range == 0
    finally:
        g.close()


# ---------------------------------------------------------------------------------------------------- 5. the Python surface
def test_env_overview_and_chase():
    from megaverse_b200.megaverse_env import MegaverseEnv

    env = MegaverseEnv("TowerBuilding", 2, 2, 2)
    try:
        env.seed(3)
        env.reset()
        env.step([[1, 0, 0, 0, 0, 0]] * 4)
        ov = env.overview([0, 1], 256, 144)
        assert ov.shape == (2, 144, 256, 3) and ov.dtype == np.uint8 and ov.any()
        ch = env.chase([0, 3])
        assert ch.shape == (2, 432, 768, 3) and ch.dtype == np.uint8 and ch.any()
        own = env.render_cameras([0], env.env.get_views()[[0]], 128, 72)
        assert np.array_equal(own[0], np.transpose(env.observations()[0], (1, 2, 0)))
        frame = env.render(mode="rgb_array")
        assert frame.shape == (2 * 432, 2 * 768, 3)
    finally:
        env.close()
