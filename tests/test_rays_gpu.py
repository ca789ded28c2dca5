"""Ray sensors (mv_set_rays) on the GPU: the engine's rays equal the oracle's restatement of the hit definition bit for bit in lockstep for
every scenario; terminal rays equal the rays of a twin whose episode went on; every drawing path (action repeat, active sets, restarts,
state loads, mixed and level-set engines, the asynchronous loop at four level slots) delivers the same rays to the host and to HBM; every
other output is byte-identical to a twin with rays off; pixel-centre rays agree with the engine's own segmentation and depth; misuse is
refused with the documented codes."""
import numpy as np
import pytest

import helpers
from test_cameras_gpu import SCENARIOS, _params

pytestmark = pytest.mark.gpu

MAXD = 60.0
SEG_AGENT = 4


def _dirs():
    from megaverse_b200 import rays

    return np.concatenate([rays.fan(64, 180.0), rays.ring(8, 50.0), rays.ring(8, -50.0)])


def _engine(name, E, A, seed=1000, params=None, dirs=None, depth=True, seg=True, **opts):
    from megaverse_b200 import capi

    g = capi.Engine(name, E, A, 128, 72, num_threads=4, params=params, depth=depth, segmentation=seg)
    for k, v in opts.items():
        g.set_option(k, v)
    if dirs is not None:
        g.set_rays(dirs, MAXD)
    for e in range(E):
        g.seed_env(e, seed + 7919 * e)
    g.reset()
    return g


def _rays(g):
    d, t = g.rays()
    return np.array(d), np.array(t)


def _same(tag, got, want):
    assert np.array_equal(got[0].view(np.uint32), want[0].view(np.uint32)), "%s: distance differs on %d rays" % (tag, int((got[0] != want[0]).sum()))
    assert np.array_equal(got[1], want[1]), "%s: tag differs on %d rays" % (tag, int((got[1] != want[1]).sum()))


def _device_rays(g, final=False):
    import torch

    p = "final_" if final else ""
    torch.cuda.synchronize()
    return (torch.as_tensor(g.device_array(p + "rays_dist"), device="cuda").cpu().numpy(),
            torch.as_tensor(g.device_array(p + "rays_tag"), device="cuda").cpu().numpy())


# ---------------------------------------------------------------------------------------------------- 1. lockstep against the oracle
@pytest.mark.parametrize("name", SCENARIOS)
def test_rays_equal_the_oracle_in_lockstep(name):
    import orc
    import orc_rays

    E, A, seed = 4, 2, 1000  # test_cameras_gpu's identity run: natural ends within 50 steps in every scenario
    dirs = _dirs()
    o = orc.Oracle(name, E, A, render=False, params=_params(name))
    g = _engine(name, E, A, seed=seed, params=_params(name), dirs=dirs, final_obs=1)
    try:
        for e in range(E):
            o.seed_env(e, seed + 7919 * e)
        o.reset()
        _same("%s reset" % name, _rays(g), orc_rays.rays_all(o, dirs, MAXD))
        rng = np.random.default_rng(11)
        ends, hits = 0, 0
        prev_final = [np.array(x) for x in g.final_rays()]
        for t in range(50):
            acts = helpers.purposeful_actions(rng, E * A, t)
            o.step(acts)
            g.step(acts)
            got = _rays(g)
            _same("%s step %d" % (name, t), got, orc_rays.rays_all(o, dirs, MAXD))
            hits += int((got[1] != 0).sum())
            dn = np.repeat(np.array(g.dones()) != 0, A)
            fin = [np.array(x) for x in g.final_rays()]
            for k in range(2):  # terminal rays: rows of envs that did not end are left alone
                assert np.array_equal(fin[k][~dn], prev_final[k][~dn]), "%s step %d: a terminal row without an end changed" % (name, t)
            if dn.any():
                assert (fin[1][dn] != 0).any(), "%s step %d: no terminal ray hit anything" % (name, t)
            ends += int(dn.sum())
            prev_final = fin
        assert ends > 0, "no natural end in 50 steps"
        assert hits > 0
    finally:
        o.close()
        g.close()


# ---------------------------------------------------------------------------------------------------- 2. terminal rays
def test_terminal_rays_equal_the_twin_that_went_on():
    """one engine asked to end envs through d_ends, a twin that is not: at each honoured request the terminal rays equal the twin's live
    rays (the scene the twin went on from, which test 1 holds equal to the oracle's); the twin then restarts the env and both go on equal"""
    import torch

    name, E, A, M = "HexExplore", 6, 2, 40
    params = {"episodeLengthSec": 60.0}
    dirs = _dirs()
    g = _engine(name, E, A, params=params, dirs=dirs, final_obs=1)
    ref = _engine(name, E, A, params=params, dirs=dirs)
    try:
        rng = np.random.default_rng(3)
        acts = np.stack([helpers.purposeful_actions(rng, E * A, t) for t in range(M)]).astype(np.int32)
        dacts = torch.from_numpy(acts).cuda()
        last = np.zeros(E, dtype=np.int64)
        honoured_total = 0
        for t in range(M):
            req = [e for e in range(E) if rng.random() < 0.25]
            ends = torch.zeros(E, dtype=torch.uint8, device="cuda")
            if req:
                ends[req] = 1
            torch.cuda.synchronize()
            g.step_device(dacts[t].data_ptr(), ends.data_ptr())
            ref.step(acts[t])
            g.sync()
            g.fetch_obs()
            last += 1
            honoured = [e for e in req if last[e] >= 3]
            assert list(np.flatnonzero(np.array(g.dones()))) == honoured
            fin, want = [np.array(x) for x in g.final_rays()], _rays(ref)
            for e in honoured:
                rows = slice(e * A, (e + 1) * A)
                _same("step %d env %d terminal" % (t, e), (fin[0][rows], fin[1][rows]), (want[0][rows], want[1][rows]))
                last[e] = 0
            _same("step %d terminal, device" % t, _device_rays(g, final=True), tuple(fin))
            honoured_total += len(honoured)
            if honoured:
                ref.reset_envs(honoured)
            _same("step %d live" % t, _rays(g), _rays(ref))
        assert honoured_total > 5
    finally:
        g.close()
        ref.close()


# ---------------------------------------------------------------------------------------------------- 3. every drawing path
PATHS = {
    "repeat4": ("Collect", dict(action_repeat=4, level_slots=4)),
    "slots4": ("ObstaclesHard", dict(level_slots=4)),
    "level_set": ("Sokoban", dict(level_set=16)),
    "mixed": (["TowerBuilding", "Collect", "HexMemory", "ObstaclesEasy"], dict(level_slots=4)),
}


@pytest.mark.parametrize("path", list(PATHS))
def test_device_loop_paths_and_a_twin_with_rays_off(path):
    """the mv_step_device loop with end requests and an active mask every third call: host rays (after mv_fetch_obs) equal the HBM rays,
    inactive envs keep theirs, and every other output and the launch count (less the ray launches) equal a twin with rays off"""
    import torch

    name, opts = PATHS[path]
    E, A, M = 4, 2, 30
    dirs = _dirs()
    g = _engine(name, E, A, dirs=dirs, final_obs=1, **opts)
    ref = _engine(name, E, A, final_obs=1, **opts)
    try:
        n0 = g.kernel_launches() - ref.kernel_launches()
        assert n0 == 1  # the reset's ray launch
        rng = np.random.default_rng(5)
        casts = 0
        for t in range(M):
            acts = torch.from_numpy(helpers.purposeful_actions(rng, E * A, t).astype(np.int32)).cuda()
            ends = torch.from_numpy((rng.random(E) < 0.1).astype(np.uint8)).cuda()
            active = None
            if t % 3 == 2:
                active = torch.from_numpy(np.array([1, 0, 1, 0], dtype=np.uint8)).cuda()
            before = _device_rays(g)
            for eng in (g, ref):
                if active is None:
                    eng.step_device(acts.data_ptr(), ends.data_ptr())
                else:
                    eng.step_device_active(acts.data_ptr(), ends.data_ptr(), active.data_ptr())
            casts += 2 if opts.get("final_obs", 1) else 1
            after = _device_rays(g)
            if active is not None:
                for e in (1, 3):
                    rows = slice(e * A, (e + 1) * A)
                    _same("step %d inactive env %d" % (t, e), (after[0][rows], after[1][rows]), (before[0][rows], before[1][rows]))
        for eng in (g, ref):
            eng.sync()
            eng.fetch_obs()
        _same(path + " host vs device", _rays(g), _device_rays(g))
        _same(path + " final host vs device", tuple(np.array(x) for x in g.final_rays()), _device_rays(g, final=True))
        assert (_rays(g)[1] != 0).any()
        for what in ("obs", "depth", "segmentation", "rewards", "dones", "done_reasons", "true_objectives", "final_obs"):
            assert np.array_equal(np.array(getattr(g, what)()), np.array(getattr(ref, what)())), "%s: %s differs" % (path, what)
        assert g.kernel_launches() - ref.kernel_launches() == n0 + casts
    finally:
        g.close()
        ref.close()


def test_restarts_state_loads_and_host_paths():
    """mv_reset_envs with seeds gives the rays of a fresh engine so seeded; mv_states_load gives back the rays of the saved step; mv_step_envs
    keeps the rays of inactive envs; action repeat and mv_step_begin / end deliver what mv_step does"""
    name, E, A = "Collect", 4, 2
    dirs = _dirs()
    g = _engine(name, E, A, dirs=dirs, state_tensors=1)
    try:
        rng = np.random.default_rng(9)
        for t in range(8):
            g.step(helpers.purposeful_actions(rng, E * A, t))
        store = g.states_create(E)
        g.states_save(store, list(range(E)), list(range(E)))
        saved = _rays(g)
        for t in range(5):
            g.step(helpers.purposeful_actions(rng, E * A, 8 + t))
        assert not np.array_equal(_rays(g)[0], saved[0])
        g.states_load(store, list(range(E)), list(range(E)))
        _same("state load", _rays(g), saved)
        before = _rays(g)
        g.step_envs(helpers.purposeful_actions(rng, E * A, 20), [0, 2])
        after = _rays(g)
        for e in (1, 3):
            rows = slice(e * A, (e + 1) * A)
            _same("step_envs inactive %d" % e, (after[0][rows], after[1][rows]), (before[0][rows], before[1][rows]))
        g.reset_envs([1, 2], seeds=[77, 78])
        fresh = _engine(name, E, A, dirs=dirs, state_tensors=1)
        try:
            fresh.reset_envs([1, 2], seeds=[77, 78])
            got, want = _rays(g), _rays(fresh)
            rows = slice(1 * A, 3 * A)
            _same("reset_envs", (got[0][rows], got[1][rows]), (want[0][rows], want[1][rows]))
        finally:
            fresh.close()
    finally:
        g.close()
    # action repeat and the split host call against mv_step
    a, b = _engine(name, E, A, dirs=dirs, action_repeat=4), _engine(name, E, A, dirs=dirs, action_repeat=4)
    try:
        for t in range(6):
            acts = helpers.purposeful_actions(rng, E * A, t)
            a.step(acts)
            b.step_begin(acts)
            b.step_end()
            _same("repeat 4 step %d" % t, _rays(a), _rays(b))
    finally:
        a.close()
        b.close()


# ---------------------------------------------------------------------------------------------------- 4. against the engine's own frames
AGREEMENT = 0.995  # tests/test_rays_cpu.py: the oracle's rays and rasteriser agree on >= 99.99 % of pixels


@pytest.mark.parametrize("name", SCENARIOS)
def test_pixel_centre_rays_agree_with_the_engine_frames(name):
    from megaverse_b200 import cameras

    W, H, E, A = 128, 72, 2, 2
    p00, p11, _, _ = cameras.projection(W, H)
    px, py = np.meshgrid(np.arange(4, W, 8), np.arange(2, H, 72 // 16)[:16])
    px, py = px.reshape(-1), py.reshape(-1)
    nx, ny = (px + 0.5 - W / 2) / (W / 2), (py + 0.5 - H / 2) / (H / 2)
    dirs = np.stack([nx / float(p00), ny / float(p11), -np.ones_like(nx)], -1).astype(np.float32)
    assert len(dirs) == 256
    g = _engine(name, E, A, params=_params(name), dirs=dirs, fast_shading=0)
    try:
        rng = np.random.default_rng(4)
        total = agree = 0
        for t in range(20):
            g.step(helpers.purposeful_actions(rng, E * A, t))
            dist, tag = _rays(g)
            seg, depth = np.array(g.segmentation())[:, py, px], np.array(g.depth())[:, py, px]
            own = (SEG_AGENT << 8) | (np.arange(E * A) % A)[:, None]
            keep = (seg != own) & (depth < MAXD)
            ok = keep & (tag == seg) & (np.abs(dist - depth) <= 0.01 * depth)
            total += int(keep.sum())
            agree += int(ok.sum())
        assert agree >= AGREEMENT * total, "%s: %d of %d pixels agree" % (name, agree, total)
    finally:
        g.close()


# ---------------------------------------------------------------------------------------------------- 5. misuse
def test_misuse_returns_the_documented_errors():
    import ctypes as C

    from megaverse_b200 import capi

    L = capi.lib()
    g = capi.Engine("Empty", 2, 1, 128, 72)
    try:
        d = np.array([[0, 0, -1]] * 300, dtype=np.float32)
        for n, dd, m in ((-1, d, 10.0), (257, d, 10.0), (1, d, 0.0), (1, d, -1.0), (1, d, float("inf")), (1, d, float("nan")), (2, None, 10.0)):
            assert L.mv_set_rays(g._h, None if dd is None else dd.ctypes.data, n, m) == capi.MV_ERR_ARG, (n, m)
        for bad in ([0, 0, 0], [float("nan"), 0, -1], [0, float("inf"), -1]):
            b = np.array([[0, 0, -1], bad], dtype=np.float32)
            assert L.mv_set_rays(g._h, b.ctypes.data, 2, 10.0) == capi.MV_ERR_ARG, bad
        p, q = C.c_void_p(), C.c_void_p()
        for name in ("mv_rays_host", "mv_rays_device", "mv_final_rays_host", "mv_final_rays_device"):
            assert getattr(L, name)(g._h, C.byref(p), C.byref(q)) == capi.MV_ERR_ARG, name  # rays off
        assert L.mv_set_rays(g._h, d.ctypes.data, 256, 10.0) == capi.MV_OK
        assert L.mv_rays_host(g._h, C.byref(p), C.byref(q)) == capi.MV_ERR_STATE  # before the reset
        assert L.mv_final_rays_host(g._h, C.byref(p), C.byref(q)) == capi.MV_ERR_ARG  # final_obs off
        assert L.mv_set_rays(g._h, d.ctypes.data, 0, 10.0) == capi.MV_OK  # off again
        g.set_rays(d[:3], 10.0)
        g.reset()
        assert L.mv_set_rays(g._h, d.ctypes.data, 3, 10.0) == capi.MV_ERR_STATE
        assert L.mv_rays_host(g._h, C.byref(p), C.byref(q)) == capi.MV_OK and L.mv_rays_host(g._h, None, None) == capi.MV_OK
        assert L.mv_final_rays_device(g._h, C.byref(p), C.byref(q)) == capi.MV_ERR_ARG
        assert g.rays()[0].shape == (2, 3)
    finally:
        g.close()


def test_rays_off_changes_nothing_and_the_env_surface():
    from megaverse_b200 import rays
    from megaverse_b200.megaverse_env import MegaverseEnv

    g = _engine("Collect", 2, 2)
    try:
        n = g.kernel_launches()
        g.step(np.zeros(4, dtype=np.int32))
        assert g.kernel_launches() - n == 2  # the step and raster kernels, as without the feature
        assert g.last_rays_ms() == 0.0
    finally:
        g.close()
    E, A = 4, 2  # test_final_obs_gpu's run with episode ends
    env = MegaverseEnv("Collect", E, A, 2, final_observation=True, ray_directions=rays.ring(16), ray_max_distance=30.0,
                       params={"episodeLengthSec": -45.0})
    try:
        env.seed(23)
        env.reset()
        dist, tag = env.ray_observations()
        assert dist.shape == (E * A, 16) and tag.shape == (E * A, 16) and (tag != 0).any()
        rng = np.random.default_rng(4)
        seen = False
        for _ in range(120):
            obs, rew, dones, infos = env.step(rng.integers(0, [3, 3, 3, 2, 2, 3], size=(E * A, 6)))
            assert len(obs) == E * A and len(rew) == E * A
            for d, info in zip(dones, infos):
                if d:
                    fd, ft = info["final_rays"]
                    assert fd.shape == (16,) and ft.dtype == np.uint16
                    seen = True
        assert seen
    finally:
        env.close()
