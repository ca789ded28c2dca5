"""Option "segmentation": the class and index of the drawable behind every pixel, drawn by the rasteriser.  Compared byte for byte with the
oracle's own segmentation (tags taken from its scene objects) at every step of warped rollouts in every scenario family, at action repeat,
and across every raster partitioning, scheduling and delivery path, the re-renders, the mixed batch and terminal frames; with the option on
every other output is byte-identical to the option off."""
import numpy as np
import pytest

import helpers
import orc_seg
import test_action_repeat_gpu as ar
import test_events_gpu as ev
from test_final_obs_gpu import MEGAVERSE8

pytestmark = pytest.mark.gpu
SEG_OBJECT, SEG_AGENT, SEG_REWARD = 3, 4, 5


def _armed(base_cls):
    """construct base_cls with the engine's option segmentation on (the runs build their engine themselves)"""
    from megaverse_b200 import capi

    class Armed(capi.Engine):
        def __init__(self, *a, **kw):
            super().__init__(*a, **kw)
            self.set_option("segmentation", 1)

    def make(*a, **kw):
        base = capi.Engine
        capi.Engine = Armed
        try:
            return base_cls(*a, **kw)
        finally:
            capi.Engine = base

    return make


def _check_seg(run, tag):
    (so, sd), sg = orc_seg.segmentation(run.o), np.array(run.g.segmentation())
    assert np.array_equal(sd.view(np.uint32), run.o.depth().view(np.uint32)), tag  # the oracle's own depth: the same winners
    assert np.array_equal(so, sg), "%s: segmentation differs in %d pixels (oracle %s, engine %s)" % (
        tag, int((so != sg).sum()), np.unique(so[so != sg])[:6], np.unique(sg[so != sg])[:6])
    assert np.array_equal(sg == 0, np.array(run.g.depth()) == 0), tag
    run.seg_classes |= set(np.unique(sg >> 8).tolist())
    run.seg_checks += 1


class SegRun(ev.Run):
    def checkpoint(self, tag, frames=True):
        super().checkpoint(tag, frames)
        if frames:
            _check_seg(self, tag)


class SegRepeatRun(ar.RepeatRun):
    def checkpoint(self, tag, frames=True):
        super().checkpoint(tag, frames)
        if frames:
            _check_seg(self, tag)


CASES = [
    # scenario, A, E, ticks, seed, fast shading
    ("TowerBuilding", 1, 8, 160, 201, False),
    ("TowerBuilding", 4, 4, 120, 202, True),
    ("ObstaclesEasy", 1, 6, 100, 203, False),
    ("ObstaclesMedium", 4, 4, 100, 204, True),
    ("ObstaclesHard", 1, 6, 100, 205, False),
    ("ObstaclesWalls", 4, 3, 80, 206, False),
    ("ObstaclesSteps", 1, 6, 80, 207, True),
    ("ObstaclesLava", 4, 3, 80, 208, False),
    ("Collect", 1, 6, 140, 209, False),
    ("Collect", 4, 4, 120, 210, True),
    ("Collect", 8, 3, 80, 211, False),
    ("Sokoban", 1, 6, 100, 212, False),
    ("Sokoban", 4, 3, 80, 213, True),
    ("Rearrange", 1, 6, 200, 214, False),
    ("Rearrange", 4, 3, 100, 215, True),
    ("HexExplore", 1, 6, 100, 216, True),
    ("HexExplore", 4, 3, 80, 217, False),
    ("HexMemory", 1, 6, 160, 218, False),
    ("HexMemory", 4, 3, 80, 219, True),
    ("Empty", 4, 4, 70, 220, False),
    ("Empty", 8, 2, 70, 221, True),
]


@pytest.mark.parametrize("scenario,A,E,ticks,seed,fast", CASES, ids=["%s-A%d%s" % (c[0], c[1], "-fast" if c[5] else "") for c in CASES])
def test_segmentation_matches_the_oracle_at_every_step(built, scenario, A, E, ticks, seed, fast):
    # several episode ends in the window: TowerBuilding, Collect and HexMemory add to the parameter per object, reward or good object
    params = {"episodeLengthSec": {"tower": -180.0, "collect": -1.5, "hexmemory": -7.0}.get(ev.family(scenario), 4.0)}
    run = _armed(SegRun)(scenario, E, A, seed, params=params, fast_shading=fast)
    run.seg_classes, run.seg_checks = set(), 0
    try:
        run.checkpoint("%s reset" % scenario)
        ev.drive(run, ticks, np.random.default_rng(seed), check_every=1)
        assert run.dones > 0, "the window is meant to cross episode ends"
        assert run.seg_checks >= ticks
        assert SEG_AGENT in run.seg_classes or A == 1
        if run.fam == "tower":
            assert run.counts["picked_up"] > 0 and SEG_OBJECT in run.seg_classes, run.table()  # carried objects were drawn
        if run.fam in ("collect", "hexmemory"):
            assert run.counts["good"] > 0 and SEG_REWARD in run.seg_classes, run.table()  # rewards were collected
    finally:
        run.close()


@pytest.mark.parametrize("scenario,A,E,calls,k,seed,params", [
    ("TowerBuilding", 4, 4, 60, 4, 301, {"episodeLengthSec": -180.0}),
    ("Collect", 4, 4, 40, 4, 302, {"episodeLengthSec": -1.5}),
    ("ObstaclesHard", 1, 6, 50, 4, 303, {"episodeLengthSec": 3.0, "obstaclesMinNumPlatforms": 0, "obstaclesMaxNumPlatforms": 0}),
])
def test_segmentation_at_action_repeat(built, scenario, A, E, calls, k, seed, params):
    run = _armed(SegRepeatRun)(scenario, E, A, seed, params, k)
    run.seg_classes, run.seg_checks = set(), 0
    try:
        run.checkpoint("%s reset" % scenario)
        ev.drive(run, calls, np.random.default_rng(seed))
        assert run.dones > 0 and run.seg_checks > 3
    finally:
        run.close()


# ------------------------------------------------------------------------------------------------ 2. the same tensor on every path
def _engine(scenario, E, A, seed=5, params=None, seg=True, depth=False, final=False, **options):
    from megaverse_b200 import capi

    g = capi.Engine(scenario, E, A, 128, 72, num_threads=4, params=params, depth=depth, segmentation=seg)
    if final:
        g.set_option("final_obs", 1)
    for k, v in options.items():
        g.set_option(k, v)
    g.seed(seed)
    g.reset()
    return g


def _acts(n, steps, seed=9):
    rng = np.random.default_rng(seed)
    return [helpers.purposeful_actions(rng, n, t).astype(np.int32) for t in range(steps)]


def _host_run(scenario, E, A, steps, params=None, **options):
    g = _engine(scenario, E, A, params=params, **options)
    out = [np.array(g.segmentation())]
    for a in _acts(E * A, steps):
        g.step(a)
        out.append(np.array(g.segmentation()))
    assert g.faults() == 0
    g.close()
    return out


PARTITIONS = [{"tri_cap": 32}, {"raster_bands": 1}, {"raster_bands": 2}, {"raster_bands": 3}, {"raster_sched": 0}, {"raster_sched": 1},
              {"raster_sched": 2}, {"tri_cap": 32, "raster_bands": 3, "raster_sched": 2}]


@pytest.mark.parametrize("scenario,E,A", [("Collect", 32, 4), ("HexMemory", 16, 2), ("TowerBuilding", 64, 1)])
def test_partitioning_and_scheduling_change_nothing(built, scenario, E, A):
    params = {"episodeLengthSec": 3.0}
    ref = _host_run(scenario, E, A, 40, params)
    assert any(((s >> 8) == SEG_AGENT).any() or ((s >> 8) == SEG_REWARD).any() for s in ref)
    for opts in PARTITIONS:
        got = _host_run(scenario, E, A, 40, params, **opts)
        for t, (a, b) in enumerate(zip(ref, got)):
            assert np.array_equal(a, b), "%s step %d: %d pixels differ" % (opts, t, int((a != b).sum()))


def test_every_delivery_path_gives_the_same_tensor(built):
    import torch

    E, A, steps, params = 64, 4, 30, {"episodeLengthSec": 2.0}
    ref = _host_run("Collect", E, A, steps, params, zero_copy=1)
    for opts in ({"zero_copy": 0, "host_slices": 0}, {"zero_copy": 0, "host_slices": 4}, {"zero_copy": 0, "host_slices": 16}):
        got = _host_run("Collect", E, A, steps, params, **opts)
        assert all(np.array_equal(a, b) for a, b in zip(ref, got)), opts
    # obs_to_host 0: the device tensor, copied down by mv_fetch_obs
    g = _engine("Collect", E, A, params=params, obs_to_host=0)
    for t, a in enumerate(_acts(E * A, steps)):
        g.step(a)
        g.fetch_obs()
        assert np.array_equal(np.array(g.segmentation()), ref[t + 1]), "obs_to_host 0, step %d" % t
    g.close()
    # mv_step_device at level_slots 4, read in stream order: each call's tensor cloned on the engine stream
    g = _engine("Collect", E, A, params=params, level_slots=4, obs_to_host=0)  # the first frame in HBM too
    d = torch.as_tensor(g.device_array("segmentation"), device="cuda")
    s = torch.cuda.ExternalStream(g.stream())
    act = torch.zeros(E * A, dtype=torch.int32, device="cuda")
    got = []
    with torch.cuda.stream(s):
        for a in _acts(E * A, steps):
            act.copy_(torch.from_numpy(a))
            g.step_device(act.data_ptr())
            got.append(d.clone())
    g.sync()
    for t, x in enumerate(got):
        assert np.array_equal(x.view(torch.int16).cpu().numpy().view(np.uint16), ref[t + 1]), "mv_step_device, call %d" % t
    g.close()


def test_re_renders(built):
    E, A, params = 16, 2, {"episodeLengthSec": 4.0}
    acts = _acts(E * A, 30)
    g = _engine("TowerBuilding", E, A, params=params)
    for a in acts[:10]:
        g.step(a)
    store = g.states_create(E)
    g.states_save(store, list(range(E)), list(range(E)))
    saved = np.array(g.segmentation()).copy()
    for a in acts[10:]:
        g.step(a)
    g.states_load(store, list(range(E)), list(range(E)))
    assert np.array_equal(np.array(g.segmentation()), saved), "mv_states_load"
    # mv_reset_envs with seeds: those envs' views equal a fresh engine's first frame
    envs, seeds = [1, 5, 12], [71, 72, 73]
    g.reset_envs(envs, seeds)
    seg = np.array(g.segmentation()).copy()
    g.close()
    from megaverse_b200 import capi

    f = capi.Engine("TowerBuilding", E, A, 128, 72, num_threads=4, params=params, segmentation=True)
    for e, s in zip(envs, seeds):
        f.seed_env(e, s)
    f.reset()
    fresh = np.array(f.segmentation())
    for e in envs:
        assert np.array_equal(seg[e * A:(e + 1) * A], fresh[e * A:(e + 1) * A]), "mv_reset_envs env %d" % e
    f.close()


def test_mixed_batch_equals_the_per_scenario_engines(built):
    from megaverse_b200 import capi

    E, A, steps = 16, 1, 20
    names = [MEGAVERSE8[i % 8] for i in range(E)]
    params = {"episodeLengthSec": 3.0}
    acts = _acts(E * A, steps)
    g = capi.Engine(names, E, A, 128, 72, num_threads=4, params=params, segmentation=True)
    for e in range(E):
        g.seed_env(e, 1000 + e)
    g.reset()
    mixed = [np.array(g.segmentation()).copy()]
    for a in acts:
        g.step(a)
        mixed.append(np.array(g.segmentation()).copy())
    g.close()
    for s in sorted(set(names)):
        envs = [e for e in range(E) if names[e] == s]
        h = capi.Engine(s, len(envs), A, 128, 72, num_threads=4, params=params, segmentation=True)
        for i, e in enumerate(envs):
            h.seed_env(i, 1000 + e)
        h.reset()
        assert np.array_equal(np.array(h.segmentation()), mixed[0][envs]), s
        for t, a in enumerate(acts):
            h.step(a.reshape(E, A)[envs].reshape(-1))
            assert np.array_equal(np.array(h.segmentation()), mixed[t + 1][envs]), "%s step %d" % (s, t)
        h.close()


def test_terminal_frames_leave_the_live_tensor_alone(built):
    import torch

    E, A, steps, params = 32, 2, 40, {"episodeLengthSec": 3.0}
    runs = []
    for final in (False, True):
        g = _engine("Collect", E, A, params=params, final=final, level_slots=4, obs_to_host=0)
        d = torch.as_tensor(g.device_array("segmentation"), device="cuda")
        s = torch.cuda.ExternalStream(g.stream())
        act, ends = torch.zeros(E * A, dtype=torch.int32, device="cuda"), torch.zeros(E, dtype=torch.uint8, device="cuda")
        out = []
        with torch.cuda.stream(s):
            for t, a in enumerate(_acts(E * A, steps)):
                act.copy_(torch.from_numpy(a))
                ends.copy_(torch.from_numpy((np.arange(E) % 5 == t % 5).astype(np.uint8)))
                g.step_device(act.data_ptr(), ends.data_ptr())
                out.append(d.clone())
        g.sync()
        runs.append([x.view(torch.int16).cpu().numpy() for x in out])
        g.close()
    for t, (a, b) in enumerate(zip(*runs)):
        assert np.array_equal(a, b), "call %d" % t


# ------------------------------------------------------------------------------------------------ 3. option off vs on
NO_CHANGE = [
    # case, scenario, E, A, depth, path, options
    ("config2", "TowerBuilding", 256, 1, False, "host", {}),
    ("config2-k4", "TowerBuilding", 256, 1, False, "host", {"action_repeat": 4}),
    ("config3", "ObstaclesHard", 2048, 1, True, "host", {"zero_copy": 0}),
    ("config3-k4-device", "ObstaclesHard", 2048, 1, True, "device", {"action_repeat": 4, "level_slots": 4}),
    ("config4", "Collect", 1024, 4, False, "host", {}),
    ("config4-k4-device", "Collect", 1024, 4, False, "device", {"action_repeat": 4, "level_slots": 4}),
]


@pytest.mark.parametrize("case,scenario,E,A,depth,path,options", NO_CHANGE, ids=[c[0] for c in NO_CHANGE])
def test_option_on_changes_nothing_else(built, case, scenario, E, A, depth, path, options):
    import torch

    acts = _acts(E * A, 32)
    # natural ends in the window: TowerBuilding and Collect add to the parameter per object / reward, Obstacles per platform
    params = {"TowerBuilding": {"episodeLengthSec": -180.0}, "Collect": {"episodeLengthSec": -1.5}}.get(
        scenario, {"episodeLengthSec": 1.0, "obstaclesMinNumPlatforms": 0, "obstaclesMaxNumPlatforms": 0})
    runs = []
    for seg in (False, True):
        g = _engine(scenario, E, A, seed=17, params=params, seg=seg, depth=depth, final=True, **options)
        rec = []
        for a in acts:
            if path == "host":
                g.step(a)
            else:
                d = torch.from_numpy(a).cuda()
                torch.cuda.synchronize()
                g.step_device(d.data_ptr())
                g.sync()
                g.fetch_obs()
            r = {"obs": np.array(g.obs()).copy(), "rewards": np.array(g.rewards()).copy(), "dones": np.array(g.dones()).copy(),
                 "reasons": np.array(g.done_reasons()).copy(), "true_obj": np.array(g.true_objectives()).copy(), "final": np.array(g.final_obs()).copy()}
            if depth:
                r["depth"] = np.array(g.depth()).copy()
                r["final_depth"] = np.array(g.final_depth()).copy()
            rec.append(r)
        assert g.faults() == 0
        runs.append(rec)
        g.close()
    assert any(r["dones"].any() for r in runs[0]), "the window is meant to hold episode ends"
    for t, (a, b) in enumerate(zip(*runs)):
        for k in a:
            assert np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)), "%s step %d: %s" % (case, t, k)


def test_option_values_order_and_getters(built):
    from megaverse_b200 import capi

    L = capi.lib()
    g = capi.Engine("Collect", 2, 1, 128, 72, num_threads=1)
    for bad in (2, -1, 7):
        with pytest.raises(capi.MegaverseError) as e:
            g.set_option("segmentation", bad)
        assert e.value.code == capi.MV_ERR_ARG
    g.set_option("segmentation", 0)
    g.seed(1)
    g.reset()
    for fn in ("segmentation",):
        with pytest.raises(capi.MegaverseError) as e:
            getattr(g, fn)()
        assert e.value.code == capi.MV_ERR_ARG
    with pytest.raises(capi.MegaverseError) as e:
        g.device_ptr("segmentation")
    assert e.value.code == capi.MV_ERR_ARG
    for v in (0, 1):
        assert L.mv_set_option(g._h, b"segmentation", v) == capi.MV_ERR_STATE
    g.close()
    # on: the host tensor after the first reset; the device pointer is refused while the HBM tensor is stale (zero-copy delivery)
    g = _engine("Collect", 2, 1)
    assert np.array(g.segmentation()).dtype == np.uint16
    with pytest.raises(capi.MegaverseError) as e:
        g.device_ptr("segmentation")
    assert e.value.code == capi.MV_ERR_STATE
    g.step_device()
    g.sync()
    assert g.device_ptr("segmentation")
    g.close()


def test_megaverse_env_segmentation(built):
    from megaverse_b200.megaverse_env import MegaverseEnv

    env = MegaverseEnv("Collect", 2, 2, 1, segmentation=True)
    obs = env.reset()
    seg = env.segmentation()
    assert len(seg) == len(obs) == 4 and seg[0].shape == (72, 128) and seg[0].dtype == np.uint16
    out = env.step([[0, 0, 1, 0, 0, 0]] * 4)
    assert len(out) == 4 and set(out[3][0]) <= {"true_reward"}
    assert all(((s >> 8) <= SEG_REWARD).all() for s in env.segmentation())
    env.close()
