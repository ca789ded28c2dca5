"""Terminal frames (option "final_obs") and end reasons: the frame an episode ended on, drawn before the flip to the next level, and why it
ended (1 time limit, 2 solved, 3 requested).  Checked against the oracle's scene before its Env::reset, against a twin engine whose episode
did not end, through a sentinel fill of the buffers, and for byte-identical other outputs with the option on."""
import ctypes as C

import numpy as np
import pytest

import helpers
import test_events_gpu as ev

pytestmark = pytest.mark.gpu


def _engine(scenario, E, A, seed, params=None, depth=False, final=True, env_seeds=None, **options):
    from megaverse_b200 import capi

    g = capi.Engine(scenario, E, A, 128, 72, num_threads=2, params=params, depth=depth)
    if final:
        g.set_option("final_obs", 1)
    for k, v in options.items():
        g.set_option(k, v)
    g.seed(seed)
    for e, s in (env_seeds or {}).items():
        g.seed_env(e, s)
    g.reset()
    return g


def _actions(n, steps, seed=7):
    rng = np.random.default_rng(seed)
    return np.stack([helpers.purposeful_actions(rng, n, t) for t in range(steps)]).astype(np.int32)


def _ends(E, envs):
    import torch

    m = np.zeros(E, dtype=np.uint8)
    m[list(envs)] = 1
    return torch.from_numpy(m).cuda()


def _healthy(g):
    assert g.fault_word() == 0
    assert g.faults() == 0


def _frames_match(a, b, fast, tag):
    if fast:
        diff = np.abs(a.astype(np.int16) - b.astype(np.int16))
        assert diff.max() <= 1, "%s: max RGB diff %d" % (tag, diff.max())
    else:
        assert np.array_equal(a, b), "%s: frames differ in %d bytes" % (tag, int((a != b).sum()))


# ------------------------------------------------------------------------------------------------ 1. against the oracle
class FinalRun(ev.Run):
    """test_events_gpu's warped run with the engine armed for terminal frames, and a mirror oracle driven env by env (orc_scen_step) whose
    ended env is drawn BEFORE its Env::reset -- the scene the oracle's orc_step throws away"""

    def __init__(self, scenario, E, A, seed, params, fast_shading=False, static_cap=None):
        import orc
        from megaverse_b200 import capi

        base = capi.Engine

        class Armed(base):
            def __init__(self, *a, **k):
                super().__init__(*a, **k)
                self.set_option("final_obs", 1)
                if static_cap:
                    self.set_option("static_cap", static_cap)

        capi.Engine = Armed
        try:
            super().__init__(scenario, E, A, seed, params=params, fast_shading=fast_shading)
        finally:
            capi.Engine = base
        L = self.O
        L.orc_scen_step.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        L.orc_scen_reset.argtypes = [C.c_void_p, C.c_int]
        self.m = orc.Oracle(scenario, E, A, params=params, render=False, depth=True, threads=1)
        for e in range(E):
            self.m.seed_env(e, seed + 7919 * e)
        self.m.reset()
        self.reasons = {1: 0, 2: 0, 3: 0}
        self.static_cap0 = static_cap

    def close(self):
        self.m.close()
        super().close()

    def warp(self, e, a, x, y, z, yaw):
        self.O.orc_scen_warp(self.m.h_, e, a, float(x), float(y), float(z), float(yaw))
        super().warp(e, a, x, y, z, yaw)

    def terminal(self, e):
        """the mirror's env e as it stands (after the step, before the reset): A frames and depth maps"""
        inst = np.zeros(18 * 4096, dtype=np.float32)
        n = self.O.orc_get_instances(self.m.h_, e, inst.ctypes.data, inst.size)
        assert n >= 0
        rgba = np.zeros((self.A, 72, 128, 4), dtype=np.uint8)
        depth = np.zeros((self.A, 72, 128), dtype=np.float32)
        view = np.zeros(16, dtype=np.float32)
        for a in range(self.A):
            self.O.orc_get_view(self.m.h_, e, a, view.ctypes.data)
            self.O.orc_render_instances(view.ctypes.data, inst.ctypes.data, n // 18, 128, 72, rgba[a].ctypes.data, depth[a].ctypes.data)
        return rgba, depth

    def step(self, acts, tag, host=True):
        d = super().step(acts, tag, host)  # the oracle and the engine step; rewards, dones and true objectives compared
        acts = np.ascontiguousarray(acts, dtype=np.int32)
        E, A = self.E, self.A
        for e in range(E):
            self.O.orc_scen_step(self.m.h_, e, acts[e * A:].ctypes.data)
        to = self.o.true_objectives()
        want = np.array([0 if not d[e] else (1 if self.fam == "tower" or to[e * A] == 0 else 2) for e in range(E)], dtype=np.uint8)
        got = np.array(self.g.done_reasons())
        assert np.array_equal(got, want), "%s: reasons %s, oracle %s" % (tag, got, want)
        if d.any():
            fo, fd = np.array(self.g.final_obs()), np.array(self.g.final_depth())
            for e in np.flatnonzero(d):
                self.reasons[int(want[e])] += 1
                rgba, depth = self.terminal(e)
                _frames_match(rgba, fo[e * A:(e + 1) * A], self.fast, "%s env %d terminal frame" % (tag, e))
                assert np.array_equal(depth.view(np.uint32), fd[e * A:(e + 1) * A].view(np.uint32)), "%s env %d terminal depth" % (tag, e)
                self.O.orc_scen_reset(self.m.h_, e)
        return d


ORACLE_CASES = [
    # scenario, A, E, ticks, seed, params, fast shading, static_cap
    ("TowerBuilding", 4, 4, 160, 301, {"episodeLengthSec": -180.0}, False, None),
    ("ObstaclesHard", 1, 8, 200, 302, {"episodeLengthSec": 4.0, "obstaclesMinNumPlatforms": 0, "obstaclesMaxNumPlatforms": 0}, False, None),
    ("ObstaclesEasy", 4, 4, 160, 303, {"episodeLengthSec": 4.0}, False, None),
    ("Collect", 8, 4, 160, 304, {"episodeLengthSec": -45.0}, False, None),
    ("Sokoban", 1, 8, 200, 305, {"episodeLengthSec": 4.0}, False, None),
    ("Rearrange", 1, 8, 240, 306, {"episodeLengthSec": 5.0}, False, None),
    ("HexExplore", 4, 6, 160, 307, {"episodeLengthSec": 3.0}, False, 16),
    ("HexMemory", 1, 8, 200, 308, {"episodeLengthSec": -50.0}, False, None),
    ("Empty", 8, 2, 100, 309, {"episodeLengthSec": 1.0}, False, None),
    ("Collect", 4, 4, 120, 310, {"episodeLengthSec": -45.0}, True, None),
]


@pytest.mark.parametrize("scenario,A,E,ticks,seed,params,fast,static_cap", ORACLE_CASES,
                         ids=["%s-A%d%s" % (c[0], c[1], "-fast" if c[6] else "") for c in ORACLE_CASES])
def test_terminal_frames_and_reasons_match_the_oracle(built, scenario, A, E, ticks, seed, params, fast, static_cap):
    """every done step: the terminal frames byte-exact (+-1 LSB with fast shading) and depth exact against the oracle's scene before its reset;
    reasons, rewards, dones and true objectives every tick; solved ends appear where a rule can solve the level"""
    run = FinalRun(scenario, E, A, seed, params, fast_shading=fast, static_cap=static_cap)
    try:
        run.checkpoint("%s reset" % scenario)
        ev.drive(run, ticks, np.random.default_rng(seed))
        print(run.table(), run.reasons)
        assert run.dones > 0, "the window is meant to hold episode ends"
        # the reasons were checked tick by tick above; Run's clock-jump count misses solves in an episode's last 0.3 s
        assert run.reasons[2] >= run.early_ends
        if run.fam in ev.SOLVED and run.fam != "hexmemory":  # a HexMemory solve needs every good object: test_events_gpu warps for it
            assert run.reasons[2] > 0, "no solved end in the window\n" + run.table()
        if static_cap:  # the first maze already has more walls than static_cap: the arrays grew with the terminal rows allocated
            assert run.g.static_cap() > run.static_cap0, "the run is meant to grow the static arrays while armed"
    finally:
        run.close()


# ------------------------------------------------------------------------------------------------ 2. against a twin whose episode did not end
MEGAVERSE8 = ["TowerBuilding", "ObstaclesEasy", "ObstaclesHard", "Collect", "Sokoban", "HexMemory", "HexExplore", "Rearrange"]
TWINS = {"hex": ("HexExplore", 6, 2, {"episodeLengthSec": 60.0}), "megaverse8": (MEGAVERSE8, 8, 1, {"episodeLengthSec": 60.0})}


@pytest.mark.parametrize("fast", [0, 1], ids=["exact", "fast"])
@pytest.mark.parametrize("case", list(TWINS))
def test_requested_end_frame_equals_the_twin_that_went_on(built, case, fast):
    """two engines on the same actions, one asked to end envs through d_ends: at each honoured request the terminal frame equals the other's
    obs byte for byte and the reason is 3; the twin then restarts the env (mv_reset_envs) and both go on equal.  Requests before an episode's
    third step write no row."""
    import torch

    scenario, E, A, params = TWINS[case]
    M = 60
    g = _engine(scenario, E, A, 14, params, depth=True, fast_shading=fast)
    ref = _engine(scenario, E, A, 14, params, depth=True, final=False, fast_shading=fast)
    acts = _actions(E * A, M, seed=11)
    dacts = torch.from_numpy(acts).cuda()
    rng = np.random.default_rng(3)
    last = np.zeros(E, dtype=np.int64)  # num_frames of the current episode after the step
    torch.as_tensor(g.device_array("final_obs"), device="cuda").fill_(0x5A)
    torch.cuda.synchronize()
    prev = None
    honoured_total = ignored_total = 0
    for t in range(M):
        req = [e for e in range(E) if rng.random() < 0.25]
        masks = _ends(E, req)
        torch.cuda.synchronize()
        g.step_device(dacts[t].data_ptr(), masks.data_ptr())
        ref.step(acts[t])
        g.sync()
        g.fetch_obs()
        last += 1
        honoured = [e for e in req if last[e] >= 3]
        ignored = [e for e in req if last[e] < 3]
        dn, why = np.array(g.dones()), np.array(g.done_reasons())
        assert list(np.flatnonzero(dn)) == honoured, "step %d: dones %s, honoured %s" % (t, np.flatnonzero(dn), honoured)
        assert (why[honoured] == 3).all() and (why[dn == 0] == 0).all(), "step %d reasons %s" % (t, why)
        fo, fd, want, wantd = np.array(g.final_obs()), np.array(g.final_depth()), np.array(ref.obs()), np.array(ref.depth())
        for e in honoured:
            assert np.array_equal(fo[e * A:(e + 1) * A], want[e * A:(e + 1) * A]), "step %d env %d: terminal frame vs the twin" % (t, e)
            assert np.array_equal(fd[e * A:(e + 1) * A].view(np.uint32), wantd[e * A:(e + 1) * A].view(np.uint32)), "step %d env %d depth" % (t, e)
            last[e] = 0
        if prev is not None:  # envs that did not end, ignored requests included: rows as before
            for e in range(E):
                if e not in honoured:
                    assert np.array_equal(fo[e * A:(e + 1) * A], prev[e * A:(e + 1) * A]), "step %d env %d: a row without an end changed" % (t, e)
        prev = fo.copy()
        honoured_total += len(honoured)
        ignored_total += len(ignored)
        if honoured:
            ref.reset_envs(honoured)
        out, want = np.array(g.obs()), np.array(ref.obs())
        assert np.array_equal(out, want), "step %d: obs after the end / restart" % t
    assert honoured_total > 5 and ignored_total > 0
    _healthy(g)
    g.close(); ref.close()


# ------------------------------------------------------------------------------------------------ 3. sentinel
@pytest.mark.parametrize("path", ["host", "device"])
def test_exactly_the_ended_envs_rows_change(built, path):
    """the final buffers are filled with a pattern before every step: afterwards exactly the views of the envs that ended differ from it"""
    import torch

    E, A, M = 12, 2, 90
    # host: short natural episodes; device: long ones, staggered requested ends (the asynchronous call needs episodes of >= 3 steps)
    g = _engine("Collect", E, A, 5, {"episodeLengthSec": -45.0 if path == "host" else 600.0}, depth=True)
    acts = _actions(E * A, M, seed=12)
    dacts = torch.from_numpy(acts).cuda()
    bank = torch.stack([_ends(E, [e for e in range(E) if (e + t) % 7 == 0]) for t in range(7)])
    if path == "device":
        fo, fd = torch.as_tensor(g.device_array("final_obs"), device="cuda"), torch.as_tensor(g.device_array("final_depth"), device="cuda")
    ended = 0
    for t in range(M):
        if path == "host":
            h_o, h_d = g.final_obs(), g.final_depth()
            h_o[...] = 0xA5
            h_d[...] = np.float32(-7.25)
            g.step(acts[t])
        else:
            fo.fill_(0xA5); fd.fill_(-7.25)
            torch.cuda.synchronize()
            g.step_device(dacts[t].data_ptr(), bank[t % 7].data_ptr())
            g.sync()
            g.fetch_obs()
        o, d, dn = np.array(g.final_obs()), np.array(g.final_depth()), np.array(g.dones())
        changed = np.array([(o[v] != 0xA5).any() for v in range(E * A)])
        changed_d = np.array([(d[v] != np.float32(-7.25)).any() for v in range(E * A)])
        want = np.repeat(dn != 0, A)
        assert np.array_equal(changed, want) and np.array_equal(changed_d, want), "step %d: rows changed %s, ended %s" % (t, changed, want)
        if dn.any():
            assert (o[want][..., 3] == 255).all()
        ended += int(dn.sum())
    assert ended >= 4
    _healthy(g)
    g.close()


# ------------------------------------------------------------------------------------------------ 4. the option changes nothing else
NO_CHANGE = [
    # case, scenario, E, A, path, depth, options
    ("config2-host-hbm", "TowerBuilding", 256, 1, "host", False, {"zero_copy": 0}),  # natural ends: episodeLengthSec -180 below
    ("config2-device", "TowerBuilding", 256, 1, "device", False, {}),
    ("config4-host-hbm", "Collect", 1024, 4, "host", False, {"zero_copy": 0}),  # 151 MB per step: four slices by size
    ("config4-device", "Collect", 1024, 4, "device", False, {}),
    ("megaverse8-host-depth", [MEGAVERSE8[i % 8] for i in range(64)], 64, 1, "host", True, {}),
    ("megaverse8-device-depth", [MEGAVERSE8[i % 8] for i in range(64)], 64, 1, "device", True, {}),
]


@pytest.mark.parametrize("case,scenario,E,A,path,depth,options", NO_CHANGE, ids=[c[0] for c in NO_CHANGE])
def test_option_on_changes_nothing_else(built, case, scenario, E, A, path, depth, options):
    """obs, depth, rewards, dones and true objectives byte-identical with the option on and off over 200 steps with episode ends (natural
    ones, and on the device path also requested ones for every env every 10 steps)"""
    import torch

    steps = 200
    params = {"episodeLengthSec": -180.0 if case == "config2-host-hbm" else 1.0}
    on = _engine(scenario, E, A, 9, params, depth=depth, final=True, **options)
    off = _engine(scenario, E, A, 9, params, depth=depth, final=False, **options)
    rng = np.random.default_rng(6)
    acts = np.stack([helpers.random_bit_actions(rng, E * A) for _ in range(steps)]).astype(np.int32)
    dacts = torch.from_numpy(acts).cuda()
    bank = torch.stack([_ends(E, [e for e in range(E) if (e + t) % 10 == 0]) for t in range(10)])
    torch.cuda.synchronize()
    dones = 0
    for t in range(steps):
        for g in (on, off):
            if path == "host":
                g.step(acts[t])
            else:
                g.step_device(dacts[t].data_ptr(), bank[t % 10].data_ptr())
                g.sync()
        keys = ["rewards", "dones", "true_objectives"]
        if path == "host" or t % 20 == 19:
            if path == "device":
                for g in (on, off):
                    g.fetch_obs()
            keys += ["obs"] + (["depth"] if depth else [])
        for k in keys:
            a, b = np.array(getattr(on, k)()), np.array(getattr(off, k)())
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), "%s step %d: %s differs" % (case, t, k)
        dones += int(np.array(on.dones()).sum())
    assert dones > 0, "the window is meant to hold episode ends"
    for g in (on, off):
        _healthy(g)
        g.close()


# ------------------------------------------------------------------------------------------------ 5. other paths
def test_asynchronous_loop_with_ends_and_restarts(built):
    """300 mv_step_device_ends steps with requests every 3 to 7 steps and restarts between them: after mv_sync + mv_fetch_obs every env's
    terminal row equals the frame a host-stepped twin showed at that env's last end"""
    import torch

    E, A, steps = 8, 1, 300
    params = {"episodeLengthSec": 60.0}
    g = _engine("HexExplore", E, A, 21, params)
    ref = _engine("HexExplore", E, A, 21, params, final=False)
    acts = _actions(E * A, steps, seed=5)
    dacts = torch.from_numpy(acts).cuda()
    rng = np.random.default_rng(8)
    period = rng.integers(3, 8, size=E)
    restarts = {50: ([1, 5], [71, 72]), 120: ([0, 3, 6], None), 200: (list(range(E)), list(range(300, 300 + E)))}
    last = np.full(E, -1)
    sched, ends_at = [], []
    for t in range(steps):
        req = [e for e in range(E) if t - last[e] >= period[e]]
        for e in req:
            last[e] = t
        if t in restarts:
            for e in restarts[t][0]:
                last[e] = t
        sched.append(_ends(E, req)); ends_at.append(req)
    torch.cuda.synchronize()
    expect = {}
    for t in range(steps):
        g.step_device(dacts[t].data_ptr(), sched[t].data_ptr())
        ref.step(acts[t])
        if ends_at[t]:
            o = np.array(ref.obs())
            for e in ends_at[t]:
                expect[e] = o[e * A:(e + 1) * A].copy()
            ref.reset_envs(ends_at[t])
        if t in restarts:
            g.reset_envs(*restarts[t]); ref.reset_envs(*restarts[t])
    g.sync()
    g.fetch_obs()
    fo = np.array(g.final_obs())
    assert len(expect) == E
    for e, want in expect.items():
        assert np.array_equal(fo[e * A:(e + 1) * A], want), "env %d: terminal row of its last end" % e
    assert np.array_equal(np.array(g.done_reasons()) != 0, np.array(g.dones()) != 0)
    assert (np.array(g.done_reasons())[np.array(g.dones()) != 0] == 3).all()
    assert np.array_equal(np.array(g.obs()), np.array(ref.obs()))
    _healthy(g)
    g.close(); ref.close()


def test_reasons_through_the_state_store_and_restarts_and_device_arrays(built):
    """a state row carries the reasons (after mv_states_load they read as after the saved step), mv_reset_envs gives 0 for the restarted envs,
    the device arrays of reasons and true objectives equal the host ones, and "final_obs" after the first reset is MV_ERR_STATE"""
    import torch

    from megaverse_b200 import capi

    E, A = 8, 2
    g = _engine("Collect", E, A, 2, {"episodeLengthSec": -45.0})
    with pytest.raises(capi.MegaverseError) as ei:
        g.set_option("final_obs", 0)
    assert ei.value.code == capi.MV_ERR_STATE
    acts = _actions(E * A, 200, seed=13)
    store = g.states_create(E)
    saved = None
    for t in range(200):
        g.step(acts[t])
        why = np.array(g.done_reasons())
        assert np.array_equal(why != 0, np.array(g.dones()) != 0)
        dr = torch.as_tensor(g.device_array("done_reasons"), device="cuda").cpu().numpy()
        to = torch.as_tensor(g.device_array("true_objectives"), device="cuda").cpu().numpy()
        assert np.array_equal(dr, why) and np.array_equal(to.view(np.uint32), np.array(g.true_objectives()).view(np.uint32)), "step %d" % t
        if saved is None and why.any():
            g.states_save(store, range(E), range(E))
            saved = why.copy()
    assert saved is not None, "the window is meant to hold an end"
    g.states_load(store, range(E), range(E))
    assert np.array_equal(np.array(g.done_reasons()), saved), "reasons after the load"
    ended = list(np.flatnonzero(saved))
    g.reset_envs(ended)
    assert not np.array(g.done_reasons())[ended].any() and not np.array(g.dones())[ended].any()
    _healthy(g)
    g.close()


def test_megaverse_env_infos(built):
    """final_observation=True: infos of done agents carry the terminal frame (CHW), terminated and truncated; without it the infos are as
    before, and observations, rewards and dones agree between the two"""
    from megaverse_b200 import MegaverseEnv

    E, A = 4, 2
    params = {"episodeLengthSec": -45.0}
    on = MegaverseEnv("Collect", E, A, 2, params=params, final_observation=True)
    off = MegaverseEnv("Collect", E, A, 2, params=params)
    for env in (on, off):
        env.seed(23)
        env.reset()
    rng = np.random.default_rng(4)
    ends = 0
    for _ in range(120):
        a = rng.integers(0, [3, 3, 3, 2, 2, 3], size=(E * A, 6))
        o1, r1, d1, i1 = on.step(a)
        o2, r2, d2, i2 = off.step(a)
        assert r1 == r2 and d1 == d2 and all(np.array_equal(x, y) for x, y in zip(o1, o2))
        final = np.array(on.env.get_final_observations())
        reasons = np.array(on.env.get_done_reasons())
        for i in range(E * A):
            assert set(i2[i]) == ({"true_reward"} if d2[i] else set())
            if not d1[i]:
                assert i1[i] == {}
                continue
            ends += 1
            assert set(i1[i]) == {"true_reward", "final_observation", "terminated", "truncated"}
            assert i1[i]["true_reward"] == i2[i]["true_reward"]
            fo = i1[i]["final_observation"]
            assert fo.shape == (3, 72, 128) and np.array_equal(fo, np.transpose(final[i, :, :, :3], (2, 0, 1)))
            r = int(reasons[i // A])
            assert i1[i]["terminated"] == (r == 2) and i1[i]["truncated"] == (r in (1, 3)) and r in (1, 2)
    assert ends > 0
    on.close(); off.close()
