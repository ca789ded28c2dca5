"""Option "level_slots" 4: one live and three staged level slots per env, so that the asynchronous mv_step_device[_ends] takes episodes of
any length at any action_repeat k and honours every end request.

The engine under test is stepped asynchronously and never synchronised between calls (the level pipeline then runs as deep as it goes):
each call's device outputs are copied on the engine stream into preallocated history tensors and compared after the loop with a twin at
level_slots 2 stepped synchronously with mv_step on the same seeds and masks (fast_shading 0: frames byte for byte).  Every env's live level
after its ends is checked against capi.generate_level for consecutive episodes of its stream, which catches levels generated out of order."""
import numpy as np
import pytest

import helpers
import test_final_obs_gpu as fin

pytestmark = pytest.mark.gpu

KEYS = ("rewards", "dones", "done_reasons", "true_objectives")
MEGAVERSE8 = fin.MEGAVERSE8
SCENARIOS = ["TowerBuilding", "Collect", "Rearrange", "Sokoban", "HexExplore", "HexMemory", "Empty", "ObstaclesEasy", "ObstaclesMedium",
             "ObstaclesHard", "ObstaclesWalls", "ObstaclesSteps", "ObstaclesLava"]


def _engine(scenario, E, A, slots, k, params, seeds, final=False, device=False, **opts):
    """an engine at level_slots `slots` (None: option not set), action_repeat k, exact shading, env e seeded seeds[e]; device=True keeps
    frames in HBM (obs_to_host 0) so that the asynchronous loop reads them there from the reset on"""
    from megaverse_b200 import capi

    g = capi.Engine(scenario, E, A, 128, 72, num_threads=4, params=params)
    if slots is not None:
        g.set_option("level_slots", slots)
    g.set_option("action_repeat", k)
    g.set_option("fast_shading", 0)
    if final:
        g.set_option("final_obs", 1)
    if device:
        g.set_option("obs_to_host", 0)
    for key, v in opts.items():
        g.set_option(key, v)
    for e, s in enumerate(seeds):
        g.seed_env(e, int(s))
    g.reset()
    return g


class Recorder:
    """the device outputs of every asynchronous call, copied on the engine stream (no host synchronisation): rewards, dones, reasons, true
    objectives in full, and frames in full or as per-view byte sums; terminal frames in full with option final_obs"""

    def __init__(self, g, calls, sums=False, final=False):
        import torch

        self.torch, self.g, self.sums, self.final = torch, g, sums, final
        self.stream = torch.cuda.ExternalStream(g.stream())
        self.src = {key: torch.as_tensor(g.device_array(key), device="cuda") for key in KEYS}
        self.src["obs"] = torch.as_tensor(g.device_array("obs"), device="cuda")
        if final:
            self.src["final_obs"] = torch.as_tensor(g.device_array("final_obs"), device="cuda")
        shapes = {key: tuple(v.shape) for key, v in self.src.items()}
        if sums:
            shapes["obs"] = (g.N,)
        self.hist = {key: torch.empty((calls,) + s, dtype=torch.int64 if (sums and key == "obs") else self.src[key].dtype, device="cuda")
                     for key, s in shapes.items()}

    def record(self, t):
        with self.torch.cuda.stream(self.stream):
            for key, h in self.hist.items():
                if key == "obs" and self.sums:
                    h[t].copy_(self.src["obs"].view(self.g.N, -1).sum(1, dtype=self.torch.int64))
                else:
                    h[t].copy_(self.src[key])

    def numpy(self):
        self.g.sync()
        self.torch.cuda.synchronize()
        return {key: h.cpu().numpy() for key, h in self.hist.items()}


def _true_objective(twin, e, scenario):
    """what the step kernel reports at an end of env e: the tower's height, else whether the episode was solved"""
    st = twin.state(e)
    return np.float32(st[3]) if scenario.lower() == "towerbuilding" else np.float32(st[-8] != 0)


def _twin_call(twin, acts, requested, scenarios, sums=False, final=False, k=1):
    """one mv_step of the level_slots 2 twin; a requested end its own step did not make reads like a timer end (test_episode_control_gpu):
    done 1, reason 3, the episode's true objective, the step's frame as terminal frame, then mv_reset_envs and its first frame.  The reward
    is 0 at k = 1; at k > 1 it is the sum of the ticks before the ending one, which the twin does not single out: "free" lists those rows"""
    import torch

    twin.step(acts)
    A = twin.A
    out = {key: np.array(getattr(twin, key)()).copy() for key in KEYS}
    restart = [e for e in requested if not out["dones"][e]]
    frames = np.array(twin.obs()).copy() if not sums else None
    if final:
        out["final_obs"] = np.array(twin.final_obs()).copy()
    out["free"] = restart if k > 1 else []
    for e in restart:
        out["rewards"][e * A:(e + 1) * A] = 0.0
        out["dones"][e], out["done_reasons"][e] = 1, 3
        out["true_objectives"][e * A:(e + 1) * A] = _true_objective(twin, e, scenarios[e])
        if final:
            out["final_obs"][e * A:(e + 1) * A] = frames[e * A:(e + 1) * A]
    if restart:
        twin.reset_envs(restart)
    if sums:
        obs = torch.as_tensor(twin.device_array("obs"), device="cuda")
        out["obs"] = obs.view(twin.N, -1).sum(1, dtype=torch.int64).cpu().numpy()
    else:
        out["obs"] = np.array(twin.obs()).copy()
    return out


def _compare(got, want, A, final=False):
    """got: the recorder's history; want: the twin's calls.  Terminal frames only where the env ended"""
    for t, w in enumerate(want):
        for key in KEYS + ("obs",):
            a, b = got[key][t], w[key]
            if key == "rewards" and w["free"]:
                a = a.copy()
                for e in w["free"]:
                    a[e * A:(e + 1) * A] = b[e * A:(e + 1) * A]
            if not np.array_equal(a.view(np.uint8), b.view(np.uint8)):
                bad = np.flatnonzero((a != b).reshape(a.shape[0], -1).any(1))
                raise AssertionError("call %d: %s differs at rows %s" % (t, key, bad[:8]))
        if final:
            for e in np.flatnonzero(w["dones"]):
                assert np.array_equal(got["final_obs"][t][e * A:(e + 1) * A], w["final_obs"][e * A:(e + 1) * A]), "call %d env %d: terminal frame" % (t, e)


def _check_levels(g, scenarios, A, seeds, episodes, params):
    """env e's live level is episode episodes[e] of its stream"""
    from megaverse_b200 import capi

    g.sync()
    for e in range(g.E):
        lvl = g.level(e)
        want = capi.generate_level(scenarios[e], A, int(seeds[e]), int(episodes[e]), params)[:lvl.size]
        assert np.array_equal(lvl, want), "env %d: live level is not episode %d of its stream" % (e, episodes[e])


def _run(scenario, E, A, k, params, calls, requests=None, final=False, sums=False, seed=0, level_every=0):
    """the level_slots 4 engine asynchronously against the twin; requests: call -> env list.  Returns the outputs and ends per env"""
    import torch

    scenarios = [scenario] * E if isinstance(scenario, str) else list(scenario)
    seeds = 1000 + 37 * seed + np.arange(E)
    g = _engine(scenario, E, A, 4, k, params, seeds, final=final, device=True)
    twin = _engine(scenario, E, A, 2, k, params, seeds, final=final, device=sums)
    rec = Recorder(g, calls, sums=sums, final=final)
    rng = np.random.default_rng(seed)
    acts = np.stack([helpers.purposeful_actions(rng, E * A, t) for t in range(calls)]).astype(np.int32)
    dacts = torch.from_numpy(acts).cuda()
    requests = requests or {}
    masks = {t: fin._ends(E, envs) for t, envs in requests.items()}
    none = fin._ends(E, [])
    torch.cuda.synchronize()
    want = []
    for t in range(calls):
        g.step_device(dacts[t].data_ptr(), masks.get(t, none).data_ptr())
        rec.record(t)
        want.append(_twin_call(twin, acts[t], requests.get(t, []), scenarios, sums=sums, final=final, k=k))
        if level_every and t % level_every == level_every - 1:  # an occasional synchronisation point: the generation-order check mid-run
            _check_levels(g, scenarios, A, seeds, sum(w["dones"].astype(np.int64) for w in want), params)
    got = rec.numpy()
    _compare(got, want, A, final=final)
    ends = got["dones"].astype(np.int64).sum(0)
    _check_levels(g, scenarios, A, seeds, ends, params)
    for x in (g, twin):
        fin._healthy(x)
        x.close()
    return got, ends


# ------------------------------------------------------------------------------------------------ 1. what level_slots 2 refuses
@pytest.mark.parametrize("k", [1, 4])
def test_every_call_ends(built, k):
    """TowerBuilding with every episode ending on its first tick and an all-ones end mask on every call (the case the asynchronous call
    refuses at level_slots 2): 300 calls, no MV_ERR_STATE, no fault bit, every output equal to the twin's, the live levels those of
    consecutive episodes"""
    E, A, calls = 8, 1, 300
    got, ends = _run("TowerBuilding", E, A, k, {"episodeLengthSec": -400.0}, calls, requests={t: range(E) for t in range(calls)}, level_every=100)
    assert (got["dones"] == 1).all() and (ends == calls).all()


def _bench_actions(E, A):
    rng = np.random.default_rng(1)  # bench.py's action stream: one uniformly random action bit per agent per call
    return (1 << rng.integers(0, 11, size=(64, E * A))).astype(np.int32)


@pytest.mark.parametrize("k", [2, 4])
def test_bench_workload_with_action_repeat(built, k):
    """Collect 1 024 x 4 on bench.py's seeds (42 + env) and action stream at k = 2 and 4: the asynchronous level_slots 4 engine equals the
    level_slots 2 engine stepped with mv_step, bit for bit (frames as per-view byte sums), over 100 calls.  Episodes shorter than three calls
    (a level solved at once) are counted and printed; these 100 calls are not long enough to be sure of one"""
    import torch

    E, A, calls = 1024, 4, 100
    seeds = 42 + np.arange(E)
    g = _engine("Collect", E, A, 4, k, None, seeds, device=True, fast_shading=1)
    twin = _engine("Collect", E, A, 2, k, None, seeds, device=True, fast_shading=1)
    rec = Recorder(g, calls, sums=True)
    acts = _bench_actions(E, A)
    dacts = torch.from_numpy(acts).cuda()
    torch.cuda.synchronize()
    want = []
    for t in range(calls):
        g.step_device(dacts[t % 64].data_ptr())
        rec.record(t)
        want.append(_twin_call(twin, acts[t % 64], [], ["Collect"] * E, sums=True))
    got = rec.numpy()
    _compare(got, want, A)
    d = got["dones"].astype(bool)
    short = 0
    for e in range(E):
        t = np.flatnonzero(d[:, e])
        short += int((np.diff(t) < 3).sum())
    print("k=%d: %d ends, %d episodes shorter than three calls" % (k, int(d.sum()), short))
    _check_levels(g, ["Collect"] * E, A, seeds, d.sum(0), None)
    for x in (g, twin):
        fin._healthy(x)
        x.close()


# ------------------------------------------------------------------------------------------------ 2. every scenario family
FAMILIES = SCENARIOS + ["megaverse8"]
SHORT = {"episodeLengthSec": 0.5, "obstaclesMinNumPlatforms": 0, "obstaclesMaxNumPlatforms": 0}  # 8 ticks where the length is the parameter


def _short(scenario):
    """episodes of a few ticks: TowerBuilding, Collect and HexMemory add time per object to the parameter, so theirs end on their first tick"""
    return {"episodeLengthSec": -1000.0} if scenario in ("TowerBuilding", "Collect", "HexMemory") else SHORT


@pytest.mark.parametrize("A,k", [(1, 1), (1, 4), (4, 1), (4, 4)], ids=["A1-k1", "A1-k4", "A4-k1", "A4-k4"])
@pytest.mark.parametrize("scenario", FAMILIES)
def test_every_family_with_natural_ends(built, scenario, A, k):
    """short episodes (two calls or fewer at k = 4) with natural ends only, against the twin"""
    E = 8
    scen = [MEGAVERSE8[i % 8] for i in range(E)] if scenario == "megaverse8" else scenario
    got, ends = _run(scen, E, A, k, _short(scenario), 30, seed=FAMILIES.index(scenario))
    assert ends.sum() > 0


# ------------------------------------------------------------------------------------------------ 3. requests and terminal frames
@pytest.mark.parametrize("k", [1, 4])
def test_requests_in_any_call(built, k):
    """HexExplore: a request in the first call after the reset, in a new episode's first call and in consecutive calls, all honoured,
    against the twin that restarts the env with mv_reset_envs"""
    E, A, calls = 6, 1, 30
    requests = {0: [4], 5: [3], 6: [3], 10: [2], 11: [2, 3], 12: [2], 13: [2, 5]}
    got, ends = _run("HexExplore", E, A, k, {"episodeLengthSec": 3.0}, calls, requests=requests)
    for t, envs in requests.items():
        assert all(got["dones"][t][e] == 1 for e in envs), "call %d: a request was not honoured" % t


def test_terminal_frames_at_every_end(built):
    """final_obs at k = 4: HexExplore with 0.5 s episodes and requests on top, terminal frames and reasons at every end equal the twin's"""
    E, A, calls = 8, 2, 30
    requests = {t: [(t * 3) % E, (t * 5 + 1) % E] for t in range(0, calls, 3)}
    got, ends = _run("HexExplore", E, A, 4, SHORT, calls, requests=requests, final=True)
    assert set(np.unique(got["done_reasons"])) >= {1, 3}


# ------------------------------------------------------------------------------------------------ 4. reseeding
def test_reset_envs_mid_run(built):
    """level_slots 4, HexExplore with episodes of two calls, asynchronous: mv_reset_envs with seeds makes envs play as the same envs of a fresh engine
    seeded so; mv_reset_envs without seeds continues the env's stream.  Every live level is checked against the streams"""
    import torch

    E, A, k, calls = 6, 2, 4, 20
    params = SHORT
    seeds = 500 + np.arange(E)
    g = _engine("HexExplore", E, A, 4, k, params, seeds, device=True)
    rng = np.random.default_rng(3)
    acts = torch.from_numpy(np.stack([helpers.purposeful_actions(rng, E * A, t) for t in range(2 * calls)]).astype(np.int32)).cuda()
    torch.cuda.synchronize()
    rec = Recorder(g, calls)
    for t in range(calls):
        g.step_device(acts[t].data_ptr())
        rec.record(t)
    ends = rec.numpy()["dones"].astype(np.int64).sum(0)
    g.reset_envs([1, 4], [77, 78])
    g.reset_envs([2])
    ends[2] += 1
    fresh_seeds = seeds.copy()
    fresh_seeds[1], fresh_seeds[4] = 77, 78
    _check_levels(g, ["HexExplore"] * E, A, fresh_seeds, np.where(np.isin(np.arange(E), [1, 4]), 0, ends), params)
    fresh = _engine("HexExplore", E, A, 4, k, params, fresh_seeds, device=True)
    ra, rb = Recorder(g, calls), Recorder(fresh, calls)
    for t in range(calls, 2 * calls):
        for x, r in ((g, ra), (fresh, rb)):
            x.step_device(acts[t].data_ptr())
            r.record(t - calls)
    a, b = ra.numpy(), rb.numpy()
    for e in (1, 4):
        for key in KEYS + ("obs",):
            per = 1 if key in ("dones", "done_reasons") else A
            assert np.array_equal(a[key][:, e * per:(e + 1) * per].view(np.uint8), b[key][:, e * per:(e + 1) * per].view(np.uint8)), "env %d: %s" % (e, key)
    assert a["dones"][:, [1, 4]].sum() >= 4, "the restarted envs are meant to end a few times"
    _check_levels(g, ["HexExplore"] * E, A, fresh_seeds, np.where(np.isin(np.arange(E), [1, 4]), 0, ends) + a["dones"].astype(np.int64).sum(0), params)
    for x in (g, fresh):
        fin._healthy(x)
        x.close()


def test_seed_env_and_seed_redraw_every_staged_level(built):
    """after the reset, mv_seed_env redraws all three staged levels from the new stream in order, and mv_seed redraws every env's: with
    every call ending every episode, the levels after the reseed are episodes 0, 1, 2, 3, 4 of the new streams"""
    from megaverse_b200 import capi

    E, A = 4, 1
    params = {"episodeLengthSec": -400.0}
    seeds = 300 + np.arange(E)
    g = _engine("TowerBuilding", E, A, 4, 1, params, seeds)
    acts = np.zeros(E * A, dtype=np.int32)
    for _ in range(3):
        g.step(acts)
    g.seed_env(2, 99)
    for ep in range(5):
        g.step(acts)
        assert np.array_equal(g.level(2), capi.generate_level("TowerBuilding", A, 99, ep, params)[:g.level(2).size]), "episode %d" % ep
        assert np.array_equal(g.level(1), capi.generate_level("TowerBuilding", A, 301, 4 + ep, params)[:g.level(1).size])
    # mv_seed: the same env streams as a fresh engine seeded so, whose reset plays their episode 0
    g.seed(7)
    ref = capi.Engine("TowerBuilding", E, A, 128, 72, num_threads=2, params=params)
    ref.set_option("level_slots", 4)
    ref.seed(7)
    ref.reset()
    for ep in range(5):
        g.step(acts)
        for e in range(E):
            assert np.array_equal(g.level(e), ref.level(e)), "env %d, episode %d of the new stream" % (e, ep)
        ref.step(acts)
    for x in (g, ref):
        fin._healthy(x)
        x.close()


# ------------------------------------------------------------------------------------------------ 5. state store and static growth
def test_state_store_replays_and_clones(built):
    """level_slots 4, HexExplore at k = 4 with episodes of two calls: envs saved mid-episode and loaded back replay the same 30 asynchronous calls
    bit for bit, across more ends than the three staged levels; a row loaded into two envs makes them play alike"""
    import torch

    E, A, k, calls = 8, 2, 4, 30
    g = _engine("HexExplore", E, A, 4, k, SHORT, 700 + np.arange(E), device=True)
    rng = np.random.default_rng(5)
    acts = np.stack([helpers.purposeful_actions(rng, E * A, t) for t in range(10 + calls)]).astype(np.int32)
    acts[:, 2:4] = acts[:, 0:2]  # envs 0 and 1 take the same masks
    dacts = torch.from_numpy(acts).cuda()
    torch.cuda.synchronize()
    for t in range(10):
        g.step_device(dacts[t].data_ptr())
    store = g.states_create(E)
    g.states_save(store, range(E), range(E))
    runs = []
    for _ in range(2):
        rec = Recorder(g, calls)
        for t in range(calls):
            g.step_device(dacts[10 + t].data_ptr())
            rec.record(t)
        runs.append(rec.numpy())
        g.states_load(store, range(E), range(E))
    for key in KEYS + ("obs",):
        assert np.array_equal(runs[0][key].view(np.uint8), runs[1][key].view(np.uint8)), "the replay differs in %s" % key
    assert runs[0]["dones"].sum(0).min() >= 4, "every env is meant to go past its three staged levels"
    g.states_load(store, [0, 0], [0, 1])  # clone env 0 into env 1
    rec = Recorder(g, calls)
    for t in range(calls):
        g.step_device(dacts[10 + t].data_ptr())
        rec.record(t)
    c = rec.numpy()
    for key in KEYS + ("obs",):
        per = 1 if key in ("dones", "done_reasons") else A
        assert np.array_equal(c[key][:, 0:per].view(np.uint8), c[key][:, per:2 * per].view(np.uint8)), "the clone differs in %s" % key
    assert np.array_equal(c["dones"][:, 0], runs[0]["dones"][:, 0])
    fin._healthy(g)
    g.close()


def test_state_row_bytes_grow_by_two_slots(built):
    """TowerBuilding: a level slot is an MvLevel (33 248 B), static_cap static boxes (32 B) and rotations (8 B), one decoration (80 B) and
    three bit planes of 588 words (the grid's 18 750 cells rounded up to a multiple of 128)"""
    from megaverse_b200 import capi

    rows = {}
    for d in (2, 4):
        g = capi.Engine("TowerBuilding", 2, 1, 128, 72, num_threads=1)
        g.set_option("level_slots", d)
        rows[d] = g.state_row_bytes()
        g.close()
    assert rows[4] - rows[2] == 2 * (33248 + 40 * 768 + 80 + 12 * 588)


def test_static_growth(built):
    """static_cap 16, HexExplore (levels need hundreds of boxes): the arrays of all four slots are re-pitched while three of them hold staged
    levels, the outputs equal the twin's, and a state store saved at the grown pitch loads back"""
    import torch

    E, A, calls = 4, 1, 30
    params = {"episodeLengthSec": 0.5}
    seeds = 40 + np.arange(E)
    g = _engine("HexExplore", E, A, 4, 4, params, seeds, device=True, static_cap=16)
    twin = _engine("HexExplore", E, A, 2, 4, params, seeds, static_cap=16)
    assert g.static_cap() > 16 and g.static_cap() == twin.static_cap()
    store = g.states_create(E)
    g.states_save(store, range(E), range(E))
    rec = Recorder(g, calls)
    rng = np.random.default_rng(9)
    acts = np.stack([helpers.purposeful_actions(rng, E * A, t) for t in range(calls)]).astype(np.int32)
    dacts = torch.from_numpy(acts).cuda()
    torch.cuda.synchronize()
    want = []
    for t in range(calls):
        g.step_device(dacts[t].data_ptr())
        rec.record(t)
        want.append(_twin_call(twin, acts[t], [], ["HexExplore"] * E))
    _compare(rec.numpy(), want, A)
    g.states_load(store, range(E), range(E))  # the store kept the engine's pitch
    g.sync()
    for e in range(E):
        assert g.state(e)[2] == 0  # the saved env's tick counter, right after the reset
    for x in (g, twin):
        fin._healthy(x)
        x.close()


# ------------------------------------------------------------------------------------------------ 6. the option itself
def test_option_values_and_order(built):
    from megaverse_b200 import capi

    g = capi.Engine("Collect", 2, 2, num_threads=2)
    for bad in (0, 1, 3, 5, 8):
        with pytest.raises(capi.MegaverseError) as ei:
            g.set_option("level_slots", bad)
        assert ei.value.code == capi.MV_ERR_ARG
    for good in (4, 2, 4):
        g.set_option("level_slots", good)
    g.seed(1)
    g.reset()
    with pytest.raises(capi.MegaverseError) as ei:
        g.set_option("level_slots", 4)
    assert ei.value.code == capi.MV_ERR_STATE
    g.close()


@pytest.mark.parametrize("scenario,E,A", [("TowerBuilding", 256, 1), ("Collect", 1024, 4)], ids=["config2", "config4"])
def test_two_slots_change_nothing(built, scenario, E, A):
    """level_slots 2 set explicitly: every output byte-identical to an engine that never saw the option, over 60 asynchronous calls with
    requested ends every ten calls"""
    import torch

    steps = 60
    on = fin._engine(scenario, E, A, 9, {"episodeLengthSec": 1.0}, final=False, level_slots=2)
    off = fin._engine(scenario, E, A, 9, {"episodeLengthSec": 1.0}, final=False)
    rng = np.random.default_rng(6)
    acts = torch.from_numpy(np.stack([helpers.purposeful_actions(rng, E * A, t) for t in range(steps)]).astype(np.int32)).cuda()
    bank = torch.stack([fin._ends(E, [e for e in range(E) if (e + t) % 10 == 0]) for t in range(10)])
    torch.cuda.synchronize()
    dones = 0
    for t in range(steps):
        for g in (on, off):
            g.step_device(acts[t].data_ptr(), bank[t % 10].data_ptr())
            g.sync()
        keys = list(KEYS)
        if t % 10 == 9:
            for g in (on, off):
                g.fetch_obs()
            keys.append("obs")
        for key in keys:
            a, b = np.array(getattr(on, key)()), np.array(getattr(off, key)())
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), "step %d: %s differs" % (t, key)
        dones += int(np.array(on.dones()).sum())
    assert dones > 0
    for g in (on, off):
        fin._healthy(g)
        g.close()
