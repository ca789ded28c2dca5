"""Per-env episode control: mv_reset_envs restarts chosen envs now (optionally reseeded) and mv_step_device_ends ends chosen envs' episodes
from a device mask.  A reseeded env equals that env of a fresh engine, an unseeded one continues its level stream, a requested end reads
like a timer end, and every env that was not named is byte-identical to an engine that made no call."""
import ctypes as C

import numpy as np
import pytest

import helpers

pytestmark = pytest.mark.gpu


def _engine(scenario, E, A, seed, params=None, depth=False, env_seeds=None, **options):
    from megaverse_b200 import capi

    g = capi.Engine(scenario, E, A, 128, 72, num_threads=2, params=params, depth=depth)
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


def _outputs(g, envs, dumps=True):
    """everything a step delivers, and the debug dumps of `envs` (float dumps as bit patterns)"""
    out = {"obs": np.array(g.obs()), "rewards": np.array(g.rewards()).view(np.uint32), "dones": np.array(g.dones()),
           "true_objectives": np.array(g.true_objectives()).view(np.uint32)}
    if dumps:
        for e in envs:
            out["state%d" % e] = g.state(e).view(np.uint32)
            out["voxels%d" % e] = g.voxels(e)
            out["instances%d" % e] = g.instances(e).view(np.uint32)
            out["level%d" % e] = g.level(e)
    return out


def _env(out, e, A, keys=("obs", "rewards", "dones", "true_objectives", "state", "voxels", "instances", "level")):
    """env e's part of _outputs, keyed without the env index"""
    r = {}
    for k in keys:
        if k == "dones":
            r[k] = out[k][e:e + 1]
        elif k in ("obs", "rewards", "true_objectives"):
            r[k] = out[k][e * A:(e + 1) * A]
        else:
            r[k] = out["%s%d" % (k, e)]
    return r


def _assert_equal(a, b, tag):
    assert a.keys() == b.keys(), tag
    for k in a:
        assert a[k].shape == b[k].shape and np.array_equal(a[k], b[k]), "%s: %s differs (%d elements)" % (
            tag, k, int((a[k] != b[k]).sum()) if a[k].shape == b[k].shape else -1)


def _healthy(g):
    assert g.fault_word() == 0
    assert g.faults() == 0


def _oracle_restart(o, e):
    """the oracle's Env::reset of env e alone, then a render (the other envs draw the same frames again)"""
    import orc

    L = orc.lib()
    L.orc_scen_reset.argtypes = [C.c_void_p, C.c_int]
    L.orc_scen_reset(o.h_, e)
    L.orc_render_now(o.h_)


def _ends(E, envs):
    """the device end mask: uint8[E] in HBM (the tests upload it with torch; the product takes a plain device pointer)"""
    import torch

    m = np.zeros(E, dtype=np.uint8)
    m[list(envs)] = 1
    return torch.from_numpy(m).cuda()


# short episodes, so that turnovers fall inside the window (the state store's replay cases)
ROUND_TRIP = [
    ("TowerBuilding", 1, {"episodeLengthSec": -180.0}),
    ("ObstaclesHard", 1, {"episodeLengthSec": 2.0, "obstaclesMinNumPlatforms": 0, "obstaclesMaxNumPlatforms": 0}),
    ("Collect", 4, {"episodeLengthSec": -45.0}),
    ("Sokoban", 1, {"episodeLengthSec": 2.0}),
    ("Rearrange", 1, {"episodeLengthSec": 2.0}),
    ("HexExplore", 1, {"episodeLengthSec": 1.0}),
    ("HexMemory", 1, {"episodeLengthSec": -50.0}),
    ("Empty", 1, {"episodeLengthSec": 1.0}),
]


@pytest.mark.parametrize("scenario,A,params", ROUND_TRIP, ids=[c[0] for c in ROUND_TRIP])
def test_reseeded_restart_equals_a_fresh_env(built, scenario, A, params):
    """two of six envs restarted with seeds at t0: from then on they equal those envs of a fresh engine given mv_seed_env and mv_reset,
    through turnovers; the other four equal an engine that made no call, byte for byte, at every step"""
    E, t0, M, restarted, seeds = 6, 4, 90, [1, 4], [1001, 2002]
    others = [e for e in range(E) if e not in restarted]
    g = _engine(scenario, E, A, 31, params)
    ref = _engine(scenario, E, A, 31, params)
    acts = _actions(E * A, t0 + M)
    for t in range(t0):
        g.step(acts[t]); ref.step(acts[t])
    g.reset_envs(restarted, seeds)
    fresh = _engine(scenario, E, A, 31, params, env_seeds=dict(zip(restarted, seeds)))
    # the true objective is the last finished episode's (it stays through a restart, as through mv_reset): compared once both ended one
    ended = {e: False for e in restarted}
    turnovers = 0
    for t in range(t0, t0 + M + 1):
        if t > t0:
            for x in (g, ref, fresh):
                x.step(acts[t - 1])
        out, want, new = _outputs(g, range(E)), _outputs(ref, others), _outputs(fresh, restarted)
        for e in others:
            _assert_equal(_env(out, e, A), _env(want, e, A), "step %d, env %d (not restarted)" % (t, e))
        for e in restarted:
            ended[e] = ended[e] or bool(out["dones"][e])
            keys = ("obs", "rewards", "dones", "state", "voxels", "instances", "level") + (("true_objectives",) if ended[e] else ())
            _assert_equal(_env(out, e, A, keys), _env(new, e, A, keys), "step %d, restarted env %d" % (t, e))
            turnovers += int(out["dones"][e])
        if t == t0:
            assert not out["dones"][restarted].any() and not out["rewards"].reshape(E, A)[restarted].any()
    assert turnovers >= 2, "the window is meant to hold turnovers of the restarted envs (%d)" % turnovers
    _healthy(g)
    for x in (g, ref, fresh):
        x.close()


def test_unseeded_restart_continues_the_stream_and_matches_the_oracle(built):
    """an env restarted in episode k plays episode k+1 of its own stream (capi.generate_level), and equals the oracle's env after
    Env::reset at the same step, through later turnovers"""
    import orc
    from megaverse_b200 import capi

    E, A, t0, M, e = 6, 1, 20, 40, 2
    params = {"episodeLengthSec": 1.0}
    env_seeds = {i: 500 + i for i in range(E)}
    g = _engine("HexExplore", E, A, 12, params, env_seeds=env_seeds, fast_shading=0)
    o = orc.Oracle("HexExplore", E, A, 128, 72, params=params)
    o.seed(12)
    for i, s in env_seeds.items():
        o.seed_env(i, s)
    o.reset()
    acts = _actions(E * A, t0 + M, seed=3)
    k = 0
    for t in range(t0):
        g.step(acts[t]); o.step(acts[t])
        k += int(g.dones()[e])
    assert k >= 1, "the restart is meant to come after a turnover"
    g.reset_envs([e])
    _oracle_restart(o, e)
    lvl = g.level(e)
    assert np.array_equal(lvl, capi.generate_level("HexExplore", A, env_seeds[e], k + 1, params)[:lvl.size]), "episode %d of the stream" % (k + 1)
    assert g.rewards()[e] == 0 and g.dones()[e] == 0
    turnovers = 0
    for t in range(t0, t0 + M + 1):
        if t > t0:
            g.step(acts[t - 1]); o.step(acts[t - 1])
            assert np.array_equal(g.rewards().view(np.uint32), o.rewards().view(np.uint32)), "step %d rewards" % t
            assert np.array_equal(g.dones(), o.dones()), "step %d dones" % t
            turnovers += int(g.dones()[e])
        for i in range(E):
            assert np.array_equal(g.state(i).view(np.uint32), o.state(i).view(np.uint32)), "step %d: state of env %d" % (t, i)
        diff = np.abs(np.array(g.obs()).astype(np.int16) - o.obs().astype(np.int16))
        assert diff.max() <= 1, "step %d: max RGB diff %d" % (t, diff.max())
    assert turnovers >= 1
    _healthy(g)
    g.close(); o.close()


def test_device_end_request_reads_like_a_timer_end(built):
    """d_ends[e] = 1 at step t1: done 1, reward 0, the true objective of the finished episode, the new level's first frame; afterwards the
    env equals an engine that stepped normally and then called mv_reset_envs([e]), and the oracle.  Requests 1 and 2 steps after that end
    are ignored, one 3 steps after it is honoured."""
    import orc
    import torch

    E, A, M, e, t1 = 6, 1, 30, 2, 10
    params = {"episodeLengthSec": 3.0}  # 45 steps: no natural end in the window
    g = _engine("HexExplore", E, A, 12, params, fast_shading=0)
    ref = _engine("HexExplore", E, A, 12, params, fast_shading=0)
    o = orc.Oracle("HexExplore", E, A, 128, 72, params=params)
    o.seed(12)
    o.reset()
    acts = _actions(E * A, M, seed=4)
    dacts = torch.from_numpy(acts).cuda()
    requested = {t1: [e], t1 + 1: [e], t1 + 2: [e], t1 + 3: [e]}
    honoured = {t1, t1 + 3}
    masks = {t: _ends(E, envs) for t, envs in requested.items()}
    none = _ends(E, [])
    torch.cuda.synchronize()
    for t in range(M):
        g.step_device(dacts[t].data_ptr(), masks.get(t, none).data_ptr())
        g.sync()
        g.fetch_obs()
        ref.step(acts[t]); o.step(acts[t])
        out = _outputs(g, range(E))
        assert not o.dones().any() and not ref.dones().any(), "the window holds no natural end"
        if t in honoured:
            ostate = o.state(e)
            assert out["dones"][e] == 1 and out["rewards"][e] == 0, "step %d" % t
            assert out["true_objectives"][e] == np.float32(ostate[-8]).view(np.uint32), "true objective (solved) at step %d" % t
            ref.reset_envs([e])
            _oracle_restart(o, e)
        else:
            assert out["dones"][e] == 0, "step %d: a request %d steps into the episode is ignored" % (t, t - t1)
        want = _outputs(ref, range(E))
        for k in ("dones", "true_objectives"):
            out[k][e * (A if k != "dones" else 1)] = want[k][e * (A if k != "dones" else 1)]
        _assert_equal(out, want, "step %d against the host-stepped engine with mv_reset_envs" % t)
        keep = [i for i in range(E) if not (t in honoured and i == e)]  # the oracle's reward of a restarted env is its last step's
        assert np.array_equal(out["rewards"][keep], o.rewards().view(np.uint32)[keep]), "step %d oracle rewards" % t
        for i in range(E):
            assert np.array_equal(out["state%d" % i], o.state(i).view(np.uint32)), "step %d: oracle state of env %d" % (t, i)
        diff = np.abs(out["obs"].astype(np.int16) - o.obs().astype(np.int16))
        assert diff.max() <= 1, "step %d: max RGB diff %d" % (t, diff.max())
    _healthy(g)
    for x in (g, ref, o):
        x.close()


MEGAVERSE8 = ["TowerBuilding", "ObstaclesEasy", "ObstaclesHard", "Collect", "Sokoban", "HexMemory", "HexExplore", "Rearrange"]
NO_CHANGE = {"config2": ("TowerBuilding", 256, 1), "config4": ("Collect", 1024, 4), "megaverse8": ([MEGAVERSE8[i % 8] for i in range(64)], 64, 1)}


@pytest.mark.parametrize("case", list(NO_CHANGE))
def test_step_device_ends_without_requests_changes_nothing(built, case):
    """mv_step_device_ends with NULL and with an all-zero mask: obs, rewards, dones and true objectives byte-identical to mv_step_device
    over 200 steps"""
    import torch

    scenario, E, A = NO_CHANGE[case]
    steps = 200
    params = {"episodeLengthSec": 1.0}
    gs = [_engine(scenario, E, A, 9, params) for _ in range(3)]
    rng = np.random.default_rng(6)
    acts = torch.from_numpy(np.stack([helpers.random_bit_actions(rng, E * A) for _ in range(steps)])).cuda()
    zeros = _ends(E, [])
    torch.cuda.synchronize()
    obs = None
    dones = 0
    for t in range(steps):
        ptr = acts[t].data_ptr()
        gs[0].step_device(ptr)
        gs[1].step_device(ptr, 0)  # d_ends = NULL
        gs[2].step_device(ptr, zeros.data_ptr())
        for g in gs:
            g.sync()
        if obs is None:  # the HBM tensors hold frames from the first device-resident step on
            obs = [torch.as_tensor(g.device_array("obs"), device="cuda") for g in gs]
        assert torch.equal(obs[0], obs[1]) and torch.equal(obs[0], obs[2]), "step %d obs" % t
        for k in ("rewards", "dones", "true_objectives"):
            a = np.array(getattr(gs[0], k)())
            for g in gs[1:]:
                assert np.array_equal(a.view(np.uint8), np.array(getattr(g, k)()).view(np.uint8)), "step %d %s" % (t, k)
        dones += int(np.array(gs[0].dones()).sum())
    if case == "megaverse8":
        assert dones > 0, "the window is meant to hold episode ends"
    for g in gs:
        _healthy(g)
        g.close()


def test_asynchronous_loop_with_restarts_and_end_requests(built):
    """300 mv_step_device_ends steps, envs asked to end every 3 to 7 steps (and some asked 1 step after an end, which is ignored), restarts
    between steps: mv_sync succeeds, no fault, and the outputs equal a host-stepped replay that restarts the ended envs"""
    import torch

    E, A, steps = 8, 1, 300
    params = {"episodeLengthSec": 60.0}  # the ends come from the schedule only
    g = _engine("HexExplore", E, A, 21, params)
    ref = _engine("HexExplore", E, A, 21, params)
    acts = _actions(E * A, steps, seed=5)
    dacts = torch.from_numpy(acts).cuda()
    rng = np.random.default_rng(8)
    period = rng.integers(3, 8, size=E)
    restarts = {50: ([1, 5], [71, 72]), 120: ([0, 3, 6], None), 200: (list(range(E)), list(range(300, 300 + E)))}
    last = np.full(E, -1)  # step after which the env's current episode began
    sched, ends_at = [], []
    for t in range(steps):
        req = [e for e in range(E) if t - last[e] >= period[e]]
        honoured = list(req)
        req += [e for e in range(E) if t - last[e] == 1 and e % 2]  # too early: ignored
        for e in honoured:
            last[e] = t
        if t in restarts:
            for e in restarts[t][0]:
                last[e] = t
        sched.append(_ends(E, req)); ends_at.append(honoured)
    torch.cuda.synchronize()
    n_ends = 0
    for t in range(steps):
        g.step_device(dacts[t].data_ptr(), sched[t].data_ptr())
        ref.step(acts[t])
        if ends_at[t]:
            ref.reset_envs(ends_at[t])
            n_ends += len(ends_at[t])
        if t in restarts:
            g.reset_envs(*restarts[t]); ref.reset_envs(*restarts[t])
            out, want = _outputs(g, range(E)), _outputs(ref, range(E))
            for k in ("dones", "true_objectives"):
                del out[k], want[k]
            _assert_equal(out, want, "after the restart behind step %d" % t)
    g.sync()
    g.fetch_obs()
    out, want = _outputs(g, range(E)), _outputs(ref, range(E))
    assert list(np.flatnonzero(out["dones"])) == sorted(ends_at[-1])
    for k in ("dones", "true_objectives"):
        del out[k], want[k]
    _assert_equal(out, want, "after %d asynchronous steps" % steps)
    assert n_ends > 300
    _healthy(g)
    g.close(); ref.close()


@pytest.mark.parametrize("mode", ["zero_copy", "hbm", "caller_buffer"])
def test_restart_delivers_frames_and_depth_like_a_step(built, mode):
    """after mv_reset_envs the host buffer, the engine's HBM tensor or the caller's tensor hold the new frames and depth: those of an engine
    delivering to the host that made the same call"""
    import torch

    E, A, t0 = 4, 2, 12
    params = {"episodeLengthSec": -2.0}
    g = _engine("Collect", E, A, 4, params, depth=True)
    ref = _engine("Collect", E, A, 4, params, depth=True)
    if mode != "zero_copy":
        g.set_option("obs_to_host", 0)
    if mode == "caller_buffer":
        obs_buf = torch.zeros((E * A, 72, 128, 4), dtype=torch.uint8, device="cuda")
        depth_buf = torch.zeros((E * A, 72, 128), dtype=torch.float32, device="cuda")
        g.set_obs_buffer(obs_buf.data_ptr(), depth_buf.data_ptr())

    def frames():
        if mode == "zero_copy":
            return np.array(g.obs()), np.array(g.depth()).view(np.uint32)
        if mode == "caller_buffer":
            torch.cuda.synchronize()
            return obs_buf.cpu().numpy(), depth_buf.cpu().numpy().view(np.uint32)
        obs = torch.as_tensor(g.device_array("obs"), device="cuda").cpu().numpy()
        depth = torch.as_tensor(g.device_array("depth"), device="cuda").cpu().numpy()
        return obs, depth.view(np.uint32)

    acts = _actions(E * A, t0, seed=2)
    for t in range(t0):
        g.step(acts[t]); ref.step(acts[t])
    before, _ = frames()
    if mode == "caller_buffer":
        obs_buf.zero_(); depth_buf.zero_()
        torch.cuda.synchronize()  # the engine writes on its own stream
    g.reset_envs([1, 3], [11, 12]); ref.reset_envs([1, 3], [11, 12])
    obs, depth = frames()
    assert np.array_equal(obs, np.array(ref.obs())), "frames after the restart"
    assert np.array_equal(depth, np.array(ref.depth()).view(np.uint32)), "depth after the restart"
    assert (obs[..., 3] == 255).all()
    assert np.array_equal(obs[[0, 1, 4, 5]], before[[0, 1, 4, 5]]), "views of envs that were not restarted"
    assert not np.array_equal(obs[[2, 3]], before[[2, 3]]) and not np.array_equal(obs[[6, 7]], before[[6, 7]]), "views of the restarted envs"
    _healthy(g)
    g.close(); ref.close()


def test_restart_in_a_mixed_engine_and_the_state_store(built):
    """one env of each Megaverse-8 scenario restarted with a seed equals env 0 of a single-scenario fresh engine; a save after the restart
    and a load replay bit for bit"""
    E, A, t0, M = 8, 1, 5, 40
    params = {"episodeLengthSec": 2.0}
    g = _engine(MEGAVERSE8, E, A, 3, params)
    acts = _actions(E * A, t0 + 2 * M, seed=9)
    for t in range(t0):
        g.step(acts[t])
    seeds = [900 + e for e in range(E)]
    g.reset_envs(list(range(E)), seeds)
    fresh = [_engine(MEGAVERSE8[e], 1, A, 3, params, env_seeds={0: seeds[e]}) for e in range(E)]
    for t in range(t0, t0 + M + 1):
        if t > t0:
            g.step(acts[t - 1])
            for e in range(E):
                fresh[e].step(acts[t - 1][e * A:(e + 1) * A])
        out = _outputs(g, range(E))
        for e in range(E):
            keys = ("obs", "rewards", "dones", "state", "voxels", "instances", "level")
            _assert_equal(_env(out, e, A, keys), _env(_outputs(fresh[e], [0]), 0, A, keys), "step %d, %s env %d" % (t, MEGAVERSE8[e], e))
    store = g.states_create(E)
    g.states_save(store, range(E), range(E))
    at_save = _outputs(g, range(E))
    g.reset_envs([2, 6])
    recorded = []
    for t in range(t0 + M, t0 + 2 * M):
        g.step(acts[t])
        recorded.append(_outputs(g, range(E)))
    g.states_load(store, range(E), range(E))
    _assert_equal(at_save, _outputs(g, range(E)), "after load")
    g.reset_envs([2, 6])
    for i, t in enumerate(range(t0 + M, t0 + 2 * M)):
        g.step(acts[t])
        _assert_equal(recorded[i], _outputs(g, range(E)), "replayed step %d" % t)
    _healthy(g)
    g.close()
    for f in fresh:
        f.close()


def test_restart_that_grows_the_static_arrays(built):
    """a reseeded HexExplore env whose first maze has more walls than the static-box arrays hold: the call grows them, and the env equals a
    fresh engine's"""
    from megaverse_b200 import capi

    E, A, M = 2, 1, 40
    params = {"episodeLengthSec": 1.0}

    def walls(seed, ep):
        d = capi.generate_level("HexExplore", A, seed, ep, params)
        return int(d[9 + 8 * d[0] + 7 * d[1] + 3 * d[2] + 3 * A + 2])

    small = [s for s in range(1, 200) if walls(s, 0) <= 120 and walls(s, 1) <= 120][:2]
    big = next(s for s in range(1, 200) if walls(s, 0) > 256)
    g = _engine("HexExplore", E, A, 1, params, env_seeds={0: small[0], 1: small[1]}, static_cap=16)
    cap = g.static_cap()
    assert cap <= 256
    acts = _actions(E * A, M, seed=10)
    g.step(acts[0])
    g.reset_envs([1], [big])
    assert g.static_cap() > cap and g.static_cap() >= walls(big, 0), "the restart is meant to grow the arrays"
    fresh = _engine("HexExplore", E, A, 1, params, env_seeds={0: small[0], 1: big}, static_cap=16)
    for t in range(1, M + 1):
        if t > 1:
            g.step(acts[t - 1]); fresh.step(acts[t - 1])
        keys = ("obs", "rewards", "dones", "state", "voxels", "instances", "level")
        _assert_equal(_env(_outputs(g, [1]), 1, A, keys), _env(_outputs(fresh, [1]), 1, A, keys), "step %d" % t)
    _healthy(g)
    g.close(); fresh.close()


def test_reset_envs_refuses_bad_arguments_and_call_order(built):
    """MV_ERR_STATE before mv_reset and while mv_step_begin is outstanding; MV_ERR_ARG for n < 0, a null list, an env out of range or listed
    twice.  A refused call changes no output or dump; n == 0 does nothing."""
    from megaverse_b200 import capi

    E, A = 4, 1
    g = capi.Engine("Collect", E, A, 128, 72, num_threads=2)
    L = capi.lib()

    def code(fn, *args):
        with pytest.raises(capi.MegaverseError) as ei:
            fn(*args)
        return ei.value.code

    assert code(g.reset_envs, [0]) == capi.MV_ERR_STATE
    g.seed(5); g.reset()
    ref = _engine("Collect", E, A, 5)
    acts = _actions(E * A, 12, seed=1)
    for t in range(4):
        g.step(acts[t]); ref.step(acts[t])
    before = _outputs(g, range(E))
    one = (C.c_int32 * 1)(0)
    assert L.mv_reset_envs(g._h, one, None, -1) == capi.MV_ERR_ARG
    assert L.mv_reset_envs(g._h, None, None, 1) == capi.MV_ERR_ARG
    assert code(g.reset_envs, [E]) == capi.MV_ERR_ARG
    assert code(g.reset_envs, [-1], [3]) == capi.MV_ERR_ARG
    assert code(g.reset_envs, [1, 2, 1]) == capi.MV_ERR_ARG
    g.reset_envs([])
    assert L.mv_reset_envs(g._h, None, None, 0) == capi.MV_OK
    _assert_equal(before, _outputs(g, range(E)), "after the refused calls")
    g.step_begin(acts[4])
    assert code(g.reset_envs, [0]) == capi.MV_ERR_STATE
    g.step_end()
    ref.step(acts[4])
    for t in range(5, 12):
        g.step(acts[t]); ref.step(acts[t])
        _assert_equal(_outputs(ref, range(E)), _outputs(g, range(E)), "step %d after the refused calls" % t)
    _healthy(g)
    g.close(); ref.close()


def test_megaverse_env_reset_envs(built):
    """MegaverseEnv.reset_envs returns every agent's observations; the reseeded env equals a fresh engine's, and the dones and infos of the
    following steps agree with each other"""
    from megaverse_b200 import MegaverseEnv, capi

    E, A = 3, 2
    params = {"episodeLengthSec": -45.0}
    env = MegaverseEnv("Collect", E, A, 2, params=params)
    env.seed(17)
    env.reset()
    rng = np.random.default_rng(4)
    actions = [rng.integers(0, [3, 3, 3, 2, 2, 3], size=(env.num_agents, 6)) for _ in range(60)]
    for a in actions[:5]:
        env.step(a)
    obs = env.reset_envs([1], seeds=[99])
    fresh = capi.Engine("Collect", E, A, 128, 72, num_threads=2, params=params)
    fresh.seed(17); fresh.seed_env(1, 99); fresh.reset()

    def same(o, eng):
        f = np.transpose(np.array(eng.obs())[:, :, :, :3], (0, 3, 1, 2))
        return all(np.array_equal(o[v], f[v]) for v in (2, 3))

    assert len(obs) == env.num_agents and same(obs, fresh)
    done_seen = False
    for a in actions[5:]:
        o, r, d, info = env.step(a)
        fresh.step(np.array([helpers.encode(x) for x in a], dtype=np.int32))
        assert same(o, fresh) and r[2:4] == list(np.array(fresh.rewards())[2:4]) and d[2] == bool(fresh.dones()[1])
        for i in range(env.num_agents):
            assert d[i] == d[i - i % A] and (("true_reward" in info[i]) == d[i])
            if d[i]:
                assert info[i]["true_reward"] == env.env.true_objective(i // A, i % A)
        done_seen = done_seen or any(d)
    assert done_seen, "the window is meant to hold an episode end"
    env.close(); fresh.close()
