"""Env state store (mv_states_*): save envs mid-episode, rewind or clone them, and the envs continue bit for bit as the saved ones would
have -- frames, depth, rewards, dones, true objectives and the debug dumps -- across episode turnovers, array growth, the asynchronous loop
and every frame delivery mode."""
import numpy as np
import pytest

import helpers

pytestmark = pytest.mark.gpu


def _engine(scenario, E, A, seed, params=None, depth=False, **options):
    from megaverse_b200 import capi

    g = capi.Engine(scenario, E, A, 128, 72, num_threads=2, params=params, depth=depth)
    for k, v in options.items():
        g.set_option(k, v)
    g.seed(seed)
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


def _assert_equal(a, b, tag):
    assert a.keys() == b.keys(), tag
    for k in a:
        assert a[k].shape == b[k].shape and np.array_equal(a[k], b[k]), "%s: %s differs (%d elements)" % (
            tag, k, int((a[k] != b[k]).sum()) if a[k].shape == b[k].shape else -1)


def _healthy(g):
    assert g.fault_word() == 0
    assert g.faults() == 0


# short episodes, so that turnovers (and the generation of the levels after them) fall inside the replayed window
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
def test_rewind_replays_bit_identical(built, scenario, A, params):
    """save every env at t0, record M steps, load, replay the same actions: every output and dump is bit-identical, across turnovers, and
    the frame load returns is the frame of step t0"""
    E, t0, M = 4, 6, 90
    g = _engine(scenario, E, A, 31, params)
    acts = _actions(E * A, t0 + M)
    for t in range(t0):
        g.step(acts[t])
    at_t0 = _outputs(g, range(E))
    store = g.states_create(E)
    g.states_save(store, range(E), range(E))
    _assert_equal(at_t0, _outputs(g, range(E)), "save changed the engine's outputs")
    recorded, turnovers = [], 0
    for t in range(t0, t0 + M):
        g.step(acts[t])
        recorded.append(_outputs(g, range(E)))
        turnovers += int(recorded[-1]["dones"].sum())
    assert turnovers >= 2, "the window is meant to hold episode turnovers (%d)" % turnovers
    g.states_load(store, range(E), range(E))
    _assert_equal(at_t0, _outputs(g, range(E)), "after load")
    for i, t in enumerate(range(t0, t0 + M)):
        g.step(acts[t])
        _assert_equal(recorded[i], _outputs(g, range(E)), "replayed step %d" % t)
    _healthy(g)
    g.close()


def test_clone_runs_the_saved_env_and_matches_the_oracle(built):
    """env a's row loaded into envs b and c: given a's actions, b and c equal a in every output and dump through turnovers (same level
    stream), the other envs equal an engine that never loaded, and b equals the oracle's env a step by step"""
    import orc

    E, A, t0, M, a, b, c = 6, 1, 5, 160, 1, 3, 4
    params = {"episodeLengthSec": 1.0}
    g = _engine("HexExplore", E, A, 12, params, fast_shading=0)
    ref = _engine("HexExplore", E, A, 12, params, fast_shading=0)
    o = orc.Oracle("HexExplore", E, A, 128, 72, params=params)
    o.seed(12)
    o.reset()
    acts = _actions(E * A, t0 + M, seed=3)
    for t in range(t0):
        for x in (g, ref, o):
            x.step(acts[t])
    store = g.states_create(1)
    g.states_save(store, [a], [0])
    g.states_load(store, [0, 0], [b, c])
    loaded = np.array(g.obs())
    assert np.array_equal(loaded[b], loaded[a]) and np.array_equal(loaded[c], loaded[a])
    others = [e for e in range(E) if e not in (b, c)]
    turnovers = 0
    for t in range(t0, t0 + M):
        m = acts[t].copy()
        m[b] = m[c] = m[a]
        for x in (g, ref, o):
            x.step(m)
        out, want = _outputs(g, range(E)), _outputs(ref, range(E))
        turnovers += int(out["dones"][a])
        for k in ("obs", "rewards", "true_objectives"):
            for e in (b, c):
                assert np.array_equal(out[k][e], out[k][a]), "step %d: %s of clone %d" % (t, k, e)
            assert np.array_equal(out[k][others], want[k][others]), "step %d: %s of an env that was not loaded" % (t, k)
        assert out["dones"][b] == out["dones"][c] == out["dones"][a] and np.array_equal(out["dones"][others], want["dones"][others]), "step %d" % t
        for kind in ("state", "voxels", "instances", "level"):
            for e in (b, c):
                assert np.array_equal(out["%s%d" % (kind, e)], out["%s%d" % (kind, a)]), "step %d: %s of clone %d" % (t, kind, e)
            for e in others:
                assert np.array_equal(out["%s%d" % (kind, e)], want["%s%d" % (kind, e)]), "step %d: %s of env %d" % (t, kind, e)
        # the clone against the oracle's env a
        assert out["rewards"][b] == o.rewards().view(np.uint32)[a] and bool(out["dones"][b]) == bool(o.dones()[a]), "step %d oracle" % t
        assert np.array_equal(out["state%d" % b], o.state(a).view(np.uint32)), "step %d oracle state" % t
        diff = np.abs(out["obs"][b].astype(np.int16) - o.obs()[a].astype(np.int16))
        assert diff.max() <= 1, "step %d oracle frame: max RGB diff %d" % (t, diff.max())
    assert turnovers >= 2, turnovers
    _healthy(g)
    for x in (g, ref, o):
        x.close()


def test_load_after_the_static_arrays_grew(built):
    """save with 16-box static arrays' first growth behind, run until a later level grows them again (the store is re-pitched with the
    engine), load and replay: identical"""
    _load_after_growth(2, 48)  # (master seed 48: env 0's third maze has 281 walls)


def test_load_after_the_static_arrays_grew_four_slots(built):
    """the same with four level slots: the store's level slabs, four per env, are re-pitched too"""
    _load_after_growth(4, 1)  # (master seed 1: no env's first four mazes have more than 211 walls, env 0's fifth has 267)


def _load_after_growth(slots, seed):
    """the reset stages the first `slots` levels of each env and grows the 16-box arrays to 256 boxes; a later maze has more walls"""
    E, A, t0, M = 2, 2, 2, 120
    params = {"episodeLengthSec": 0.6}
    g = _engine("HexExplore", E, A, seed, params, static_cap=16, level_slots=slots)
    acts = _actions(E * A, t0 + M, seed=8)
    for t in range(t0):
        g.step(acts[t])
    at_t0 = _outputs(g, range(E))
    store = g.states_create(E)
    g.states_save(store, range(E), range(E))
    cap, row_bytes = g.static_cap(), g.state_row_bytes()
    recorded = []
    for t in range(t0, t0 + M):
        g.step(acts[t])
        recorded.append(_outputs(g, range(E)))
    assert g.static_cap() > cap and g.state_row_bytes() > row_bytes, "the case is meant to grow the arrays after the save"
    g.states_load(store, range(E), range(E))
    _assert_equal(at_t0, _outputs(g, range(E)), "after load")
    for i, t in enumerate(range(t0, t0 + M)):
        g.step(acts[t])
        _assert_equal(recorded[i], _outputs(g, range(E)), "replayed step %d" % t)
    _healthy(g)
    g.close()


def test_asynchronous_loop_around_save_and_load(built):
    """mv_step_device before and after save and load: the asynchronous results equal a host-facing engine's, and the loaded envs' recent
    episode ends never trip the asynchronous call's contract check"""
    import torch

    E, A, t0, M = 8, 1, 30, 160
    params = {"episodeLengthSec": 1.0}  # episodes of 15 steps: >= 4, the asynchronous call's contract
    g = _engine("HexExplore", E, A, 21, params)
    ref = _engine("HexExplore", E, A, 21, params)
    acts = _actions(E * A, t0 + M, seed=5)
    dacts = torch.from_numpy(acts).cuda()
    torch.cuda.synchronize()
    expect = {}
    for t in range(t0 + M):
        ref.step(acts[t])
        if t in (t0 - 1, t0 + M - 1):
            expect[t] = _outputs(ref, range(E))
    for t in range(t0):
        g.step_device(dacts.data_ptr() + t * E * A * 4)
    store = g.states_create(E)
    g.states_save(store, range(E), range(E))  # retires the outstanding steps
    g.fetch_obs()
    _assert_equal(expect[t0 - 1], _outputs(g, range(E)), "asynchronous steps up to the save")
    for rewind in range(2):
        for t in range(t0, t0 + M):
            g.step_device(dacts.data_ptr() + t * E * A * 4)
        g.sync()
        g.fetch_obs()
        _assert_equal(expect[t0 + M - 1], _outputs(g, range(E)), "asynchronous run %d after the save" % rewind)
        g.states_load(store, range(E), range(E))
        _assert_equal(expect[t0 - 1], _outputs(g, range(E)), "after load %d" % rewind)
    _healthy(g)
    g.close(); ref.close()


@pytest.mark.parametrize("mode", ["zero_copy", "hbm", "caller_buffer"])
def test_load_delivers_frames_and_depth_like_a_step(built, mode):
    """the re-render after a load delivers as a step does: zero-copy into the host buffer, into the engine's HBM tensor, or into a caller's
    tensor (mv_set_obs_buffer) -- frames and depth equal the saved step's"""
    import torch

    E, A, t0 = 4, 2, 12
    g = _engine("Collect", E, A, 4, {"episodeLengthSec": -2.0}, depth=True)
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

    acts = _actions(E * A, t0 + 20, seed=2)
    for t in range(t0):
        g.step(acts[t])
    saved_obs, saved_depth = frames()
    assert (saved_obs[..., 3] == 255).all()
    saved = _outputs(g, range(E), dumps=False)
    store = g.states_create(E)
    g.states_save(store, range(E), range(E))
    for t in range(t0, t0 + 20):
        g.step(acts[t])
    if mode == "caller_buffer":
        obs_buf.zero_(); depth_buf.zero_()
        torch.cuda.synchronize()  # the engine writes on its own stream
    g.states_load(store, range(E), range(E))
    obs, depth = frames()
    assert np.array_equal(obs, saved_obs), "frames after load"
    assert np.array_equal(depth, saved_depth), "depth after load"
    after = _outputs(g, range(E), dumps=False)
    for k in ("rewards", "dones", "true_objectives"):
        assert np.array_equal(after[k], saved[k]), k
    _healthy(g)
    g.close()


def test_state_calls_refuse_bad_arguments_and_call_order(built):
    """MV_ERR_STATE before mv_reset and while mv_step_begin is outstanding; MV_ERR_ARG for a bad store, an env or row out of range, a
    destination named twice, a row never saved.  A refused call changes nothing: the engine steps on like one that never saw it."""
    from megaverse_b200 import capi

    E, A = 4, 1
    g = capi.Engine("Collect", E, A, 128, 72, num_threads=2)

    def code(fn, *args):
        with pytest.raises(capi.MegaverseError) as ei:
            fn(*args)
        return ei.value.code

    assert code(g.states_create, 2) == capi.MV_ERR_STATE
    assert code(g.states_save, 0, [0], [0]) == capi.MV_ERR_STATE
    assert code(g.states_load, 0, [0], [0]) == capi.MV_ERR_STATE
    g.seed(5); g.reset()
    ref = _engine("Collect", E, A, 5)
    acts = _actions(E * A, 12, seed=1)
    for t in range(4):
        g.step(acts[t]); ref.step(acts[t])
    assert code(g.states_create, 0) == capi.MV_ERR_ARG
    store = g.states_create(2)
    assert g.state_row_bytes() > 0
    assert code(g.states_save, store + 1, [0], [0]) == capi.MV_ERR_ARG
    assert code(g.states_save, store, [E], [0]) == capi.MV_ERR_ARG
    assert code(g.states_save, store, [-1], [0]) == capi.MV_ERR_ARG
    assert code(g.states_save, store, [0], [2]) == capi.MV_ERR_ARG
    assert code(g.states_save, store, [0, 1], [1, 1]) == capi.MV_ERR_ARG  # two envs into one row
    assert code(g.states_load, store, [0], [0]) == capi.MV_ERR_ARG  # row 0 was never saved
    g.states_save(store, [2, 2], [0, 1])  # one env into two rows is fine
    assert code(g.states_load, store, [0, 1], [3, 3]) == capi.MV_ERR_ARG  # env 3 loaded twice
    assert code(g.states_load, store, [0], [E]) == capi.MV_ERR_ARG
    assert code(g.states_load, store, [2], [0]) == capi.MV_ERR_ARG
    g.step_begin(acts[4])
    assert code(g.states_save, store, [0], [0]) == capi.MV_ERR_STATE
    assert code(g.states_load, store, [0], [0]) == capi.MV_ERR_STATE
    g.step_end()
    ref.step(acts[4])
    for t in range(5, 12):
        g.step(acts[t]); ref.step(acts[t])
        _assert_equal(_outputs(ref, range(E)), _outputs(g, range(E)), "step %d after the refused calls" % t)
    g.states_destroy(store)
    assert code(g.states_destroy, store) == capi.MV_ERR_ARG
    assert code(g.states_save, store, [0], [0]) == capi.MV_ERR_ARG
    _healthy(g)
    g.close(); ref.close()


def test_megaverse_env_save_and_load_state(built):
    """MegaverseEnv.save_state / load_state: load returns the saved step's observations, and the steps after it return what they returned
    after the save"""
    from megaverse_b200 import MegaverseEnv

    env = MegaverseEnv("Collect", 3, 2, 2, params={"episodeLengthSec": -45.0})
    env.seed(17)
    obs = env.reset()
    rng = np.random.default_rng(4)
    actions = [rng.integers(0, [3, 3, 3, 2, 2, 3], size=(env.num_agents, 6)) for _ in range(60)]
    for a in actions[:5]:
        obs, _, _, _ = env.step(a)
    saved_obs = [np.array(o) for o in obs]
    state = env.save_state()
    after = []
    for a in actions[5:]:
        o, r, d, info = env.step(a)
        after.append(([np.array(x) for x in o], list(r), list(d), info))
    assert any(any(d) for _, _, d, _ in after), "the window is meant to hold an episode end"
    loaded = env.load_state(state)
    assert len(loaded) == env.num_agents and all(np.array_equal(x, y) for x, y in zip(loaded, saved_obs))
    for a, (o0, r0, d0, i0) in zip(actions[5:], after):
        o, r, d, info = env.step(a)
        assert all(np.array_equal(x, y) for x, y in zip(o, o0)) and r == r0 and d == d0 and info == i0
    clone = env.load_state(state, envs=[2], rows=[0])  # env 0's saved state into env 2
    assert np.array_equal(clone[4], saved_obs[0]) and np.array_equal(clone[5], saved_obs[1])
    state.close()
    env.close()
