"""Option "level_set": a fixed bank of levels in HBM shared by the envs; the step kernel chooses each env's next level at an episode end (the
caller's choice from the next-level array, else mv_level_set_pick) and reports it in level_ids; the host does nothing per end.

Level j of a set seeded s is the first level of a generator seeded s + j (test_level_set_cpu pins that against the oracle), so an oracle
env -- or an env of a stream engine -- seeded s + j and reset plays the same level.  Engines draw with fast_shading 0: frames byte for byte."""
import ctypes as C

import numpy as np
import pytest

import helpers

pytestmark = pytest.mark.gpu

MEGAVERSE8 = ['TowerBuilding', 'ObstaclesEasy', 'ObstaclesHard', 'Collect', 'Sokoban', 'HexMemory', 'HexExplore', 'Rearrange']


def _engine(scenario, E, A, L, s=0, params=None, seeds=None, reset=True, **opts):
    """an engine with a level set of L levels seeded s (L = 0: a stream engine), exact shading, env e's seed seeds[e] (default 42 + e)"""
    from megaverse_b200 import capi

    g = capi.Engine(scenario, E, A, 128, 72, num_threads=4, params=params)
    g.set_option("fast_shading", 0)
    if L:
        g.set_option("level_set_seed", s)
        g.set_option("level_set", L)
    for k, v in opts.items():
        g.set_option(k, v)
    for e in range(E):
        g.seed_env(e, int(42 + e if seeds is None else seeds[e]))
    if reset:
        g.reset()
    return g


def _healthy(g):
    assert g.fault_word() == 0
    assert g.faults() == 0


def _ends(E, envs):
    import torch

    m = np.zeros(E, dtype=np.uint8)
    m[list(envs)] = 1
    return torch.from_numpy(m).cuda()


def _actions(n, steps, seed=7):
    rng = np.random.default_rng(seed)
    return np.stack([helpers.purposeful_actions(rng, n, t) for t in range(steps)]).astype(np.int32)


def _pick(seed, episode, L):
    from megaverse_b200 import capi

    return capi.level_set_pick(seed, episode, L)


def _level_is(g, e, scenario, A, s, j, params=None):
    from megaverse_b200 import capi

    lvl = g.level(e)
    return np.array_equal(lvl, capi.generate_level(scenario, A, s + int(j), 0, params)[:lvl.size])


def _oracle_restart(o, e, seed):
    """the oracle's env e alone onto the first level of seed `seed`, then a render"""
    import orc

    L = orc.lib()
    L.orc_scen_reset.argtypes = [C.c_void_p, C.c_int]
    o.seed_env(e, seed)
    L.orc_scen_reset(o.h_, e)
    L.orc_render_now(o.h_)


# ------------------------------------------------------------------------------------------------ 1. bank content
@pytest.mark.parametrize("scenario,A", [("Collect", 2), ("TowerBuilding", 1), ("ObstaclesHard", 1), ("HexExplore", 1), ("Sokoban", 1)])
def test_bank_rows_are_the_levels_of_seeds_s_plus_j(built, scenario, A):
    """whenever level_ids[e] reads j, the env's live level is generate_level(scenario, A, s + j, 0); requested ends turn the levels over
    until every env has been on at least three"""
    E, L, s = 4, 8, 100
    g = _engine(scenario, E, A, L, s)
    ends = _ends(E, range(E))
    seen = [set() for _ in range(E)]
    for call in range(60):
        ids = np.array(g.level_ids())
        assert ((ids >= 0) & (ids < L)).all()
        for e in range(E):
            assert _level_is(g, e, scenario, A, s, ids[e]), "call %d env %d: not level %d" % (call, e, ids[e])
            seen[e].add(int(ids[e]))
        if min(len(x) for x in seen) >= 3:
            break
        g.step_device(None, ends.data_ptr())
        g.sync()
        assert np.array(g.dones()).all(), "a level set honours every end request"
    assert min(len(x) for x in seen) >= 3
    _healthy(g)
    g.close()


# ------------------------------------------------------------------------------------------------ 2. parity with the oracle across turnovers
@pytest.mark.parametrize("A", [1, 4])
@pytest.mark.parametrize("device", [False, True], ids=["mv_step", "mv_step_device"])
def test_oracle_parity_across_turnovers(built, A, device):
    """an oracle env per env, put on level s + level_ids[e] at the reset and at every reported end: rewards, dones, true objectives, states
    and frames equal the oracle's at every step through at least three episodes per env"""
    import orc
    import torch

    E, L, s, steps = 3, 5, 300, 56
    params = {"episodeLengthSec": 1.0}
    g = _engine("HexExplore", E, A, L, s, params)
    o = orc.Oracle("HexExplore", E, A, 128, 72, params=params)
    ids = np.array(g.level_ids())
    for e in range(E):
        o.seed_env(e, s + int(ids[e]))
    o.reset()
    acts = _actions(E * A, steps)
    dacts = torch.from_numpy(acts).cuda()
    episodes = np.zeros(E, dtype=int)
    for t in range(steps + 1):
        if t:
            if device:
                g.step_device(dacts[t - 1].data_ptr())
                g.fetch_obs()
            else:
                g.step(acts[t - 1])
            o.step(acts[t - 1])
            for key in ("rewards", "dones", "true_objectives"):
                a, b = np.array(getattr(g, key)()), getattr(o, key)()
                assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), "step %d: %s" % (t, key)
            ids = np.array(g.level_ids())
            for e in np.flatnonzero(np.array(g.dones())):
                _oracle_restart(o, int(e), s + int(ids[e]))
                episodes[e] += 1
        for e in range(E):
            assert np.array_equal(g.state(e).view(np.uint32), o.state(e).view(np.uint32)), "step %d: state of env %d" % (t, e)
        assert np.array_equal(np.array(g.obs()), o.obs()), "step %d: frames" % t
    assert episodes.min() >= 3
    _healthy(g)
    g.close(); o.close()


# ------------------------------------------------------------------------------------------------ 3. the pick
def _id_history(g, calls, ends):
    hist, frames = [np.array(g.level_ids()).copy()], []
    for _ in range(calls):
        g.step_device(None, ends.data_ptr())
        g.fetch_obs()
        hist.append(np.array(g.level_ids()).copy())
        frames.append(np.array(g.obs()).copy())
    return np.stack(hist), np.stack(frames)


def test_pick_sequence_follows_the_hash_and_the_seeds(built):
    E, A, L, calls = 6, 1, 16, 12
    ends = _ends(E, range(E))
    g = _engine("TowerBuilding", E, A, L, 7)
    hist, frames = _id_history(g, calls, ends)
    for t in range(calls + 1):  # every call ends every env: after call t the envs are in episode t
        assert [int(j) for j in hist[t]] == [_pick(42 + e, t, L) for e in range(E)], "episode %d" % t
    twin = _engine("TowerBuilding", E, A, L, 7)
    hist2, frames2 = _id_history(twin, calls, ends)
    assert np.array_equal(hist, hist2) and np.array_equal(frames, frames2), "engines built alike play the same levels and draw the same bytes"
    # mv_seed: one pick seed per env from the master stream; another master seed gives other sequences, the same one the same
    seqs = []
    for master in (1, 2, 1):
        x = _engine("TowerBuilding", E, A, L, 7, reset=False)
        x.seed(master)
        x.reset()
        seqs.append(_id_history(x, calls, ends)[0])
        x.close()
    assert np.array_equal(seqs[0], seqs[2]) and not np.array_equal(seqs[0], seqs[1])
    # a reseed after the reset changes the picks, not the bank
    g.seed_env(2, 4242)
    g.step_device(None, ends.data_ptr())
    g.sync()
    assert int(g.level_ids()[2]) == _pick(4242, calls + 1, L) and int(g.level_ids()[3]) == _pick(45, calls + 1, L)
    assert _level_is(g, 2, "TowerBuilding", A, 7, g.level_ids()[2])
    for x in (g, twin):
        _healthy(x)
        x.close()


# ------------------------------------------------------------------------------------------------ 4. the next-level array
def test_next_levels_host_and_device_forms(built):
    import torch
    from megaverse_b200 import capi

    E, A, L, s = 6, 1, 16, 3
    g = _engine("TowerBuilding", E, A, L, s)
    ends = _ends(E, range(E))
    nl = torch.as_tensor(g.device_array("next_levels"), device="cuda")
    stream = torch.cuda.ExternalStream(g.stream())
    assert (nl.cpu().numpy() == -1).all()

    def call():
        g.step_device(None, ends.data_ptr())
        g.sync()
        return np.array(g.level_ids()).copy()

    # host form: played at the next end, exactly once
    want1 = [_pick(42 + e, 1, L) for e in range(E)]
    g.set_next_levels([1, 3], [(want1[1] + 5) % L, (want1[3] + 2) % L])
    ids = call()
    want1[1], want1[3] = (want1[1] + 5) % L, (want1[3] + 2) % L
    assert [int(j) for j in ids] == want1
    for e in (1, 3):
        assert _level_is(g, e, "TowerBuilding", A, s, ids[e])
    assert (nl.cpu().numpy() == -1).all()
    assert [int(j) for j in call()] == [_pick(42 + e, 2, L) for e in range(E)]
    # device form, written on the engine's stream; a value outside the set is ignored, left alone, and nothing faults
    want3 = [_pick(42 + e, 3, L) for e in range(E)]
    with torch.cuda.stream(stream):
        nl[2] = (want3[2] + 7) % L
        nl[0] = 99
        nl[5] = -7
    want3[2] = (want3[2] + 7) % L
    assert [int(j) for j in call()] == want3
    assert nl.cpu().numpy().tolist() == [99, -1, -1, -1, -1, -7]
    _healthy(g)
    # the host form refuses what the kernel ignores, and changes nothing
    for envs, levels in (([0], [L]), ([0], [-1]), ([E], [0]), ([1, -1], [0, 0])):
        with pytest.raises(capi.MegaverseError) as err:
            g.set_next_levels(envs, levels)
        assert err.value.code == capi.MV_ERR_ARG
    assert nl.cpu().numpy().tolist() == [99, -1, -1, -1, -1, -7]
    g.close()


def test_chosen_envs_start_on_chosen_levels_now(built):
    """set_next_levels + reset_envs: the listed envs start the listed levels, the others' state, frames and ids are untouched"""
    E, A, L, s = 5, 2, 8, 20
    g = _engine("Collect", E, A, L, s)
    acts = _actions(E * A, 6)
    for t in range(6):
        g.step(acts[t])
    before = {"ids": np.array(g.level_ids()).copy(), "obs": np.array(g.obs()).copy(), "state": [g.state(e).view(np.uint32).copy() for e in range(E)]}
    g.set_next_levels([4, 1], [6, 2])
    g.reset_envs([4, 1])
    ids = np.array(g.level_ids())
    assert ids[4] == 6 and ids[1] == 2
    o = _engine("Collect", E, A, 0, seeds=[s + int(j) for j in ids])  # a stream engine whose env e starts on the same level
    for e in range(E):
        if e in (1, 4):
            assert _level_is(g, e, "Collect", A, s, ids[e])
            assert np.array_equal(np.array(g.obs())[e * A:(e + 1) * A], np.array(o.obs())[e * A:(e + 1) * A]), "env %d: first frame of the chosen level" % e
            assert g.state(e)[2] == 0 and not np.array(g.dones())[e]
        else:
            assert ids[e] == before["ids"][e]
            assert np.array_equal(np.array(g.obs())[e * A:(e + 1) * A], before["obs"][e * A:(e + 1) * A])
            assert np.array_equal(g.state(e).view(np.uint32), before["state"][e])
    _healthy(g)
    g.close(); o.close()


# ------------------------------------------------------------------------------------------------ 5. no host in the loop
@pytest.mark.parametrize("k", [1, 4])
@pytest.mark.parametrize("final", [0, 1])
def test_two_tick_episodes_asynchronously(built, k, final):
    """episodes of two ticks -- what mv_step_device refuses with level slots 2 -- for 300 unsynchronised calls: no error, no fault, every
    output equal to a twin stepped with mv_step, and exactly two kernel launches per call (three with terminal frames)"""
    import torch

    E, A, L, calls = 6, 1, 8, 300
    params = {"episodeLengthSec": 0.1}
    g = _engine("HexExplore", E, A, L, 11, params, action_repeat=k, final_obs=final, obs_to_host=0)
    twin = _engine("HexExplore", E, A, L, 11, params, action_repeat=k, final_obs=final)
    acts = _actions(E * A, calls, seed=5)
    dacts = torch.from_numpy(acts).cuda()
    keys = ("rewards", "dones", "done_reasons", "true_objectives", "level_ids")
    src = {key: torch.as_tensor(g.device_array(key), device="cuda") for key in keys}
    obs = torch.as_tensor(g.device_array("obs"), device="cuda")
    hist = {key: torch.empty((calls,) + tuple(v.shape), dtype=v.dtype, device="cuda") for key, v in src.items()}
    sums = torch.empty((calls, g.N), dtype=torch.int64, device="cuda")
    stream = torch.cuda.ExternalStream(g.stream())
    torch.cuda.synchronize()
    launches = g.kernel_launches()
    for t in range(calls):
        g.step_device(dacts[t].data_ptr())
        with torch.cuda.stream(stream):
            for key in keys:
                hist[key][t].copy_(src[key])
            sums[t].copy_(obs.view(g.N, -1).sum(1, dtype=torch.int64))
    assert g.kernel_launches() - launches == (3 if final else 2) * calls
    g.sync()
    torch.cuda.synchronize()
    assert np.array_equal(np.array(g.level_ids()), hist["level_ids"][-1].cpu().numpy()), "the retired ids are the last call's"
    ended = 0
    for t in range(calls):
        twin.step(acts[t])
        for key in keys:
            a, b = hist[key][t].cpu().numpy(), np.array(getattr(twin, key)())
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), "call %d: %s" % (t, key)
        assert np.array_equal(sums[t].cpu().numpy(), np.array(twin.obs()).reshape(g.N, -1).sum(1, dtype=np.int64)), "call %d: frames" % t
        ended += int(np.array(twin.dones()).sum())
    assert ended >= E * calls // 2
    for x in (g, twin):
        _healthy(x)
        x.close()


# ------------------------------------------------------------------------------------------------ 6. state store
def test_saved_envs_replay_later_levels_and_clones_agree(built):
    E, A, L, s, t0, M = 4, 2, 8, 60, 10, 50
    params = {"episodeLengthSec": 1.0}
    sizes = {}
    for name, opts in (("off", {}), ("off4", {"level_slots": 4}), ("on", {"level_set": L})):
        x = _engine("Collect", E, A, 0, params=params, reset=False, **opts)
        sizes[name] = x.state_row_bytes()
        x.close()
    slabs = (sizes["off4"] - sizes["off"]) // 2  # one level slot of every level array
    assert sizes["on"] == sizes["off"] - 2 * slabs + 4, "a row holds its level id instead of two level slots"

    g = _engine("HexExplore", E, A, L, s, params)
    acts = _actions(E * A, t0 + M)
    for t in range(t0):
        g.step(acts[t])
    store = g.states_create(E)
    g.states_save(store, range(E), range(E))

    def run():
        out = []
        for t in range(t0, t0 + M):
            g.step(acts[t])
            out.append([np.array(x).copy() for x in (g.rewards(), g.dones(), g.level_ids(), g.obs())])
        return out

    first = run()
    assert sum(int(o[1].sum()) for o in first) >= 3 * E, "three episodes on"
    g.states_load(store, range(E), range(E))
    for t, (a, b) in enumerate(zip(first, run())):
        for x, y, key in zip(a, b, ("rewards", "dones", "level_ids", "obs")):
            assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), "replayed step %d: %s" % (t, key)
    # one row into all four envs: the same levels, frames and rewards under the same actions
    g.states_load(store, [1] * E, range(E))
    ids0 = np.array(g.level_ids())
    assert (ids0 == ids0[0]).all(), "a loaded env reports its level before it is stepped"
    turnovers = 0
    for t in range(M):
        g.step(np.tile(acts[t0 + t][:A], E))
        ids, obs, rew = np.array(g.level_ids()), np.array(g.obs()).reshape(E, A, -1), np.array(g.rewards()).reshape(E, A)
        assert (ids == ids[0]).all() and (obs == obs[0]).all() and (rew == rew[0]).all(), "clones diverged at step %d" % t
        turnovers += int(np.array(g.dones())[0])
    assert turnovers >= 3
    g.states_destroy(store)
    _healthy(g)
    g.close()


# ------------------------------------------------------------------------------------------------ 7. mixed engine
def test_mixed_engine_keeps_every_env_in_its_scenarios_rows(built):
    """Megaverse-8 in one engine, L = 4: through five ends per env the live level is a level of the env's own scenario, and every env is
    byte-identical to the same env of a single-scenario engine with the same options and seeds"""
    E, A, L, s, calls = 8, 1, 4, 9, 15
    g = _engine(MEGAVERSE8, E, A, L, s)
    acts = _actions(E * A, calls, seed=2)
    ends = {t: _ends(E, range(E) if t % 3 == 2 else []) for t in range(calls)}
    import torch

    dacts = torch.from_numpy(acts).cuda()
    hist = []
    for t in range(calls):
        g.step_device(dacts[t].data_ptr(), ends[t].data_ptr())
        g.fetch_obs()
        ids = np.array(g.level_ids()).copy()
        for e in range(E):
            assert _level_is(g, e, MEGAVERSE8[e], A, s, ids[e]), "call %d: env %d left its scenario's rows" % (t, e)
        hist.append((ids, np.array(g.obs()).copy(), np.array(g.rewards()).copy(), np.array(g.dones()).copy()))
    assert sum(h[3].astype(int) for h in hist).min() >= 5
    _healthy(g)
    g.close()
    for e, name in enumerate(MEGAVERSE8):
        one = _engine(name, E, A, L, s)
        for t in range(calls):
            one.step_device(dacts[t].data_ptr(), ends[t].data_ptr())
            one.fetch_obs()
            got = (np.array(one.level_ids())[e], np.array(one.obs())[e * A:(e + 1) * A], np.array(one.rewards())[e * A:(e + 1) * A], np.array(one.dones())[e])
            want = (hist[t][0][e], hist[t][1][e * A:(e + 1) * A], hist[t][2][e * A:(e + 1) * A], hist[t][3][e])
            for x, y in zip(got, want):
                assert np.array_equal(x, y), "%s env %d, call %d" % (name, e, t)
        one.close()


# ------------------------------------------------------------------------------------------------ 8. with the other options
def test_first_episode_equals_a_stream_engine_on_the_same_level(built):
    """final_obs, segmentation and mv_set_obs_buffer with a level set: env e, on level j, against env e of a stream engine seeded s + j (the
    same level as its episode 0) through the episode's end -- frames in a caller's tensor, segmentation, and at the end the terminal
    frame of the old level and its reason"""
    import torch

    E, A, L, s = 4, 2, 8, 70
    params = {"episodeLengthSec": 1.0}
    g = _engine("HexExplore", E, A, L, s, params, final_obs=1, segmentation=1, obs_to_host=0)
    ids = np.array(g.level_ids()).copy()
    ref = _engine("HexExplore", E, A, 0, params=params, seeds=[s + int(j) for j in ids], final_obs=1, segmentation=1)
    mine = torch.zeros((g.N, 72, 128, 4), dtype=torch.uint8, device="cuda")
    g.set_obs_buffer(mine.data_ptr())
    acts = _actions(E * A, 20)
    dacts = torch.from_numpy(acts).cuda()
    seg = torch.as_tensor(g.device_array("segmentation"), device="cuda")
    done = False
    for t in range(20):
        g.step_device(dacts[t].data_ptr())
        g.fetch_obs()
        ref.step(acts[t])
        assert np.array_equal(np.array(g.dones()), np.array(ref.dones())) and np.array_equal(np.array(g.done_reasons()), np.array(ref.done_reasons()))
        assert np.array_equal(np.array(g.rewards()).view(np.uint32), np.array(ref.rewards()).view(np.uint32))
        if np.array(g.dones()).any():
            assert np.array(g.dones()).all() and (np.array(g.done_reasons()) == 1).all()
            assert np.array_equal(np.array(g.final_obs()), np.array(ref.final_obs())), "terminal frames of the old levels"
            assert (np.array(g.level_ids()) == [_pick(42 + e, 1, L) for e in range(E)]).all()
            done = True
            break
        assert np.array_equal(mine.cpu().numpy(), np.array(ref.obs())), "step %d: frames in the caller's tensor" % t
        assert np.array_equal(seg.cpu().numpy(), np.array(ref.segmentation())), "step %d: segmentation" % t
    assert done
    g.sync()
    for x in (g, ref):
        _healthy(x)
        x.close()


def test_inactive_envs_keep_level_frame_and_state(built):
    E, A, L = 5, 1, 8
    g = _engine("HexExplore", E, A, L, 5, {"episodeLengthSec": 0.5})
    acts = _actions(E * A, 40, seed=9)
    ended = np.zeros(E, dtype=int)
    for t in range(40):
        active = [e for e in range(E) if (e + t) % 3]
        idle = [e for e in range(E) if e not in active]
        ids, obs = np.array(g.level_ids()).copy(), np.array(g.obs()).copy()
        states = {e: g.state(e).view(np.uint32).copy() for e in idle}
        g.step_envs(acts[t], active)
        for e in idle:
            assert g.level_ids()[e] == ids[e] and not g.dones()[e]
            assert np.array_equal(np.array(g.obs())[e * A:(e + 1) * A], obs[e * A:(e + 1) * A])
            st = g.state(e).view(np.uint32).copy()
            rw = 8 + 26 * np.arange(A) + 24  # the state dump's copy of this call's reward: 0 for an inactive env
            st[rw], states[e][rw] = 0, 0
            assert np.array_equal(st, states[e])
        for e in np.flatnonzero(np.array(g.dones())):
            ended[e] += 1
            assert int(g.level_ids()[e]) == _pick(42 + int(e), int(ended[e]), L)
    assert ended.min() >= 2
    _healthy(g)
    g.close()


# ------------------------------------------------------------------------------------------------ 9. Python surface
def test_python_env_reports_levels(built):
    from megaverse_b200.megaverse_env import MegaverseEnv

    env = MegaverseEnv("HexExplore", 3, 2, 2, params={"episodeLengthSec": 1.0}, num_levels=4, start_level=7)
    env.seed(3)
    env.reset()
    playing = env.level_ids()
    assert len(playing) == 3 and all(0 <= j < 4 for j in playing)
    finished = 0
    for t in range(40):
        obs, rewards, dones, infos = env.step([[0, 0, 0, 0, 0, 0]] * env.num_agents)
        for i, (d, info) in enumerate(zip(dones, infos)):
            if d:
                assert info['level'] == playing[i // 2], "the level the finished episode was played on"
                finished += 1
            else:
                assert 'level' not in info
        playing = env.level_ids()
    assert finished >= 6
    env.set_next_levels([0, 2], [3, 1])
    env.reset_envs([0, 2])
    assert env.level_ids()[0] == 3 and env.level_ids()[2] == 1
    env.close()

    plain = MegaverseEnv("HexExplore", 2, 1, 2, params={"episodeLengthSec": 0.5})
    plain.reset()
    for t in range(12):
        _, _, dones, infos = plain.step([[0, 0, 0, 0, 0, 0]] * plain.num_agents)
        assert all('level' not in info for info in infos)
    with pytest.raises(RuntimeError):
        plain.level_ids()
    plain.close()


# ------------------------------------------------------------------------------------------------ 10. off means off
def test_accessors_need_the_option(built):
    from megaverse_b200 import capi

    g = _engine("TowerBuilding", 2, 1, 0)
    for call in (g.level_ids, lambda: g.device_ptr("level_ids"), lambda: g.device_ptr("next_levels"), lambda: g.set_next_levels([0], [0])):
        with pytest.raises(capi.MegaverseError) as err:
            call()
        assert err.value.code == capi.MV_ERR_STATE and "level_set" in str(err.value)
    with pytest.raises(capi.MegaverseError) as err:
        g.set_option("level_set", 4)  # after the first reset
    assert err.value.code == capi.MV_ERR_STATE
    g.close()
