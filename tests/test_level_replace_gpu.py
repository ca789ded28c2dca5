"""Replaceable level-set rows (mv_replace_levels, mv_level_rows): a requested row retires at the next kernel-enqueuing call (no flip lands
on it, a next-level entry naming it waits), envs on it finish their episodes on the old level, and the row is rewritten at the start of
the first call whose published level ids are at or after the request's call and show no env on it.  Engines draw with fast_shading 0."""
import numpy as np
import pytest

from test_level_replace_cpu import pick_with_probe
from test_level_set_gpu import _actions, _ends, _engine, _healthy, _pick

pytestmark = pytest.mark.gpu


def _is_seed_level(g, e, scenario, A, seed, params=None):
    from megaverse_b200 import capi

    lvl = g.level(e)
    return np.array_equal(lvl, capi.generate_level(scenario, A, int(seed), 0, params)[:lvl.size])


def _outputs(g):
    return {"obs": np.array(g.obs()).copy(), "rewards": np.array(g.rewards()).copy(), "dones": np.array(g.dones()).copy(),
            "reasons": np.array(g.done_reasons()).copy(), "ids": np.array(g.level_ids()).copy(), "launches": g.kernel_launches()}


def _equal(a, b, what):
    for k in a:
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), "%s: %s" % (what, k)


def _turn(g, ends):
    """one asynchronous call with the given end requests, then every call retired"""
    g.step_device(None, ends.data_ptr())
    g.sync()


# ------------------------------------------------------------------------------------------------ 1. identity
@pytest.mark.parametrize("device", [False, True], ids=["mv_step", "mv_step_device"])
def test_reading_the_rows_changes_nothing(built, device):
    import torch

    E, A, L, calls = 8, 2, 16, 300
    params = {"episodeLengthSec": 1.0}
    g, t = _engine("Collect", E, A, L, 10, params), _engine("Collect", E, A, L, 10, params)
    acts = _actions(E * A, calls)
    dacts = torch.from_numpy(acts).cuda()
    rng = np.random.default_rng(3)
    for c in range(calls):
        ends = _ends(E, np.flatnonzero(rng.random(E) < 0.1))
        for x in (g, t):
            if device:
                x.step_device(dacts[c].data_ptr(), ends.data_ptr())
                x.fetch_obs()
            else:
                x.step(acts[c])
        seeds, retiring = g.level_rows()
        assert seeds.tolist() == list(range(10, 10 + L)) and not retiring.any()
        _equal(_outputs(g), _outputs(t), "call %d" % c)
    _healthy(g)
    g.close(); t.close()


# ------------------------------------------------------------------------------------------------ 2. content of a replaced row
@pytest.mark.parametrize("scenario,A", [("Collect", 2), ("TowerBuilding", 1), ("ObstaclesHard", 1), ("HexExplore", 1), ("Sokoban", 1)])
def test_replaced_row_holds_the_new_seeds_level(built, scenario, A):
    """after the rewrite an env sent to the row plays the first level of the new seed, in lockstep with an oracle env on that seed"""
    import orc

    E, L, s, row, seed, steps = 4, 4, 100, 2, 5000, 40
    g = _engine(scenario, E, A, L, s)
    every = _ends(E, range(E))
    g.replace_levels([row], [seed])
    seeds, retiring = g.level_rows()
    assert seeds[row] == s + row and retiring[row]
    _turn(g, every)  # the row retires: every env ends and the probe keeps them off it
    assert row not in np.array(g.level_ids()).tolist()
    _turn(g, every)  # the published ids show the row empty: rewritten ahead of this call's kernel
    seeds, retiring = g.level_rows()
    assert seeds[row] == seed and not retiring.any()
    g.set_next_levels([0], [row])
    g.reset_envs([0])
    assert int(g.level_ids()[0]) == row
    assert _is_seed_level(g, 0, scenario, A, seed)
    o = orc.Oracle(scenario, 1, A, 128, 72)
    o.seed_env(0, seed)
    o.reset()
    assert np.array_equal(np.array(g.obs())[:A], o.obs()), "first frame"
    acts = _actions(E * A, steps)
    for t in range(steps):
        g.step(acts[t])
        o.step(acts[t][:A])
        for key in ("rewards", "true_objectives"):
            a, b = np.array(getattr(g, key)())[:A], getattr(o, key)()
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), "step %d: %s" % (t, key)
        assert bool(np.array(g.dones())[0]) == bool(o.dones()[0]), "step %d: done" % t
        if o.dones()[0]:
            break
        assert np.array_equal(np.array(g.obs())[:A], o.obs()), "step %d: frames" % t
    _healthy(g)
    g.close(); o.close()


# ------------------------------------------------------------------------------------------------ 3. live envs, the probe, deferred entries
def test_envs_on_a_replaced_row_play_on_untouched(built):
    """env 0 is on the row when it is replaced: byte-identical to a twin's env 0 until its episode ends; envs that have not ended since
    the request are identical as well"""
    E, A, L, s = 6, 1, 8, 30
    params = {"episodeLengthSec": 1.0}
    g, t = _engine("Collect", E, A, L, s, params), _engine("Collect", E, A, L, s, params)
    acts = _actions(E * A, 200, seed=4)
    for x in (g, t):
        x.step(acts[0])
    j0 = int(g.level_ids()[0])
    g.replace_levels([j0], [777])
    untouched = set(range(E))
    for c in range(1, 200):
        g.step(acts[c]); t.step(acts[c])
        a, b = _outputs(g), _outputs(t)
        for e in untouched:  # up to and including the call that ends them
            for k, rows in (("rewards", slice(e * A, (e + 1) * A)), ("dones", e), ("reasons", e)):
                assert np.array_equal(a[k][rows], b[k][rows]), "call %d env %d: %s" % (c, e, k)
        untouched -= set(np.flatnonzero(a["dones"]).tolist())
        for e in untouched:
            assert np.array_equal(a["obs"][e * A:(e + 1) * A], b["obs"][e * A:(e + 1) * A]), "call %d env %d" % (c, e)
            assert np.array_equal(g.state(e).view(np.uint32), t.state(e).view(np.uint32)), "call %d: state of env %d" % (c, e)
        if a["dones"][0]:
            break
        assert g.level_rows()[1][j0] and g.level_rows()[0][j0] == s + j0, "env 0 still holds the row"
    assert a["dones"][0], "env 0's episode ended"
    _healthy(g)
    g.close(); t.close()


def test_probe_and_deferred_next_level(built):
    """every call ends every env but the holder (so after call c the others are in episode c): pick seeds are chosen so that the hash
    lands on the retiring row, and the probe lands where the restatement says; an entry naming the row is honoured on exactly the call
    that rewrites it"""
    E, A, L, s, hold_calls = 6, 1, 8, 50, 4
    g = _engine("TowerBuilding", E, A, L, s)
    others = [e for e in range(1, E)]
    j0 = 5
    g.set_next_levels([0], [j0])
    g.reset_envs([0])  # env 0 (the holder) is on row j0
    ends = _ends(E, others)
    g.replace_levels([j0, (j0 + 1) % L], [900, 901])
    g.set_next_levels([1], [j0])
    rewritten_at = None
    for c in range(1, hold_calls + 4):
        ep = c  # the others' episode index after this call
        seeds = {e: next(x for x in range(10 ** 6) if _pick(x, ep, L) in (j0, (j0 + 1) % L) and x % 7 == e) for e in others[1:]}
        for e, x in seeds.items():
            g.seed_env(e, x)
        if c == hold_calls + 1:
            ends = _ends(E, range(E))  # the end request releases the holder
        _turn(g, ends)
        ids = np.array(g.level_ids())
        rows, retiring = g.level_rows()
        pickable = [not r for r in retiring]  # a rewrite precedes its call's kernel
        for e, x in seeds.items():
            assert ids[e] == pick_with_probe(x, ep, L, pickable)[0], "call %d env %d" % (c, e)
        if rewritten_at is None and not retiring[j0]:
            rewritten_at = c
        if rewritten_at is None:
            assert c > hold_calls or ids[0] == j0, "the holder stays"
            assert ids[1] != j0, "the entry waits while the row retires"
            assert j0 not in [ids[e] for e in seeds]
        elif rewritten_at == c:
            assert ids[1] == j0, "the entry is honoured on the rewrite call"
            assert _is_seed_level(g, 1, "TowerBuilding", A, 900)
    # the holder left at call hold_calls + 1 (published by the sync), so the rewrite is the next call
    assert rewritten_at == hold_calls + 2
    _healthy(g)
    g.close()


# ------------------------------------------------------------------------------------------------ 4. the rewrite call
def _predict(requests, kinds, ids_after, L, E_bank):
    """first call c > request call whose published call (host: the previous call; device: three back in a run, per `kinds`) is at or after
    the request call and whose published ids show no env on the row.  ids_after[c]: level_ids() right after call c (what was published)"""
    published_after, done = [], -1
    for c, k in enumerate(kinds):
        done = c if k == "host" else max(done, c - 2)
        published_after.append(done)
    out = {}
    for row, req in requests.items():
        for c in range(req + 1, len(kinds)):
            p = published_after[c - 1]
            if p >= req and row not in [int(j) for j in ids_after[c - 1]]:
                out[row] = c
                break
    return out


@pytest.mark.parametrize("kind", ["host", "device", "device_active"])
def test_rewrite_call_follows_the_rule(built, kind):
    import torch

    E, A, L, s, calls = 8, 1, 6, 70, 40
    params = {"episodeLengthSec": 1.0}
    g = _engine("HexExplore", E, A, L, s, params)
    acts = _actions(E * A, calls, seed=9)
    dacts = torch.from_numpy(acts).cuda()
    rng = np.random.default_rng(11)
    requests, seen_rewrite, ids_after, kinds = {}, {}, [], []
    prev_seeds = g.level_rows()[0].copy()
    holder, keep = 0, []
    for c in range(calls):
        if c in (2, 9, 17) and len(requests) < 3:
            row = int(g.level_ids()[holder]) if c == 2 else int(rng.integers(0, L))
            seeds, retiring = g.level_rows()
            if not retiring[row] and row not in requests:
                g.replace_levels([row], [4000 + c])
                requests[row] = c
        if kind == "host":
            g.step(acts[c])
        else:
            ends = _ends(E, [e for e in range(E) if rng.random() < 0.15] + ([holder] if c == 12 else []))
            active = np.ones(E, dtype=np.uint8)
            if kind == "device_active" and c < 12:
                active[holder] = 0  # the inactive holder keeps the row until its end request at call 12
            dact = torch.from_numpy(active).cuda()
            keep.append((ends, dact))  # read by the engine's stream later
            g.step_device_active(dacts[c].data_ptr(), ends.data_ptr(), dact.data_ptr())
        kinds.append("host" if kind == "host" else "device")
        ids_after.append(np.array(g.level_ids()).copy())
        seeds = g.level_rows()[0].copy()
        for row in np.flatnonzero(seeds != prev_seeds):
            seen_rewrite[int(row)] = c
        prev_seeds = seeds
    want = _predict(requests, kinds, ids_after, L, E)
    assert seen_rewrite == want, (seen_rewrite, want, requests)
    assert len(want) >= 2
    if kind == "device_active":
        assert want[min(requests, key=requests.get)] > 12, "the inactive holder held the row until its end"
    _healthy(g)
    g.close()


# ------------------------------------------------------------------------------------------------ 5. worker timing
def test_thread_count_does_not_matter(built):
    import torch
    from megaverse_b200 import capi

    E, A, L, calls = 32, 1, 32, 60
    engines = []
    for threads in (1, 16):
        g = capi.Engine("ObstaclesHard", E, A, 128, 72, num_threads=threads)
        g.set_option("fast_shading", 0)
        g.set_option("level_set", L)
        for e in range(E):
            g.seed_env(e, 42 + e)
        g.reset()
        engines.append(g)
    rng = np.random.default_rng(5)
    acts = torch.from_numpy(_actions(E * A, calls)).cuda()
    for c in range(calls):
        ends = _ends(E, np.flatnonzero(rng.random(E) < 0.2))
        retiring = engines[0].level_rows()[1]
        free = [r for r in range(L) if not retiring[r]]
        rows = rng.choice(free, size=min(6, len(free) - 1), replace=False)
        seeds = rng.integers(0, 1 << 30, size=rows.size)
        outs = []
        for g in engines:
            g.replace_levels(rows, seeds)
            g.step_device(acts[c].data_ptr(), ends.data_ptr())
            g.fetch_obs()
            o = _outputs(g)
            o["rows"], o["retiring"] = g.level_rows()
            outs.append(o)
        _equal(outs[0], outs[1], "call %d" % c)
    for g in engines:
        _healthy(g)
        g.close()


# ------------------------------------------------------------------------------------------------ 6. mixed engines
def test_mixed_engine_blocks(built):
    names = ["Collect", "TowerBuilding", "Collect", "TowerBuilding"]
    E, A, L, s = 4, 1, 4, 10
    g, t = _engine(names, E, A, L, s), _engine(names, E, A, L, s)
    every = _ends(E, range(E))
    g.replace_levels([1 * L + 2], [6001])
    for c in range(3):
        _turn(g, every); _turn(t, every)
        a, b = _outputs(g), _outputs(t)
        for e in (0, 2):  # Collect envs never see the TowerBuilding block
            assert a["ids"][e] == b["ids"][e] and np.array_equal(a["obs"][e], b["obs"][e]), "call %d env %d" % (c, e)
    assert g.level_rows()[0].tolist() == [10, 11, 12, 13, 10, 11, 6001, 13]
    g.set_next_levels([1], [2])
    g.reset_envs([1])
    assert _is_seed_level(g, 1, "TowerBuilding", A, 6001)
    _healthy(g)
    g.close(); t.close()


# ------------------------------------------------------------------------------------------------ 7. state store
def test_state_store_refuses_rewritten_and_retiring_rows(built):
    from megaverse_b200 import capi

    E, A, L, s, K = 4, 1, 8, 20, 10
    g = _engine("Collect", E, A, L, s)
    g.set_next_levels([0, 1], [3, 6])
    g.reset_envs([0, 1])
    acts = _actions(E * A, 2 * K + 10)
    g.step(acts[0])
    store = g.states_create(2)
    g.states_save(store, [0, 1], [0, 1])
    recorded = []
    for t in range(1, K + 1):
        g.step(acts[t])
        recorded.append((np.array(g.obs())[A:2 * A].copy(), np.array(g.rewards())[A:2 * A].copy()))
    g.replace_levels([3], [8888])
    before = _outputs(g)
    for rows, envs in (([0], [0]), ([0], [2])):
        with pytest.raises(capi.MegaverseError) as err:
            g.states_load(store, rows, envs)
        assert err.value.code == capi.MV_ERR_ARG and "row 0" in str(err.value)
        _equal(_outputs(g), before, "a refused load changes nothing")
    every = _ends(E, range(E))
    _turn(g, every); _turn(g, every); _turn(g, every)
    assert g.level_rows()[0][3] == 8888
    with pytest.raises(capi.MegaverseError) as err:
        g.states_load(store, [0], [0])
    assert err.value.code == capi.MV_ERR_ARG
    g.states_load(store, [1], [1])  # row 6 was never touched
    assert int(g.level_ids()[1]) == 6
    for t in range(1, K + 1):
        g.step(acts[t])
        obs, rew = recorded[t - 1]
        assert np.array_equal(np.array(g.obs())[A:2 * A], obs) and np.array_equal(np.array(g.rewards())[A:2 * A], rew), "replay %d" % t
    _healthy(g)
    g.close()


# ------------------------------------------------------------------------------------------------ 8. growth with a store present
def test_growth_store_loads_and_replays(built):
    """the store's instance rows are re-pitched with the arrays: a state saved before a growing rewrite loads and replays bit for bit"""
    from megaverse_b200 import capi

    E, A, L, M = 2, 1, 2, 15
    params = {"episodeLengthSec": 3.0}

    def walls(seed):
        d = capi.generate_level("HexExplore", A, seed, 0, params)
        return int(d[9 + 8 * d[0] + 7 * d[1] + 3 * d[2] + 3 * A + 2])

    small = next(x for x in range(1, 300) if walls(x) <= 120 and walls(x + 1) <= 120)
    big = next(x for x in range(1, 300) if walls(x) > 256)
    g = _engine("HexExplore", E, A, L, small, params, static_cap=16)
    g.set_next_levels([0, 1], [0, 0])
    g.reset_envs([0, 1])
    cap = g.static_cap()
    acts = _actions(E * A, 2 * M + 2, seed=6)
    g.step(acts[0])
    store = g.states_create(E)
    g.states_save(store, range(E), range(E))
    recorded = []
    for c in range(1, M + 1):
        g.step(acts[c])
        recorded.append(_outputs(g))
    g.replace_levels([1], [big])
    g.step(acts[M + 1]); g.step(acts[M + 1])
    if g.level_rows()[1][1]:
        g.reset_envs([e for e in range(E) if int(g.level_ids()[e]) == 1])
        g.step(acts[M + 1])
    assert g.level_rows()[0][1] == big and g.static_cap() > cap, "the rewrite grew the arrays"
    g.states_load(store, range(E), range(E))
    for c in range(1, M + 1):
        g.step(acts[c])
        a = _outputs(g)
        for k in ("obs", "rewards", "dones", "ids"):
            assert np.array_equal(a[k], recorded[c - 1][k]), "replayed call %d: %s" % (c, k)
        if a["dones"].any():  # the next level may be a rewritten row
            break
    _healthy(g)
    g.close()


# ------------------------------------------------------------------------------------------------ 9. refusals
def test_refusals_change_nothing(built):
    from megaverse_b200 import capi

    E, A, L = 4, 1, 4
    off = _engine("Collect", E, A, 0)
    with pytest.raises(capi.MegaverseError) as err:
        off.replace_levels([0], [1])
    assert err.value.code == capi.MV_ERR_STATE
    off.close()
    fresh = _engine("Collect", E, A, L, reset=False)
    with pytest.raises(capi.MegaverseError) as err:
        fresh.replace_levels([0], [1])
    assert err.value.code == capi.MV_ERR_STATE
    fresh.close()
    g = _engine("Collect", E, A, L, 5)
    g.step_begin(np.zeros(E * A, dtype=np.int32))
    with pytest.raises(capi.MegaverseError) as err:
        g.replace_levels([0], [1])
    assert err.value.code == capi.MV_ERR_STATE
    g.step_end()
    g.replace_levels([1], [77])
    before = (g.level_rows()[0].copy(), g.level_rows()[1].copy())
    for rows in ([L], [-1], [0, 0], [1], [0, 2, 3]):
        with pytest.raises(capi.MegaverseError) as err:
            g.replace_levels(rows, [9] * len(rows))
        assert err.value.code == capi.MV_ERR_ARG, rows
        assert np.array_equal(g.level_rows()[0], before[0]) and np.array_equal(g.level_rows()[1], before[1])
    g.replace_levels([0, 2], [8, 9])  # leaves row 3 pickable
    _healthy(g)
    g.close()


# ------------------------------------------------------------------------------------------------ 10. Python
def test_python_surface(built):
    """replace_levels / level_seeds on MegaverseEnv: level_seeds()[info['level']], read after step(), is the finished episode's seed"""
    from megaverse_b200.megaverse_env import MegaverseEnv

    env = MegaverseEnv("HexExplore", 3, 2, 2, params={"episodeLengthSec": 1.0}, num_levels=4, start_level=30)
    env.seed(3)
    env.reset()
    assert env.level_seeds() == [30, 31, 32, 33]
    seed_of_episode = [env.level_seeds()[j] for j in env.level_ids()]
    rng = np.random.default_rng(0)
    replaced, checked = 0, 0
    for t in range(120):
        if t % 5 == 0:
            retiring = env.env.get_level_rows()[1]
            j = int(rng.integers(0, 4))
            if not retiring[j] and int((retiring == 0).sum()) > 1:
                env.replace_levels([j], [1000 + t])
                replaced += 1
        _, _, dones, infos = env.step([[0, 0, 0, 0, 0, 0]] * env.num_agents)
        for i, (d, info) in enumerate(zip(dones, infos)):
            if d:
                assert env.level_seeds()[info['level']] == seed_of_episode[i // 2], "the finished episode's level seed"
                checked += 1
        seed_of_episode = [env.level_seeds()[j] for j in env.level_ids()]
    assert replaced >= 5 and checked >= 12 and any(x >= 1000 for x in env.level_seeds())
    env.close()


# ------------------------------------------------------------------------------------------------ 11. faults
def test_no_faults_under_heavy_replacement(built):
    import torch

    E, A, L, calls = 256, 2, 64, 120
    g = _engine("Collect", E, A, L, 0)
    rng = np.random.default_rng(1)
    acts = torch.from_numpy(_actions(E * A, calls)).cuda()
    keep = []
    for c in range(calls):
        retiring = g.level_rows()[1]
        free = [r for r in range(L) if not retiring[r]]
        rows = rng.choice(free, size=min(10, len(free) - 1), replace=False)
        g.replace_levels(rows, rng.integers(0, 1 << 30, size=rows.size))
        keep.append(_ends(E, np.flatnonzero(rng.random(E) < 0.1)))  # read by the engine's stream later
        g.step_device(acts[c].data_ptr(), keep[-1].data_ptr())
        assert g.fault_word() == 0
    g.sync()
    assert (g.level_rows()[0] != np.arange(L)).sum() > L // 2
    _healthy(g)
    g.close()
