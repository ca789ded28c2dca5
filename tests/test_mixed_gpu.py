"""Mixed-scenario engine (mv_create_mixed): every env of one engine runs its own scenario and behaves exactly as the same env of a
single-scenario engine of its name, seeded the same -- frames, depth, rewards, dones, true objectives and the debug dumps, bit for bit --
in every delivery mode, with reward shaping per scenario, growing static arrays and the env state store."""
import numpy as np
import pytest

import helpers

pytestmark = pytest.mark.gpu

# every registered name
NAMES = ["ObstaclesEasy", "ObstaclesMedium", "ObstaclesHard", "ObstaclesWalls", "ObstaclesSteps", "ObstaclesLava", "Test",
         "TowerBuilding", "Collect", "Sokoban", "Rearrange", "HexExplore", "HexMemory", "Empty"]
MEGAVERSE8 = ["TowerBuilding", "ObstaclesEasy", "ObstaclesHard", "Collect", "Sokoban", "HexMemory", "HexExplore", "Rearrange"]
# one dict for every env: a negative base ends the TowerBuilding, Collect, HexMemory and fixed-length episodes after one step, Obstacles
# chains without platforms last a few seconds -- every env turns over many times in the window
SHORT = {"episodeLengthSec": -200.0, "obstaclesMinNumPlatforms": 0.0, "obstaclesMaxNumPlatforms": 0.0}
# episodes of 3 s (45 steps) and more: gameplay between the resets, and long enough for the asynchronous call's contract
PLAY = {"episodeLengthSec": 3.0}


def _layout(names, copies, kind):
    n = len(names)
    if kind == "interleaved":
        return [names[e % n] for e in range(n * copies)]
    return [names[e // copies] for e in range(n * copies)]


def _seed(names, name, j):
    return 1000 + 10 * names.index(name) + j


class Mixed:
    """a mixed engine and, per scenario name, a single-scenario engine whose env j is the j-th env of that name in the mixed one"""

    def __init__(self, names, copies, kind, A, params, depth=False, **options):
        from megaverse_b200 import capi

        self.names, self.A = names, A
        self.layout = _layout(names, copies, kind)
        self.E = len(self.layout)
        self.g = capi.Engine(self.layout, self.E, A, 128, 72, num_threads=2, params=params, depth=depth)
        self.refs = {n: capi.Engine(n, copies, A, 128, 72, num_threads=1, params=params, depth=depth) for n in names}
        self.slot = []  # env e -> (name, j)
        seen = {}
        for e, n in enumerate(self.layout):
            j = seen.get(n, 0)
            seen[n] = j + 1
            self.slot.append((n, j))
            self.g.seed_env(e, _seed(names, n, j))
        for n, r in self.refs.items():
            for j in range(copies):
                r.seed_env(j, _seed(names, n, j))
        for x in self.engines():
            for k, v in options.items():
                x.set_option(k, v)
            x.reset()

    def engines(self):
        return [self.g] + list(self.refs.values())

    def ref_masks(self, masks):
        """the mixed engine's masks [E*A] split into each single engine's [copies*A]"""
        out = {n: np.zeros(r.N, dtype=np.int32) for n, r in self.refs.items()}
        for e, (n, j) in enumerate(self.slot):
            out[n][j * self.A:(j + 1) * self.A] = masks[e * self.A:(e + 1) * self.A]
        return out

    def step(self, masks):
        self.g.step(masks)
        for n, m in self.ref_masks(masks).items():
            self.refs[n].step(m)

    def close(self):
        for x in self.engines():
            x.close()


def _actions(n, steps, seed=7):
    rng = np.random.default_rng(seed)
    return np.stack([helpers.purposeful_actions(rng, n, t) for t in range(steps)]).astype(np.int32)


def _outputs(g, envs, dumps=True, depth=False):
    out = {"obs": np.array(g.obs()), "rewards": np.array(g.rewards()).view(np.uint32), "dones": np.array(g.dones()),
           "true_objectives": np.array(g.true_objectives()).view(np.uint32)}
    if depth:
        out["depth"] = np.array(g.depth()).view(np.uint32)
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
        assert a[k].shape == b[k].shape and np.array_equal(a[k], b[k]), "%s: %s differs" % (tag, k)


def _compare(m, tag, dumps=True, depth=False):
    """every output of every mixed env against its single-scenario engine; returns the mixed engine's outputs"""
    A = m.A
    mine = _outputs(m.g, range(m.E), dumps=dumps, depth=depth)
    theirs = {n: _outputs(r, range(r.E), dumps=dumps, depth=depth) for n, r in m.refs.items()}
    for e, (n, j) in enumerate(m.slot):
        t = theirs[n]
        for k in ("obs", "rewards", "true_objectives") + (("depth",) if depth else ()):
            assert np.array_equal(mine[k][e * A:(e + 1) * A], t[k][j * A:(j + 1) * A]), "%s: env %d (%s) %s" % (tag, e, n, k)
        assert mine["dones"][e] == t["dones"][j], "%s: env %d (%s) dones" % (tag, e, n)
        if dumps:
            for kind in ("state", "voxels", "instances", "level"):
                assert np.array_equal(mine["%s%d" % (kind, e)], t["%s%d" % (kind, j)]), "%s: env %d (%s) %s" % (tag, e, n, kind)
    return mine


def _healthy(*engines):
    for g in engines:
        assert g.fault_word() == 0
        assert g.faults() == 0


CASES = [("interleaved", 1, "short"), ("blocked", 1, "short"), ("interleaved", 4, "short"), ("blocked", 1, "play")]


@pytest.mark.parametrize("kind,A,params", CASES, ids=["%s-A%d-%s" % c for c in CASES])
def test_every_scenario_in_one_engine_matches_single_engines(built, kind, A, params):
    """all 14 registered names, two envs each, in one engine: every env equals its single-scenario engine step by step"""
    short = params == "short"
    m = Mixed(NAMES, 2, kind, A, SHORT if short else PLAY)
    _compare(m, "after reset")
    T = 60 if short else 120
    acts = _actions(m.E * A, T, seed=3)
    turnovers = np.zeros(m.E, dtype=np.int64)
    for t in range(T):
        m.step(acts[t])
        out = _compare(m, "step %d" % t, dumps=(t % 3 == 0))
        turnovers += out["dones"]
    if short:
        assert (turnovers >= 2).all(), "every env is meant to turn over at least twice: %s" % turnovers.tolist()
    else:
        assert turnovers.sum() > 0
    _healthy(*m.engines())
    m.close()


@pytest.mark.parametrize("mode", ["zero_copy", "hbm_copy", "begin_end", "device_async"])
def test_delivery_modes_with_depth(built, mode):
    """depth on; the host zero-copy stores, option zero_copy 0, mv_step_begin / mv_step_end and the asynchronous step_device + sync
    loop all deliver what the single-scenario engines deliver; draw_hires too"""
    import torch

    options = {"zero_copy": 0} if mode == "hbm_copy" else {}
    m = Mixed(MEGAVERSE8, 2, "interleaved", 1, PLAY, depth=True, **options)
    T = 70
    acts = _actions(m.E, T, seed=11)
    if mode == "device_async":
        dacts = torch.from_numpy(acts).cuda()
        torch.cuda.synchronize()
        for t in range(T):
            m.g.step_device(dacts.data_ptr() + t * m.E * 4)
            for n, mk in m.ref_masks(acts[t]).items():
                m.refs[n].step(mk)
            if t in (30, T - 1):
                m.g.sync()
                m.g.fetch_obs()
                _compare(m, "asynchronous step %d" % t, depth=True)
    else:
        for t in range(T):
            if mode == "begin_end":
                m.g.step_begin(acts[t])
                m.g.step_end()
                for n, mk in m.ref_masks(acts[t]).items():
                    m.refs[n].step(mk)
            else:
                m.step(acts[t])
            _compare(m, "step %d" % t, dumps=(t % 10 == 0), depth=True)
    hi = np.array(m.g.draw_hires(256, 144))
    for n, r in m.refs.items():
        rh = np.array(r.draw_hires(256, 144))
        for e, (n2, j) in enumerate(m.slot):
            if n2 == n:
                assert np.array_equal(hi[e], rh[j]), "draw_hires env %d (%s)" % (e, n)
    _healthy(*m.engines())
    m.close()


def test_static_arrays_grow_in_a_mixed_engine(built):
    """static_cap 16: the first HexExplore mazes and Collect landscapes outgrow it at once; the grown engine still matches"""
    m = Mixed(["HexExplore", "Collect"], 2, "interleaved", 2, {"episodeLengthSec": 0.6}, static_cap=16)
    acts = _actions(m.E * 2, 60, seed=8)
    for t in range(60):
        m.step(acts[t])
        _compare(m, "step %d" % t, dumps=(t % 5 == 0))
    assert m.g.static_cap() > 16
    _healthy(*m.engines())
    m.close()


def test_reward_shaping_per_scenario(built):
    """get returns the env's own scenario's keys; a scheme of another scenario is refused; a changed scheme changes only that env's
    rewards, which equal a single engine given the same scheme"""
    from megaverse_b200 import capi

    m = Mixed(MEGAVERSE8, 2, "interleaved", 1, PLAY)
    for e, (n, j) in enumerate(m.slot):
        assert m.g.get_reward_shaping(e, 0) == m.refs[n].get_reward_shaping(j, 0), (e, n)
    tower = m.layout.index("TowerBuilding")
    collect = m.layout.index("Collect")
    scheme = m.g.get_reward_shaping(collect, 0)
    with pytest.raises(capi.MegaverseError) as ei:
        m.g.set_reward_shaping(tower, 0, scheme)  # lacks the TowerBuilding keys
    assert ei.value.code == capi.MV_ERR_ARG and "towerbuilding" in str(ei.value)
    assert m.g.get_reward_shaping(tower, 0) == m.refs["TowerBuilding"].get_reward_shaping(0, 0)
    scheme = dict(scheme, collectSingleGood=3.5, collectSingleBad=-0.25, teamSpirit=0.3)
    m.g.set_reward_shaping(collect, 0, scheme)
    m.refs["Collect"].set_reward_shaping(m.slot[collect][1], 0, scheme)
    acts = _actions(m.E, 150, seed=5)
    rewarded = 0.0
    for t in range(150):
        m.step(acts[t])
        out = _compare(m, "step %d" % t, dumps=False)
        rewarded += abs(float(out["rewards"].view(np.float32)[collect]))
    assert rewarded > 0, "the shaped env is meant to collect rewards in the window"
    _healthy(*m.engines())
    m.close()


def test_state_store_in_a_mixed_engine(built):
    """rewind replays bit-identically across turnovers; a clone into another env of the same name runs the saved env; a row of another
    scenario is refused and changes nothing"""
    from megaverse_b200 import capi

    m = Mixed(NAMES, 2, "interleaved", 1, SHORT)
    g = m.g
    E, t0, M = m.E, 4, 90
    acts = _actions(E, t0 + M + 20, seed=9)
    for t in range(t0):
        m.step(acts[t])
    at_t0 = _outputs(g, range(E))
    store = g.states_create(E)
    g.states_save(store, range(E), range(E))
    recorded, turnovers = [], np.zeros(E, dtype=np.int64)
    for t in range(t0, t0 + M):
        g.step(acts[t])
        recorded.append(_outputs(g, range(E)))
        turnovers += recorded[-1]["dones"]
    for n in NAMES:  # the replayed window holds turnovers of every scenario
        assert max(turnovers[e] for e in range(E) if m.layout[e] == n) >= 2, (n, turnovers.tolist())
    g.states_load(store, range(E), range(E))
    _assert_equal(at_t0, _outputs(g, range(E)), "after load")
    for i, t in enumerate(range(t0, t0 + M)):
        g.step(acts[t])
        _assert_equal(recorded[i], _outputs(g, range(E)), "replayed step %d" % t)

    # a cross-scenario load is refused and leaves every output as it was
    before = _outputs(g, range(E))
    tower, obst = m.layout.index("TowerBuilding"), m.layout.index("ObstaclesHard")
    with pytest.raises(capi.MegaverseError) as ei:
        g.states_load(store, [obst, 0], [tower, 0])
    assert ei.value.code == capi.MV_ERR_ARG
    assert "obstacleshard" in str(ei.value) and "towerbuilding" in str(ei.value), str(ei.value)
    _assert_equal(before, _outputs(g, range(E)), "after the refused load")

    # clone: env a's saved row into env b of the same name; with a's actions b runs exactly as a
    a = m.layout.index("Collect")
    b = len(NAMES) + a  # the second Collect env
    assert m.layout[b] == "Collect"
    clone = g.states_create(1)
    g.states_save(clone, [a], [0])
    g.states_load(clone, [0], [b])
    out = _outputs(g, [a, b])
    assert np.array_equal(out["obs"][b], out["obs"][a])
    for t in range(t0 + M, t0 + M + 20):
        mk = acts[t].copy()
        mk[b] = mk[a]
        g.step(mk)
        out = _outputs(g, [a, b])
        for k in ("obs", "rewards", "true_objectives", "dones"):
            assert np.array_equal(out[k][b], out[k][a]), "step %d: %s of the clone" % (t, k)
        for kind in ("state", "voxels", "instances", "level"):
            assert np.array_equal(out["%s%d" % (kind, b)], out["%s%d" % (kind, a)]), "step %d: %s of the clone" % (t, kind)
    _healthy(g)
    m.close()


def test_megaverse_env_with_a_list_and_make_env_mixed(built):
    """MegaverseEnv over a list of names and make_env_mixed: step / reset / render run, and every env's observations equal the same env
    of a single-scenario MegaverseEnv seeded the same (mv_seed draws env e's seed by index, whatever the scenario)"""
    from megaverse_b200 import MegaverseEnv, make_env_mixed

    E = 16
    mixed = make_env_mixed("multitask_megaverse8", E, 1, 2)
    assert mixed.scenarios == [s.casefold() for s in (MEGAVERSE8 * 2)]
    listed = MegaverseEnv(MEGAVERSE8 * 2, E, 1, 2)
    singles = {s: MegaverseEnv(s, E, 1, 1) for s in MEGAVERSE8}
    for env in [mixed, listed] + list(singles.values()):
        env.seed(77)
    obs = {id(env): env.reset() for env in [mixed, listed] + list(singles.values())}
    rng = np.random.default_rng(6)
    for t in range(25):
        for e, s in enumerate(MEGAVERSE8 * 2):
            for x in (mixed, listed):
                assert np.array_equal(obs[id(x)][e], obs[id(singles[s])][e]), "step %d env %d (%s)" % (t, e, s)
        actions = rng.integers(0, [3, 3, 3, 2, 2, 3], size=(E, 6))
        for env in [mixed, listed] + list(singles.values()):
            obs[id(env)], rewards, dones, infos = env.step(actions)
            assert len(rewards) == len(dones) == len(infos) == E
    for e, s in enumerate(MEGAVERSE8 * 2):
        assert mixed.get_default_reward_shaping(e) == singles[s].get_default_reward_shaping(), (e, s)
    assert mixed.get_default_reward_shaping() == singles["TowerBuilding"].get_default_reward_shaping()
    frame = mixed.render(mode="rgb_array")
    assert frame.shape == (E * 432, 768, 3)
    for env in [mixed, listed] + list(singles.values()):
        env.close()
