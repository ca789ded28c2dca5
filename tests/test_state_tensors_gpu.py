"""State tensors (option "state_tensors"): the agent, env, object and reward rows the step kernel writes beside the frames, bit for bit
against the oracle stepped env by env (live rows after every call, terminal rows before the oracle's Env::reset), against the engine's own
host-side state dump (restarts, the state store, active sets, mixed and level-set engines), and for byte-identical other outputs."""
import ctypes as C

import numpy as np
import pytest

import helpers
import state_rows

pytestmark = pytest.mark.gpu

ALL = ["TowerBuilding", "Collect", "Rearrange", "Sokoban", "HexExplore", "HexMemory", "Empty", "ObstaclesEasy", "ObstaclesMedium",
       "ObstaclesHard", "ObstaclesWalls", "ObstaclesSteps", "ObstaclesLava"]
KEYS = ("agents", "envs", "objects", "rewards")


def _engine(scenario, E, A, seed, params=None, state=True, final=True, **options):
    from megaverse_b200 import capi

    g = capi.Engine(scenario, E, A, 128, 72, num_threads=2, params=params)
    if state:
        g.set_option("state_tensors", 1)
    if final:
        g.set_option("final_obs", 1)
    for k, v in options.items():
        g.set_option(k, v)
    g.seed(seed)
    g.reset()
    return g


def _env_rows(t, e, A):
    """env e's rows of a state-tensor dict, copied"""
    return {"agents": np.array(t["agents"][e * A:(e + 1) * A]), "envs": np.array(t["envs"][e]), "objects": np.array(t["objects"][e]),
            "rewards": np.array(t["rewards"][e])}


def _engine_dump(g, e, what):
    from megaverse_b200 import capi

    cap = 1 << 16
    dt = np.float32 if what == "state" else np.int32
    out = np.zeros(cap, dtype=dt)
    n = getattr(capi.lib(), "mv_debug_get_" + what)(g._h, e, out.ctypes.data, cap)
    assert n >= 0
    return out[:n].copy()


def _check_against_dump(g, name, tag, envs=None, tensors=None):
    """the rows against the engine's own host-side dump of its HBM state (mv_debug_get_state / _level), every env or the listed ones"""
    t = tensors or g.state_tensors()
    names = [name] * g.E if isinstance(name, str) else name
    for e in (range(g.E) if envs is None else envs):
        want, known, sign = state_rows.expected_rows(names[e], g.A, _engine_dump(g, e, "state"), _engine_dump(g, e, "level"))
        state_rows.compare("%s env %d" % (tag, e), _env_rows(t, e, g.A), want, known, sign)


class Mirror:
    """the oracle driven env by env (orc_scen_step / orc_scen_reset), so that an ended env can be read before its reset and ended on request"""

    def __init__(self, scenario, E, A, seed, params=None):
        import orc

        self.L = orc.lib()
        self.L.orc_scen_step.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        self.L.orc_scen_reset.argtypes = [C.c_void_p, C.c_int]
        self.o = orc.Oracle(scenario, E, A, params=params, render=False)
        self.o.seed(seed)
        self.o.reset()
        self.name, self.E, self.A = scenario, E, A

    def close(self):
        self.o.close()

    def tick(self, e, acts):
        a = np.ascontiguousarray(acts[e * self.A:(e + 1) * self.A], dtype=np.int32)
        self.L.orc_scen_step(self.o.h_, e, a.ctypes.data)
        return self.o.state(e)[7] != 0  # the env's done flag

    def step(self, acts, repeat=1, envs=None):
        """one engine call: up to `repeat` ticks per env (Interact on the first only), stopping at the env's end"""
        for e in (range(self.E) if envs is None else envs):
            for k in range(repeat):
                if self.tick(e, acts if k == 0 else acts & ~np.int32(1 << 8)):
                    break

    def expected(self, e):
        return state_rows.expected_rows(self.name, self.A, self.o.state(e), self.o.level(e))

    def check(self, g, dones, tag, tensors=None, final=None):
        """terminal rows of the ended envs (then their reset), and every env's live rows"""
        for e in np.flatnonzero(dones):
            if final is not None:
                want, known, sign = self.expected(e)
                state_rows.compare("%s env %d terminal" % (tag, e), _env_rows(final, e, self.A), want, known, sign)
            self.L.orc_scen_reset(self.o.h_, e)
        t = tensors if tensors is not None else g.state_tensors()
        for e in range(self.E):
            want, known, sign = self.expected(e)
            state_rows.compare("%s env %d" % (tag, e), _env_rows(t, e, self.A), want, known, sign)


def _params(name):
    """short episodes, so that every run crosses episode ends (Collect's length grows with its object count, Obstacles' with its platforms)"""
    if name == "Rearrange":
        return {"episodeLengthSec": 8.0}
    if name == "Collect":
        return {"episodeLengthSec": -45.0}
    if name.startswith("Obstacles"):
        return {"episodeLengthSec": 4.0, "obstaclesMinNumPlatforms": 0, "obstaclesMaxNumPlatforms": 0}
    return {"episodeLengthSec": 4.0}


# ------------------------------------------------------------------------------------------------ 1. + 2. lockstep, terminal rows
@pytest.mark.parametrize("name", ALL)
def test_lockstep_against_the_oracle(built, name):
    A = 1 + ALL.index(name) % 4
    if name == "Rearrange":
        A = 2
    E, steps, seed = 3, 220, 41 + ALL.index(name)
    g = _engine(name, E, A, seed, _params(name))
    m = Mirror(name, E, A, seed, _params(name))
    try:
        m.check(g, np.zeros(E, dtype=np.uint8), "%s reset" % name)
        rng = np.random.default_rng(seed)
        ends = carried = 0
        for t in range(steps):
            if name == "Rearrange":
                acts = np.concatenate([helpers.rearrange_controller(m.o, e, A) for e in range(E)]).astype(np.int32)
            else:
                acts = helpers.purposeful_actions(rng, E * A, t)
            g.step(acts)
            m.step(acts)
            d = np.array(g.dones())
            m.check(g, d, "%s t=%d" % (name, t), final=g.final_state_tensors())
            ends += int(d.sum())
            carried += int((g.state_tensors()["objects"][:, :, 3] >= 0).sum())
        assert ends > 0 or name == "TowerBuilding", "no episode ended"  # TowerBuilding's episode length follows its object count
        if name == "Rearrange":
            assert carried > 0, "the solver never carried an object"
        assert g.fault_word() == 0
    finally:
        m.close()
        g.close()


# ------------------------------------------------------------------------------------------------ 2. requested ends, 5. the device loop
@pytest.mark.parametrize("name", ["Collect", "ObstaclesHard", "HexMemory"])
def test_device_loop_with_requested_ends(built, name):
    import torch

    E, A, seed, steps = 6, 2, 77, 120
    g = _engine(name, E, A, seed, _params(name), level_slots=4)
    m = Mirror(name, E, A, seed, _params(name))
    try:
        rng = np.random.default_rng(3)
        dev = {k: torch.as_tensor(g.device_array("state_" + k), device="cuda") for k in KEYS}
        reasons = set()
        for t in range(steps):
            acts = helpers.purposeful_actions(rng, E * A, t)
            req = np.zeros(E, dtype=np.uint8)
            if t % 9 == 4:
                req[rng.integers(0, E)] = 1
            d_acts = torch.from_numpy(acts).cuda()
            d_ends = torch.from_numpy(req).cuda()
            g.step_device(d_acts.data_ptr(), d_ends.data_ptr())
            g.fetch_obs()
            d = np.array(g.dones())
            reasons |= set(int(x) for x in np.array(g.done_reasons())[d != 0])
            m.step(acts)
            host = {k: np.array(v) for k, v in g.state_tensors().items()}
            for k in KEYS:  # HBM in stream order, and mv_fetch_obs brought it down
                hbm = dev[k].cpu().numpy()
                assert np.array_equal(hbm.view(np.uint32), host[k].view(np.uint32)), "%s t=%d: HBM %s differ from the fetched rows" % (name, t, k)
            m.check(g, d, "%s device t=%d" % (name, t), tensors=host, final=g.final_state_tensors())
        assert 3 in reasons and (1 in reasons or name == "HexMemory"), reasons  # HexMemory's clock outlasts the run
    finally:
        m.close()
        g.close()


# ------------------------------------------------------------------------------------------------ 3. action repeat, active sets, restarts
@pytest.mark.parametrize("k", [2, 4])
def test_action_repeat(built, k):
    name, E, A, seed = "Collect", 4, 2, 90 + k
    g = _engine(name, E, A, seed, _params(name), action_repeat=k)
    m = Mirror(name, E, A, seed, _params(name))
    try:
        rng = np.random.default_rng(k)
        ends = 0
        for t in range(90):
            acts = helpers.purposeful_actions(rng, E * A, t)
            g.step(acts)
            m.step(acts, repeat=k)
            d = np.array(g.dones())
            ends += int(d.sum())
            m.check(g, d, "repeat %d t=%d" % (k, t), final=g.final_state_tensors())
        assert ends > 0
    finally:
        m.close()
        g.close()


def test_active_sets(built):
    name, E, A, seed = "ObstaclesEasy", 6, 2, 123
    g = _engine(name, E, A, seed, _params(name))
    m = Mirror(name, E, A, seed, _params(name))
    try:
        rng = np.random.default_rng(8)
        for t in range(80):
            acts = helpers.purposeful_actions(rng, E * A, t)
            active = sorted(rng.choice(E, size=int(rng.integers(1, E)), replace=False).tolist())
            before = {k: np.array(v) for k, v in g.state_tensors().items()}
            g.step_envs(acts, active)
            m.step(acts, envs=active)
            after = g.state_tensors()
            for e in set(range(E)) - set(active):
                for k, v in _env_rows(after, e, A).items():
                    assert np.array_equal(v.view(np.uint32), _env_rows(before, e, A)[k].view(np.uint32)), "t=%d inactive env %d %s changed" % (t, e, k)
            m.check(g, np.array(g.dones()), "active t=%d" % t, final=g.final_state_tensors())
    finally:
        m.close()
        g.close()


def test_restarts(built):
    name, E, A = "Collect", 6, 2
    g = _engine(name, E, A, 5, _params(name))
    try:
        rng = np.random.default_rng(1)
        for t in range(30):
            g.step(helpers.purposeful_actions(rng, E * A, t))
        _check_against_dump(g, name, "after steps")
        g.reset_envs([1, 4])
        _check_against_dump(g, name, "unseeded reset_envs")
        assert (np.array(g.state_tensors()["envs"])[[1, 4], 2] == 0).all()  # num_frames of the new episodes
        g.reset_envs([0, 5], seeds=[17, 18])
        _check_against_dump(g, name, "seeded reset_envs")
        g.reset()
        _check_against_dump(g, name, "mv_reset")
        assert (np.array(g.state_tensors()["envs"])[:, 2] == 0).all()
    finally:
        g.close()


# ------------------------------------------------------------------------------------------------ 4. the state store
def test_state_store(built):
    name, E, A = "Rearrange", 4, 2
    g = _engine(name, E, A, 9, _params(name))
    off = _engine(name, E, A, 9, _params(name), state=False)
    try:
        assert g.state_row_bytes() - off.state_row_bytes() == 64 * A + 4160
        m = Mirror(name, E, A, 9, _params(name))
        try:
            for t in range(60):
                acts = np.concatenate([helpers.rearrange_controller(m.o, e, A) for e in range(E)]).astype(np.int32)
                g.step(acts)
                m.step(acts)
                m.check(g, np.array(g.dones()), "store warm-up t=%d" % t)
        finally:
            m.close()
        store = g.states_create(E)
        g.states_save(store, list(range(E)), list(range(E)))
        saved = {k: np.array(v) for k, v in g.state_tensors().items()}
        rng = np.random.default_rng(2)
        for t in range(25):
            g.step(helpers.purposeful_actions(rng, E * A, t))
        g.states_load(store, list(range(E)), list(range(E)))
        for k, v in g.state_tensors().items():
            assert np.array_equal(np.array(v).view(np.uint32), saved[k].view(np.uint32)), "loaded %s differ from the saved step's" % k
        g.states_load(store, [0, 0], [2, 3])  # clones of env 0
        t2 = g.state_tensors()
        for e in (2, 3):
            for k, v in _env_rows(t2, e, A).items():
                assert np.array_equal(v.view(np.uint32), _env_rows(saved, 0, A)[k].view(np.uint32)), "clone into env %d: %s" % (e, k)
        _check_against_dump(g, name, "after load")
    finally:
        g.close()
        off.close()


# ------------------------------------------------------------------------------------------------ 5. mixed and level-set engines
def test_mixed_and_level_set_engines(built):
    from megaverse_b200 import capi

    names = ["TowerBuilding", "ObstaclesHard", "Collect", "Sokoban", "HexExplore", "HexMemory", "Rearrange", "ObstaclesEasy"]
    mixed = capi.Engine(names, len(names), 2, 128, 72, num_threads=2, params={"episodeLengthSec": 3.0})
    mixed.set_option("state_tensors", 1)
    mixed.seed(4)
    mixed.reset()
    ls = _engine("Collect", 6, 2, 4, _params("Collect"), level_set=5)
    try:
        rng = np.random.default_rng(6)
        for t in range(70):
            mixed.step(helpers.purposeful_actions(rng, mixed.N, t))
            ls.step(helpers.purposeful_actions(rng, ls.N, t))
            if t % 5 == 0 or np.array(mixed.dones()).any() or np.array(ls.dones()).any():
                _check_against_dump(mixed, names, "mixed t=%d" % t)
                _check_against_dump(ls, "Collect", "level set t=%d" % t)
        assert (np.array(mixed.state_tensors()["envs"])[:, 3] == [state_rows.scenario_code(n) for n in names]).all()
    finally:
        mixed.close()
        ls.close()


# ------------------------------------------------------------------------------------------------ 6. every other output is unchanged
def test_other_outputs_identical(built):
    E, A, steps = 256, 4, 300
    from megaverse_b200 import capi

    engines = []
    for s in (False, True):
        g = capi.Engine("Collect", E, A, 128, 72, num_threads=4, params=_params("Collect"), depth=True, segmentation=True)
        g.set_option("final_obs", 1)
        if s:
            g.set_option("state_tensors", 1)
        g.seed(31)
        g.reset()
        engines.append(g)
    try:
        rng = np.random.default_rng(12)
        ended = 0
        for t in range(steps):
            acts = helpers.purposeful_actions(rng, E * A, t)
            for g in engines:
                g.step(acts)
            a, b = engines
            for what in ("obs", "depth", "segmentation", "rewards", "dones", "done_reasons", "true_objectives", "final_obs", "final_depth"):
                x, y = np.array(getattr(a, what)()), np.array(getattr(b, what)())
                assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), "t=%d: %s differ with the option on" % (t, what)
            ended += int(np.array(a.dones()).sum())
        assert ended > 0
    finally:
        for g in engines:
            g.close()


# ------------------------------------------------------------------------------------------------ 7. Python
def test_python_surface(built):
    from megaverse_b200 import capi
    from megaverse_b200.megaverse_env import MegaverseEnv

    E, A = 4, 2
    env = MegaverseEnv("Collect", E, A, 2, params={"episodeLengthSec": -45.0}, final_observation=True, state_tensors=True)
    twin = capi.Engine("Collect", E, A, 128, 72, num_threads=2, params={"episodeLengthSec": -45.0})
    twin.set_option("state_tensors", 1)
    twin.set_option("final_obs", 1)
    try:
        env.seed(21)
        twin.seed(21)
        env.reset()
        twin.reset()
        rng = np.random.default_rng(4)
        seen_final = 0
        for t in range(60):
            heads = np.stack([[rng.integers(0, s) for s in helpers.SIZES] for _ in range(E * A)]).astype(np.int32)
            _, _, dones, infos = env.step(heads)
            twin.step(np.array([helpers.encode(h) for h in heads], dtype=np.int32))
            mine, theirs = env.state_tensors(), twin.state_tensors()
            assert set(mine) == set(KEYS)
            for k in KEYS:
                assert np.array_equal(np.asarray(mine[k]).view(np.uint32), np.asarray(theirs[k]).view(np.uint32)), "t=%d %s" % (t, k)
            fin = twin.final_state_tensors()["agents"]
            for v, (d, info) in enumerate(zip(dones, infos)):
                if d:
                    assert np.array_equal(info["final_state"].view(np.uint32), np.asarray(fin[v]).view(np.uint32))
                    seen_final += 1
                else:
                    assert "final_state" not in info
        assert seen_final > 0
    finally:
        env.close()
        twin.close()


# ------------------------------------------------------------------------------------------------ 8. misuse
def test_misuse(built):
    from megaverse_b200 import capi

    g = capi.Engine("Collect", 2, 1, 128, 72)
    try:
        with pytest.raises(capi.MegaverseError) as ex:
            g.set_option("state_tensors", 2)
        assert ex.value.code == capi.MV_ERR_ARG
        g.set_option("state_tensors", 1)
        with pytest.raises(capi.MegaverseError) as ex:
            g.state_tensors()
        assert ex.value.code == capi.MV_ERR_STATE  # before mv_reset
        with pytest.raises(capi.MegaverseError) as ex:
            g.final_state_tensors()
        assert ex.value.code == capi.MV_ERR_ARG  # final_obs is off
        g.reset()
        assert g.state_tensors()["agents"].shape == (2, 16)
        with pytest.raises(capi.MegaverseError) as ex:
            g.set_option("state_tensors", 0)
        assert ex.value.code == capi.MV_ERR_STATE
    finally:
        g.close()
    off = _engine("Collect", 2, 1, 3, state=False, final=True)
    try:
        for fn in (off.state_tensors, off.final_state_tensors):
            with pytest.raises(capi.MegaverseError) as ex:
                fn()
            assert ex.value.code == capi.MV_ERR_ARG
        with pytest.raises(capi.MegaverseError) as ex:
            off.device_array("state_agents")
        assert ex.value.code == capi.MV_ERR_ARG
    finally:
        off.close()
