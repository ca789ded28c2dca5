"""Reward components (option "reward_components"): the step rows against the oracle's per-slot columns bit for bit (masked-weight oracle
twins, tests/reward_components.py), the episode rows against the call-order float32 sums of the step rows, every rule in its own column
on the scripted event scenes of test_events_gpu, action repeat, active sets, restarts, requested ends in the device loop, the state store,
mixed engines, byte-identical other outputs, the misuse refusals and MegaverseEnv's infos."""
import ctypes as C

import numpy as np
import pytest

import helpers
import reward_components as rc

pytestmark = pytest.mark.gpu

INTERACT = 1 << 8


def _engine(scenario, E, A, seeds, params=None, on=True, depth=False, segmentation=False, **options):
    from megaverse_b200 import capi

    g = capi.Engine(scenario, E, A, 128, 72, num_threads=2, params=params, depth=depth, segmentation=segmentation)
    if on:
        g.set_option("reward_components", 1)
    for k, v in options.items():
        g.set_option(k, v)
    for e, s in enumerate(seeds):
        g.seed_env(e, s)
    return g


def _rows(g):
    step, ep = g.reward_components()
    return np.array(step), np.array(ep)


def _check_sum(g, step, tag):
    r = np.array(g.rewards(), dtype=np.float64)
    s = step.astype(np.float64).sum(axis=1)
    assert np.all(np.abs(s - r) <= 1e-5 + 1e-6 * np.abs(r)), "%s: columns sum %s, rewards %s" % (tag, s, r)
    assert not step[:, 0].any(), "%s: column 0 paid" % tag


def _short(scenario):
    """short episodes: the length's base at 1 s (TowerBuilding, Collect and HexMemory add time per object, Obstacles 35 s per platform, so
    those courses get at most two platforms)"""
    p = {"episodeLengthSec": 1.0}
    if rc.family(scenario) == "obstacles":
        p["obstaclesMaxNumPlatforms"] = 2.0
        p["obstaclesMinNumPlatforms"] = 1.0
    return p


# ------------------------------------------------------------------------------------------------ lockstep against the oracle
LOCKSTEP = [(n, 2, "random") for n in rc.NAMES] + [("TowerBuilding", 1, "default"), ("Collect", 4, "random"), ("ObstaclesHard", 4, "default"),
                                                   ("Sokoban", 1, "random"), ("HexMemory", 4, "random"), ("Rearrange", 4, "default")]


@pytest.mark.parametrize("scenario,A,shaping_kind", LOCKSTEP)
def test_step_rows_match_the_oracle(built, scenario, A, shaping_kind):
    E, cap = 4, 2500
    rng = np.random.default_rng(7 + A)
    params = _short(scenario)
    seeds = [400 + 13 * e for e in range(E)]
    shaping = [d for _ in range(E) for d in rc.random_shaping(rng, scenario, A)] if shaping_kind == "random" else None
    ref = rc.SlotOracles(scenario, E, A, params=params, shaping=shaping)
    g = _engine(scenario, E, A, seeds, params=params)
    try:
        for e, s in enumerate(seeds):
            ref.seed_env(e, s)
        if shaping is not None:
            for v, d in enumerate(shaping):
                g.set_reward_shaping(v // A, v % A, d)
        ref.reset()
        g.reset()
        step, ep = _rows(g)
        assert not step.any() and not ep.any()
        mine, theirs = rc.Totals(E * A, A), rc.Totals(E * A, A)
        ends = 0
        for t in range(cap):
            if t >= 100 and ends >= 3:
                break
            acts = helpers.purposeful_actions(rng, E * A, t) if rc.family(scenario) != "rearrange" else np.concatenate(
                [helpers.rearrange_controller(ref.main, e, A) for e in range(E)]).astype(np.int32)
            ref.step(acts)
            g.step(acts)
            tag = "%s A=%d t=%d" % (scenario, A, t)
            rc.same_bits(g.rewards(), ref.rewards(), tag + " rewards")
            assert np.array_equal(np.array(g.dones()), ref.dones()), tag
            step, ep = _rows(g)
            rc.same_bits(step, ref.columns(), tag + " step rows")
            _check_sum(g, step, tag)
            mine.add(step, g.dones())
            theirs.add(ref.columns(), ref.dones())
            mine.check(ep, tag)
            theirs.check(ep, tag + " (oracle sums)")
            ends += int(np.count_nonzero(g.dones()))
        assert ends > 0
        assert g.faults() == 0
    finally:
        ref.close()
        g.close()


def test_mixed_engine_rows_equal_single_scenario_engines(built):
    """MEGAVERSE8 in one engine: env e's rows equal those of env j of a single-scenario engine of its name, seeded the same"""
    from test_mixed_gpu import MEGAVERSE8, Mixed

    A, copies = 2, 2
    rng = np.random.default_rng(3)
    m = Mixed(MEGAVERSE8, copies, "interleaved", A, {"episodeLengthSec": 3.0}, reward_components=1)
    try:
        shaping = {}
        for n in MEGAVERSE8:
            shaping[n] = rc.random_shaping(rng, n, A)
        for e, (n, j) in enumerate(m.slot):
            for a in range(A):
                m.g.set_reward_shaping(e, a, shaping[n][a])
                m.refs[n].set_reward_shaping(j, a, shaping[n][a])
        tot = rc.Totals(m.E * A, A)
        ends = 0
        for t in range(100):
            acts = helpers.purposeful_actions(rng, m.E * A, t)
            m.g.step(acts)
            for n, r in m.refs.items():
                sub = np.concatenate([acts[e * A:(e + 1) * A] for e, (nn, _) in enumerate(m.slot) if nn == n])
                r.step(sub)
            step, ep = _rows(m.g)
            for e, (n, j) in enumerate(m.slot):
                rs, re_ = _rows(m.refs[n])
                tag = "t=%d env %d (%s %d)" % (t, e, n, j)
                rc.same_bits(step[e * A:(e + 1) * A], rs[j * A:(j + 1) * A], tag + " step")
                rc.same_bits(ep[e * A:(e + 1) * A], re_[j * A:(j + 1) * A], tag + " episode")
            _check_sum(m.g, step, "mixed t=%d" % t)
            tot.add(step, m.g.dones())
            tot.check(ep, "mixed t=%d" % t)
            ends += int(np.count_nonzero(m.g.dones()))
        assert ends > 0
    finally:
        for x in m.engines():
            x.close()


# ------------------------------------------------------------------------------------------------ every rule in its own column
def _event_run_class():
    import test_events_gpu as ev

    class RCRun(ev.Run):
        """test_events_gpu's warped coverage run with option reward_components on: every tick, every slot's column of every agent is
        the decoded count of its event times the slot's weight"""

        def __init__(self, *args, **kw):
            from megaverse_b200 import capi

            real = capi.Engine

            class On(real):
                def reset(self):
                    if not getattr(self, "_rc_on", False):
                        self.set_option("reward_components", 1)
                        self._rc_on = True
                    super().reset()

            capi.Engine = On
            try:
                super().__init__(*args, **kw)
            finally:
                capi.Engine = real
            self.col_paid = np.zeros(rc.R_COUNT, dtype=np.int64)
            self.fall_paid = 0
            self.totals = rc.Totals(self.E * self.A, self.A)

        def step(self, acts, tag, host=True):
            falls = self.counts.get("fall", 0)
            d = super().step(acts, tag, host)
            if not host:
                return d
            step, ep = _rows(self.g)
            r = self.o.rewards()
            slots = rc.KEY_SLOTS[self.fam]
            for v in range(self.E * self.A):
                a = v % self.A
                val = float(r[v]) / 2.0 ** a
                if self.fam == "tower":
                    val = round(val)
                for k, key in enumerate(self.keys):
                    s = slots[key]
                    if self.fam == "tower" and key == "towerBuildingReward":
                        continue
                    want = np.float32(((int(val) >> (4 * k)) & 15) * 16.0 ** k * 2.0 ** a)
                    assert step[v, s] == want, "%s view %d: column %d (%s) %r, want %r" % (tag, v, s, key, float(step[v, s]), float(want))
            self.col_paid += np.count_nonzero(step, axis=0)
            if self.fam == "collect" and self.counts.get("fall", 0) > falls and step[:, slots["collectSingleBad"]].any():
                self.fall_paid += 1
            _check_sum(self.g, step, tag)
            self.totals.add(step, self.g.dones())
            self.totals.check(ep, tag)
            return d

    return ev, RCRun


EVENT_RUNS = [("TowerBuilding", 2, 12, 320, 101), ("ObstaclesHard", 3, 8, 240, 104), ("ObstaclesWalls", 2, 10, 240, 105),
              ("Collect", 2, 12, 320, 109), ("Sokoban", 2, 12, 240, 111), ("Rearrange", 2, 8, 450, 113), ("HexExplore", 2, 12, 200, 114),
              ("HexMemory", 2, 8, 260, 117)]


@pytest.mark.parametrize("scenario,A,E,ticks,seed", EVENT_RUNS)
def test_every_rule_pays_in_its_own_column(built, scenario, A, E, ticks, seed):
    ev, RCRun = _event_run_class()
    run = RCRun(scenario, E, A, seed, params={"episodeLengthSec": 30.0})
    try:
        run.seen_rewards = any(len(run.level_rewards(e)) for e in range(E)) if run.fam in ("obstacles", "collect") else False
        run.seen_objects = any(len(run.objects(e)) for e in range(E))
        run.seen_lava = any(len(ev.cells(run, e, 0x200)) for e in range(E)) if run.fam == "obstacles" else False
        ev.drive(run, ticks, np.random.default_rng(seed))
        names = dict(zip(ev.EVENTS[run.fam], run.keys))
        for event in ev.required_events(run):
            if event in names:
                s = rc.KEY_SLOTS[run.fam][names[event]]
                assert run.col_paid[s] > 0, "%s: column %d (%s) never paid\n%s" % (scenario, s, names[event], run.table())
        unused = [s for s in range(rc.R_COUNT) if s not in rc.KEY_SLOTS[run.fam].values()]
        assert not run.col_paid[unused].any(), "%s: a column without a key paid: %s" % (scenario, run.col_paid)
        if run.fam == "collect":
            assert run.fall_paid > 0, "no Collect fall paid under collectSingleBad\n%s" % run.table()
            assert run.col_paid[rc.KEY_SLOTS["collect"]["collectAbyss"]] == 0
    finally:
        run.close()


# ------------------------------------------------------------------------------------------------ action repeat
@pytest.mark.parametrize("k", [2, 4])
@pytest.mark.parametrize("scenario", ["Collect", "TowerBuilding", "ObstaclesMedium"])
def test_action_repeat_sums_oracle_ticks_in_tick_order(built, scenario, k):
    """per env an oracle of its own (the envs end at different ticks): up to k ticks per call, Interact on the first only, the ending tick
    paying nothing; the call's columns are the tick columns summed in tick order from 0.0f"""
    E, A, cap = 3, 2, 1500
    rng = np.random.default_rng(50 + k)
    params = _short(scenario)
    seeds = [900 + e for e in range(E)]
    shaping = [d for _ in range(E) for d in rc.random_shaping(rng, scenario, A)]
    refs = [rc.SlotOracles(scenario, 1, A, params=params, shaping=shaping[e * A:(e + 1) * A]) for e in range(E)]
    g = _engine(scenario, E, A, seeds, params=params, action_repeat=k)
    try:
        for v, d in enumerate(shaping):
            g.set_reward_shaping(v // A, v % A, d)
        for e in range(E):
            refs[e].seed_env(0, seeds[e])
            refs[e].reset()
        g.reset()
        tot = rc.Totals(E * A, A)
        ends = 0
        for t in range(cap):
            if t >= 40 and ends >= 2:
                break
            acts = helpers.purposeful_actions(rng, E * A, t)
            g.step(acts)
            want = np.zeros((E * A, rc.R_COUNT), dtype=np.float32)
            for e in range(E):
                for j in range(k):
                    m = acts[e * A:(e + 1) * A].copy()
                    if j > 0:
                        m &= ~INTERACT
                    refs[e].step(m)
                    if refs[e].dones()[0]:
                        break
                    want[e * A:(e + 1) * A] = (want[e * A:(e + 1) * A] + refs[e].columns()).astype(np.float32)
            step, ep = _rows(g)
            tag = "%s k=%d call %d" % (scenario, k, t)
            rc.same_bits(step, want, tag)
            _check_sum(g, step, tag)
            tot.add(step, g.dones())
            tot.check(ep, tag)
            ends += int(np.count_nonzero(g.dones()))
        assert ends > 0
    finally:
        for r in refs:
            r.close()
        g.close()


# ------------------------------------------------------------------------------------------------ active sets, restarts
def test_active_sets_and_restarts(built):
    """inactive envs: step rows 0, running totals and episode rows kept; mv_reset_envs zeroes only the restarted envs' running totals,
    writes step rows 0 for them and no episode row"""
    E, A = 6, 2
    rng = np.random.default_rng(8)
    g = _engine("Collect", E, A, [70 + e for e in range(E)], params=_short("Collect"))
    try:
        g.reset()
        tot = rc.Totals(E * A, A)
        ends = subset_ends = 0
        for t in range(3000):
            if t >= 150 and ends >= 3 and subset_ends >= 1:
                break
            acts = helpers.purposeful_actions(rng, E * A, t)
            tag = "t=%d" % t
            if t % 37 == 36:
                envs = sorted(rng.choice(E, size=2, replace=False).tolist())
                before_step, before_ep = _rows(g)
                g.reset_envs(envs)
                step, ep = _rows(g)
                for e in range(E):
                    rows = slice(e * A, (e + 1) * A)
                    if e in envs:
                        assert not step[rows].any(), tag + " restarted env %d" % e
                    else:
                        rc.same_bits(step[rows], before_step[rows], tag + " untouched env %d" % e)
                rc.same_bits(ep, before_ep, tag + " episode rows after a restart")
                tot.restart(envs)
                tot.check(ep, tag)
                continue
            if t % 3 == 1:
                active = sorted(rng.choice(E, size=3, replace=False).tolist())
                g.step_envs(acts, active)
            else:
                active = list(range(E))
                g.step(acts)
            step, ep = _rows(g)
            for e in set(range(E)) - set(active):
                assert not step[e * A:(e + 1) * A].any(), tag + " inactive env %d" % e
            _check_sum(g, step, tag)
            tot.add(step, g.dones())
            tot.check(ep, tag)
            ends += int(np.count_nonzero(g.dones()))
            if t % 3 == 1:
                subset_ends += int(np.count_nonzero(g.dones()))
        assert ends > 0 and subset_ends > 0
    finally:
        g.close()


# ------------------------------------------------------------------------------------------------ the device loop with requested ends
@pytest.mark.parametrize("mode", ["level_slots", "level_set"])
def test_requested_ends_in_the_device_loop(built, mode):
    """mv_step_device_ends: the HBM rows equal what mv_fetch_obs copies down, and a requested end writes its episode rows like any end"""
    import torch

    from megaverse_b200 import capi

    E, A = 8, 2
    rng = np.random.default_rng(21)
    opts = {"level_slots": 4} if mode == "level_slots" else {"level_set": 5}
    g = _engine("Collect", E, A, [300 + e for e in range(E)], params={"episodeLengthSec": 4.0}, **opts)
    try:
        g.reset()
        tot = rc.Totals(E * A, A)
        d_acts = torch.zeros(E * A, dtype=torch.int32, device="cuda")
        d_ends = torch.zeros(E, dtype=torch.uint8, device="cuda")
        requested = 0
        for t in range(80):
            acts = helpers.purposeful_actions(rng, E * A, t)
            ends = (rng.random(E) < 0.08).astype(np.uint8)
            d_acts.copy_(torch.from_numpy(acts))
            d_ends.copy_(torch.from_numpy(ends))
            torch.cuda.synchronize()
            g.step_device(d_acts.data_ptr(), d_ends.data_ptr())
            g.fetch_obs()
            step, ep = _rows(g)
            hbm_step = torch.as_tensor(g.device_array("reward_components"), device="cuda").cpu().numpy()
            hbm_ep = torch.as_tensor(g.device_array("episode_reward_components"), device="cuda").cpu().numpy()
            tag = "%s t=%d" % (mode, t)
            rc.same_bits(step, hbm_step, tag + " step rows host vs HBM")
            rc.same_bits(ep, hbm_ep, tag + " episode rows host vs HBM")
            _check_sum(g, step, tag)
            tot.add(step, g.dones())
            tot.check(ep, tag)
            requested += int(np.count_nonzero(np.array(g.done_reasons()) == capi.MV_END_REQUESTED))
        assert requested > 0
    finally:
        g.close()


# ------------------------------------------------------------------------------------------------ the state store
def test_save_load_and_clone_replay(built):
    E, A = 4, 2
    rng = np.random.default_rng(12)
    g = _engine("Test", E, A, [40 + e for e in range(E)])
    try:
        g.reset()
        base = g.state_row_bytes()
        for t in range(20):
            g.step(helpers.purposeful_actions(rng, E * A, t))
        saved = _rows(g)
        store = g.states_create(2)
        g.states_save(store, [0, 1], [0, 1])
        acts = [helpers.purposeful_actions(rng, E * A, 20 + t) for t in range(150)]
        first, ended = [], 0
        for a in acts:
            g.step(a)
            first.append(_rows(g))
            ended += int(np.count_nonzero(np.array(g.dones())[:2]))
        # load: rows read as after the saved step, and the next calls replay bit for bit
        g.states_load(store, [0, 1], [0, 1])
        step, ep = _rows(g)
        rc.same_bits(step[:2 * A], saved[0][:2 * A], "after load: step rows")
        rc.same_bits(ep[:2 * A], saved[1][:2 * A], "after load: episode rows")
        for i, a in enumerate(acts):
            g.step(a)
            step, ep = _rows(g)
            rc.same_bits(step[:2 * A], first[i][0][:2 * A], "replay call %d step" % i)
            rc.same_bits(ep[:2 * A], first[i][1][:2 * A], "replay call %d episode" % i)
        # clone: env 0's saved row into envs 0 and 2; with the same actions env 2's rows are env 0's
        g.states_load(store, [0, 0], [0, 2])
        for i, a in enumerate(acts):
            a = a.copy()
            a[2 * A:3 * A] = a[0:A]
            g.step(a)
            step, ep = _rows(g)
            rc.same_bits(step[2 * A:3 * A], step[0:A], "clone call %d step" % i)
            rc.same_bits(ep[2 * A:3 * A], ep[0:A], "clone call %d episode" % i)
        assert ended > 0, "no episode of envs 0, 1 ended in the replay window"
        off = _engine("Test", E, A, [40 + e for e in range(E)], on=False)
        off.reset()
        assert base - off.state_row_bytes() == 96 * A
        off.close()
    finally:
        g.close()


# ------------------------------------------------------------------------------------------------ nothing else changes
@pytest.mark.parametrize("path", ["host", "device"])
def test_every_other_output_is_byte_identical(built, path):
    import torch

    from megaverse_b200 import rays

    E, A = 6, 2
    seeds = [600 + e for e in range(E)]
    params = {"episodeLengthSec": -20.0}  # 2 s per reward object less 20: from one-call episodes to a few seconds
    engines = []
    for on in (False, True):
        g = _engine("Collect", E, A, seeds, params=params, on=on, depth=True, segmentation=True, state_tensors=1, final_obs=1,
                    level_slots=4)
        g.set_rays(rays.fan(16, 90.0), 60.0)
        g.reset()
        engines.append(g)
    rng = np.random.default_rng(2)
    d_acts = torch.zeros(E * A, dtype=torch.int32, device="cuda")
    try:
        for t in range(120):
            acts = helpers.purposeful_actions(rng, E * A, t)
            for g in engines:
                if path == "host":
                    g.step(acts)
                else:
                    d_acts.copy_(torch.from_numpy(acts))
                    torch.cuda.synchronize()
                    g.step_device(d_acts.data_ptr())
                    g.fetch_obs()
            a, b = engines
            outs = [("obs", lambda g: g.obs()), ("depth", lambda g: g.depth()), ("seg", lambda g: g.segmentation()),
                    ("rewards", lambda g: g.rewards()), ("dones", lambda g: g.dones()), ("reasons", lambda g: g.done_reasons()),
                    ("true objectives", lambda g: g.true_objectives()), ("final obs", lambda g: g.final_obs()),
                    ("final depth", lambda g: g.final_depth()), ("rays", lambda g: g.rays()[0]), ("tags", lambda g: g.rays()[1]),
                    ("final rays", lambda g: g.final_rays()[0])]
            for name, f in outs:
                x, y = np.array(f(a)), np.array(f(b))
                assert x.tobytes() == y.tobytes(), "%s t=%d: %s differs" % (path, t, name)
            for which in ("state_tensors", "final_state_tensors"):
                sa, sb = getattr(a, which)(), getattr(b, which)()
                for k in sa:
                    assert np.array(sa[k]).tobytes() == np.array(sb[k]).tobytes(), "%s t=%d: %s %s differs" % (path, t, which, k)
    finally:
        for g in engines:
            g.close()


# ------------------------------------------------------------------------------------------------ misuse
def test_refusals(built):
    from megaverse_b200 import capi

    L = capi.lib()
    p, q = C.c_void_p(), C.c_void_p()
    g = capi.Engine("Collect", 2, 2, num_threads=1)
    try:
        assert L.mv_set_option(g._h, b"reward_components", 2) == capi.MV_ERR_ARG
        assert L.mv_set_option(g._h, b"reward_components", -1) == capi.MV_ERR_ARG
        assert L.mv_reward_components_host(g._h, C.byref(p), C.byref(q)) == capi.MV_ERR_ARG  # off
        assert L.mv_set_option(g._h, b"reward_components", 1) == capi.MV_OK
        assert L.mv_reward_components_host(g._h, C.byref(p), C.byref(q)) == capi.MV_ERR_STATE  # before mv_reset
        assert L.mv_reward_components_device(g._h, C.byref(p), C.byref(q)) == capi.MV_ERR_STATE
        g.reset()
        assert L.mv_set_option(g._h, b"reward_components", 0) == capi.MV_ERR_STATE
        assert L.mv_reward_components_host(g._h, None, None) == capi.MV_OK
        assert L.mv_reward_components_device(g._h, C.byref(p), None) == capi.MV_OK and p.value
        step, ep = g.reward_components()
        assert step.shape == (4, 8) and ep.shape == (4, 8) and not step.any() and not ep.any()
    finally:
        g.close()
    off = capi.Engine("Collect", 2, 2, num_threads=1)
    try:
        off.reset()
        assert L.mv_reward_components_host(off._h, C.byref(p), C.byref(q)) == capi.MV_ERR_ARG
        assert L.mv_reward_components_device(off._h, C.byref(p), C.byref(q)) == capi.MV_ERR_ARG
        with pytest.raises(capi.MegaverseError):
            off.reward_components()
    finally:
        off.close()


# ------------------------------------------------------------------------------------------------ MegaverseEnv
def test_megaverse_env_infos_carry_episode_totals(built):
    from megaverse_b200.megaverse_env import MegaverseEnv

    E, A = 4, 2
    env = MegaverseEnv("Collect", E, A, 2, params={"episodeLengthSec": -20.0}, reward_components=True)
    plain = MegaverseEnv("Collect", E, A, 2, params={"episodeLengthSec": -20.0})
    try:
        env.seed(5)
        plain.seed(5)
        env.reset()
        plain.reset()
        keys = env.reward_component_keys(0)
        assert keys == rc.keys8("Collect")
        rng = np.random.default_rng(0)
        tot = rc.Totals(E * A, A)
        seen = 0
        for t in range(80):
            acts = [[int(rng.integers(0, s)) for s in helpers.SIZES] for _ in range(E * A)]
            obs, rew, dones, infos = env.step(acts)
            obs2, rew2, dones2, infos2 = plain.step(acts)
            assert np.array_equal(np.asarray(rew), np.asarray(rew2)) and list(dones) == list(dones2)
            assert all(np.array_equal(x, y) for x, y in zip(obs, obs2))
            step = np.array(env.reward_components())
            assert step.shape == (E * A, 8)
            env_dones = np.array(dones[::A], dtype=np.uint8)
            tot.add(step, env_dones)
            for v in range(E * A):
                if dones[v]:
                    got = infos[v]["reward_components"]
                    assert list(got) == [k for k in keys if k]
                    for c, k in enumerate(keys):
                        if k:
                            assert np.float32(got[k]) == tot.episode[v, c], (t, v, k)
                    assert "reward_components" not in infos2[v]
                    seen += 1
                else:
                    assert "reward_components" not in infos[v]
        assert seen > 0
    finally:
        env.close()
        plain.close()
