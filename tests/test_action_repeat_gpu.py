"""Action repeat (option "action_repeat" k): every step call runs up to k physics ticks with the same masks (Interact on the first tick only),
stops at an episode end and draws once; rewards are the float32 sums of the ticks before the end.

Checked against a per-env mirror of the oracle (orc_scen_step / orc_scen_reset) that steps each env up to k ticks and stops at its done tick,
against a k = 1 twin engine stepped k times per call, for byte-identical outputs at k = 1, for requested ends and for the asynchronous
loop, the state store and MegaverseEnv."""
import ctypes as C

import numpy as np
import pytest

import helpers
import test_events_gpu as ev
import test_final_obs_gpu as fin

pytestmark = pytest.mark.gpu

INTERACT = 1 << 8
AG = ev.AG


# ------------------------------------------------------------------------------------------------ 1. against the oracle
class RepeatRun(ev.Run):
    """test_events_gpu's warped run with the engine at action_repeat k (and final_obs), its oracle stepped env by env: up to k ticks per
    call, tick 0 with the full masks and the rest without Interact, stopping at the env's done tick (drawn there, then Env::reset)"""

    def __init__(self, scenario, E, A, seed, params, k, fast_shading=False):
        from megaverse_b200 import capi

        base = capi.Engine

        class Armed(base):
            def __init__(self, *a, **kw):
                super().__init__(*a, **kw)
                self.set_option("action_repeat", k)
                self.set_option("final_obs", 1)

        capi.Engine = Armed
        try:
            super().__init__(scenario, E, A, seed, params=params, fast_shading=fast_shading)
        finally:
            capi.Engine = base
        self.O.orc_scen_step.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        self.O.orc_scen_reset.argtypes = [C.c_void_p, C.c_int]
        self.k = k
        self.to = np.zeros(E * A, dtype=np.float32)  # true objectives hold their value between ends, as the engine's do
        self.offsets = [0] * k  # episode ends by the tick of the call they fell on
        self.reasons = {1: 0, 2: 0}
        self.carry_events = 0   # pick-ups and put-downs
        self.call_rewards = np.zeros(E * A, dtype=np.float32)

    def terminal(self, e):
        """the oracle's env e as it stands after its done tick, before Env::reset"""
        import orc

        inst = self.o.instances(e)
        rgba = np.zeros((self.A, 72, 128, 4), dtype=np.uint8)
        depth = np.zeros((self.A, 72, 128), dtype=np.float32)
        for a in range(self.A):
            rgba[a], depth[a] = orc.render_instances(self.o.view(e, a), inst, 128, 72, want_depth=True)
        return rgba, depth

    def compare_state(self, e, tag):
        """as test_events_gpu's, except that the engine reports the call's summed reward where the oracle holds its last tick's"""
        so, sg = self.o.state(e), self.g.state(e)
        assert so.shape == sg.shape, "%s env %d: state size %d vs %d" % (tag, e, so.size, sg.size)
        so[8 + AG * np.arange(self.A) + 24] = self.call_rewards[e * self.A:(e + 1) * self.A]
        if not np.array_equal(so.view(np.uint32), sg.view(np.uint32)):
            bad = np.nonzero(so.view(np.uint32) != sg.view(np.uint32))[0]
            raise AssertionError("%s env %d: state words %s differ: oracle %s device %s" % (tag, e, bad[:8], so[bad[:8]], sg[bad[:8]]))
        assert np.array_equal(self.o.voxels(e), self.g.voxels(e)), "%s env %d: voxels" % (tag, e)

    def step(self, acts, tag, host=True):
        acts = np.ascontiguousarray(acts, dtype=np.int32)
        self.g.step(acts)
        rew, done, why, term = self.mirror(acts)
        g = self.g
        assert np.array_equal(rew.view(np.uint32), np.array(g.rewards()).view(np.uint32)), "%s: rewards %s vs %s" % (tag, rew, np.array(g.rewards()))
        assert np.array_equal(done, np.array(g.dones())), "%s: dones" % tag
        assert np.array_equal(why, np.array(g.done_reasons())), "%s: reasons %s vs %s" % (tag, why, np.array(g.done_reasons()))
        assert np.array_equal(self.to.view(np.uint32), np.array(g.true_objectives()).view(np.uint32)), "%s: true objectives" % tag
        if term:
            fo, fd = np.array(g.final_obs()), np.array(g.final_depth())
            for e, (rgba, depth) in term.items():
                fin._frames_match(rgba, fo[e * self.A:(e + 1) * self.A], self.fast, "%s env %d terminal frame" % (tag, e))
                assert np.array_equal(depth.view(np.uint32), fd[e * self.A:(e + 1) * self.A].view(np.uint32)), "%s env %d terminal depth" % (tag, e)
        return done

    def mirror(self, acts):
        """the oracle's side of one call: per env up to k ticks, stopping at the done tick; returns rewards, dones, reasons, terminal frames"""
        E, A, k = self.E, self.A, self.k
        rew = np.zeros(E * A, dtype=np.float32)
        done = np.zeros(E, dtype=np.uint8)
        why = np.zeros(E, dtype=np.uint8)
        term = {}
        for e in range(E):
            masks = acts[e * A:(e + 1) * A].copy()
            total = np.zeros(A, dtype=np.float32)
            prev = self.states[e]
            for t in range(k):
                self.O.orc_scen_step(self.o.h_, e, masks.ctypes.data)
                st = self.o.state(e)
                self.carry_events += sum(int(prev[8 + AG * a + 22] != st[8 + AG * a + 22]) for a in range(A))
                prev = st
                if st[7]:  # Env::done: this tick ends the episode and pays 0
                    done[e] = 1
                    self.offsets[t] += 1
                    solved = self.fam != "tower" and st[-8] != 0
                    self.to[e * A:(e + 1) * A] = st[3] if self.fam == "tower" else np.float32(solved)
                    why[e] = 2 if solved else 1
                    self.reasons[int(why[e])] += 1
                    term[e] = self.terminal(e)
                    self.O.orc_scen_reset(self.o.h_, e)
                    break
                total += st[8 + AG * np.arange(A) + 24]  # lastReward, float32 in tick order
                masks &= ~np.int32(INTERACT)
            rew[e * A:(e + 1) * A] = total
        self.states = [self.o.state(e) for e in range(E)]
        self.call_rewards = rew
        self.dones += int(done.sum())
        return rew, done, why, term


ORACLE_CASES = [
    # scenario, A, E, calls, k, seed, params, fast shading.  The lengths make the ends of each k fall on every tick offset of a call across
    # its cases: a level's clock end comes after a fixed number of ticks, so the offset varies with the level's length (objects, rewards)
    # and with the tick a rule solved it (the end follows 0.3 s later)
    ("TowerBuilding", 4, 4, 90, 2, 501, {"episodeLengthSec": -180.0}, False),
    ("ObstaclesHard", 1, 8, 70, 3, 502, {"episodeLengthSec": 3.0, "obstaclesMinNumPlatforms": 0, "obstaclesMaxNumPlatforms": 0}, False),
    ("ObstaclesEasy", 4, 4, 60, 4, 503, {"episodeLengthSec": 1.0, "obstaclesMinNumPlatforms": 0, "obstaclesMaxNumPlatforms": 0}, False),
    ("Collect", 8, 4, 50, 4, 504, {"episodeLengthSec": -1.5}, False),
    ("Sokoban", 1, 8, 100, 2, 505, {"episodeLengthSec": 4.0}, False),
    ("Rearrange", 1, 8, 80, 3, 506, {"episodeLengthSec": 5.0}, False),
    ("HexExplore", 4, 6, 80, 2, 507, {"episodeLengthSec": 3.0}, False),
    ("HexMemory", 1, 8, 60, 4, 508, {"episodeLengthSec": -5.0}, False),
    ("Empty", 4, 2, 40, 3, 509, {"episodeLengthSec": 1.0}, False),
    ("Collect", 4, 4, 50, 4, 510, {"episodeLengthSec": -1.5}, True),
]
CARRY = ("tower", "rearrange", "obstacles")
SOLVES = ("obstacles", "collect", "hexexplore")  # families whose warps solve levels within these windows
OFFSETS = {}  # k -> ends by tick offset, summed over the oracle cases run so far
CASES_RUN = []


@pytest.mark.parametrize("scenario,A,E,calls,k,seed,params,fast", ORACLE_CASES,
                         ids=["%s-A%d-k%d%s" % (c[0], c[1], c[4], "-fast" if c[7] else "") for c in ORACLE_CASES])
def test_repeat_matches_the_oracle(built, scenario, A, E, calls, k, seed, params, fast):
    """every call: rewards (float32 sums), dones, reasons and true objectives bit for bit; state, voxels, frames and depth at checkpoints and
    every done; terminal frames of every end.  Solved ends appear where the warps solve levels, and objects are carried with Interact held
    over consecutive calls"""
    run = RepeatRun(scenario, E, A, seed, params, k, fast_shading=fast)
    try:
        run.checkpoint("%s reset" % scenario)
        ev.drive(run, calls, np.random.default_rng(seed))
        print("%s k=%d offsets=%s reasons=%s carry_events=%d" % (run.table(), k, run.offsets, run.reasons, run.carry_events))
        assert run.dones > 0, "the window is meant to hold episode ends"
        if run.fam in SOLVES:
            assert run.reasons[2] > 0, "no solved end in the window\n" + run.table()
        if run.fam in CARRY:
            assert run.carry_events > 0, "no object was picked up or put down"
        OFFSETS[k] = [a + b for a, b in zip(OFFSETS.get(k, [0] * k), run.offsets)]
        CASES_RUN.append((scenario, A, k, fast))
    finally:
        run.close()


def test_ends_land_on_every_tick_offset(built):
    """over the oracle cases of each k, episode ends fell on every tick 0 .. k-1 of a call"""
    if len(CASES_RUN) < len(ORACLE_CASES):
        pytest.skip("needs every case of test_repeat_matches_the_oracle in the same session")
    print("ends by tick offset:", OFFSETS)
    for k, counts in OFFSETS.items():
        assert all(counts), "k=%d: ends by tick offset %s" % (k, counts)


# ------------------------------------------------------------------------------------------------ 2. k = 1 changes nothing
MEGAVERSE8 = fin.MEGAVERSE8
NO_CHANGE = [
    # case, scenario, E, A, path, depth
    ("config2-host", "TowerBuilding", 256, 1, "host", False),
    ("config2-device", "TowerBuilding", 256, 1, "device", False),
    ("config4-host", "Collect", 1024, 4, "host", False),
    ("config4-device", "Collect", 1024, 4, "device", False),
    ("megaverse8-host-depth", [MEGAVERSE8[i % 8] for i in range(64)], 64, 1, "host", True),
    ("megaverse8-device-depth", [MEGAVERSE8[i % 8] for i in range(64)], 64, 1, "device", True),
]


@pytest.mark.parametrize("case,scenario,E,A,path,depth", NO_CHANGE, ids=[c[0] for c in NO_CHANGE])
def test_repeat_one_changes_nothing(built, case, scenario, E, A, path, depth):
    """action_repeat 1 set explicitly: obs, depth, rewards, dones, reasons and true objectives byte-identical to an engine that never saw the
    option, over 60 steps with natural (and on the device path requested) ends"""
    import torch

    steps = 60
    # host: short natural episodes (lengths from the level, some shorter than three steps); device: requested ends every ten steps
    params = {"episodeLengthSec": {"config2-host": -180.0, "config4-host": -45.0}.get(case, 1.0)}
    on = fin._engine(scenario, E, A, 9, params, depth=depth, final=False, action_repeat=1)
    off = fin._engine(scenario, E, A, 9, params, depth=depth, final=False)
    rng = np.random.default_rng(6)
    acts = np.stack([helpers.purposeful_actions(rng, E * A, t) for t in range(steps)]).astype(np.int32)
    dacts = torch.from_numpy(acts).cuda()
    bank = torch.stack([fin._ends(E, [e for e in range(E) if (e + t) % 10 == 0]) for t in range(10)])
    torch.cuda.synchronize()
    dones = 0
    for t in range(steps):
        for g in (on, off):
            if path == "host":
                g.step(acts[t])
            else:
                g.step_device(dacts[t].data_ptr(), bank[t % 10].data_ptr())
                g.sync()
        keys = ["rewards", "dones", "done_reasons", "true_objectives"]
        if path == "host" or t % 10 == 9:
            if path == "device":
                for g in (on, off):
                    g.fetch_obs()
            keys += ["obs"] + (["depth"] if depth else [])
        for key in keys:
            a, b = np.array(getattr(on, key)()), np.array(getattr(off, key)())
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), "%s step %d: %s differs" % (case, t, key)
        dones += int(np.array(on.dones()).sum())
    assert dones > 0, "the window is meant to hold episode ends"
    for g in (on, off):
        fin._healthy(g)
        g.close()


# ------------------------------------------------------------------------------------------------ 3. engine against engine at scale
def test_repeat_four_equals_four_single_ticks(built):
    """Collect 256 x 4, long episodes, fast shading: every k = 4 call equals a k = 1 twin stepped four times with Interact cleared after the
    first -- rewards the float32 sums of the twin's four, obs byte for byte, the states at the end.  An env whose episode ends (a level with
    few good rewards can be solved) ends on the same tick in both and is left out from then on: the twin goes on ticking its next episode"""
    E, A, calls = 256, 4, 25
    params = {"episodeLengthSec": 600.0}
    g4 = fin._engine("Collect", E, A, 17, params, final=False, action_repeat=4)
    g1 = fin._engine("Collect", E, A, 17, params, final=False)
    rng = np.random.default_rng(17)
    live = np.ones(E, dtype=bool)  # envs without an end so far
    for c in range(calls):
        acts = helpers.purposeful_actions(rng, E * A, c)
        g4.step(acts)
        total = np.zeros(E * A, dtype=np.float32)
        ended = np.zeros(E, dtype=bool)
        m = acts.copy()
        for t in range(4):
            g1.step(m)
            total += np.array(g1.rewards())
            ended |= np.array(g1.dones()) != 0
            m = m & ~np.int32(INTERACT)
        assert np.array_equal((np.array(g4.dones()) != 0)[live], ended[live]), "call %d: dones" % c
        same = np.repeat(live & ~ended, A)
        assert np.array_equal(total[same].view(np.uint32), np.array(g4.rewards())[same].view(np.uint32)), "call %d: rewards" % c
        assert np.array_equal(np.array(g4.obs())[same], np.array(g1.obs())[same]), "call %d: obs" % c
        live &= ~ended
    assert live.sum() >= E * 9 // 10
    reward_words = 8 + AG * np.arange(A) + 24  # the dump's reward of the last call: the sum at k = 4, the last tick's in the twin
    for e in np.flatnonzero(live):
        s4, s1 = g4.state(e), g1.state(e)
        s4[reward_words] = s1[reward_words] = 0
        assert np.array_equal(s4.view(np.uint32), s1.view(np.uint32)), "env %d: state" % e
    for g in (g4, g1):
        fin._healthy(g)
        g.close()


# ------------------------------------------------------------------------------------------------ 4. requested ends
def test_requests_before_three_calls_are_no_ops(built):
    """k = 3, Empty with long episodes: a request ends the episode after the call's last tick once it has run 3k ticks (three calls), with
    reason 3 and reward 0; earlier requests change nothing"""
    import torch

    E, A, k, calls = 12, 2, 3, 60
    g = fin._engine("Empty", E, A, 4, {"episodeLengthSec": 60.0}, final=False, action_repeat=k)
    acts = np.stack([helpers.purposeful_actions(np.random.default_rng(t), E * A, t) for t in range(calls)]).astype(np.int32)
    dacts = torch.from_numpy(acts).cuda()
    rng = np.random.default_rng(2)
    ran = np.zeros(E, dtype=np.int64)  # calls of the current episode, this one included
    honoured_total = ignored_total = 0
    for t in range(calls):
        req = [e for e in range(E) if rng.random() < 0.3]
        masks = fin._ends(E, req)
        torch.cuda.synchronize()
        g.step_device(dacts[t].data_ptr(), masks.data_ptr())
        g.sync()
        ran += 1
        honoured = [e for e in req if ran[e] >= 3]
        dn, why, r = np.array(g.dones()), np.array(g.done_reasons()), np.array(g.rewards()).reshape(E, A)
        assert list(np.flatnonzero(dn)) == honoured, "call %d: dones %s, honoured %s" % (t, np.flatnonzero(dn), honoured)
        assert (why[honoured] == 3).all() and (why[dn == 0] == 0).all() and not r[honoured].any(), "call %d" % t
        for e in honoured:
            assert g.state(e)[2] == 0  # the new episode's tick counter
            ran[e] = 0
        honoured_total += len(honoured)
        ignored_total += len(req) - len(honoured)
    assert honoured_total > 5 and ignored_total > 5
    fin._healthy(g)
    g.close()


def test_request_in_a_call_that_already_ended_is_ignored(built):
    """k = 4, Empty episodes of 1.2 s: a request sent in exactly the calls where the episode ends by its clock changes nothing -- the end
    stands with reason 1, and the run equals a twin that never sends requests"""
    import torch

    E, A, k, calls = 8, 2, 4, 40
    params = {"episodeLengthSec": 1.2}
    g = fin._engine("Empty", E, A, 5, params, final=False, action_repeat=k)
    twin = fin._engine("Empty", E, A, 5, params, final=False, action_repeat=k)
    acts = np.stack([helpers.purposeful_actions(np.random.default_rng(100 + t), E * A, t) for t in range(calls)]).astype(np.int32)
    dacts = torch.from_numpy(acts).cuda()
    ignored = 0
    for t in range(calls):
        twin.step(acts[t])
        tdn = np.array(twin.dones()).copy()
        masks = fin._ends(E, list(np.flatnonzero(tdn)))
        torch.cuda.synchronize()
        g.step_device(dacts[t].data_ptr(), masks.data_ptr())
        g.sync()
        g.fetch_obs()
        for key in ("dones", "done_reasons", "rewards", "true_objectives", "obs"):
            a, b = np.array(getattr(g, key)()), np.array(getattr(twin, key)())
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), "call %d: %s" % (t, key)
        assert (np.array(g.done_reasons())[tdn != 0] == 1).all()
        ignored += int(tdn.sum())
    assert ignored >= E
    for x in (g, twin):
        fin._healthy(x)
        x.close()


# ------------------------------------------------------------------------------------------------ 5. loops and state
def test_asynchronous_loop_with_ends_requests_and_restarts(built):
    """300 mv_step_device_ends calls at k = 4 with natural ends (Empty, 2 s = 30 ticks: the eighth call), requests every 3 to 12 calls per env
    and mv_reset_envs between them, never synchronised in between: no fault bit, no MV_ERR_STATE, and both kinds of end happen"""
    import torch

    E, A, k, calls = 16, 2, 4, 300
    g = fin._engine("Empty", E, A, 31, {"episodeLengthSec": 2.0}, final=True, action_repeat=k)
    acts = torch.from_numpy(np.stack([helpers.purposeful_actions(np.random.default_rng(t), E * A, t) for t in range(20)]).astype(np.int32)).cuda()
    rng = np.random.default_rng(31)
    period = rng.integers(3, 13, size=E)
    bank = [fin._ends(E, [e for e in range(E) if t % period[e] == period[e] - 1]) for t in range(calls)]
    torch.cuda.synchronize()
    reasons = {0: 0, 1: 0, 3: 0}
    for t in range(calls):
        g.step_device(acts[t % 20].data_ptr(), bank[t].data_ptr())
        if t % 50 == 49:
            g.reset_envs([t % E, (t + 5) % E], [t, t + 1] if t % 100 == 49 else None)
        why = np.array(g.done_reasons())  # the host buffers hold the call the pipeline retired last
        for r in reasons:
            reasons[r] += int((why == r).sum())
    g.sync()
    assert reasons[1] > 0 and reasons[3] > 0, reasons
    fin._healthy(g)
    g.close()


def test_state_save_and_load_replays_at_k3(built):
    """k = 3: envs saved mid-episode and loaded back replay the same calls bit for bit (rewards, dones, reasons, obs, state)"""
    E, A = 8, 2
    g = fin._engine("Collect", E, A, 23, {"episodeLengthSec": -45.0}, depth=True, final=False, action_repeat=3)
    rng = np.random.default_rng(23)
    acts = np.stack([helpers.purposeful_actions(rng, E * A, t) for t in range(50)]).astype(np.int32)
    for t in range(20):
        g.step(acts[t])
    store = g.states_create(E)
    g.states_save(store, range(E), range(E))
    first = []
    for t in range(20, 50):
        g.step(acts[t])
        first.append([np.array(getattr(g, key)()).copy() for key in ("rewards", "dones", "done_reasons", "true_objectives", "obs", "depth")])
    states = [g.state(e).copy() for e in range(E)]
    assert sum(int(f[1].sum()) for f in first) > 0, "the replayed window is meant to hold ends"
    g.states_load(store, range(E), range(E))
    for t in range(20, 50):
        g.step(acts[t])
        again = [np.array(getattr(g, key)()) for key in ("rewards", "dones", "done_reasons", "true_objectives", "obs", "depth")]
        for a, b in zip(first[t - 20], again):
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), "call %d replays differently" % t
    for e in range(E):
        assert np.array_equal(states[e].view(np.uint32), g.state(e).view(np.uint32))
    fin._healthy(g)
    g.close()


def test_option_range_and_order(built):
    from megaverse_b200 import capi

    g = capi.Engine("Collect", 2, 2, num_threads=2)
    for bad in (0, -1, 5, 100):
        with pytest.raises(capi.MegaverseError) as ei:
            g.set_option("action_repeat", bad)
        assert ei.value.code == capi.MV_ERR_ARG
    for good in (1, 4, 2):
        g.set_option("action_repeat", good)
    g.seed(1)
    g.reset()
    with pytest.raises(capi.MegaverseError) as ei:
        g.set_option("action_repeat", 2)
    assert ei.value.code == capi.MV_ERR_STATE
    g.close()


def test_megaverse_env_returns_summed_rewards(built):
    """MegaverseEnv(action_repeat=3): each step's rewards are the float32 sums of three single ticks of a k = 1 env (Interact on the first),
    observations equal"""
    from megaverse_b200 import MegaverseEnv

    E, A = 4, 2
    rep = MegaverseEnv("Collect", E, A, 2, action_repeat=3)
    one = MegaverseEnv("Collect", E, A, 2)
    for env in (rep, one):
        env.seed(29)
        env.reset()
    rng = np.random.default_rng(29)
    paid = 0
    for _ in range(40):
        a = rng.integers(0, [3, 3, 3, 2, 2, 3], size=(E * A, 6))
        o3, r3, d3, _ = rep.step(a)
        total = np.zeros(E * A, dtype=np.float32)
        b = a.copy()
        for t in range(3):
            o1, r1, d1, _ = one.step(b)
            assert not any(d1)
            total += np.float32(r1)
            b[:, 4] = 0  # the Interact head
        assert not any(d3)
        assert np.array_equal(np.float32(r3).view(np.uint32), total.view(np.uint32))
        assert all(np.array_equal(x, y) for x, y in zip(o3, o1))
        paid += int((total != 0).sum())
    assert paid > 0, "the window is meant to pay rewards"
    rep.close(); one.close()
