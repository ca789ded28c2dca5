"""Autoreset modes (option "autoreset") on the GPU.

Next-step (1) is checked against a same-step twin with final_obs (0), whose terminal path the suite already checks against the oracle.
The twin A is driven with an active mask that leaves out the envs B was awaiting on before the call, so A skips exactly B's reset calls.
After every call: for an env that ended, B's frame, state rows, rays and level id equal A's terminal frame, terminal rows, terminal rays and
the level A was on before the call; everything else B reports equals A's own output.  Disabled (2) is checked against a next-step engine
whose active mask leaves out its own awaiting envs, one-episode evaluation against a same-step engine's first episodes, then the state
store, level replacement, the refusals and MegaverseEnv."""
import ctypes as C

import numpy as np
import pytest

import helpers

pytestmark = pytest.mark.gpu

MEGAVERSE8 = ["TowerBuilding", "ObstaclesEasy", "ObstaclesHard", "Collect", "Sokoban", "HexMemory", "HexExplore", "Rearrange"]
# episodes of a few calls: the episode length is a base plus a per-level term in some scenarios (4 s per block in TowerBuilding, 2 s per
# reward in Collect, 3 s per good object in HexMemory), which the negative bases take back; Obstacles chains without platforms are short
NO_PLATFORMS = {"obstaclesMinNumPlatforms": 0.0, "obstaclesMaxNumPlatforms": 0.0}
SHORT = {"Collect": {"episodeLengthSec": -60.0}, "TowerBuilding": {"episodeLengthSec": -180.0}, "HexMemory": {"episodeLengthSec": -5.0},
         "ObstaclesHard": dict(NO_PLATFORMS, episodeLengthSec=1.0), "Sokoban": {"episodeLengthSec": 1.0}}
# a negative base ends the timed episodes after a step or two
SHORT_MIXED = dict(NO_PLATFORMS, episodeLengthSec=-200.0)
L = 16
HOST_CALLS = ["step", "step_envs", "begin_end"]
DEVICE_CALLS = ["device_ends", "device_active"]
STREAM_CALLS = ["stream"]


def _engine(scenario, A, repeat, mode, slots=2, level_set=0, E=8, final=None):
    from megaverse_b200 import capi
    from megaverse_b200 import rays

    mixed = scenario == "mixed"
    names = [MEGAVERSE8[e % 8] for e in range(E)] if mixed else scenario
    g = capi.Engine(names, E, A, 128, 72, num_threads=4, params=SHORT_MIXED if mixed else SHORT[scenario], segmentation=True)
    g.set_option("fast_shading", 0)
    g.set_option("zero_copy", 0)
    opts = [("state_tensors", 1), ("reward_components", 1), ("action_repeat", repeat), ("level_slots", slots)]
    opts += [("final_obs", 1)] if (mode == 0 if final is None else final) else []
    opts += [("autoreset", mode)] if mode else []
    for k, v in opts:
        g.set_option(k, v)
    if level_set:
        g.set_option("level_set_seed", 5)
        g.set_option("level_set", level_set)
    g.set_rays(rays.fan(6, 90.0, -10.0), 20.0)
    for e in range(E):
        g.seed_env(e, 300 + 7 * e)
    return g


def _snap(g, level_set, terminal=False):
    """copies of everything g reports after its last call (host arrays: call fetch_obs first after a device call)"""
    s = {"obs": np.array(g.obs()), "seg": np.array(g.segmentation()), "rewards": np.array(g.rewards()), "dones": np.array(g.dones()),
         "reasons": np.array(g.done_reasons()), "to": np.array(g.true_objectives())}
    s.update({"st_" + k: np.array(v) for k, v in g.state_tensors().items()})
    s["rd"], s["rt"] = (np.array(x) for x in g.rays())
    s["rc_step"], s["rc_ep"] = (np.array(x) for x in g.reward_components())
    s["levels"] = np.array(g.level_ids()) if level_set else None
    if terminal:
        s["f_obs"] = np.array(g.final_obs())
        s.update({"f_st_" + k: np.array(v) for k, v in g.final_state_tensors().items()})
        s["f_rd"], s["f_rt"] = (np.array(x) for x in g.final_rays())
    return s


SCENE = ["obs", "st_agents", "st_envs", "st_objects", "st_rewards", "rd", "rt"]  # what describes the scene: the terminal one after an end
PER_AGENT = {"obs", "seg", "rewards", "to", "st_agents", "rd", "rt", "rc_step", "rc_ep"}


def _rows(key, e, A):
    return slice(e * A, (e + 1) * A) if key in PER_AGENT else slice(e, e + 1)


def _eq(a, b, tag):
    assert a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8)), tag


def _check(sa, sb, prev_b, b_await_before, b_await, a_levels_before, A, tag):
    """B (next-step or disabled) after a call against A (same-step + final_obs) after its masked twin call; prev_b: B before the call"""
    E = len(sb["dones"])
    for k in ("rewards", "dones", "reasons", "to", "rc_step", "rc_ep"):
        _eq(sb[k], sa[k], "%s: %s" % (tag, k))
    for e in range(E):
        if sb["dones"][e]:  # ended in this call: B shows the terminal scene, and the finished episode's level
            assert b_await[e], "%s: env %d ended without awaiting" % (tag, e)
            for k in SCENE:
                _eq(sb[k][_rows(k, e, A)], sa["f_" + k][_rows(k, e, A)], "%s: env %d ended, %s is not the terminal one" % (tag, e, k))
            if sb["levels"] is not None:
                assert sb["levels"][e] == a_levels_before[e], "%s: env %d ended, level id" % (tag, e)
        elif b_await_before[e] and b_await[e]:  # still awaiting: nothing changed
            for k in SCENE + ["seg"] + (["levels"] if sb["levels"] is not None else []):
                _eq(sb[k][_rows(k, e, A)], prev_b[k][_rows(k, e, A)], "%s: awaiting env %d, %s changed" % (tag, e, k))
        else:  # stepped, restarted or inactive: as A
            for k in SCENE + ["seg"] + (["levels"] if sb["levels"] is not None else []):
                _eq(sb[k][_rows(k, e, A)], sa[k][_rows(k, e, A)], "%s: env %d, %s" % (tag, e, k))
        if b_await_before[e]:  # restarted or still awaiting: nothing paid, nothing ended
            assert not sb["rewards"][_rows("rewards", e, A)].any() and not sb["dones"][e], "%s: awaiting env %d" % (tag, e)


class Twin:
    def __init__(self, scenario, A, repeat, slots=2, level_set=0, E=8):
        self.a = _engine(scenario, A, repeat, 0, slots, level_set, E)
        self.b = _engine(scenario, A, repeat, 1, slots, level_set, E)
        self.A, self.E, self.N, self.ls = A, E, E * A, level_set
        self.a.reset()
        self.b.reset()
        self.prev_b = _snap(self.b, level_set)
        self.await_b = np.zeros(E, dtype=np.uint8)
        self.ends = 0
        self.restarts = 0

    def close(self):
        self.a.close()
        self.b.close()

    def call(self, kind, masks, ends, active, tag):
        """one call of `kind` on B, the masked equivalent on A, then the check"""
        import torch

        a, b = self.a, self.b
        before = self.await_b.copy()
        a_levels = np.array(a.level_ids()) if self.ls else None
        act_b = active if kind in ("step_envs", "device_active", "stream") else np.ones(self.E, dtype=np.uint8)
        act_a = (act_b & (before == 0)).astype(np.uint8)
        if kind in HOST_CALLS:
            if kind == "step":
                b.step(masks)
            elif kind == "step_envs":
                b.step_envs(masks, np.flatnonzero(act_b).astype(np.int32))
            else:
                b.step_begin(masks)
                b.step_end()
            a.step_envs(masks, np.flatnonzero(act_a).astype(np.int32))
        else:
            dm = torch.from_numpy(np.ascontiguousarray(masks, dtype=np.int32)).cuda()
            de = torch.from_numpy(ends).cuda()
            dab, daa = torch.from_numpy(act_b).cuda(), torch.from_numpy(act_a).cuda()
            torch.cuda.synchronize()
            if kind == "device_ends":
                b.step_device(dm.data_ptr(), de.data_ptr())
            elif kind == "device_active":
                b.step_device_active(dm.data_ptr(), de.data_ptr(), dab.data_ptr())
            else:
                b.step_stream(torch.cuda.current_stream().cuda_stream, dm.data_ptr(), de.data_ptr(), dab.data_ptr())
            a.step_device_active(dm.data_ptr(), de.data_ptr(), daa.data_ptr())
            torch.cuda.synchronize()
            a.fetch_obs()
            b.fetch_obs()
        sa, sb = _snap(a, self.ls, terminal=True), _snap(b, self.ls)
        aw = np.array(b.awaiting_reset())
        _check(sa, sb, self.prev_b, before, aw, a_levels, self.A, tag)
        self.ends += int(sb["dones"].sum())
        self.restarts += int((before & (aw == 0) & (act_b != 0)).sum())
        self.await_b, self.prev_b = aw, sb

    def healthy(self):
        for g in (self.a, self.b):
            assert g.fault_word() == 0 and g.faults() == 0


def _inputs(E, N, steps, seed):
    rng = np.random.default_rng(seed)
    acts = [helpers.purposeful_actions(rng, N, t).astype(np.int32) for t in range(steps)]
    ends = [(rng.random(E) < 0.08).astype(np.uint8) for _ in range(steps)]
    active = [(rng.random(E) < (0.75 if t % 3 == 2 else 1.0)).astype(np.uint8) for t in range(steps)]
    return acts, ends, active


# (scenario, A, action_repeat, level_slots, level_set, E, calls)
CASES = [
    ("Collect", 2, 1, 2, 0, 8, HOST_CALLS),
    ("ObstaclesHard", 1, 3, 2, 0, 8, HOST_CALLS),
    ("TowerBuilding", 4, 1, 4, 0, 6, HOST_CALLS + DEVICE_CALLS),
    ("HexMemory", 1, 3, 4, 0, 8, DEVICE_CALLS),
    ("Collect", 2, 3, 2, L, 8, HOST_CALLS + DEVICE_CALLS + STREAM_CALLS),
    ("Sokoban", 4, 1, 2, L, 6, DEVICE_CALLS + STREAM_CALLS),
    ("mixed", 2, 1, 2, L, 16, HOST_CALLS + DEVICE_CALLS + STREAM_CALLS),
    ("mixed", 1, 3, 4, 0, 16, HOST_CALLS + DEVICE_CALLS),
]
IDS = ["collect-a2-d2", "obstacleshard-r3-d2", "tower-a4-d4", "hexmemory-r3-d4", "collect-r3-set", "sokoban-a4-set", "megaverse8-set",
       "megaverse8-r3-d4"]


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_next_step_against_same_step_twin(built, case):
    scenario, A, repeat, slots, level_set, E, calls = case
    t = Twin(scenario, A, repeat, slots, level_set, E)
    try:
        steps = 72
        acts, ends, active = _inputs(E, E * A, steps, 17)
        for i in range(steps):
            kind = calls[i % len(calls)]
            t.call(kind, acts[i], ends[i], active[i], "%s call %d (%s)" % (scenario, i, kind))
        assert t.ends >= 8 and t.restarts >= 4, (t.ends, t.restarts)
        t.healthy()
    finally:
        t.close()


def test_next_step_graph_against_same_step_twin(built):
    """a graph of K next-step stream steps with active masks, replayed on refilled inputs, against the same-step twin driven call by call"""
    import torch

    A, E, K = 2, 8, 8
    t = Twin("Collect", A, 1, 2, L, E)
    try:
        b = t.b
        dv = {k: torch.as_tensor(b.device_array(k), device="cuda") for k in ("rewards", "dones", "awaiting_reset")}
        masks = torch.zeros((K, t.N), dtype=torch.int32, device="cuda")
        ends = torch.zeros((K, E), dtype=torch.uint8, device="cuda")
        active = torch.ones((K, E), dtype=torch.uint8, device="cuda")
        static = {k: torch.zeros((K,) + tuple(v.shape), dtype=v.dtype, device="cuda") for k, v in dv.items()}
        acts, ends_in, act_in = _inputs(E, t.N, 1 + K * 6, 29)
        t.call("stream", acts[0], ends_in[0], act_in[0], "eager stream step")  # warms up, starts stream mode
        for k, v in dv.items():
            static[k][0].copy_(v)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            s = torch.cuda.current_stream().cuda_stream
            for k in range(K):
                b.step_stream(s, masks[k].data_ptr(), ends[k].data_ptr(), active[k].data_ptr())
                for key, v in dv.items():
                    static[key][k].copy_(v)
        for r in range(6):
            base = 1 + K * r
            masks.copy_(torch.from_numpy(np.stack(acts[base:base + K])))
            ends.copy_(torch.from_numpy(np.stack(ends_in[base:base + K])))
            active.copy_(torch.from_numpy(np.stack(act_in[base:base + K])))
            graph.replay()
            torch.cuda.synchronize()
            got = {k: v.cpu().numpy() for k, v in static.items()}
            for k in range(K):  # the twin, call by call, against what each captured step left
                before = t.await_b.copy()
                act_a = (act_in[base + k] & (before == 0)).astype(np.uint8)
                dm = torch.from_numpy(acts[base + k]).cuda()
                de, da = torch.from_numpy(ends_in[base + k]).cuda(), torch.from_numpy(act_a).cuda()
                torch.cuda.synchronize()
                t.a.step_device_active(dm.data_ptr(), de.data_ptr(), da.data_ptr())
                t.a.sync()
                tag = "replay %d step %d" % (r, k)
                _eq(got["rewards"][k], np.array(t.a.rewards()), tag + ": rewards")
                _eq(got["dones"][k], np.array(t.a.dones()), tag + ": dones")
                assert np.array_equal(got["awaiting_reset"][k], (before & ~act_in[base + k].astype(bool)) | got["dones"][k]), tag
                t.ends += int(got["dones"][k].sum())
                t.await_b = got["awaiting_reset"][k].astype(np.uint8)
                if k < K - 1:
                    continue
                t.a.fetch_obs()
                b.fetch_obs()
                sa, sb = _snap(t.a, L, terminal=True), _snap(b, L)
                aw = np.array(b.awaiting_reset())
                assert np.array_equal(aw, t.await_b), tag
                for e in range(E):  # envs that ended in this last step: terminal scene; others as A (those awaiting longer: as before)
                    if sb["dones"][e]:
                        for key in SCENE:
                            _eq(sb[key][_rows(key, e, A)], sa["f_" + key][_rows(key, e, A)], "%s: env %d %s" % (tag, e, key))
                    elif not aw[e]:
                        for key in SCENE + ["seg", "levels"]:
                            _eq(sb[key][_rows(key, e, A)], sa[key][_rows(key, e, A)], "%s: env %d %s" % (tag, e, key))
                for key in ("rewards", "dones", "reasons", "to", "rc_step", "rc_ep"):
                    _eq(sb[key], sa[key], "%s: %s" % (tag, key))
        assert t.ends >= 8
        t.healthy()
    finally:
        t.close()


def test_disabled_against_next_step(built):
    """a disabled engine C against a next-step engine B that never steps its own awaiting envs: byte-equal throughout, with C's awaiting
    envs restarted (by both) now and then"""
    A, E = 2, 8
    b = _engine("Collect", A, 1, 1, 2, L, E)
    c = _engine("Collect", A, 1, 2, 2, L, E)
    try:
        b.reset()
        c.reset()
        acts, _, active = _inputs(E, E * A, 90, 41)
        held, longest = np.zeros(E, dtype=np.int64), 0
        restarted = 0
        for i in range(90):
            aw = np.array(c.awaiting_reset())
            _eq(aw, np.array(b.awaiting_reset()), "call %d: awaiting" % i)
            held = np.where(aw != 0, held + 1, 0)
            longest = max(longest, int(held.max()))
            if i % 15 == 14 and aw.any():  # restart the envs awaiting longest, with and without seeds
                envs = np.flatnonzero(aw).astype(np.int32)[:3]
                seeds = None if i % 30 == 14 else [500 + int(e) for e in envs]
                b.reset_envs(envs, seeds)
                c.reset_envs(envs, seeds)
                restarted += len(envs)
            else:
                on = active[i] & (aw == 0)
                c.step_envs(acts[i], np.flatnonzero(active[i]).astype(np.int32))
                b.step_envs(acts[i], np.flatnonzero(on).astype(np.int32))
            sb, sc = _snap(b, L), _snap(c, L)
            for k in sb:
                _eq(sc[k], sb[k], "call %d: %s" % (i, k))
            aw_after = np.array(c.awaiting_reset())
            for e in np.flatnonzero(aw & aw_after):
                assert not sc["dones"][e] and not sc["rewards"][_rows("rewards", e, A)].any(), "call %d: awaiting env %d" % (i, e)
        assert restarted >= 3 and longest >= 5
        for g in (b, c):
            assert g.fault_word() == 0 and g.faults() == 0
    finally:
        b.close()
        c.close()


def test_one_episode_evaluation(built):
    """a level set with L = E, every env assigned its own level again after each pick; run until every env awaits: each level's return,
    reason and true objective equal the first episode of a same-step engine started on that level"""
    A, E = 2, 8
    for scenario in ("ObstaclesHard", "Sokoban"):
        c = _engine(scenario, A, 1, 2, 2, E, E)
        s = _engine(scenario, A, 1, 0, 2, E, E, final=False)
        try:
            for g in (c, s):
                g.set_next_levels(range(E), range(E))
                g.reset()
            assert list(c.level_ids()) == list(range(E)) and list(s.level_ids()) == list(range(E))
            rng = np.random.default_rng(3)
            ret_c, ret_s = np.zeros(E * A), np.zeros(E * A)
            done_s = np.zeros(E, dtype=bool)
            res_c, res_s = {}, {}
            for t in range(400):
                acts = helpers.purposeful_actions(rng, E * A, t)
                c.step(acts)
                s.step_envs(acts, np.flatnonzero(~done_s).astype(np.int32))
                for g, ret, res, live in ((c, ret_c, res_c, None), (s, ret_s, res_s, done_s)):
                    ret += np.array(g.rewards())
                    for e in np.flatnonzero(np.array(g.dones())):
                        res[int(e)] = (ret[e * A:(e + 1) * A].copy(), int(g.done_reasons()[e]), np.array(g.true_objectives()[e * A:(e + 1) * A]))
                        if live is not None:
                            live[e] = True
                if np.array(c.awaiting_reset()).all() and done_s.all():
                    break
            assert np.array(c.awaiting_reset()).all() and len(res_c) == E and len(res_s) == E
            assert list(c.level_ids()) == list(range(E))
            for e in range(E):
                _eq(res_c[e][0].astype(np.float32), res_s[e][0].astype(np.float32), "%s level %d: return" % (scenario, e))
                assert res_c[e][1] == res_s[e][1], "%s level %d: reason" % (scenario, e)
                _eq(res_c[e][2], res_s[e][2], "%s level %d: true objective" % (scenario, e))
            for _ in range(3):  # and they stay put
                c.step(helpers.purposeful_actions(rng, E * A, 0))
                assert not np.array(c.dones()).any() and not np.array(c.rewards()).any()
            for g in (c, s):
                assert g.fault_word() == 0 and g.faults() == 0
        finally:
            c.close()
            s.close()


@pytest.mark.parametrize("level_set", [0, L], ids=["streams", "level-set"])
def test_state_store(built, level_set):
    """an awaiting env saved, loaded into itself and into another env: under next-step both restart on their next call, equal to the
    un-rewound run"""
    A, E = 1, 4
    g = _engine("Collect", A, 1, 1, 4, level_set, E)
    try:
        g.reset()
        rng = np.random.default_rng(5)
        zeros = np.zeros(E * A, dtype=np.int32)
        for t in range(150):
            g.step_envs(helpers.purposeful_actions(rng, E * A, t), [0, 1, 2, 3] if not np.array(g.awaiting_reset())[0] else [1, 2, 3])
            if np.array(g.awaiting_reset())[0]:
                break
        assert np.array(g.awaiting_reset())[0]
        store = g.states_create(1)
        g.states_save(store, [0], [0])
        saved = _snap(g, level_set)
        g.step(zeros)  # the un-rewound run: env 0 restarts
        assert not np.array(g.awaiting_reset())[0] and not g.dones()[0] and g.rewards()[0] == 0
        want = _snap(g, level_set)
        g.states_load(store, [0, 0], [0, 3])  # back into itself, and a clone into env 3
        aw = np.array(g.awaiting_reset())
        assert aw[0] and aw[3]
        now = _snap(g, level_set)
        for k in SCENE:
            for e in (0, 3):
                _eq(now[k][_rows(k, e, A)], saved[k][_rows(k, 0, A)], "loaded env %d: %s" % (e, k))
        g.step_envs(zeros, [0, 3])
        after = _snap(g, level_set)
        assert not np.array(g.awaiting_reset())[[0, 3]].any()
        for k in SCENE + ["rewards", "dones", "reasons", "to", "rc_step"]:
            _eq(after[k][_rows(k, 0, A)], want[k][_rows(k, 0, A)], "rewound env 0: %s" % k)
        if level_set:
            assert after["levels"][0] == want["levels"][0] and after["levels"][3] == want["levels"][0]
        assert g.fault_word() == 0 and g.faults() == 0
    finally:
        g.close()


def test_level_replacement_waits_for_a_restart(built):
    """a level-set row under a disabled awaiting env is not rewritten until the env is restarted (one env: no other can hold the row)"""
    g = _engine("ObstaclesHard", 1, 1, 2, 2, L, 1)
    try:
        g.reset()
        rng = np.random.default_rng(8)
        for t in range(60):
            g.step(helpers.purposeful_actions(rng, 1, t))
            if g.awaiting_reset()[0]:
                break
        assert g.awaiting_reset()[0]
        row = int(g.level_ids()[0])
        g.replace_levels([row], [977])
        for t in range(8):
            g.step(helpers.purposeful_actions(rng, 1, t))
            seeds, retiring = (np.array(x) for x in g.level_rows())
            assert retiring[row] and seeds[row] != 977, "the row was rewritten under an awaiting env"
            assert int(g.level_ids()[0]) == row and g.awaiting_reset()[0]
        g.reset_envs([0])  # the restart releases the row; the hash probes past it
        assert int(g.level_ids()[0]) != row
        for t in range(4):
            g.step(np.zeros(1, dtype=np.int32))
        seeds, retiring = (np.array(x) for x in g.level_rows())
        assert not retiring[row] and seeds[row] == 977
        assert g.fault_word() == 0 and g.faults() == 0
    finally:
        g.close()


def test_refusals(built):
    from megaverse_b200 import capi

    Lb = capi.lib()
    p = C.c_void_p()
    g = _engine("Collect", 1, 1, 0, 2, 0, 4)
    try:
        # mode 0: no getter, and final_obs is on
        assert Lb.mv_awaiting_reset_host(g._h, C.byref(p)) == capi.MV_ERR_ARG
        assert Lb.mv_awaiting_reset_device(g._h, C.byref(p)) == capi.MV_ERR_ARG
        for v in (1, 2):
            assert Lb.mv_set_option(g._h, b"autoreset", v) == capi.MV_ERR_ARG
        for v in (-1, 3, 99):
            assert Lb.mv_set_option(g._h, b"autoreset", v) == capi.MV_ERR_ARG
        g.reset()
        assert Lb.mv_set_option(g._h, b"autoreset", 0) == capi.MV_ERR_STATE
        assert Lb.mv_set_option(g._h, b"autoreset", 1) == capi.MV_ERR_STATE
        assert Lb.mv_awaiting_reset_host(g._h, C.byref(p)) == capi.MV_ERR_ARG
        g.step(np.zeros(g.N, dtype=np.int32))
        assert g.faults() == 0
    finally:
        g.close()
    g = _engine("ObstaclesHard", 1, 1, 1, 2, 0, 4)
    try:
        assert Lb.mv_set_option(g._h, b"final_obs", 1) == capi.MV_ERR_ARG
        assert Lb.mv_awaiting_reset_host(g._h, C.byref(p)) == capi.MV_ERR_STATE  # before mv_reset
        assert Lb.mv_awaiting_reset_device(g._h, C.byref(p)) == capi.MV_ERR_STATE
        assert Lb.mv_awaiting_reset_host(g._h, None) == capi.MV_ERR_ARG
        assert Lb.mv_set_option(g._h, b"autoreset", 4) == capi.MV_ERR_ARG
        g.reset()  # still next-step, final_obs still off
        assert Lb.mv_set_option(g._h, b"autoreset", 2) == capi.MV_ERR_STATE
        assert Lb.mv_set_option(g._h, b"final_obs", 1) == capi.MV_ERR_STATE
        assert Lb.mv_final_obs_host(g._h, C.byref(p)) == capi.MV_ERR_ARG
        rng = np.random.default_rng(1)
        saw = False
        for t in range(30):
            g.step(helpers.purposeful_actions(rng, g.N, t))
            d, aw = np.array(g.dones()), np.array(g.awaiting_reset())
            assert np.array_equal(d != 0, (aw != 0) & (d != 0))
            saw = saw or bool(d.any())
        assert saw
        assert Lb.mv_awaiting_reset_device(g._h, C.byref(p)) == capi.MV_OK and p.value
        assert g.fault_word() == 0 and g.faults() == 0
    finally:
        g.close()


def test_megaverse_env_modes(built):
    from megaverse_b200.megaverse_env import MegaverseEnv

    E, A = 4, 1
    env = MegaverseEnv("ObstaclesHard", E, A, 2, params=SHORT["ObstaclesHard"], autoreset_mode="next_step", num_levels=8)
    try:
        assert env.metadata["autoreset_mode"] == "next_step"
        env.seed(3)
        env.reset()
        rng = np.random.default_rng(0)
        seen = 0
        for t in range(60):
            acts = rng.integers(0, 2, size=(E * A, 6))
            levels_before = env.level_ids()
            obs, rew, dones, infos = env.step(acts)
            aw = env.awaiting_reset()
            for e in range(E):
                if dones[e]:
                    seen += 1
                    assert aw[e] and infos[e]["level"] == levels_before[e] == env.level_ids()[e]
                    assert infos[e]["terminated"] != infos[e]["truncated"] and "true_reward" in infos[e]
                    frame = obs[e].copy()
                    obs2, rew2, dones2, infos2 = env.step(acts)  # the restart: reward 0, not done, a new frame
                    assert rew2[e] == 0 and not dones2[e] and not env.awaiting_reset()[e]
                    assert not np.array_equal(obs2[e], frame)
                    break
            if seen >= 2:
                break
        assert seen >= 2
        env.check_faults()
    finally:
        env.close()
    env = MegaverseEnv("ObstaclesHard", E, A, 2, params=SHORT["ObstaclesHard"], autoreset_mode="disabled")
    try:
        env.seed(4)
        env.reset()
        for t in range(40):
            env.step(np.zeros((E * A, 6), dtype=np.int32))
        assert all(env.awaiting_reset())
        frame = env.observations()[0].copy()
        obs, rew, dones, infos = env.step(np.zeros((E * A, 6), dtype=np.int32))
        assert not any(dones) and not np.any(rew) and np.array_equal(obs[0], frame)
        obs = env.reset_envs([0])
        assert not env.awaiting_reset()[0] and all(env.awaiting_reset()[1:])
        env.check_faults()
    finally:
        env.close()
