"""Steps with an active set (mv_step_envs, mv_step_device_active): an inactive env runs nothing and keeps its frames, an active env is
stepped exactly as by the full call.  The reference for env e is env e of a twin engine with the same seeds and options that is stepped by
the full call only at the calls where e was active, so no test assumes that an env behaves independently of its index."""
import ctypes as C

import numpy as np
import pytest

import helpers
from test_episode_control_gpu import MEGAVERSE8, ROUND_TRIP

pytestmark = pytest.mark.gpu

E = 6


def _engine(scenario, A, seed, params, depth=False, seg=False, **options):
    from megaverse_b200 import capi

    g = capi.Engine(scenario, E, A, 128, 72, num_threads=2, params=params, depth=depth, segmentation=seg)
    for k, v in options.items():
        g.set_option(k, v)
    g.seed(seed)
    g.reset()
    return g


def _dev(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _active_sets(T, seed):
    """seeded random active sets at densities 0.1, 0.5 and 0.9, with all-inactive and all-active calls among them"""
    rng = np.random.default_rng(seed)
    sets = []
    for t in range(T):
        if t % 13 == 5:
            sets.append(np.zeros(E, dtype=np.uint8))
        elif t % 17 == 8:
            sets.append(np.ones(E, dtype=np.uint8))
        else:
            sets.append((rng.random(E) < (0.1, 0.5, 0.9)[t % 3]).astype(np.uint8))
    return sets


class Twins:
    """engine `a`, and per env e a twin b[e] that takes the full call whenever e is active in a"""

    def __init__(self, make, A, depth=False, seg=False, final=False):
        self.a, self.b, self.A = make(), [make() for _ in range(E)], A
        self.depth, self.seg, self.final = depth, seg, final

    def all(self):
        return [self.a] + self.b

    def host(self, acts, active):
        """mv_step_envs on a (active None: mv_step), mv_step on the twins of the active envs"""
        if active is None:
            self.a.step(acts)
        else:
            self.a.step_envs(acts, np.flatnonzero(active))
        for e in range(E):
            if active is None or active[e]:
                self.b[e].step(acts)

    def device(self, dacts, dends, active, dactive):
        """mv_step_device_active on a (active None: mv_step_device_ends), mv_step_device_ends on the twins of the active envs; each followed
        by mv_sync and mv_fetch_obs"""
        ends = dends.data_ptr() if dends is not None else None
        self.a.step_device_active(dacts.data_ptr(), ends or 0, dactive.data_ptr() if dactive is not None else 0)
        self.a.sync(); self.a.fetch_obs()
        for e in range(E):
            if active is None or active[e]:
                self.b[e].step_device(dacts.data_ptr(), ends)
                self.b[e].sync(); self.b[e].fetch_obs()

    def rows(self, g, e):
        A = self.A
        v = slice(e * A, (e + 1) * A)
        r = {"obs": np.array(g.obs()[v]), "true_objectives": np.array(g.true_objectives()[v]).view(np.uint32),
             "state": g.state(e).view(np.uint32), "voxels": g.voxels(e), "instances": g.instances(e).view(np.uint32), "level": g.level(e)}
        if self.depth:
            r["depth"] = np.array(g.depth()[v]).view(np.uint32)
        if self.seg:
            r["segmentation"] = np.array(g.segmentation()[v])
        if self.final:
            r["final_obs"] = np.array(g.final_obs()[v])
        return r

    def check(self, tag, active):
        """every env's rows in a against its twin's; at an inactive call reward 0, done 0 and reason 0"""
        A = self.A
        rew, dones, why = np.array(self.a.rewards()).view(np.uint32), np.array(self.a.dones()), np.array(self.a.done_reasons())
        for e in range(E):
            b = self.b[e]
            mine, want = self.rows(self.a, e), self.rows(b, e)
            if not (active is None or active[e]):  # the state dump carries each agent's reward of the call: 0 here, the twin's last one there
                slot = [8 + 26 * i + 24 for i in range(A)]
                assert not mine["state"][slot].any(), "%s, inactive env %d: reward in the state dump" % (tag, e)
                mine["state"][slot] = want["state"][slot]
            for k in mine:
                assert mine[k].shape == want[k].shape and np.array_equal(mine[k], want[k]), "%s, env %d: %s differs" % (tag, e, k)
            if active is None or active[e]:
                assert np.array_equal(rew[e * A:(e + 1) * A], np.array(b.rewards()[e * A:(e + 1) * A]).view(np.uint32)), "%s, env %d rewards" % (tag, e)
                assert dones[e] == b.dones()[e] and why[e] == b.done_reasons()[e], "%s, env %d done / reason" % (tag, e)
            else:
                assert not rew[e * A:(e + 1) * A].any() and dones[e] == 0 and why[e] == 0, "%s, inactive env %d reports" % (tag, e)
        return dones, why

    def healthy(self):
        for g in self.all():
            assert g.fault_word() == 0 and g.faults() == 0

    def close(self):
        for g in self.all():
            g.close()


def _host_run(scenario, A, params, T=156, depth=False, seg=False, final=False, seed=31, **options):
    tw = Twins(lambda: _engine(scenario, A, seed, params, depth, seg, final_obs=int(final), **options), A, depth, seg, final)
    rng = np.random.default_rng(seed)
    ends = 0
    for t, active in enumerate(_active_sets(T, seed)):
        tw.host(helpers.purposeful_actions(rng, E * A, t), active)
        dones, _ = tw.check("call %d" % t, active)
        ends += int(dones.sum())
    assert ends >= 2, "the window is meant to hold turnovers (%d)" % ends
    tw.healthy()
    tw.close()


HOST_CASES = [(s, A, p) for s, A, p in ROUND_TRIP] + [(MEGAVERSE8[:E], 1, {"episodeLengthSec": 2.0}), (MEGAVERSE8[2:2 + E], 1, {"episodeLengthSec": 2.0})]


@pytest.mark.parametrize("scenario,A,params", HOST_CASES, ids=[c[0] if isinstance(c[0], str) else "mixed_" + c[0][0] for c in HOST_CASES])
def test_step_envs_equals_twins_stepped_at_the_active_calls(built, scenario, A, params):
    """mv_step_envs with zero-copy delivery: every env against its twin over 156 calls of random active sets"""
    _host_run(scenario, A, params)


def test_step_envs_sliced_download_with_depth_and_terminal_frames(built):
    """mv_step_envs with option zero_copy 0 and host_slices 3 (HBM, then the copy engine per slice), depth and final_obs on"""
    _host_run("Collect", 4, {"episodeLengthSec": -45.0}, depth=True, final=True, zero_copy=0, host_slices=3)


def test_step_envs_segmentation_and_action_repeat(built):
    """mv_step_envs with segmentation and action_repeat 4 in a mixed batch"""
    _host_run(MEGAVERSE8[:E], 1, {"episodeLengthSec": 2.0}, seg=True, action_repeat=4)


DEVICE_CASES = {
    "slots2_repeat1_overlap1": ("HexExplore", 1, {"episodeLengthSec": 1.0}, dict(level_slots=2, action_repeat=1, overlap=1), {}),
    "slots2_repeat1_overlap0_final": ("HexExplore", 1, {"episodeLengthSec": 1.0}, dict(level_slots=2, action_repeat=1, overlap=0), {"final": True}),
    "slots4_repeat4_overlap0_depth": ("ObstaclesHard", 1, {"episodeLengthSec": 2.0, "obstaclesMinNumPlatforms": 0, "obstaclesMaxNumPlatforms": 0},
                                      dict(level_slots=4, action_repeat=4, overlap=0), {"depth": True, "final": True}),
    "slots4_repeat1_overlap1_mixed_seg": (MEGAVERSE8[2:2 + E], 1, {"episodeLengthSec": 2.0}, dict(level_slots=4, action_repeat=1, overlap=1), {"seg": True}),
    "slots4_repeat4_overlap1": ("Collect", 4, {"episodeLengthSec": -45.0}, dict(level_slots=4, action_repeat=4, overlap=1), {}),
}


@pytest.mark.parametrize("case", list(DEVICE_CASES))
def test_step_device_active_equals_twins_stepped_at_the_active_calls(built, case):
    """mv_step_device_active + mv_sync + mv_fetch_obs with end requests: every env against its twin (mv_step_device_ends with the same end
    bytes at the calls where the env was active) over 156 calls; requests to inactive envs are ignored"""
    scenario, A, params, options, extra = DEVICE_CASES[case]
    T, seed = 156, 23
    tw = Twins(lambda: _engine(scenario, A, seed, params, extra.get("depth", False), extra.get("seg", False), final_obs=int(extra.get("final", False)),
                               **options), A, extra.get("depth", False), extra.get("seg", False), extra.get("final", False))
    rng = np.random.default_rng(seed)
    sets = _active_sets(T, seed)
    acts = [_dev(helpers.purposeful_actions(rng, E * A, t)) for t in range(T)]
    ends = [(rng.random(E) < 0.12).astype(np.uint8) for t in range(T)]
    dends, dact = [_dev(x) for x in ends], [_dev(x) for x in sets]
    import torch

    torch.cuda.synchronize()
    requested = ignored = done = 0
    for t in range(T):
        tw.device(acts[t], dends[t], sets[t], dact[t])
        dones, why = tw.check("call %d" % t, sets[t])
        requested += int((why == 3).sum())
        done += int(dones.sum())
        ignored += int((ends[t] & (1 - sets[t])).sum())
    assert requested >= 1 and ignored >= 1 and done >= 3, "the window is meant to hold natural and requested ends (%d, %d, %d)" % (done, requested, ignored)
    tw.healthy()
    tw.close()


def test_freshness_across_interleaved_calls(built):
    """the raster leaves the inactive rows of a destination only when they hold the current frames: a zero-copy mv_step then
    mv_step_device_active (HBM rows complete), mv_step_device then mv_step_envs (host rows complete), a caller's buffer (every row drawn),
    and mv_reset_envs and mv_states_load between subset calls -- every row against the twins"""
    import torch

    A, seed = 2, 5
    params = {"episodeLengthSec": -45.0}
    tw = Twins(lambda: _engine("Collect", A, seed, params, True, True, level_slots=4), A, True, True)
    rng = np.random.default_rng(seed)
    sets = _active_sets(60, seed)

    def acts(t):
        return helpers.purposeful_actions(rng, E * A, t)

    def hbm(g):
        torch.cuda.synchronize()
        return [torch.as_tensor(g.device_array(k), device="cuda").cpu().numpy() for k in ("obs", "depth", "segmentation")]

    def against_twins(tag, mine):
        """rows of a's HBM tensors (or the caller's) against each twin's host rows, which are current after its last call"""
        for e in range(E):
            v = slice(e * A, (e + 1) * A)
            want = [np.array(tw.b[e].obs()), np.array(tw.b[e].depth()), np.array(tw.b[e].segmentation())]
            for m, w in zip(mine, want):
                assert np.array_equal(m[v], w[v]), "%s: device rows of env %d" % (tag, e)

    def device_calls(n, tag, t):
        for _ in range(n):
            a = _dev(acts(t))
            tw.device(a, None, sets[t], _dev(sets[t]))
            tw.check("%s %d" % (tag, t), sets[t])
            against_twins("%s %d" % (tag, t), hbm(tw.a))
            t += 1
        return t

    def host_calls(n, tag, t):
        for _ in range(n):
            tw.host(acts(t), sets[t]); tw.check("%s %d" % (tag, t), sets[t]); t += 1
        return t

    t = host_calls(4, "zero-copy host", 0)  # the HBM tensors go stale
    t = device_calls(4, "device after zero-copy host", t)  # the first asynchronous subset call draws every view into HBM
    full = _dev(acts(t))  # a full asynchronous step without a fetch: the host rows go stale
    for g in tw.all():
        g.step_device(full.data_ptr())
    for g in tw.all():
        g.sync()
    for b in tw.b:  # the twins' host rows are the reference
        b.fetch_obs()
    t = host_calls(4, "host after device", t + 1)
    # restarts and a state load between subset calls
    store = [g.states_create(E) for g in tw.all()]
    for g, s in zip(tw.all(), store):
        g.states_save(s, range(E), range(E))
    at_save = sets[t - 1]  # a row carries the rewards, done and reason of the saved call: 0 for the envs inactive in it
    t = host_calls(5, "host", t)
    for g in tw.all():
        g.reset_envs([1, 4], [77, 78])
    tw.check("after mv_reset_envs", sets[t - 1] | np.isin(np.arange(E), [1, 4]))  # the others still report their last call
    t = device_calls(5, "device after mv_reset_envs", t)
    for g, s in zip(tw.all(), store):
        g.states_load(s, [0, 2, 3], [0, 2, 3])
    tw.check("after mv_states_load", np.where(np.isin(np.arange(E), [0, 2, 3]), at_save, sets[t - 1]))
    t = host_calls(5, "host after mv_states_load", t)
    # a caller's buffer, zeroed before every call: every row is drawn
    obs_buf = torch.zeros((E * A, 72, 128, 4), dtype=torch.uint8, device="cuda")
    depth_buf = torch.zeros((E * A, 72, 128), dtype=torch.float32, device="cuda")
    tw.a.set_obs_buffer(obs_buf.data_ptr(), depth_buf.data_ptr())
    for _ in range(5):
        obs_buf.zero_(); depth_buf.zero_()
        torch.cuda.synchronize()
        a = _dev(acts(t))
        tw.device(a, None, sets[t], _dev(sets[t]))
        tw.check("caller buffer %d" % t, sets[t])
        torch.cuda.synchronize()
        against_twins("caller buffer %d" % t, [obs_buf.cpu().numpy(), depth_buf.cpu().numpy(), hbm(tw.a)[2]])
        t += 1
    tw.a.set_obs_buffer(None, None)  # back to the engine's own tensors, which the caller's steps left stale: every row is drawn again
    t = device_calls(3, "own tensors again", t)
    tw.healthy()
    tw.close()


def test_neutral_masks(built):
    """d_active = NULL is mv_step_device_ends (outputs and kernel launches), an all-ones mask gives the full step's outputs, and mv_step_envs
    over every env equals mv_step"""
    import torch

    A, T = 1, 40
    params = {"episodeLengthSec": 1.0}
    gs = [_engine(MEGAVERSE8[:E], A, 9, params, final_obs=1) for _ in range(3)]
    hs = [_engine(MEGAVERSE8[:E], A, 9, params, final_obs=1) for _ in range(2)]
    rng = np.random.default_rng(6)
    ones = _dev(np.ones(E, dtype=np.uint8))
    for t in range(T):
        a = helpers.purposeful_actions(rng, E * A, t)
        da, de = _dev(a), _dev((rng.random(E) < 0.1).astype(np.uint8))
        torch.cuda.synchronize()
        n0 = [g.kernel_launches() for g in gs]
        gs[0].step_device(da.data_ptr(), de.data_ptr())
        gs[1].step_device_active(da.data_ptr(), de.data_ptr(), 0)
        gs[2].step_device_active(da.data_ptr(), de.data_ptr(), ones.data_ptr())
        assert gs[0].kernel_launches() - n0[0] == gs[1].kernel_launches() - n0[1], "call %d: launches" % t
        hs[0].step(a)
        hs[1].step_envs(a, range(E))
        assert hs[0].kernel_launches() == hs[1].kernel_launches()
        for g in gs:
            g.sync(); g.fetch_obs()
        for group in (gs, hs):
            for k in ("obs", "rewards", "dones", "done_reasons", "true_objectives", "final_obs"):
                x = np.array(getattr(group[0], k)())
                for g in group[1:]:
                    assert np.array_equal(x.view(np.uint8), np.array(getattr(g, k)()).view(np.uint8)), "call %d: %s" % (t, k)
    for g in gs + hs:
        assert g.fault_word() == 0
        g.close()


def test_step_envs_refuses_bad_arguments_and_call_order(built):
    """MV_ERR_STATE before mv_reset and with mv_step_begin outstanding; MV_ERR_ARG for n < 0, a null list, an env out of range or listed
    twice.  A refused call changes nothing: the engine equals a twin that made no call"""
    from megaverse_b200 import capi

    A = 1
    params = {"episodeLengthSec": 1.0}
    g = capi.Engine("HexExplore", E, A, 128, 72, num_threads=2, params=params)
    L = capi.lib()
    one = (C.c_int32 * 1)(0)
    assert L.mv_step_envs(g._h, one, 1) == capi.MV_ERR_STATE
    g.seed(5); g.reset()
    ref = _engine("HexExplore", A, 5, params)
    rng = np.random.default_rng(2)
    acts = [helpers.purposeful_actions(rng, E * A, t) for t in range(12)]
    for t in range(4):
        g.step(acts[t]); ref.step(acts[t])

    def same(tag):
        for e in range(E):
            for k, x, y in (("state", g.state(e), ref.state(e)), ("instances", g.instances(e), ref.instances(e)), ("level", g.level(e), ref.level(e))):
                assert np.array_equal(x.view(np.uint32), y.view(np.uint32)), "%s: env %d %s" % (tag, e, k)
        for k in ("obs", "rewards", "dones", "done_reasons", "true_objectives"):
            assert np.array_equal(np.array(getattr(g, k)()).view(np.uint8), np.array(getattr(ref, k)()).view(np.uint8)), "%s: %s" % (tag, k)

    L.mv_set_actions(g._h, np.ascontiguousarray(acts[4]).ctypes.data)
    assert L.mv_step_envs(g._h, one, -1) == capi.MV_ERR_ARG
    assert L.mv_step_envs(g._h, None, 1) == capi.MV_ERR_ARG
    for bad in ([E], [-1], [1, 2, 1], [0, E + 3]):
        arr = (C.c_int32 * len(bad))(*bad)
        assert L.mv_step_envs(g._h, arr, len(bad)) == capi.MV_ERR_ARG, bad
    same("after the refused arguments")
    g.step_begin(acts[4])
    assert L.mv_step_envs(g._h, one, 1) == capi.MV_ERR_STATE
    g.step_end()
    ref.step(acts[4])
    same("after the refused call order")
    for t in range(5, 12):
        g.step(acts[t]); ref.step(acts[t])
        same("step %d after the refused calls" % t)
    assert g.fault_word() == 0
    g.close(); ref.close()


def test_megaverse_env_step_envs(built):
    """MegaverseEnv.step_envs against a MegaverseEnv twin per env: the active envs' agents return the twin's observation, reward, done and
    infos; the inactive ones reward 0, done False, {} and their previous observation"""
    from megaverse_b200 import MegaverseEnv

    n, A, T = 3, 2, 80
    params = {"episodeLengthSec": -45.0}

    def make():
        env = MegaverseEnv("Collect", n, A, 2, params=params)
        env.seed(17)
        return env

    a, twins = make(), [make() for _ in range(n)]
    prev = a.reset()
    for b in twins:
        b.reset()
    rng = np.random.default_rng(4)
    dones = 0
    for t in range(T):
        actions = rng.integers(0, [3, 3, 3, 2, 2, 3], size=(a.num_agents, 6))
        envs = [e for e in range(n) if rng.random() < (0.3, 0.7)[t % 2]]
        obs, rew, done, info = a.step_envs(envs, actions)
        assert len(obs) == len(rew) == len(done) == len(info) == a.num_agents
        for e in range(n):
            views = range(e * A, (e + 1) * A)
            if e in envs:
                o2, r2, d2, i2 = twins[e].step(actions)
                for v in views:
                    assert np.array_equal(obs[v], o2[v]) and rew[v] == r2[v] and done[v] == d2[v] and info[v] == i2[v], "call %d, agent %d" % (t, v)
                dones += int(done[e * A])
            else:
                for v in views:
                    assert np.array_equal(obs[v], prev[v]) and rew[v] == 0 and done[v] is False and info[v] == {}, "call %d, inactive agent %d" % (t, v)
        prev = [np.array(o) for o in obs]
    assert dones >= 1, "the window is meant to hold an episode end"
    for x in [a] + twins:
        x.close()
