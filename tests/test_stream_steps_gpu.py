"""Stream steps (mv_step_stream): the level-set device step enqueued on the caller's stream as device work only, so that a CUDA graph can
capture it.  Every check runs twin engines -- same seeds, options and inputs -- one taking stream steps (eager on a torch side stream, or
replayed from a torch.cuda.graph), the other mv_step_device, and asks for the same bytes after every step: frames, rewards, dones, reasons,
true objectives, level ids, terminal frames, state tensors, rays, reward components and segmentation.  Short episodes and requested ends
turn envs over throughout.  Then the host calls of stream mode against the twin, and the refusals."""
import ctypes as C

import numpy as np
import pytest

import helpers

pytestmark = pytest.mark.gpu

MEGAVERSE8 = ["TowerBuilding", "ObstaclesEasy", "ObstaclesHard", "Collect", "Sokoban", "HexMemory", "HexExplore", "Rearrange"]
# a negative base ends the timed episodes after a step or two, Obstacles chains without platforms last a few seconds
SHORT_MIXED = {"episodeLengthSec": -200.0, "obstaclesMinNumPlatforms": 0.0, "obstaclesMaxNumPlatforms": 0.0}
SHORT = {"episodeLengthSec": 0.5}
L = 16

# (scenario, A, overlap, action_repeat)
CASES = [("Collect", 2, 1, 1), ("Collect", 2, 0, 1), ("Collect", 2, 1, 3), ("Collect", 2, 0, 3), ("mixed", 2, 1, 1)]
IDS = ["overlap1-repeat1", "overlap0-repeat1", "overlap1-repeat3", "overlap0-repeat3", "megaverse8"]


def _engine(scenario, A, overlap, repeat, level_set=L):
    from megaverse_b200 import capi
    from megaverse_b200 import rays

    names = [MEGAVERSE8[e % 8] for e in range(16)] if scenario == "mixed" else scenario
    E = 16 if scenario == "mixed" else 8
    g = capi.Engine(names, E, A, 128, 72, num_threads=4, params=SHORT_MIXED if scenario == "mixed" else SHORT, segmentation=True)
    g.set_option("fast_shading", 0)
    g.set_option("zero_copy", 0)  # host-facing calls leave their frames in HBM too: the device arrays can be compared after any call
    for k, v in (("final_obs", 1), ("state_tensors", 1), ("reward_components", 1), ("overlap", overlap), ("action_repeat", repeat)):
        g.set_option(k, v)
    if level_set:
        g.set_option("level_set_seed", 5)
        g.set_option("level_set", level_set)
    g.set_rays(rays.fan(6, 90.0, -10.0), 20.0)
    for e in range(E):
        g.seed_env(e, 300 + 7 * e)
    return g


KEYS = ["obs", "segmentation", "rewards", "dones", "done_reasons", "true_objectives", "level_ids", "final_obs", "rays_dist", "rays_tag",
        "final_rays_dist", "final_rays_tag", "reward_components", "episode_reward_components"]
KEYS += ["%sstate_%s" % (p, k) for p in ("", "final_") for k in ("agents", "envs", "objects", "rewards")]


class Twins:
    """the stream engine `s` and its mv_step_device twin `d`, with torch views of every device output of both"""

    def __init__(self, scenario, A, overlap, repeat):
        import torch

        self.s = _engine(scenario, A, overlap, repeat)
        self.d = _engine(scenario, A, overlap, repeat)
        self.s.reset()
        self.d.reset()
        self.E, self.N = self.s.E, self.s.N
        self.sv = {k: torch.as_tensor(self.s.device_array(k), device="cuda") for k in KEYS}
        self.dv = {k: torch.as_tensor(self.d.device_array(k), device="cuda") for k in KEYS}
        self.side = torch.cuda.Stream()
        torch.cuda.synchronize()

    def same(self, tag, keys=KEYS):
        import torch

        torch.cuda.synchronize()
        for k in keys:
            assert torch.equal(self.sv[k], self.dv[k]), "%s: %s differs" % (tag, k)

    def same_host(self, tag):
        for fn in ("rewards", "dones", "done_reasons", "true_objectives", "level_ids"):
            a, b = np.array(getattr(self.s, fn)()), np.array(getattr(self.d, fn)())
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), "%s: host %s differs" % (tag, fn)

    def healthy(self):
        for g in (self.s, self.d):
            assert g.fault_word() == 0
            assert g.faults() == 0

    def close(self):
        self.s.close()
        self.d.close()


def _inputs(E, N, steps, seed, active=True):
    """device actions [steps, N], requested ends [steps, E] (about one env in twenty per step) and active masks [steps, E] (every env in
    two steps of three, about four in five in the third)"""
    import torch

    rng = np.random.default_rng(seed)
    acts = np.stack([helpers.purposeful_actions(rng, N, t) for t in range(steps)]).astype(np.int32)
    ends = (rng.random((steps, E)) < 0.05).astype(np.uint8)
    act = np.ones((steps, E), dtype=np.uint8)
    if active:
        act[2::3] = (rng.random((len(act[2::3]), E)) < 0.8).astype(np.uint8)
    out = torch.from_numpy(acts).cuda(), torch.from_numpy(ends).cuda(), torch.from_numpy(act).cuda()
    torch.cuda.synchronize()
    return out


@pytest.fixture(params=CASES, ids=IDS)
def twins(built, request):
    t = Twins(*request.param)
    yield t
    t.close()


def test_eager_stream_steps_equal_device_steps(twins):
    """150 eager stream steps on a torch side stream against 150 mv_step_device calls, compared after every step"""
    import torch

    t = twins
    acts, ends, act = _inputs(t.E, t.N, 150, 11)
    turnovers = 0
    for i in range(150):
        with torch.cuda.stream(t.side):
            t.s.step_stream(t.side.cuda_stream, acts[i].data_ptr(), ends[i].data_ptr(), act[i].data_ptr())
        t.d.step_device_active(acts[i].data_ptr(), ends[i].data_ptr(), act[i].data_ptr())
        t.same("step %d" % i)
        turnovers += int(t.dv["dones"].sum())
    assert turnovers >= 20
    t.healthy()


def _capture(t, K, masks, ends, active, static):
    """a graph of K stream steps on masks[k] / ends[k] / active[k], each followed by torch copies of its rewards and dones into
    static[...][k]"""
    import torch

    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        s = torch.cuda.current_stream().cuda_stream
        for k in range(K):
            t.s.step_stream(s, masks[k].data_ptr(), ends[k].data_ptr(), active[k].data_ptr())
            static["rewards"][k].copy_(t.sv["rewards"])
            static["dones"][k].copy_(t.sv["dones"])
    return g


def test_graph_replays_equal_device_steps(twins):
    """a graph of K = 8 stream steps replayed 20 times on refilled inputs, against the twin's eager steps step for step; then the host calls
    of stream mode, each against the same call on the twin"""
    import torch

    t = twins
    K, reps = 8, 20
    masks = torch.zeros((K, t.N), dtype=torch.int32, device="cuda")
    ends = torch.zeros((K, t.E), dtype=torch.uint8, device="cuda")
    active = torch.ones((K, t.E), dtype=torch.uint8, device="cuda")
    static = {"rewards": torch.zeros((K, t.N), device="cuda"), "dones": torch.zeros((K, t.E), dtype=torch.uint8, device="cuda")}
    acts, ends_in, act_in = _inputs(t.E, t.N, K * (reps + 6), 23)
    # one eager step on each first: the graph then starts from a stream-mode engine, as a trainer's would
    t.s.step_stream(None, acts[0].data_ptr())
    t.d.step_device(acts[0].data_ptr())
    t.same("eager step")
    static["rewards"][0].copy_(t.sv["rewards"])  # the copy kernels loaded before the capture
    static["dones"][0].copy_(t.sv["dones"])
    torch.cuda.synchronize()
    graph = _capture(t, K, masks, ends, active, static)
    turnovers = 0
    rnd = 0

    def replay(tag):
        nonlocal rnd
        base = 1 + K * rnd
        rnd += 1
        masks.copy_(acts[base:base + K])
        ends.copy_(ends_in[base:base + K])
        active.copy_(act_in[base:base + K])
        graph.replay()
        for k in range(K):
            t.d.step_device_active(acts[base + k].data_ptr(), ends_in[base + k].data_ptr(), act_in[base + k].data_ptr())
            torch.cuda.synchronize()
            assert torch.equal(static["rewards"][k], t.dv["rewards"]), "%s step %d: rewards differ" % (tag, k)
            assert torch.equal(static["dones"][k], t.dv["dones"]), "%s step %d: dones differ" % (tag, k)
        t.same(tag)
        return int(static["dones"].sum())

    for r in range(reps):
        turnovers += replay("replay %d" % r)
    assert turnovers >= 20

    # host calls after replays: each a synchronisation point that refreshes the mirrors
    t.d.sync()
    t.same_host("after the replays")
    envs = np.array([1, 4, 6], dtype=np.int32)
    t.s.reset_envs(envs)
    t.d.reset_envs(envs)
    t.same("reset_envs")
    t.same_host("reset_envs")
    t.s.reset_envs(envs[:2], [77, 78])
    t.d.reset_envs(envs[:2], [77, 78])
    t.same("reset_envs with seeds")
    t.same_host("reset_envs with seeds")
    sid_s, sid_d = t.s.states_create(2), t.d.states_create(2)
    t.s.states_save(sid_s, [0, 3], [0, 1])
    t.d.states_save(sid_d, [0, 3], [0, 1])
    turnovers += replay("replay after the save")
    dst = [t.E // 2, 3 + t.E // 2]  # envs of the saved envs' scenarios (the mixed engine repeats its eight names)
    t.s.states_load(sid_s, [0, 1], dst)
    t.d.states_load(sid_d, [0, 1], dst)
    t.same("states_load")
    t.same_host("states_load")
    t.s.set_next_levels([0, 2, 7], [3, 9, 15])
    t.d.set_next_levels([0, 2, 7], [3, 9, 15])
    turnovers += replay("replay after set_next_levels")
    t.d.sync()
    t.same_host("replay after set_next_levels")
    for g in (t.s, t.d):
        rs = g.get_reward_shaping(0, 0)
        g.set_reward_shaping(0, 0, {k: (v * 2.5 + 0.25 if k != "teamSpirit" else v) for k, v in rs.items()})
    turnovers += replay("replay after set_reward_shaping")
    # a regular device step and a host-facing step on both
    a = acts[-1]
    t.s.step_device(a.data_ptr())
    t.d.step_device(a.data_ptr())
    t.same("step_device in stream mode")
    t.d.sync()
    t.same_host("step_device in stream mode")
    host_acts = a.cpu().numpy()
    t.s.step(host_acts)
    t.d.step(host_acts)
    t.same_host("step in stream mode")
    assert np.array_equal(np.array(t.s.obs()), np.array(t.d.obs())), "step in stream mode: host obs differ"
    # and replays again after the host-path calls
    turnovers += replay("replay after host-path steps")
    t.d.sync()
    t.same_host("the end")
    t.healthy()


def _policy(obs, N):
    """a deterministic integer policy: one action bit per agent from a strided sum of its frame"""
    import torch

    s = obs.view(N, -1)[:, ::61].to(torch.int32).sum(1)
    return torch.bitwise_left_shift(torch.ones_like(s), s % 11).to(torch.int32)


def test_policy_inside_the_graph(twins):
    """a policy on the obs and 16 stream steps in one graph, against the same torch ops run eagerly before each mv_step_device"""
    import torch

    t = twins
    K = 16
    static = {"rewards": torch.zeros((K, t.N), device="cuda"), "dones": torch.zeros((K, t.E), dtype=torch.uint8, device="cuda"),
              "masks": torch.zeros((K, t.N), dtype=torch.int32, device="cuda")}
    t.s.step_stream(None)
    t.d.step_device(None)
    torch.cuda.synchronize()
    static["masks"][0].copy_(_policy(t.sv["obs"], t.N))  # the torch ops' kernels loaded before the capture
    static["rewards"][0].copy_(t.sv["rewards"])
    static["dones"][0].copy_(t.sv["dones"])
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        s = torch.cuda.current_stream().cuda_stream
        for k in range(K):
            static["masks"][k].copy_(_policy(t.sv["obs"], t.N))
            t.s.step_stream(s, static["masks"][k].data_ptr())
            static["rewards"][k].copy_(t.sv["rewards"])
            static["dones"][k].copy_(t.sv["dones"])
    torch.cuda.synchronize()
    for r in range(4):
        graph.replay()
        for k in range(K):
            torch.cuda.synchronize()
            m = _policy(t.dv["obs"], t.N)
            torch.cuda.synchronize()
            t.d.step_device(m.data_ptr())
            torch.cuda.synchronize()
            assert torch.equal(static["masks"][k], m), "replay %d step %d: policy differs" % (r, k)
            assert torch.equal(static["rewards"][k], t.dv["rewards"]), "replay %d step %d: rewards differ" % (r, k)
            assert torch.equal(static["dones"][k], t.dv["dones"]), "replay %d step %d: dones differ" % (r, k)
        t.same("policy replay %d" % r)
    t.healthy()


def test_eager_policy_on_the_default_stream(twins):
    """eager stream steps on torch's default stream (handle 0, the legacy default stream) whose masks come from torch ops on the obs on
    that stream, with no synchronisation between them: each step must see its policy's masks and each policy the previous step's frames"""
    import torch

    t = twins
    K = 32
    buf = {"masks": torch.zeros((K, t.N), dtype=torch.int32, device="cuda"), "rewards": torch.zeros((K, t.N), device="cuda"),
           "dones": torch.zeros((K, t.E), dtype=torch.uint8, device="cuda")}
    assert torch.cuda.current_stream().cuda_stream == 0
    for k in range(K):
        buf["masks"][k].copy_(_policy(t.sv["obs"], t.N))
        t.s.step_stream(torch.cuda.current_stream().cuda_stream, buf["masks"][k].data_ptr())
        buf["rewards"][k].copy_(t.sv["rewards"])
        buf["dones"][k].copy_(t.sv["dones"])
    torch.cuda.synchronize()
    for k in range(K):
        m = _policy(t.dv["obs"], t.N)
        torch.cuda.synchronize()
        t.d.step_device(m.data_ptr())
        torch.cuda.synchronize()
        assert torch.equal(buf["masks"][k], m), "step %d: policy differs" % k
        assert torch.equal(buf["rewards"][k], t.dv["rewards"]), "step %d: rewards differ" % k
        assert torch.equal(buf["dones"][k], t.dv["dones"]), "step %d: dones differ" % k
    t.same("after the eager policy loop")
    t.healthy()


def test_refusals(built):
    import torch

    from megaverse_b200 import capi

    Lb = capi.lib()
    stream_engine = _engine("Collect", 1, 1, 1, level_set=0)
    try:
        stream_engine.reset()
        assert Lb.mv_step_stream(stream_engine._h, None, None, None, None) == capi.MV_ERR_STATE
        assert b"level_set" in Lb.mv_last_error(stream_engine._h)
    finally:
        stream_engine.close()
    g = _engine("Collect", 1, 1, 1)
    try:
        assert Lb.mv_step_stream(g._h, None, None, None, None) == capi.MV_ERR_STATE  # before mv_reset
        g.reset()
        g.step_begin(np.zeros(g.N, dtype=np.int32))
        assert Lb.mv_step_stream(g._h, None, None, None, None) == capi.MV_ERR_STATE  # outstanding mv_step_begin
        g.step_end()
        free = sorted(set(range(L)) - set(int(x) for x in g.level_ids()))[0]  # a row no env is on: rewritten two calls on
        g.replace_levels([free], [901])
        assert Lb.mv_step_stream(g._h, None, None, None, None) == capi.MV_ERR_STATE  # pending replacement
        for _ in range(4):  # host-path steps carry the replacement out
            g.step(np.zeros(g.N, dtype=np.int32))
            if not g.level_rows()[1].any():
                break
        assert not g.level_rows()[1].any()
        g.step_stream(torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        # stream mode: what reallocates a buffer a captured launch refers to is refused, and changes nothing
        rows = np.array([3], dtype=np.int32)
        assert Lb.mv_replace_levels(g._h, rows.ctypes.data, rows.ctypes.data, 1) == capi.MV_ERR_STATE
        assert not g.level_rows()[1].any()
        cfg = g.raster_config()
        for key in (b"tri_cap", b"raster_bands"):
            assert Lb.mv_set_option(g._h, key, 1 if key == b"raster_bands" else 256) == capi.MV_ERR_STATE
        assert g.raster_config() == cfg
        for fn in ("mv_debug_step_profile", "mv_debug_raster_stats"):
            getattr(Lb, fn).argtypes = [C.c_void_p, C.c_void_p, C.c_int]
            assert getattr(Lb, fn)(g._h, None, 1) == capi.MV_ERR_STATE
        g.step_stream(None)
        g.sync()
        assert g.fault_word() == 0 and g.faults() == 0
    finally:
        g.close()
