"""Option "segmentation" without a GPU: the header documents the option, the classes and the entry points, the new names are exported, the
calls refuse a null handle, and the oracle's own segmentation (from its scene objects) is consistent with its frames.  Everything the
engine draws is compared with the oracle in test_segmentation_gpu.py."""
import ctypes as C
import inspect
import os

import numpy as np

import helpers
import orc
import orc_seg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["mv_segmentation_host", "mv_segmentation_device"]
SEG_STATIC, SEG_TERRAIN, SEG_OBJECT, SEG_AGENT, SEG_REWARD = 1, 2, 3, 4, 5


def test_segmentation_is_documented(built):
    with open(os.path.join(ROOT, "include", "megaverse_b200.h")) as f:
        header = f.read()
    assert '"segmentation" (0/1, before the first reset' in header
    for name, value in (("NONE", 0), ("STATIC", 1), ("TERRAIN", 2), ("OBJECT", 3), ("AGENT", 4), ("REWARD", 5)):
        assert "#define MV_SEG_%s %d" % (name, value) in header
    for name in NEW:
        assert "int %s(mv_handle h" % name in header
    assert "uint16[N][h][w]" in header and "18 432 B per view" in header
    for limit in ("mv_draw_hires", "mv_debug_render_instances", "mv_set_obs_buffer", "final_obs", "multi-GPU gather"):
        assert limit in header.split('Segmentation, option "segmentation"')[1].split("int mv_segmentation_host")[0], limit


def test_segmentation_exports_and_signatures(built):
    from megaverse_b200 import capi
    from megaverse_b200.extension.megaverse import MegaverseGym
    from megaverse_b200.megaverse_env import MegaverseEnv

    assert set(NEW) <= set(capi.EXPORTS)
    assert (capi.MV_SEG_NONE, capi.MV_SEG_STATIC, capi.MV_SEG_TERRAIN, capi.MV_SEG_OBJECT, capi.MV_SEG_AGENT, capi.MV_SEG_REWARD) == (0, 1, 2, 3, 4, 5)
    assert inspect.signature(capi.Engine.__init__).parameters["segmentation"].default is False
    assert list(inspect.signature(capi.Engine.segmentation).parameters) == ["self"]
    assert "segmentation" in capi.Engine.device_array.__doc__ and "<u2" in inspect.getsource(capi.Engine.device_array)
    assert "segmentation" in MegaverseGym.get_segmentation.__doc__
    params = inspect.signature(MegaverseEnv.__init__).parameters
    positional = [n for n, p in params.items() if p.kind == p.POSITIONAL_OR_KEYWORD]
    assert positional == ["self", "scenario_name", "num_envs", "num_agents_per_env", "num_simulation_threads", "use_vulkan", "params"]
    assert params["segmentation"].kind == inspect.Parameter.KEYWORD_ONLY and params["segmentation"].default is False
    assert list(inspect.signature(MegaverseEnv.segmentation).parameters) == ["self"]


def test_segmentation_calls_refuse_a_null_handle(built):
    from megaverse_b200 import capi

    L = capi.lib()
    p = C.c_void_p()
    for name in NEW:
        assert getattr(L, name)(None, C.byref(p)) == capi.MV_ERR_ARG, name
    for v in (0, 1, 2, -1):
        assert L.mv_set_option(None, b"segmentation", v) == capi.MV_ERR_ARG


def _rollout(scenario, E, A, steps, seed=3):
    o = orc.Oracle(scenario, E, A, depth=True)
    o.seed(seed)
    o.reset()
    rng = np.random.default_rng(seed)
    yield o
    for t in range(steps):
        o.step(helpers.purposeful_actions(rng, E * A, t))
        yield o
    o.close()


def test_oracle_segmentation_is_zero_exactly_where_nothing_was_drawn(built):
    for scenario, A in (("TowerBuilding", 2), ("ObstaclesHard", 1), ("Collect", 2), ("HexMemory", 1), ("Rearrange", 1)):
        classes = set()
        for o in _rollout(scenario, 2, A, 12):
            (seg, sdepth), depth = orc_seg.segmentation(o), o.depth()
            # the restated raster loop draws the oracle's own depth, bit for bit
            assert np.array_equal(sdepth.view(np.uint32), depth.view(np.uint32)), scenario
            assert np.array_equal(seg == 0, depth == 0), scenario
            classes |= set(np.unique(seg >> 8).tolist())
        assert classes <= {0, SEG_STATIC, SEG_TERRAIN, SEG_OBJECT, SEG_AGENT, SEG_REWARD}, (scenario, classes)
        assert SEG_STATIC in classes, scenario
        if scenario == "TowerBuilding":  # the building zone's slab
            assert SEG_TERRAIN in classes, scenario


def test_oracle_segmentation_names_a_reward_in_front_of_the_agent(built):
    """a Collect view where a reward object covers pixels: they carry MV_SEG_REWARD and the index of the reward object that is there"""
    o = orc.Oracle("Collect", 8, 1, depth=True)
    o.seed(11)
    o.reset()
    seg, _ = orc_seg.segmentation(o)
    hits = 0
    for v in range(8):
        rew = seg[v][(seg[v] >> 8) == SEG_REWARD]
        if rew.size == 0:
            continue
        hits += 1
        idx = np.unique(rew & 0xFF)
        # each named reward object, drawn alone from its two instances, covers pixels of this view where the tag says it does
        inst = o.instances(v)
        cones = [i for i in range(inst.shape[0]) if int(inst[i, 0]) == 3]  # Collect's rewards are the only cones: diamonds of 2 cones each
        for r in idx:
            rgba, depth = orc.render_instances(o.view(v, 0), inst[cones[2 * r]: cones[2 * r] + 2], 128, 72, want_depth=True)
            mine = seg[v] == ((SEG_REWARD << 8) | r)
            assert mine.any() and (depth[mine] > 0).all(), (v, r)
    assert hits >= 1, "no Collect view of these seeds shows a reward object"


def test_oracle_segmentation_hud_bar_carries_its_agent(built):
    """the HUD bar is under a pixel tall: where the oracle draws an agent's own bar (the bar drawn alone wins the pixel at the frame's
    depth), the pixels name that agent"""
    found = 0
    for o in _rollout("TowerBuilding", 4, 4, 30, seed=5):
        (seg, _), depth = orc_seg.segmentation(o), o.depth()
        for e in range(o.E):
            inst = o.instances(e)
            nb = int((inst[:, 0].astype(np.int32) == 0).sum())  # boxes first; the last 2A of them are the agents' eyes, then their bars
            for a in range(o.A):
                v = e * o.A + a
                _, bar = orc.render_instances(o.view(e, a), inst[nb - o.A + a: nb - o.A + a + 1], o.w, o.h, want_depth=True)
                won = (bar > 0) & (bar == depth[v])
                found += int(won.sum())
                assert (seg[v][won] == ((SEG_AGENT << 8) | a)).all(), (e, a)
    assert found >= 1, "no view of these rollouts shows its own HUD bar"
