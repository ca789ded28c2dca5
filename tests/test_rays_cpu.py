"""Ray sensors (mv_set_rays) without a GPU: the new entry points refuse a null handle and the Python surfaces exist; the direction helpers
give unit vectors in the stated order and angles; the oracle's restatement of the hit definition (tests/oracle_seg/orc_rays.cpp) gives the
analytic hits of hand-built scenes, and its rays through pixel centres agree with the oracle rasteriser's own segmentation and depth."""
import ctypes as C
import inspect
import math

import numpy as np
import pytest

import helpers

NEW = ["mv_set_rays", "mv_rays_host", "mv_rays_device", "mv_final_rays_host", "mv_final_rays_device", "mv_last_rays_ms"]
SCENARIOS = ["TowerBuilding", "Collect", "Rearrange", "Sokoban", "HexExplore", "HexMemory", "Empty", "ObstaclesEasy", "ObstaclesMedium",
             "ObstaclesHard", "ObstaclesWalls", "ObstaclesSteps", "ObstaclesLava"]
SEG_STATIC, SEG_OBJECT, SEG_AGENT = 1, 3, 4
EYE = np.eye(4, dtype=np.float32).reshape(16)  # the camera at the origin looking down -z


def test_ray_calls_refuse_a_null_handle(built):
    from megaverse_b200 import capi

    L = capi.lib()
    d = np.array([[0.0, 0.0, -1.0]], dtype=np.float32)
    assert L.mv_set_rays(None, d.ctypes.data, 1, 10.0) == capi.MV_ERR_ARG
    p, q = C.c_void_p(), C.c_void_p()
    for name in NEW[1:5]:
        assert getattr(L, name)(None, C.byref(p), C.byref(q)) == capi.MV_ERR_ARG, name
        assert getattr(L, name)(None, None, None) == capi.MV_ERR_ARG, name
    f = C.c_float()
    assert L.mv_last_rays_ms(None, C.byref(f)) == capi.MV_ERR_ARG


def test_ray_exports_and_signatures(built):
    from megaverse_b200 import capi
    from megaverse_b200.extension.megaverse import MegaverseGym
    from megaverse_b200.megaverse_env import MegaverseEnv

    assert set(NEW) <= set(capi.EXPORTS)
    for name in NEW:
        assert hasattr(capi.lib(), name)
    for name in ("rays", "final_rays"):
        assert list(inspect.signature(getattr(capi.Engine, name)).parameters) == ["self"], name
    assert list(inspect.signature(capi.Engine.set_rays).parameters) == ["self", "directions", "max_distance"]
    assert "rays_dist" in capi.Engine.device_array.__doc__ and "final_rays_tag" in capi.Engine.device_array.__doc__
    for name in ("set_rays", "get_rays", "get_final_rays"):
        assert hasattr(MegaverseGym, name), name
    params = inspect.signature(MegaverseEnv.__init__).parameters
    positional = [n for n, p in params.items() if p.kind == p.POSITIONAL_OR_KEYWORD]
    assert positional == ["self", "scenario_name", "num_envs", "num_agents_per_env", "num_simulation_threads", "use_vulkan", "params"]
    assert params["ray_directions"].kind == inspect.Parameter.KEYWORD_ONLY and params["ray_directions"].default is None
    assert params["ray_max_distance"].kind == inspect.Parameter.KEYWORD_ONLY
    assert hasattr(MegaverseEnv, "ray_observations")


# ---------------------------------------------------------------------------------------------------- direction helpers
def _yaw_pitch(d):
    d = np.asarray(d, dtype=np.float64)
    return np.degrees(np.arctan2(d[:, 0], -d[:, 2])), np.degrees(np.arcsin(np.clip(d[:, 1], -1.0, 1.0)))


def test_fan_and_ring_directions():
    from megaverse_b200 import rays

    for d in (rays.fan(7, 120.0), rays.fan(1, 90.0), rays.ring(8), rays.ring(5, -30.0), rays.fan(16, 90.0, 15.0)):
        assert d.dtype == np.float32 and d.shape[1] == 3 and d.flags.c_contiguous
        assert np.allclose(np.linalg.norm(d.astype(np.float64), axis=1), 1.0, atol=1e-6)
    yaw, pitch = _yaw_pitch(rays.fan(7, 120.0))
    assert np.allclose(yaw, np.linspace(-60.0, 60.0, 7), atol=1e-4) and np.allclose(pitch, 0.0, atol=1e-5)  # left to right
    assert np.array_equal(rays.fan(1, 90.0), np.array([[0.0, 0.0, -1.0]], dtype=np.float32))
    yaw, pitch = _yaw_pitch(rays.fan(16, 90.0, 15.0))
    assert np.allclose(pitch, 15.0, atol=1e-4) and np.allclose(yaw, np.linspace(-45.0, 45.0, 16), atol=1e-4)
    ring = rays.ring(4)  # forward, right, back, left
    assert np.allclose(ring, [[0, 0, -1], [1, 0, 0], [0, 0, 1], [-1, 0, 0]], atol=1e-7)
    yaw, pitch = _yaw_pitch(rays.ring(5, -30.0))
    assert np.allclose(np.mod(yaw, 360.0), [0.0, 72.0, 144.0, 216.0, 288.0], atol=1e-4) and np.allclose(pitch, -30.0, atol=1e-4)
    # float64 rounded once
    a = math.radians(-60.0)
    assert rays.fan(3, 120.0)[0, 0] == np.float32(math.sin(a))
    with pytest.raises(ValueError):
        rays.fan(0, 90.0)


# ---------------------------------------------------------------------------------------------------- the definition on hand-built scenes
def _inst(mesh, translate=(0.0, 0.0, 0.0), scale=(1.0, 1.0, 1.0)):
    m = np.diag([*scale, 1.0])
    m[:3, 3] = translate
    return np.concatenate([[mesh, 0.0], m.T.reshape(16)]).astype(np.float32)


def _cast(insts, tags, dirs, max_dist=100.0, agent=-1, view=EYE):
    import orc_rays

    return orc_rays.rays_scene(view, np.stack(insts), tags, np.asarray(dirs, dtype=np.float32), max_dist, agent)


def test_axis_aligned_box_hits_its_front_face():
    box = _inst(0, (0.0, 0.0, -5.0), (1.0, 2.0, 1.0))  # front face at z = -4
    dist, tag = _cast([box], [SEG_STATIC << 8], [[0, 0, -1], [0, 0, -2], [0.2, 0.0, -1.0], [0, 0, 1], [0, 1, 0]])
    assert dist[0] == 4.0 and tag[0] == SEG_STATIC << 8
    assert dist[1] == 2.0  # distances count multiples of the direction's length
    assert dist[2] == np.float32(4.0) and tag[2] == SEG_STATIC << 8  # hits at x = 0.8: inside the face
    assert dist[3] == 0.0 and tag[3] == 0 and dist[4] == 0.0 and tag[4] == 0  # behind and beside: nothing
    # through a moved camera: the same box seen from (0, 0, 3) forward is 7 away; the view matrix maps world to camera
    view = np.eye(4, dtype=np.float32)
    view[2, 3] = -3.0
    dist, _ = _cast([box], [SEG_STATIC << 8], [[0, 0, -1]], view=view.T.reshape(16))
    assert dist[0] == 7.0


def test_max_distance_is_inclusive():
    box = _inst(0, (0.0, 0.0, -5.0))
    assert _cast([box], [256], [[0, 0, -1]], max_dist=4.0)[0][0] == 4.0
    d, t = _cast([box], [256], [[0, 0, -1]], max_dist=3.999)
    assert d[0] == 0.0 and t[0] == 0


def test_only_front_faces_count():
    # a ray that starts inside a box or a closed mesh sees only back faces: no hit; it then hits what lies beyond
    far = _inst(0, (0.0, 0.0, -20.0))
    for mesh, scale in ((0, 3.0), (2, 3.0), (4, 3.0), (1, 3.0)):
        d, t = _cast([_inst(mesh, (0.0, 0.0, 0.0), (scale,) * 3), far], [SEG_OBJECT << 8 | 1, SEG_STATIC << 8], [[0, 0, -1], [0, 1, 0], [1, 0, 0]])
        assert d[0] == 19.0 and t[0] == SEG_STATIC << 8, mesh
        assert (t[1:] == 0).all() and (d[1:] == 0).all(), mesh
    # a sphere ahead: the hit lies between the inscribed and the circumscribed sphere of the icosphere
    d, t = _cast([_inst(2, (0.0, 0.0, -5.0))], [SEG_OBJECT << 8 | 2], [[0, 0, -1]])
    assert 4.0 <= d[0] <= 4.25 and t[0] == SEG_OBJECT << 8 | 2


def test_exact_tie_goes_to_the_later_entry():
    a, b = _inst(0, (0.0, 0.0, -5.0)), _inst(0, (0.0, 0.0, -5.0))
    d, t = _cast([a, b], [SEG_OBJECT << 8 | 1, SEG_OBJECT << 8 | 2], [[0, 0, -1]])
    assert d[0] == 4.0 and t[0] == SEG_OBJECT << 8 | 2
    d, t = _cast([b, a], [SEG_OBJECT << 8 | 2, SEG_OBJECT << 8 | 1], [[0, 0, -1]])
    assert t[0] == SEG_OBJECT << 8 | 1
    # a nearer earlier entry still wins
    d, t = _cast([_inst(0, (0.0, 0.0, -3.0)), a], [SEG_OBJECT << 8 | 3, SEG_OBJECT << 8 | 1], [[0, 0, -1]])
    assert d[0] == 2.0 and t[0] == SEG_OBJECT << 8 | 3


def test_the_agents_own_drawables_are_ignored():
    body = _inst(1, (0.0, 0.0, -3.0), (0.5, 0.5, 0.5))
    eyes = _inst(0, (0.0, 0.0, -2.0), (0.1, 0.1, 0.1))
    wall = _inst(0, (0.0, 0.0, -10.0))
    insts, tags = [body, eyes, wall], [SEG_AGENT << 8 | 1, SEG_AGENT << 8 | 1, SEG_STATIC << 8]
    d, t = _cast(insts, tags, [[0, 0, -1]], agent=1)
    assert d[0] == 9.0 and t[0] == SEG_STATIC << 8
    d, t = _cast(insts, tags, [[0, 0, -1]], agent=0)  # another agent's eyes are in the way
    assert t[0] == SEG_AGENT << 8 | 1 and d[0] == np.float32(1.9)


def test_mesh_bounds_of_the_prefilter():
    import orc

    for mesh in range(1, 5):
        vtx, _ = orc.mesh(mesh)
        p = vtx[:, :3].copy().view(np.float32)
        lim = np.array([1.0, 2.0 if mesh == 1 else 1.0, 1.0], dtype=np.float32)
        assert (np.abs(p) <= lim).all(), mesh


# ---------------------------------------------------------------------------------------------------- against the oracle rasteriser
# measured on the CPU: 100 % of tags and >= 99.99 % of tags and distances (1 % relative) in every scenario at 128 x 72 after 40 steps,
# the agent's own body excluded.  The rasteriser samples snapped sub-pixel coordinates, so a pixel at an edge may name the neighbour.
AGREEMENT = 0.995


@pytest.mark.parametrize("name", SCENARIOS)
def test_pixel_centre_rays_agree_with_the_oracle_segmentation(name):
    import orc
    import orc_rays
    import orc_seg_view
    from megaverse_b200 import cameras

    W, H, E, A = 128, 72, 2, 2
    p00, p11, _, _ = cameras.projection(W, H)
    px, py = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64))
    nx, ny = (px + 0.5 - W / 2) / (W / 2), (py + 0.5 - H / 2) / (H / 2)
    dirs = np.stack([nx / float(p00), ny / float(p11), -np.ones_like(nx)], -1).reshape(-1, 3).astype(np.float32)
    o = orc.Oracle(name, E, A, render=False)
    try:
        for e in range(E):
            o.seed_env(e, 100 + e)
        o.reset()
        rng = np.random.default_rng(3)
        for t in range(40):
            o.step(helpers.purposeful_actions(rng, E * A, t))
        total = agree = 0
        for e in range(E):
            for a in range(A):
                seg, depth = orc_seg_view.segmentation_view(o, e, o.view(e, a), W, H)
                dist, tag = orc_rays.rays_env(o, e, a, dirs, 120.0)
                dist, tag = dist.reshape(H, W), tag.reshape(H, W)
                keep = seg != (SEG_AGENT << 8 | a)  # the rasteriser draws the agent's own body; its rays ignore it
                ok = keep & (tag == seg) & (np.abs(dist - depth) <= 0.01 * depth)
                total += int(keep.sum())
                agree += int(ok.sum())
        assert agree >= AGREEMENT * total, "%s: %d of %d pixels agree" % (name, agree, total)
    finally:
        o.close()
