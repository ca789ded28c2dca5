"""Spectator cameras without a GPU: every new C entry point refuses a null handle, the Python surfaces exist, and the pose helpers
(megaverse_b200.cameras) give rigid view matrices in the engine's convention that frame what they are asked to frame."""
import ctypes as C
import inspect
import math

import numpy as np
import pytest

NEW = ["mv_draw_cameras", "mv_draw_cameras_device", "mv_views_device", "mv_level_bounds", "mv_debug_view_order"]


def _matrix(v16):
    return np.asarray(v16, dtype=np.float64).reshape(4, 4).T  # column-major storage


def _check_rigid(v16, eye):
    m = _matrix(v16)
    r = m[:3, :3]
    assert np.allclose(r @ r.T, np.eye(3), atol=1e-6), "rotation block is not orthonormal"
    assert abs(np.linalg.det(r) - 1.0) < 1e-6, "not a proper rotation"
    assert np.allclose(m[3], [0.0, 0.0, 0.0, 1.0])
    assert np.allclose(m @ np.append(eye, 1.0), [0.0, 0.0, 0.0, 1.0], atol=1e-4), "the eye does not map to the origin"


def test_camera_calls_refuse_a_null_handle(built):
    from megaverse_b200 import capi

    L = capi.lib()
    envs = (C.c_int32 * 1)(0)
    views = (C.c_float * 16)()
    p = [C.c_void_p() for _ in range(3)]
    wide = C.c_uint32()
    assert L.mv_draw_cameras(None, envs, views, 1, 128, 72, 1, 1, *[C.byref(x) for x in p], C.byref(wide)) == capi.MV_ERR_ARG
    assert L.mv_draw_cameras(None, None, None, 0, 128, 72, 0, 0, None, None, None, None) == capi.MV_ERR_ARG
    ctr = C.c_void_p()
    assert L.mv_draw_cameras_device(None, envs, views, 1, 128, 72, views, None, None, C.byref(ctr)) == capi.MV_ERR_ARG
    assert L.mv_draw_cameras_device(None, None, None, 0, 128, 72, None, None, None, None) == capi.MV_ERR_ARG
    assert L.mv_views_device(None, C.byref(ctr)) == capi.MV_ERR_ARG
    out = (C.c_float * 6)()
    assert L.mv_level_bounds(None, out) == capi.MV_ERR_ARG
    words = (C.c_uint32 * 8)()
    assert L.mv_debug_view_order(None, words, 8) == capi.MV_ERR_ARG


def test_camera_exports_and_signatures(built):
    from megaverse_b200 import capi
    from megaverse_b200.extension.megaverse import MegaverseGym
    from megaverse_b200.megaverse_env import MegaverseEnv

    assert set(NEW) <= set(capi.EXPORTS)
    for name in NEW:
        assert hasattr(capi.lib(), name)
    params = inspect.signature(capi.Engine.draw_cameras).parameters
    assert list(params) == ["self", "envs", "views16", "w", "h", "depth", "seg"]
    assert params["depth"].default is False and params["seg"].default is False
    assert "views" in capi.Engine.device_array.__doc__
    for name in ("draw_cameras", "get_views", "level_bounds"):
        assert getattr(MegaverseGym, name).__doc__, name
    for name, args in (("render_cameras", ["self", "envs", "views", "w", "h"]), ("overview", ["self", "envs", "w", "h"]),
                       ("chase", ["self", "agents", "w", "h"])):
        sig = inspect.signature(getattr(MegaverseEnv, name)).parameters
        assert list(sig) == args, name
        assert sig["w"].default == 768 and sig["h"].default == 432, name
    # render() keeps its signature
    assert list(inspect.signature(MegaverseEnv.render).parameters) == ["self", "mode"]


def test_projection_matches_the_engine_constants():
    from megaverse_b200 import cameras

    p00, p11, p22, p32 = cameras.projection(128, 72)
    assert all(isinstance(x, np.float32) for x in (p00, p11, p22, p32))
    assert abs(float(p00) - 1.0 / math.tan(math.radians(50.0))) < 1e-6
    assert abs(float(p11) + (128.0 / 72.0) / math.tan(math.radians(50.0))) < 1e-5
    assert float(p22) < 0 and float(p32) < 0


def test_look_at_is_rigid_and_maps_the_eye_to_the_origin():
    from megaverse_b200 import cameras

    rng = np.random.default_rng(3)
    for _ in range(200):
        eye = rng.uniform(-50, 50, 3)
        target = eye + rng.normal(size=3) * rng.uniform(0.5, 30)
        v = cameras.look_at(eye, target)
        assert v.dtype == np.float32 and v.shape == (16,)
        _check_rigid(v, eye)
        # the target lies on the camera's -z axis
        t = _matrix(v) @ np.append(target, 1.0)
        assert abs(t[0]) < 1e-3 and abs(t[1]) < 1e-3 and t[2] < 0
    with pytest.raises(ValueError):
        cameras.look_at((0, 0, 0), (0, 5, 0))


def test_chase_views_with_no_offset_equal_the_agent_views():
    from megaverse_b200 import cameras

    rng = np.random.default_rng(7)
    agent = np.stack([cameras.look_at(rng.uniform(-20, 20, 3), rng.uniform(-20, 20, 3)) for _ in range(16)])
    same = cameras.chase_views(agent, back=0.0, up=0.0, pitch=0.0)
    assert same.dtype == np.float32 and same.shape == agent.shape
    assert (same == agent).all()


def test_chase_views_are_rigid_and_sit_behind_and_above_the_agent():
    from megaverse_b200 import cameras

    rng = np.random.default_rng(8)
    for _ in range(50):
        eye = rng.uniform(-20, 20, 3)
        agent = cameras.look_at(eye, eye + np.array([rng.normal(), 0.2 * rng.normal(), rng.normal()]))
        ch = cameras.chase_views(agent[None], back=3.0, up=1.5, pitch=0.35)[0]
        a = _matrix(agent)
        chase_eye = np.linalg.inv(a) @ np.array([0.0, 1.5, 3.0, 1.0])  # (0, up, back) in the agent's camera frame
        _check_rigid(ch, chase_eye[:3])
        # the agent's eye is in front of the chase camera, below its axis
        p = _matrix(ch) @ np.append(eye, 1.0)
        assert p[2] < 0 and p[1] < 0


def _corners(b):
    return np.array([[b[0 + 3 * i], b[1 + 3 * j], b[2 + 3 * k]] for i in (0, 1) for j in (0, 1) for k in (0, 1)], dtype=np.float64)


@pytest.mark.parametrize("w,h", [(768, 432), (256, 144), (128, 72), (128, 128), (64, 256)])
def test_overview_frames_every_corner(w, h):
    from megaverse_b200 import cameras

    p00, p11, p22, p32 = (float(x) for x in cameras.projection(w, h))
    rng = np.random.default_rng(w * 1000 + h)
    boxes = [np.array([0, 0, 0, 40, 6, 40]), np.array([-3, -1, -3, 3, 12, 3]), np.array([0, 0, 0, 1, 0.05, 1])]
    for _ in range(100):
        lo = rng.uniform(-30, 30, 3)
        boxes.append(np.concatenate([lo, lo + rng.uniform(0.1, 40, 3)]))
    views = cameras.overview_views(np.stack(boxes), w, h)
    assert views.dtype == np.float32 and views.shape == (len(boxes), 16)
    for b, v in zip(boxes, views):
        m = _matrix(v)
        centre = 0.5 * (b[:3] + b[3:])
        c = m @ np.append(centre, 1.0)
        assert abs(c[0]) < 1e-3 and c[2] < 0, "the overview does not look at the box's centre"
        for corner in _corners(b):
            x, y, z, _ = m @ np.append(corner, 1.0)
            cw = -z
            assert cw > cameras.NEAR and cw < cameras.FAR, "a corner is outside the depth range"
            assert abs(p00 * x / cw) <= 1.0 and abs(p11 * y / cw) <= 1.0, "a corner projects outside the frame"
        rot = m[:3, :3]
        assert np.allclose(rot @ rot.T, np.eye(3), atol=1e-6)
        fwd = -rot[2]  # the camera's viewing direction in world space
        assert fwd[1] < -0.5, "the overview is not pitched down"
