"""Pose helpers for the spectator cameras (mv_draw_cameras): view matrices in the engine's convention, pure numpy float32.

A view matrix maps world coordinates to camera coordinates: the camera looks down -z with +y up, as an agent's eye does.  The engine
stores it as 16 float32 in column-major order (the translation in elements 12..14), which is what these helpers return and what
`Engine.draw_cameras` and `mv_draw_cameras` take.  Every frame is drawn with the agents' projection at its size: a 100 degree horizontal
field of view, near plane 0.01, far plane 120."""
import math

import numpy as np

HFOV_DEG = 100.0
NEAR, FAR = 0.01, 120.0


def projection(w, h):
    """(p00, p11, p22, p32) of the engine's projection at w x h (fillConsts in csrc/engine.cu): clip x = p00 * x, clip y = p11 * y (y is
    flipped: rows run downwards), clip z = p22 * z + p32, clip w = -z"""
    half_tan = np.float32(math.tan(math.radians(HFOV_DEG) / 2.0))
    aspect = np.float32(w) / np.float32(h)
    p00 = np.float32(1.0) / half_tan
    p11 = -aspect / half_tan
    p22 = np.float32(FAR) / (np.float32(NEAR) - np.float32(FAR))
    p32 = np.float32(FAR) * np.float32(NEAR) / (np.float32(NEAR) - np.float32(FAR))
    return p00, p11, p22, p32


def _column_major(m4):
    return np.ascontiguousarray(np.asarray(m4, dtype=np.float64).T.reshape(16), dtype=np.float32)


def _matrix(v16):
    return np.asarray(v16, dtype=np.float64).reshape(4, 4).T


def look_at(eye, target, up=(0.0, 1.0, 0.0)):
    """float32[16]: the view matrix of a camera at `eye` looking at `target`, with `up` as close to its +y as the direction allows"""
    eye, target, up = (np.asarray(v, dtype=np.float64).reshape(3) for v in (eye, target, up))
    f = target - eye
    f /= np.linalg.norm(f)
    s = np.cross(f, up)
    if np.linalg.norm(s) < 1e-9:
        raise ValueError("look_at: the view direction is parallel to up")
    s /= np.linalg.norm(s)
    u = np.cross(s, f)
    m = np.eye(4)
    m[0, :3], m[1, :3], m[2, :3] = s, u, -f
    m[:3, 3] = -(m[:3, :3] @ eye)
    return _column_major(m)


def overview_views(bounds, w=768, h=432, pitch_deg=60.0, margin=1.05):
    """float32[E,16]: for each row {min xyz, max xyz} of `bounds` (mv_level_bounds), a camera above and in front of the box's centre,
    looking at it pitched down by pitch_deg, just far enough back that all eight corners project inside the w x h frame (with `margin` to
    spare) under the engine's projection.  A box too large for the far plane at that distance (the hex mazes at 16:9) gets the farthest
    distance that keeps the box's centre at half the far plane: its outer parts then lie beyond the frame or the far plane."""
    b = np.asarray(bounds, dtype=np.float64).reshape(-1, 6)
    p00, p11 = (abs(float(x)) for x in projection(w, h)[:2])
    pitch = math.radians(pitch_deg)
    back = np.array([0.0, math.sin(pitch), math.cos(pitch)])  # from the centre towards the eye
    up = (0.0, 1.0, 0.0) if abs(math.cos(pitch)) > 1e-6 else (0.0, 0.0, -1.0)
    rot = _matrix(look_at(back, (0.0, 0.0, 0.0), up))[:3, :3]  # the camera's orientation (rows: its axes in world space)
    out = np.zeros((b.shape[0], 16), dtype=np.float32)
    for i, row in enumerate(b):
        centre = 0.5 * (row[:3] + row[3:])
        corners = np.array([[row[3 * a], row[1 + 3 * c], row[2 + 3 * d]] for a in (0, 1) for c in (0, 1) for d in (0, 1)]) - centre
        x, y, z = (rot @ corners.T)  # camera-space offsets from the centre; the centre itself sits at depth `dist`
        # a corner's clip w is dist - z: inside the frame when |p00 x| and |p11 y| stay below w / margin, in front of the near plane
        dist = float(np.max(np.maximum(margin * p00 * np.abs(x), margin * p11 * np.abs(y)) + z))
        dist = max(dist, float(np.max(z)) + 2.0 * NEAR, 1.0)
        dist = min(dist, 0.5 * FAR)
        out[i] = look_at(centre + back * dist, centre, up)
    return out


def chase_views(agent_views, back=3.0, up=1.5, pitch=0.35):
    """float32[n,16]: a camera `back` units behind and `up` units above each agent's eye, pitched down by `pitch` radians, both in the
    agent's own camera frame -- the agent's view matrix left-multiplied by that camera-space rigid transform, so no state is needed.
    With back = up = pitch = 0 the result equals the agent's own matrix."""
    v = np.asarray(agent_views, dtype=np.float32).reshape(-1, 16)
    c, s = math.cos(pitch), math.sin(pitch)
    rot = np.array([[1.0, 0.0, 0.0, 0.0], [0.0, c, -s, 0.0], [0.0, s, c, 0.0], [0.0, 0.0, 0.0, 1.0]])  # the inverse of the camera's pitch-down
    shift = np.eye(4)
    shift[:3, 3] = [0.0, -up, -back]  # the chase eye sits at (0, up, back) in the agent's camera frame
    t = rot @ shift
    out = np.zeros_like(v)
    for i, row in enumerate(v):
        out[i] = _column_major(t @ _matrix(row))
    return out
