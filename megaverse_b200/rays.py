"""Direction helpers for the ray sensors (mv_set_rays): unit float32[n, 3] directions in camera space, pure numpy.

Camera space is the frame of an agent's view matrix: x right, y up, -z forward.  A direction at yaw a (radians, positive to the right)
and pitch p (positive up) is (sin a cos p, sin p, -cos a cos p).  Each is computed in float64 and rounded once to float32."""
import math

import numpy as np


def _directions(yaw, pitch):
    yaw, pitch = np.asarray(yaw, dtype=np.float64), np.asarray(pitch, dtype=np.float64)
    cp = np.cos(pitch)
    d = np.stack([np.sin(yaw) * cp, np.sin(pitch) * np.ones_like(yaw), -np.cos(yaw) * cp], axis=-1)
    return np.ascontiguousarray(d, dtype=np.float32).reshape(-1, 3)


def fan(n, hfov_deg, pitch_deg=0.0):
    """float32[n, 3]: n rays spread evenly over a horizontal fan of hfov_deg degrees centred on forward, left to right (yaw
    -hfov/2 .. +hfov/2; a single ray points forward), all at pitch_deg degrees (positive up)"""
    n = int(n)
    if n < 1:
        raise ValueError("fan: n must be at least 1")
    t = np.linspace(-0.5, 0.5, n) if n > 1 else np.zeros(1)
    return _directions(math.radians(float(hfov_deg)) * t, np.full(n, math.radians(float(pitch_deg))))


def ring(n, pitch_deg=0.0):
    """float32[n, 3]: n rays spread evenly all the way round, starting forward and turning right (yaw 360 * i / n degrees), all at
    pitch_deg degrees (positive up)"""
    n = int(n)
    if n < 1:
        raise ValueError("ring: n must be at least 1")
    return _directions(2.0 * math.pi * np.arange(n) / n, np.full(n, math.radians(float(pitch_deg))))
