"""Ray sensors on the oracle (test infrastructure only): tests/oracle_seg/orc_rays.cpp, built on first use into a temporary directory with
the compiler and flags of oracle/Makefile, applied to one env of an orc.Oracle's current scenes or to a hand-built instance list."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_SRC = os.path.join(_HERE, "oracle_seg", "orc_rays.cpp")
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        oracle = os.path.join(_ROOT, "oracle")
        deps = [_SRC, os.path.join(_HERE, "oracle_seg", "orc_seg.cpp")]
        deps += sorted(os.path.join(oracle, f) for f in os.listdir(oracle) if f.endswith((".hpp", ".cpp", ".inc")))
        h = hashlib.sha256()
        for d in deps:
            with open(d, "rb") as f:
                h.update(f.read())
        path = os.path.join(tempfile.gettempdir(), "megaverse_orc_rays_%s.so" % h.hexdigest()[:16])
        if not os.path.exists(path):
            tmp = "%s.%d.tmp" % (path, os.getpid())
            subprocess.check_call([os.environ.get("CXX", "g++"), "-std=c++17", "-O2", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-pthread",
                                   "-shared", "-o", tmp, _SRC])
            os.replace(tmp, path)
        L = C.CDLL(path)
        vp, ci = C.c_void_p, C.c_int
        L.orc_rays_env.argtypes = [vp, ci, ci, vp, vp, ci, C.c_float, vp, vp]
        L.orc_rays_env.restype = ci
        L.orc_rays_scene.argtypes = [vp, vp, vp, ci, ci, vp, ci, C.c_float, vp, vp]
        L.orc_rays_scene.restype = None
        _LIB = L
    return _LIB


def _dirs(dirs):
    return np.ascontiguousarray(dirs, dtype=np.float32).reshape(-1, 3)


def rays_env(o, env, agent, dirs, max_dist, view16=None):
    """(dist float32[R], tag uint16[R]) of agent `agent` of env `env` of the oracle's current scenes, cast from the oracle's own view of
    that agent (or from view16), against the oracle's tagged instances"""
    d = _dirs(dirs)
    dist = np.zeros(len(d), dtype=np.float32)
    tag = np.zeros(len(d), dtype=np.uint16)
    v = None if view16 is None else np.ascontiguousarray(view16, dtype=np.float32).reshape(16)
    if lib().orc_rays_env(o.h_, int(env), int(agent), None if v is None else v.ctypes.data, d.ctypes.data, len(d), float(max_dist),
                          dist.ctypes.data, tag.ctypes.data) != 0:
        raise RuntimeError("oracle rays: bad env or agent, or a scene object could not be tagged")
    return dist, tag


def rays_all(o, dirs, max_dist):
    """(dist float32[N, R], tag uint16[N, R]) for every view env*A + agent of the oracle's current scenes"""
    out = [rays_env(o, e, a, dirs, max_dist) for e in range(o.E) for a in range(o.A)]
    return np.stack([d for d, _ in out]), np.stack([t for _, t in out])


def rays_scene(view16, inst18, tags, dirs, max_dist, agent=-1):
    """(dist float32[R], tag uint16[R]) against a hand-built list: inst18 rows (mesh, colour, column-major model), one tag per row; agent
    -1 ignores no drawable, else the drawables tagged MV_SEG_AGENT << 8 | agent are the caster's own"""
    d = _dirs(dirs)
    inst = np.ascontiguousarray(inst18, dtype=np.float32).reshape(-1, 18)
    t = np.ascontiguousarray(tags, dtype=np.int32).reshape(-1)
    assert len(t) == len(inst)
    v = np.ascontiguousarray(view16, dtype=np.float32).reshape(16)
    dist = np.zeros(len(d), dtype=np.float32)
    tag = np.zeros(len(d), dtype=np.uint16)
    lib().orc_rays_scene(v.ctypes.data, inst.ctypes.data, t.ctypes.data, len(inst), int(agent), d.ctypes.data, len(d), float(max_dist),
                         dist.ctypes.data, tag.ctypes.data)
    return dist, tag
