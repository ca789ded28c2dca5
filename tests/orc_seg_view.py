"""Segmentation on the oracle through an arbitrary view matrix (test infrastructure only): tests/oracle_seg/orc_seg_view.cpp, built on first
use into a temporary directory with the compiler and flags of oracle/Makefile, applied to one env of an orc.Oracle's current scenes."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_SRC = os.path.join(_HERE, "oracle_seg", "orc_seg_view.cpp")
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
        path = os.path.join(tempfile.gettempdir(), "megaverse_orc_seg_view_%s.so" % h.hexdigest()[:16])
        if not os.path.exists(path):
            tmp = "%s.%d.tmp" % (path, os.getpid())
            subprocess.check_call([os.environ.get("CXX", "g++"), "-std=c++17", "-O2", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-pthread",
                                   "-shared", "-o", tmp, _SRC])
            os.replace(tmp, path)
        L = C.CDLL(path)
        L.orc_seg_render_view.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        L.orc_seg_render_view.restype = C.c_int
        _LIB = L
    return _LIB


def segmentation_view(o, env, view16, w, h):
    """(seg uint16[h,w], depth float32[h,w]) of env `env` of the oracle's current scenes through view16: class << 8 | index of the scene
    object whose fragment wins each pixel (0 where nothing was drawn), and that fragment's depth"""
    v = np.ascontiguousarray(view16, dtype=np.float32).reshape(16)
    seg = np.zeros((h, w), dtype=np.uint16)
    depth = np.zeros((h, w), dtype=np.float32)
    if lib().orc_seg_render_view(o.h_, int(env), v.ctypes.data, int(w), int(h), seg.ctypes.data, depth.ctypes.data) != 0:
        raise RuntimeError("oracle segmentation: a scene object could not be tagged")
    return seg, depth
