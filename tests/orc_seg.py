"""Segmentation on the oracle (test infrastructure only): tests/oracle_seg/orc_seg.cpp, built on first use into a temporary directory
with the compiler and flags of oracle/Makefile, applied to an orc.Oracle's current scenes."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_SRC = os.path.join(_HERE, "oracle_seg", "orc_seg.cpp")
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        oracle = os.path.join(_ROOT, "oracle")
        deps = [_SRC] + sorted(os.path.join(oracle, f) for f in os.listdir(oracle) if f.endswith((".hpp", ".cpp", ".inc")))
        h = hashlib.sha256()
        for d in deps:
            with open(d, "rb") as f:
                h.update(f.read())
        path = os.path.join(tempfile.gettempdir(), "megaverse_orc_seg_%s.so" % h.hexdigest()[:16])
        if not os.path.exists(path):
            tmp = "%s.%d.tmp" % (path, os.getpid())
            # oracle/Makefile's compiler (make's CXX: the environment's, else g++) and flags: OrcVec must have liborc.so's layout
            subprocess.check_call([os.environ.get("CXX", "g++"), "-std=c++17", "-O2", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-pthread",
                                   "-shared", "-o", tmp, _SRC])
            os.replace(tmp, path)
        L = C.CDLL(path)
        L.orc_seg_render.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.orc_seg_render.restype = C.c_int
        _LIB = L
    return _LIB


def segmentation(o):
    """(seg uint16[N,h,w], depth float32[N,h,w]) of the oracle's current scenes: class << 8 | index of the scene object whose fragment wins
    each pixel (0 where nothing was drawn), and the depth of that fragment, which equals what the oracle's renderView draws"""
    seg = np.zeros((o.N, o.h, o.w), dtype=np.uint16)
    depth = np.zeros((o.N, o.h, o.w), dtype=np.float32)
    if lib().orc_seg_render(o.h_, seg.ctypes.data, depth.ctypes.data) != 0:
        raise RuntimeError("oracle segmentation: a scene object could not be tagged")
    return seg, depth
