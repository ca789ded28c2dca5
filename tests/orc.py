"""ctypes wrapper over the ORACLE (oracle/liborc.so).  Test infrastructure only -- never imported by the product."""
import ctypes as C
import os
import subprocess
import numpy as np

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        path = os.path.join(_ROOT, "oracle", "liborc.so")
        if not os.path.exists(path):
            subprocess.check_call(["make", "-C", os.path.join(_ROOT, "oracle"), "oracle"])
        L = C.CDLL(path)
        L.orc_create.restype = C.c_void_p
        L.orc_create.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_float), C.c_int]
        for name in ("orc_obs", "orc_depth", "orc_rewards", "orc_dones", "orc_true_objectives"):
            getattr(L, name).restype = C.c_void_p
            getattr(L, name).argtypes = [C.c_void_p]
        for name in ("orc_destroy", "orc_reset", "orc_step", "orc_render_now"):
            getattr(L, name).argtypes = [C.c_void_p]
            getattr(L, name).restype = None
        L.orc_set_options.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
        L.orc_seed.argtypes = [C.c_void_p, C.c_int]
        L.orc_seed_env.argtypes = [C.c_void_p, C.c_int, C.c_int]
        L.orc_set_actions.argtypes = [C.c_void_p, C.c_void_p]
        L.orc_get_level.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int]
        L.orc_get_state.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int]
        L.orc_get_voxels.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int]
        L.orc_get_instances.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int]
        L.orc_get_view.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        L.orc_render_instances.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        L.orc_get_mesh.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int]
        L.orc_get_reward_shaping.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_char_p, C.POINTER(C.c_float)]
        L.orc_set_reward_shaping.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_char_p, C.c_float]
        L.orc_kcc_case.argtypes = [C.c_void_p] * 4 + [C.c_int, C.c_void_p, C.c_void_p]
        L.orc_kcc_case.restype = None
        _LIB = L
    return _LIB


class Oracle:
    def __init__(self, scenario, num_envs, num_agents, w=128, h=72, params=None, render=True, depth=False, threads=1):
        L = lib()
        params = params or {}
        keys = (C.c_char_p * max(1, len(params)))(*[k.encode() for k in params])
        vals = (C.c_float * max(1, len(params)))(*[float(v) for v in params.values()])
        self.h_ = L.orc_create(scenario.encode(), w, h, num_envs, num_agents, keys, vals, len(params))
        if not self.h_:
            raise ValueError("oracle: unknown scenario %r" % scenario)
        self.E, self.A, self.N, self.w, self.h = num_envs, num_agents, num_envs * num_agents, w, h
        L.orc_set_options(self.h_, int(render), int(depth), threads)

    def close(self):
        if self.h_:
            lib().orc_destroy(self.h_)
            self.h_ = None

    def seed(self, s):
        lib().orc_seed(self.h_, s)

    def seed_env(self, e, s):
        lib().orc_seed_env(self.h_, e, s)

    def reset(self):
        lib().orc_reset(self.h_)

    def step(self, masks):
        m = np.ascontiguousarray(masks, dtype=np.int32)
        assert m.size == self.N
        lib().orc_set_actions(self.h_, m.ctypes.data)
        lib().orc_step(self.h_)

    def _arr(self, fn, shape, dtype):
        ptr = getattr(lib(), fn)(self.h_)
        n = int(np.prod(shape))
        buf = (C.c_char * (n * np.dtype(dtype).itemsize)).from_address(ptr)
        return np.frombuffer(buf, dtype=dtype).reshape(shape).copy()

    def obs(self):
        return self._arr("orc_obs", (self.N, self.h, self.w, 4), np.uint8)

    def depth(self):
        return self._arr("orc_depth", (self.N, self.h, self.w), np.float32)

    def rewards(self):
        return self._arr("orc_rewards", (self.N,), np.float32)

    def dones(self):
        return self._arr("orc_dones", (self.E,), np.uint8)

    def true_objectives(self):
        return self._arr("orc_true_objectives", (self.N,), np.float32)

    def _dump(self, fn, env, dtype, cap=1 << 16):
        out = np.zeros(cap, dtype=dtype)
        n = getattr(lib(), fn)(self.h_, env, out.ctypes.data, cap)
        if n < 0:
            return self._dump(fn, env, dtype, -n)
        return out[:n].copy()

    def level(self, env):
        return self._dump("orc_get_level", env, np.int32)

    def state(self, env):
        return self._dump("orc_get_state", env, np.float32)

    def arrangement(self, env):
        return self._dump("orc_get_arrangement", env, np.int32)

    def voxels(self, env):
        return self._dump("orc_get_voxels", env, np.int32).reshape(-1, 4)

    def instances(self, env):
        return self._dump("orc_get_instances", env, np.float32).reshape(-1, 18)

    def view(self, env, agent):
        out = np.zeros(16, dtype=np.float32)
        lib().orc_get_view(self.h_, env, agent, out.ctypes.data)
        return out


def render_instances(view16, inst18, w, h, want_depth=False):
    view16 = np.ascontiguousarray(view16, dtype=np.float32)
    inst18 = np.ascontiguousarray(inst18, dtype=np.float32).reshape(-1, 18)
    rgba = np.zeros((h, w, 4), dtype=np.uint8)
    depth = np.zeros((h, w), dtype=np.float32)
    lib().orc_render_instances(view16.ctypes.data, inst18.ctypes.data, inst18.shape[0], w, h, rgba.ctypes.data, depth.ctypes.data if want_depth else None)
    return (rgba, depth) if want_depth else rgba


def kcc_cases(hdr, boxes, agents, query):
    """the oracle's convexSweep / recoverFromPenetration / KCC::playerStep over mv_debug_kcc's case layouts, every collider a candidate:
    (out_i int32[n, 8], out_f float32[n, 16]) as capi.kcc_cases returns them"""
    hdr = np.ascontiguousarray(hdr, dtype=np.int32)
    boxes = np.ascontiguousarray(boxes, dtype=np.float32)
    agents = np.ascontiguousarray(agents, dtype=np.float32)
    query = np.ascontiguousarray(query, dtype=np.float32)
    n = hdr.shape[0]
    assert boxes.shape == (n, 256, 10) and agents.shape == (n, 8, 3) and query.shape == (n, 20)
    out_i = np.zeros((n, 8), dtype=np.int32)
    out_f = np.zeros((n, 16), dtype=np.float32)
    lib().orc_kcc_case(hdr.ctypes.data, boxes.ctypes.data, agents.ctypes.data, query.ctypes.data, n, out_i.ctypes.data, out_f.ctypes.data)
    return out_i, out_f


def mesh(type_):
    vtx = np.zeros(128 * 6, dtype=np.uint32)
    idx = np.zeros(512, dtype=np.uint16)
    r = lib().orc_get_mesh(type_, vtx.ctypes.data, vtx.size, idx.ctypes.data, idx.size)
    nv, ni = r >> 16, r & 0xFFFF
    return vtx[: nv * 6].reshape(nv, 6).copy(), idx[:ni].copy()


def encode_actions(actions6):
    """MegaverseGym::setActions (megaverse.cpp:100-116): 6-tuple -> bit mask."""
    sizes = [3, 3, 3, 2, 2, 3]
    mask, idx = 0, 0
    for a, sz in zip(actions6, sizes):
        if a > 0:
            mask |= 1 << (idx + int(a))
        idx += sz - 1
    return mask
