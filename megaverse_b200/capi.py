"""ctypes binding of the C ABI (include/megaverse_b200.h).  This is the reference-side stub INTEGRATION.md describes: what a
maintainer would bind from Python if they did not want the pybind11 module.  It loads the in-tree libmegaverse_b200.so and
fails loudly when the library or a CUDA device is missing -- there is no CPU fallback in the product."""
import ctypes as C
import os

import numpy as np

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("MV_B200_LIB") or os.path.join(_PKG, "libmegaverse_b200.so")  # the override is for kernel-variant experiments (tools/)
_lib = None

MV_OK, MV_ERR_ARG, MV_ERR_CUDA, MV_ERR_CAPACITY, MV_ERR_STATE = 0, -1, -2, -3, -4
MV_END_NONE, MV_END_TIME, MV_END_SOLVED, MV_END_REQUESTED = 0, 1, 2, 3  # done_reasons(): why an episode ended
# segmentation(): a pixel is class << 8 | index of the drawable behind it, 0 where nothing was drawn
MV_SEG_NONE, MV_SEG_STATIC, MV_SEG_TERRAIN, MV_SEG_OBJECT, MV_SEG_AGENT, MV_SEG_REWARD = 0, 1, 2, 3, 4, 5
MAX_OBJECTS, MAX_AGENTS, MAX_CAND = 128, 8, 96  # MV_MAX_OBJECTS, MV_MAX_AGENTS, MV_MAX_CAND (csrc/mv_types.h)
MV_FAULT_ENVELOPE, MV_FAULT_CAND_OVERFLOW = 16, 32


class MegaverseError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("megaverse_b200 error %d: %s" % (code, msg))
        self.code = code


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError("%s is missing: run `python -m megaverse_b200._build` (needs nvcc)" % LIB_PATH)
        L = C.CDLL(LIB_PATH)
        vp, ci, cf = C.c_void_p, C.c_int, C.c_float
        L.mv_create.argtypes = [C.c_char_p, ci, ci, ci, ci, ci, ci, C.POINTER(C.c_char_p), C.POINTER(cf), ci, C.POINTER(vp)]
        L.mv_create_mixed.argtypes = [C.POINTER(C.c_char_p), ci, ci, ci, ci, ci, ci, C.POINTER(C.c_char_p), C.POINTER(cf), ci, C.POINTER(vp)]
        L.mv_last_error.argtypes = [vp]
        L.mv_last_error.restype = C.c_char_p
        for name in ("mv_reset", "mv_step", "mv_step_begin", "mv_step_end", "mv_close", "mv_sync", "mv_fetch_obs"):
            getattr(L, name).argtypes = [vp]
        L.mv_seed.argtypes = [vp, ci]
        L.mv_seed_env.argtypes = [vp, ci, ci]
        L.mv_set_actions.argtypes = [vp, vp]
        L.mv_encode_action.argtypes = [vp]
        L.mv_step_device.argtypes = [vp, vp]
        L.mv_step_device_ends.argtypes = [vp, vp, vp]
        L.mv_step_device_active.argtypes = [vp, vp, vp, vp]
        L.mv_step_envs.argtypes = [vp, vp, ci]
        L.mv_reset_envs.argtypes = [vp, vp, vp, ci]
        for name in ("mv_obs_host", "mv_depth_host", "mv_rewards", "mv_dones", "mv_true_objectives", "mv_actions_device", "mv_obs_device",
                     "mv_depth_device", "mv_rewards_device", "mv_dones_device", "mv_stream", "mv_done_reasons", "mv_done_reasons_device",
                     "mv_true_objectives_device", "mv_final_obs_host", "mv_final_depth_host", "mv_final_obs_device", "mv_final_depth_device",
                     "mv_segmentation_host", "mv_segmentation_device", "mv_level_ids", "mv_level_ids_device", "mv_next_levels_device",
                     "mv_views_device"):
            getattr(L, name).argtypes = [vp, C.POINTER(vp)]
        L.mv_get_reward_shaping.argtypes = [vp, ci, ci, C.POINTER(C.c_char_p), C.POINTER(cf), ci, C.POINTER(ci)]
        L.mv_set_reward_shaping.argtypes = [vp, ci, ci, C.POINTER(C.c_char_p), C.POINTER(cf), ci]
        L.mv_set_option.argtypes = [vp, C.c_char_p, ci]
        L.mv_faults.argtypes = [vp, C.POINTER(C.c_int32)]
        L.mv_kernel_launches.argtypes = [vp, C.POINTER(C.c_int64)]
        L.mv_last_kernel_ms.argtypes = [vp, C.POINTER(cf)]
        L.mv_last_final_ms.argtypes = [vp, C.POINTER(cf)]
        L.mv_last_rays_ms.argtypes = [vp, C.POINTER(cf)]
        L.mv_set_rays.argtypes = [vp, vp, ci, cf]
        for name in ("mv_rays_host", "mv_rays_device", "mv_final_rays_host", "mv_final_rays_device"):
            getattr(L, name).argtypes = [vp, C.POINTER(vp), C.POINTER(vp)]
        for name in ("mv_debug_get_level", "mv_debug_get_state", "mv_debug_get_voxels", "mv_debug_get_instances"):
            getattr(L, name).argtypes = [vp, ci, vp, ci]
        L.mv_debug_get_view.argtypes = [vp, ci, ci, vp]
        L.mv_debug_warp_agent.argtypes = [vp, ci, ci, vp, vp]
        L.mv_debug_render_instances.argtypes = [vp, vp, ci, ci, ci, vp, vp]
        L.mv_debug_render_instances_ex.argtypes = [vp, vp, ci, ci, ci, vp, vp, vp, vp, vp]
        L.mv_debug_cast_rays.argtypes = [vp, vp, vp, vp, ci, ci, ci, vp, ci, cf, vp, vp, vp]
        L.mv_debug_kcc.argtypes = [vp, vp, vp, vp, ci, vp, vp]
        L.mv_debug_bzset.argtypes = [vp, ci, vp, ci]
        L.mv_debug_generate_level.argtypes = [C.c_char_p, ci, ci, ci, C.POINTER(C.c_char_p), C.POINTER(cf), ci, vp, ci]
        L.mv_states_create.argtypes = [vp, ci, C.POINTER(ci)]
        L.mv_states_save.argtypes = [vp, ci, vp, vp, ci]
        L.mv_states_load.argtypes = [vp, ci, vp, vp, ci]
        L.mv_states_destroy.argtypes = [vp, ci]
        L.mv_state_row_bytes.argtypes = [vp, C.POINTER(C.c_int64)]
        L.mv_set_next_levels.argtypes = [vp, vp, vp, ci]
        L.mv_level_set_pick.argtypes = [C.c_uint32, C.c_int32, C.c_int32]
        L.mv_level_set_pick.restype = C.c_uint32
        for name in ("mv_state_tensors_host", "mv_state_tensors_device", "mv_final_state_tensors_host", "mv_final_state_tensors_device"):
            getattr(L, name).argtypes = [vp] + [C.POINTER(vp)] * 4
        L.mv_draw_cameras.argtypes = [vp, vp, vp, ci, ci, ci, ci, ci, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.POINTER(C.c_uint32)]
        L.mv_draw_cameras_device.argtypes = [vp, vp, vp, ci, ci, ci, vp, vp, vp, C.POINTER(vp)]
        L.mv_level_bounds.argtypes = [vp, vp]
        L.mv_debug_view_order.argtypes = [vp, vp, ci]
        _lib = L
    return _lib


EXPORTS = [
    "mv_create", "mv_create_mixed", "mv_last_error", "mv_seed", "mv_seed_env", "mv_reset", "mv_set_actions", "mv_encode_action", "mv_step", "mv_step_begin", "mv_step_end", "mv_obs_host", "mv_depth_host",
    "mv_rewards", "mv_dones", "mv_true_objectives", "mv_get_reward_shaping", "mv_set_reward_shaping", "mv_set_option", "mv_step_device", "mv_set_obs_buffer",
    "mv_sync", "mv_fetch_obs", "mv_draw_hires", "mv_actions_device", "mv_obs_device", "mv_depth_device", "mv_rewards_device", "mv_dones_device", "mv_stream", "mv_faults", "mv_fault_word", "mv_kernel_launches",
    "mv_last_kernel_ms", "mv_close", "mv_debug_get_level", "mv_debug_get_state", "mv_debug_get_voxels", "mv_debug_get_instances", "mv_debug_get_view", "mv_debug_warp_agent",
    "mv_debug_render_instances", "mv_debug_render_instances_ex", "mv_debug_step_profile", "mv_debug_raster_config", "mv_debug_static_cap", "mv_debug_raster_stats", "mv_debug_color_tables", "mv_debug_defaults", "mv_debug_count_unfit_levels", "mv_levels_skipped", "mv_debug_bzset", "mv_debug_generate_level",
    "mv_states_create", "mv_states_save", "mv_states_load", "mv_states_destroy", "mv_state_row_bytes", "mv_step_device_ends", "mv_reset_envs",
    "mv_done_reasons", "mv_done_reasons_device", "mv_true_objectives_device", "mv_final_obs_host", "mv_final_depth_host", "mv_final_obs_device",
    "mv_final_depth_device", "mv_last_final_ms", "mv_segmentation_host", "mv_segmentation_device", "mv_step_envs", "mv_step_device_active",
    "mv_level_ids", "mv_level_ids_device", "mv_next_levels_device", "mv_set_next_levels", "mv_level_set_pick",
    "mv_state_tensors_host", "mv_state_tensors_device", "mv_final_state_tensors_host", "mv_final_state_tensors_device",
    "mv_draw_cameras", "mv_draw_cameras_device", "mv_views_device", "mv_level_bounds", "mv_debug_view_order",
    "mv_set_rays", "mv_rays_host", "mv_rays_device", "mv_final_rays_host", "mv_final_rays_device", "mv_last_rays_ms", "mv_debug_cast_rays",
    "mv_debug_kcc",
]

STATE_TENSORS = ("agents", "envs", "objects", "rewards")  # the state tensors' order in the C calls (include/megaverse_b200.h)


class CameraFrames(tuple):
    """what Engine.draw_cameras returns: (obs uint8[n,h,w,4], depth float32[n,h,w] or None, seg uint16[n,h,w] or None, out_of_range)"""
    __slots__ = ()

    def __new__(cls, obs, depth, seg, out_of_range):
        return tuple.__new__(cls, (obs, depth, seg, out_of_range))

    obs = property(lambda self: self[0])
    depth = property(lambda self: self[1])
    seg = property(lambda self: self[2])
    out_of_range = property(lambda self: self[3])


class Engine:
    """Thin object wrapper: one method per C entry point, numpy views over engine-owned host memory."""

    def __init__(self, scenario, num_envs, num_agents, w=128, h=72, num_threads=1, device=0, params=None, depth=False, segmentation=False):
        """scenario: one name for every env, or a list of num_envs names (env e runs scenario[e]: mv_create_mixed)"""
        L = lib()
        params = params or {}
        keys = (C.c_char_p * max(1, len(params)))(*[k.encode() for k in params])
        vals = (C.c_float * max(1, len(params)))(*[float(v) for v in params.values()])
        self._h = C.c_void_p()
        if isinstance(scenario, str):
            rc = L.mv_create(scenario.encode(), w, h, num_envs, num_agents, num_threads, device, keys, vals, len(params), C.byref(self._h))
        else:
            names = list(scenario)
            if len(names) != num_envs:
                raise MegaverseError(MV_ERR_ARG, "%d scenario names for %d envs" % (len(names), num_envs))
            arr = (C.c_char_p * max(1, num_envs))(*[n.encode() for n in names])
            rc = L.mv_create_mixed(arr, w, h, num_envs, num_agents, num_threads, device, keys, vals, len(params), C.byref(self._h))
        if rc != MV_OK:
            raise MegaverseError(rc, (L.mv_last_error(None) or b"").decode())
        self.E, self.A, self.N, self.w, self.h = num_envs, num_agents, num_envs * num_agents, w, h
        self.num_rays = 0  # set_rays
        if depth:
            self._ck(L.mv_set_option(self._h, b"depth", 1))
        if segmentation:
            self._ck(L.mv_set_option(self._h, b"segmentation", 1))

    def _ck(self, rc):
        if rc != MV_OK:
            raise MegaverseError(rc, (lib().mv_last_error(self._h) or b"").decode())

    def close(self):
        if self._h:
            lib().mv_close(self._h)
            self._h = C.c_void_p()

    def set_option(self, key, value):
        self._ck(lib().mv_set_option(self._h, key.encode(), int(value)))

    def seed(self, s):
        self._ck(lib().mv_seed(self._h, int(s)))

    def seed_env(self, e, s):
        self._ck(lib().mv_seed_env(self._h, int(e), int(s)))

    def reset(self):
        self._ck(lib().mv_reset(self._h))

    def step(self, masks):
        m = np.ascontiguousarray(masks, dtype=np.int32)
        assert m.size == self.N
        self._ck(lib().mv_set_actions(self._h, m.ctypes.data))
        self._ck(lib().mv_step(self._h))

    def step_begin(self, masks):
        """first half of step(): upload the masks, enqueue kernels and device->host copies, return at once"""
        m = np.ascontiguousarray(masks, dtype=np.int32)
        assert m.size == self.N
        self._ck(lib().mv_set_actions(self._h, m.ctypes.data))
        self._ck(lib().mv_step_begin(self._h))

    def step_end(self):
        """second half: wait; obs() / rewards() / dones() are then valid as after step()"""
        self._ck(lib().mv_step_end(self._h))

    def step_device(self, d_masks_ptr=None, d_ends_ptr=None):
        """d_ends_ptr: optional device uint8[E]; a non-zero entry ends that env's episode at this step (mv_step_device_ends)"""
        m = C.c_void_p(d_masks_ptr) if d_masks_ptr else None
        if d_ends_ptr is None:
            self._ck(lib().mv_step_device(self._h, m))
        else:
            self._ck(lib().mv_step_device_ends(self._h, m, C.c_void_p(d_ends_ptr) if d_ends_ptr else None))

    def step_envs(self, masks, envs):
        """step() of the listed envs only (mv_step_envs): the others run nothing, report reward 0 and not done, and keep their frames;
        masks covers every agent, the entries of unlisted envs are ignored"""
        m = np.ascontiguousarray(masks, dtype=np.int32)
        assert m.size == self.N
        e = np.ascontiguousarray(envs, dtype=np.int32)
        self._ck(lib().mv_set_actions(self._h, m.ctypes.data))
        self._ck(lib().mv_step_envs(self._h, e.ctypes.data if e.size else None, e.size))

    def step_device_active(self, d_masks_ptr, d_ends_ptr, d_active_ptr):
        """step_device() of the envs whose byte of the device uint8[E] at d_active_ptr is non-zero (mv_step_device_active); a 0 / None
        pointer is the engine's own actions, no end requests, every env active"""
        p = [C.c_void_p(x) if x else None for x in (d_masks_ptr, d_ends_ptr, d_active_ptr)]
        self._ck(lib().mv_step_device_active(self._h, *p))

    def reset_envs(self, envs, seeds=None):
        """envs[i] start a new episode now; with seeds, env envs[i] is reseeded with seeds[i] first (mv_reset_envs).  With option level_set,
        set_next_levels(envs, levels) before it chooses the levels they start on."""
        e = np.ascontiguousarray(envs, dtype=np.int32)
        s = None if seeds is None else np.ascontiguousarray(seeds, dtype=np.int32)
        assert s is None or s.size == e.size
        self._ck(lib().mv_reset_envs(self._h, e.ctypes.data if e.size else None, None if s is None else s.ctypes.data, e.size))

    def set_obs_buffer(self, d_obs_ptr=None, d_depth_ptr=None):
        """rasterise into caller-owned device memory (a slice of a larger tensor) instead of the engine's own obs buffer"""
        lib().mv_set_obs_buffer.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        self._ck(lib().mv_set_obs_buffer(self._h, C.c_void_p(d_obs_ptr) if d_obs_ptr else None, C.c_void_p(d_depth_ptr) if d_depth_ptr else None))

    def sync(self):
        self._ck(lib().mv_sync(self._h))

    def draw_hires(self, w, h):
        """uint8[N,h,w,4] view of the engine's hi-res frame (valid until the next draw_hires)"""
        p = C.c_void_p()
        lib().mv_draw_hires.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_void_p)]
        self._ck(lib().mv_draw_hires(self._h, int(w), int(h), C.byref(p)))
        n = self.N * h * w * 4
        return np.frombuffer((C.c_char * n).from_address(p.value), dtype=np.uint8).reshape(self.N, h, w, 4)

    def draw_cameras(self, envs, views16, w, h, depth=False, seg=False):
        """spectator cameras (mv_draw_cameras): camera c draws env envs[c] through the view matrix views16[c] (16 float32, column-major;
        megaverse_b200.cameras builds them) at w x h from the last step's scene.  Returns CameraFrames(obs uint8[n,h,w,4], depth float32[n,h,w]
        or None, seg uint16[n,h,w] or None, out_of_range): copies, plus the number of triangles whose window coordinates left the range the
        rasteriser is exact in (0 means every pixel is exact)."""
        e = np.ascontiguousarray(envs, dtype=np.int32).reshape(-1)
        v = np.ascontiguousarray(views16, dtype=np.float32).reshape(-1)
        assert v.size == 16 * e.size
        n = e.size
        po, pd, ps, wide = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_uint32()
        self._ck(lib().mv_draw_cameras(self._h, e.ctypes.data if n else None, v.ctypes.data if n else None, n, int(w), int(h), int(bool(depth)),
                                       int(bool(seg)), C.byref(po), C.byref(pd), C.byref(ps), C.byref(wide)))

        def grab(ptr, shape, dtype):
            size = int(np.prod(shape)) * np.dtype(dtype).itemsize
            if size == 0:
                return np.zeros(shape, dtype=dtype)
            return np.frombuffer((C.c_char * size).from_address(ptr.value), dtype=dtype).reshape(shape).copy()

        obs = grab(po, (n, h, w, 4), np.uint8)
        dep = grab(pd, (n, h, w), np.float32) if depth else None
        sg = grab(ps, (n, h, w), np.uint16) if seg else None
        return CameraFrames(obs, dep, sg, int(wide.value))

    def draw_cameras_device(self, d_envs_ptr, d_views_ptr, n, w, h, d_obs_ptr, d_depth_ptr=None, d_seg_ptr=None):
        """asynchronous spectator cameras (mv_draw_cameras_device) on the engine stream: device int32[n] env table, float32[n,16] views and
        the caller's output buffers (uint8[n,h,w,4], optional float32[n,h,w] depth and uint16[n,h,w] segmentation).  An env outside
        [0, E) gives an all-zero frame.  Returns the device address of the engine's uint32 out-of-range counter of this launch."""
        p = [C.c_void_p(x) if x else None for x in (d_envs_ptr, d_views_ptr, d_obs_ptr, d_depth_ptr, d_seg_ptr)]
        ctr = C.c_void_p()
        self._ck(lib().mv_draw_cameras_device(self._h, p[0], p[1], int(n), int(w), int(h), p[2], p[3], p[4], C.byref(ctr)))
        return ctr.value

    def level_bounds(self):
        """float32[E,6]: {min x, y, z, max x, y, z} of each env's live level (mv_level_bounds), valid after host-facing calls and sync()"""
        out = np.zeros((self.E, 6), dtype=np.float32)
        self._ck(lib().mv_level_bounds(self._h, out.ctypes.data))
        return out

    def device_array(self, what="obs"):
        """zero-copy handle on an engine-owned device tensor for any consumer of the CUDA array interface
        (`torch.as_tensor(eng.device_array("obs"), device="cuda")`, CuPy, Numba): "obs" uint8[N,h,w,4], "depth" float32[N,h,w],
        "rewards" float32[N], "dones" uint8[E], "done_reasons" uint8[E] (MV_END_*), "true_objectives" float32[N], with option final_obs
        "final_obs" uint8[N,h,w,4] / "final_depth" float32[N,h,w] (terminal frames of mv_step_device steps), and with option segmentation
        "segmentation" uint16[N,h,w] (MV_SEG_* << 8 | index), with option state_tensors "state_agents" float32[N,16], "state_envs"
        float32[E,16], "state_objects" / "state_rewards" float32[E,128,4] and, with option final_obs too, the terminal rows "final_state_agents",
        ... (state_tensors()), and with option level_set "level_ids" int32[E] (the level each env is on) and
        "next_levels" int32[E] (writable: the level an env plays next, -1 = the engine picks; write it on the engine's stream), and "views"
        float32[N,16] (the last step's view matrices, column-major: chase cameras on the device), and with rays (set_rays) "rays_dist"
        float32[N,R] / "rays_tag" uint16[N,R] and, with option final_obs too, "final_rays_dist" / "final_rays_tag".  Valid in the engine
        stream's order (mv_stream) until mv_close."""
        frame, px = (self.N, self.h, self.w, 4), (self.N, self.h, self.w)
        shapes = {"obs": (frame, "|u1"), "depth": (px, "<f4"), "rewards": ((self.N,), "<f4"), "dones": ((self.E,), "|u1"),
                  "done_reasons": ((self.E,), "|u1"), "true_objectives": ((self.N,), "<f4"), "final_obs": (frame, "|u1"), "final_depth": (px, "<f4"),
                  "segmentation": (px, "<u2"), "level_ids": ((self.E,), "<i4"), "next_levels": ((self.E,), "<i4"), "views": ((self.N, 16), "<f4")}
        for prefix in ("state_", "final_state_"):
            for k, shp in self._state_shapes().items():
                shapes[prefix + k] = (shp, "<f4")
        for prefix in ("", "final_"):
            shapes[prefix + "rays_dist"] = ((self.N, self.num_rays), "<f4")
            shapes[prefix + "rays_tag"] = ((self.N, self.num_rays), "<u2")
        shape, typestr = shapes[what]
        if what.endswith(("rays_dist", "rays_tag")):
            ptr = self._ray_ptrs("mv_%srays_device" % ("final_" if what.startswith("final_") else ""))[0 if what.endswith("dist") else 1]
        elif what.startswith(("state_", "final_state_")):
            ptr = self._state_ptrs("mv_%s_tensors_device" % what.rsplit("_", 1)[0])[what.rsplit("_", 1)[1]]
        else:
            ptr = self.device_ptr(what)
        stream = self.stream()

        class _DeviceArray:
            __cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (ptr, False), "version": 3, "strides": None, "stream": stream or 1}

        return _DeviceArray()

    def fetch_obs(self):
        self._ck(lib().mv_fetch_obs(self._h))

    def _host(self, fn, shape, dtype):
        p = C.c_void_p()
        self._ck(getattr(lib(), fn)(self._h, C.byref(p)))
        n = int(np.prod(shape)) * np.dtype(dtype).itemsize
        return np.frombuffer((C.c_char * n).from_address(p.value), dtype=dtype).reshape(shape)

    def obs(self):
        """uint8[N,h,w,4]: a VIEW of engine memory, valid until the next step (megaverse.cpp:139-143)"""
        return self._host("mv_obs_host", (self.N, self.h, self.w, 4), np.uint8)

    def depth(self):
        return self._host("mv_depth_host", (self.N, self.h, self.w), np.float32)

    def segmentation(self):
        """uint16[N,h,w] (option segmentation): MV_SEG_* class << 8 | index of the drawable behind each pixel, 0 where nothing was drawn"""
        return self._host("mv_segmentation_host", (self.N, self.h, self.w), np.uint16)

    def rewards(self):
        return self._host("mv_rewards", (self.N,), np.float32)

    def dones(self):
        return self._host("mv_dones", (self.E,), np.uint8)

    def true_objectives(self):
        return self._host("mv_true_objectives", (self.N,), np.float32)

    def done_reasons(self):
        """uint8[E] MV_END_* of the last step: 0 not done, 1 time limit, 2 solved, 3 requested"""
        return self._host("mv_done_reasons", (self.E,), np.uint8)

    def level_ids(self):
        """int32[E] (option level_set): the level of the set each env is on after the last call; for an env that just ended, the new episode's"""
        return self._host("mv_level_ids", (self.E,), np.int32)

    def set_next_levels(self, envs, levels):
        """(option level_set) env envs[i] plays level levels[i] of the set in its next episode, once (mv_set_next_levels).  Followed by
        reset_envs(envs) it starts those envs on those levels now."""
        e, lv = np.ascontiguousarray(envs, dtype=np.int32), np.ascontiguousarray(levels, dtype=np.int32)
        assert e.size == lv.size
        self._ck(lib().mv_set_next_levels(self._h, e.ctypes.data if e.size else None, lv.ctypes.data if lv.size else None, e.size))

    def _state_shapes(self):
        return {"agents": (self.N, 16), "envs": (self.E, 16), "objects": (self.E, 128, 4), "rewards": (self.E, 128, 4)}

    def _state_ptrs(self, fn):
        p = [C.c_void_p() for _ in STATE_TENSORS]
        self._ck(getattr(lib(), fn)(self._h, *[C.byref(x) for x in p]))
        return {k: x.value for k, x in zip(STATE_TENSORS, p)}

    def _state_views(self, fn):
        shapes = self._state_shapes()
        out = {}
        for k, ptr in self._state_ptrs(fn).items():
            n = int(np.prod(shapes[k])) * 4
            out[k] = np.frombuffer((C.c_char * n).from_address(ptr), dtype=np.float32).reshape(shapes[k])
        return out

    def state_tensors(self):
        """option state_tensors: {"agents": float32[N,16], "envs": float32[E,16], "objects": float32[E,128,4], "rewards": float32[E,128,4]},
        views of the engine's pinned rows after the last host-facing call (or mv_fetch_obs); the layout is in include/megaverse_b200.h"""
        return self._state_views("mv_state_tensors_host")

    def final_state_tensors(self):
        """options state_tensors and final_obs: the same dict of terminal rows, the state each env's last episode ended on"""
        return self._state_views("mv_final_state_tensors_host")

    def set_rays(self, directions, max_distance):
        """ray sensors (mv_set_rays, before the first reset): directions float32[R,3] in camera space (x right, y up, -z forward; rays.fan /
        rays.ring build them), R in 0..MV_MAX_RAYS (0 turns them off); a hit distance counts multiples of a direction's length"""
        d = np.ascontiguousarray(directions, dtype=np.float32).reshape(-1, 3)
        self._ck(lib().mv_set_rays(self._h, d.ctypes.data if len(d) else None, len(d), float(max_distance)))
        self.num_rays = len(d)

    def _ray_ptrs(self, fn):
        dist, tag = C.c_void_p(), C.c_void_p()
        self._ck(getattr(lib(), fn)(self._h, C.byref(dist), C.byref(tag)))
        return dist.value, tag.value

    def _ray_views(self, fn):
        dist, tag = self._ray_ptrs(fn)
        n = self.N * self.num_rays
        return (np.frombuffer((C.c_char * (n * 4)).from_address(dist), dtype=np.float32).reshape(self.N, self.num_rays),
                np.frombuffer((C.c_char * (n * 2)).from_address(tag), dtype=np.uint16).reshape(self.N, self.num_rays))

    def rays(self):
        """(dist float32[N,R], tag uint16[N,R]) of the rays set by set_rays: views of the engine's pinned arrays after the last host-facing
        call (or fetch_obs).  Ray r of view env*A + agent: the distance to the first front face it meets (0: none within the maximum) and
        that drawable's MV_SEG_* class << 8 | index (0: none)"""
        return self._ray_views("mv_rays_host")

    def final_rays(self):
        """rays and option final_obs: the same pair cast from the terminal rows, the scene each env's last episode ended on"""
        return self._ray_views("mv_final_rays_host")

    def last_rays_ms(self):
        out = C.c_float()
        self._ck(lib().mv_last_rays_ms(self._h, C.byref(out)))
        return out.value

    def final_obs(self):
        """uint8[N,h,w,4] terminal frames (option final_obs): views of env e hold the frame its last episode ended on"""
        return self._host("mv_final_obs_host", (self.N, self.h, self.w, 4), np.uint8)

    def final_depth(self):
        return self._host("mv_final_depth_host", (self.N, self.h, self.w), np.float32)

    def device_ptr(self, what):
        p = C.c_void_p()
        self._ck(getattr(lib(), "mv_%s_device" % what)(self._h, C.byref(p)))
        return p.value

    def stream(self):
        p = C.c_void_p()
        self._ck(lib().mv_stream(self._h, C.byref(p)))
        return p.value

    def get_reward_shaping(self, env, agent):
        keys = (C.c_char_p * 32)()
        vals = (C.c_float * 32)()
        n = C.c_int()
        self._ck(lib().mv_get_reward_shaping(self._h, env, agent, keys, vals, 32, C.byref(n)))
        return {keys[i].decode(): float(vals[i]) for i in range(n.value)}

    def set_reward_shaping(self, env, agent, rs):
        keys = (C.c_char_p * max(1, len(rs)))(*[k.encode() for k in rs])
        vals = (C.c_float * max(1, len(rs)))(*[float(v) for v in rs.values()])
        self._ck(lib().mv_set_reward_shaping(self._h, env, agent, keys, vals, len(rs)))

    def faults(self):
        f = C.c_int32()
        self._ck(lib().mv_faults(self._h, C.byref(f)))
        return f.value

    def fault_word(self):
        """the latched fault bits without a device round trip (mv_fault_word)"""
        f = C.c_int32()
        lib().mv_fault_word.argtypes = [C.c_void_p, C.POINTER(C.c_int32)]
        self._ck(lib().mv_fault_word(self._h, C.byref(f)))
        return f.value

    def kernel_launches(self):
        n = C.c_int64()
        self._ck(lib().mv_kernel_launches(self._h, C.byref(n)))
        return n.value

    def step_profile(self, enable=True, read=True):
        out = np.zeros((self.E, 16), dtype=np.uint32)
        lib().mv_debug_step_profile.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        self._ck(lib().mv_debug_step_profile(self._h, out.ctypes.data if read else None, 1 if enable else 0))
        return out

    def static_cap(self):
        lib().mv_debug_static_cap.argtypes = [C.c_void_p]
        return int(lib().mv_debug_static_cap(self._h))

    def raster_config(self):
        out = (C.c_int32 * 4)()
        lib().mv_debug_raster_config.argtypes = [C.c_void_p, C.c_void_p]
        self._ck(lib().mv_debug_raster_config(self._h, out))
        return {"grid": out[0], "ctas_per_sm": out[1], "smem": out[2], "bands": out[3]}

    def raster_stats(self, enable=True, read=True):
        out = (C.c_ulonglong * 16)()
        lib().mv_debug_raster_stats.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        self._ck(lib().mv_debug_raster_stats(self._h, out if read else None, 1 if enable else 0))
        names = ["work_items", "instances", "visible_instances", "items", "clipped_items", "triangles", "batches", "sub_passes", "cyc_head", "cyc_tma_wait", "cyc_instance", "cyc_item", "cyc_tile", "cyc_total"]
        return {n: int(out[i]) for i, n in enumerate(names)}

    # ---- env state store (mv_states_*)
    def states_create(self, rows):
        sid = C.c_int()
        self._ck(lib().mv_states_create(self._h, int(rows), C.byref(sid)))
        return sid.value

    def states_save(self, store, envs, rows):
        """env envs[i] -> row rows[i] of the store"""
        e, r = np.ascontiguousarray(envs, dtype=np.int32), np.ascontiguousarray(rows, dtype=np.int32)
        assert e.size == r.size
        self._ck(lib().mv_states_save(self._h, int(store), e.ctypes.data, r.ctypes.data, e.size))

    def states_load(self, store, rows, envs):
        """row rows[i] of the store -> env envs[i]; obs() / rewards() / dones() then read as after the saved step"""
        r, e = np.ascontiguousarray(rows, dtype=np.int32), np.ascontiguousarray(envs, dtype=np.int32)
        assert e.size == r.size
        self._ck(lib().mv_states_load(self._h, int(store), r.ctypes.data, e.ctypes.data, e.size))

    def states_destroy(self, store):
        self._ck(lib().mv_states_destroy(self._h, int(store)))

    def state_row_bytes(self):
        n = C.c_int64()
        self._ck(lib().mv_state_row_bytes(self._h, C.byref(n)))
        return n.value

    def last_kernel_ms(self):
        out = (C.c_float * 2)()
        self._ck(lib().mv_last_kernel_ms(self._h, out))
        return float(out[0]), float(out[1])

    def last_final_ms(self):
        """device time of the last step's terminal-frame launch (mv_last_final_ms)"""
        out = C.c_float()
        self._ck(lib().mv_last_final_ms(self._h, C.byref(out)))
        return float(out.value)

    # ---- introspection (tests)
    def _dump(self, fn, env, dtype, cap=1 << 16):
        out = np.zeros(cap, dtype=dtype)
        n = getattr(lib(), fn)(self._h, env, out.ctypes.data, cap)
        if n < -8:
            return self._dump(fn, env, dtype, -n)
        if n < 0:
            self._ck(n)
        return out[:n].copy()

    def level(self, env):
        return self._dump("mv_debug_get_level", env, np.int32)

    def state(self, env):
        return self._dump("mv_debug_get_state", env, np.float32)

    def voxels(self, env):
        return self._dump("mv_debug_get_voxels", env, np.int32).reshape(-1, 4)

    def instances(self, env):
        return self._dump("mv_debug_get_instances", env, np.float32).reshape(-1, 18)

    def view(self, env, agent):
        out = np.zeros(16, dtype=np.float32)
        self._ck(lib().mv_debug_get_view(self._h, env, agent, out.ctypes.data))
        return out

    def view_order(self):
        """uint32 words of the cost-ordered raster queue (mv_debug_view_order): item costs, the next launch's env order, the exit counter"""
        out = np.zeros(self.N * (self.h // 4) + self.E + 1, dtype=np.uint32)
        n = lib().mv_debug_view_order(self._h, out.ctypes.data, out.size)
        if n < 0:
            self._ck(n)
        return out[:n].copy()

    def warp_agent(self, env, agent, pos, basis):
        """test hook (mv_debug_warp_agent): set the agent's position and basis rows, zero its velocities; drawn by the next step"""
        p = np.ascontiguousarray(pos, dtype=np.float32)
        b = np.ascontiguousarray(basis, dtype=np.float32)
        assert p.size == 3 and b.size == 9
        self._ck(lib().mv_debug_warp_agent(self._h, int(env), int(agent), p.ctypes.data, b.ctypes.data))


def render_instances(view16, inst18, w, h, want_depth=False, fast=None, segmentation=False, tri_cap=None, bands=None, stats=False):
    """debug: draw caller-supplied instances (18 floats each) with one view through the CUDA rasteriser.  Without the keyword options this
    is mv_debug_render_instances (exact shading, tri_cap 96, one or two bands); any of them selects mv_debug_render_instances_ex with
    fast (0/1), segmentation, tri_cap (0 = engine default) and bands (0 = the hi-res rule).  Returns rgba, then depth (want_depth), the
    uint16 segmentation image (instance i drawn with tag i + 1) and the kernel's 16 counters (stats), those asked for, in that order."""
    view16 = np.ascontiguousarray(view16, dtype=np.float32)
    inst18 = np.ascontiguousarray(inst18, dtype=np.float32).reshape(-1, 18)
    rgba = np.zeros((h, w, 4), dtype=np.uint8)
    depth = np.zeros((h, w), dtype=np.float32)
    out = [rgba] + ([depth] if want_depth else [])
    if fast is None and not segmentation and tri_cap is None and bands is None and not stats:
        rc = lib().mv_debug_render_instances(view16.ctypes.data, inst18.ctypes.data, inst18.shape[0], w, h, rgba.ctypes.data, depth.ctypes.data if want_depth else None)
        if rc != MV_OK:
            raise MegaverseError(rc, "mv_debug_render_instances failed")
    else:
        opts = np.array([int(bool(fast)), int(bool(segmentation)), int(tri_cap or 0), int(bands or 0)], dtype=np.int32)
        seg = np.zeros((h, w), dtype=np.uint16)
        st = np.zeros(16, dtype=np.uint64)
        rc = lib().mv_debug_render_instances_ex(view16.ctypes.data, inst18.ctypes.data, inst18.shape[0], w, h, opts.ctypes.data, rgba.ctypes.data,
                                                depth.ctypes.data if want_depth else None, seg.ctypes.data if segmentation else None,
                                                st.ctypes.data if stats else None)
        if rc != MV_OK:
            raise MegaverseError(rc, "mv_debug_render_instances_ex failed")
        out += ([seg] if segmentation else []) + ([st] if stats else [])
    return tuple(out) if len(out) > 1 else rgba


def cast_rays(views, inst18, tags, counts, dirs, max_dist, env_mask=None, dist=None, tag=None):
    """debug: cast rays over caller-supplied scenes through the engine's ray launch (mv_debug_cast_rays).  views float32[E, A, 16],
    inst18 float32[E, stride, 18], tags int32[E, stride], counts int32[E], dirs float32[R, 3]; env_mask uint8[E] or None.  dist / tag
    (float32 / uint16 [E * A, R]) are what the launch starts from (zeros when None): rows of envs the mask leaves out come back as given.
    Returns (dist, tag)."""
    views = np.ascontiguousarray(views, dtype=np.float32)
    E, A = views.shape[0], views.shape[1]
    views = views.reshape(E * A, 16)
    inst18 = np.ascontiguousarray(inst18, dtype=np.float32)
    stride = inst18.shape[1]
    tags = np.ascontiguousarray(tags, dtype=np.int32)
    counts = np.ascontiguousarray(counts, dtype=np.int32)
    dirs = np.ascontiguousarray(dirs, dtype=np.float32).reshape(-1, 3)
    assert inst18.shape == (E, stride, 18) and tags.shape == (E, stride) and counts.shape == (E,)
    R = dirs.shape[0]
    dist = np.zeros((E * A, R), dtype=np.float32) if dist is None else np.array(dist, dtype=np.float32).reshape(E * A, R)
    tag = np.zeros((E * A, R), dtype=np.uint16) if tag is None else np.array(tag, dtype=np.uint16).reshape(E * A, R)
    mask = None if env_mask is None else np.ascontiguousarray(env_mask, dtype=np.uint8).reshape(E)
    rc = lib().mv_debug_cast_rays(views.ctypes.data, inst18.ctypes.data, tags.ctypes.data, counts.ctypes.data, E, A, stride, dirs.ctypes.data, R,
                                  float(max_dist), None if mask is None else mask.ctypes.data, dist.ctypes.data, tag.ctypes.data)
    if rc != MV_OK:
        raise MegaverseError(rc, "mv_debug_cast_rays failed")
    return dist, tag


def kcc_cases(hdr, boxes, agents, query):
    """debug: contact cases through the step kernel's candidate gather, sweep, recovery and controller step (mv_debug_kcc).  hdr int32[n, 8],
    boxes float32[n, 2 * MAX_OBJECTS, 10], agents float32[n, MAX_AGENTS, 3], query float32[n, 20] in the layouts the header documents.
    Returns (out_i int32[n, 8], out_f float32[n, 16])."""
    hdr = np.ascontiguousarray(hdr, dtype=np.int32)
    n = hdr.shape[0]
    boxes = np.ascontiguousarray(boxes, dtype=np.float32)
    agents = np.ascontiguousarray(agents, dtype=np.float32)
    query = np.ascontiguousarray(query, dtype=np.float32)
    assert hdr.shape == (n, 8) and boxes.shape == (n, 2 * MAX_OBJECTS, 10) and agents.shape == (n, MAX_AGENTS, 3) and query.shape == (n, 20)
    out_i = np.zeros((n, 8), dtype=np.int32)
    out_f = np.zeros((n, 16), dtype=np.float32)
    rc = lib().mv_debug_kcc(hdr.ctypes.data, boxes.ctypes.data, agents.ctypes.data, query.ctypes.data, n, out_i.ctypes.data, out_f.ctypes.data)
    if rc != MV_OK:
        raise MegaverseError(rc, "mv_debug_kcc failed")
    return out_i, out_f


def generate_level(scenario, num_agents, env_seed, episode, params=None):
    """host-only level generation (no CUDA): int32 dump of episode `episode` of the env stream seeded with env_seed"""
    params = params or {}
    keys = (C.c_char_p * max(1, len(params)))(*[k.encode() for k in params])
    vals = (C.c_float * max(1, len(params)))(*[float(v) for v in params.values()])
    out = np.zeros(1 << 14, dtype=np.int32)
    n = lib().mv_debug_generate_level(scenario.encode(), num_agents, env_seed, episode, keys, vals, len(params), out.ctypes.data, out.size)
    if n < 0:
        raise MegaverseError(n, "mv_debug_generate_level failed")
    return out[:n].copy()


def level_set_pick(pick_seed, episode, count):
    """host-only: the level of a set of `count` an env with this pick seed plays in episode `episode` when nobody names one (mv_level_set_pick)"""
    return int(lib().mv_level_set_pick(int(pick_seed) & 0xFFFFFFFF, int(episode), int(count)))


def bzset_order(ops):
    ops = np.ascontiguousarray(ops, dtype=np.int32).reshape(-1, 4)
    out = np.zeros(3 * 256, dtype=np.int32)
    n = lib().mv_debug_bzset(ops.ctypes.data, ops.shape[0], out.ctypes.data, out.size)
    return out[: n * 3].reshape(n, 3).copy()


def encode_action(heads6):
    a = np.ascontiguousarray(heads6, dtype=np.int32)
    return int(lib().mv_encode_action(a.ctypes.data))
