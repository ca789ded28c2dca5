"""What each engine call launches and times, the raster grid cap on every delivery path, and where the options allocate.

- mv_kernel_launches per call: a step is the step kernel and one raster launch per slice of the delivery, plus the terminal-frame launch
  with option final_obs; mv_reset and mv_reset_envs the same without it; a state save its copy kernel; a load the copy kernel and the
  re-render; mv_draw_hires one launch.
- mv_last_kernel_ms / mv_last_final_ms as the header documents them for each call, with option overlap 0 and 1.
- Option raster_grid bounds every raster launch, the sliced download's and the hi-res pass's included, and frames do not depend on it.
- Options that allocate do so on the engine's device, whatever device the calling thread has current."""
import ctypes as C
import threading

import numpy as np
import pytest

import helpers

pytestmark = pytest.mark.gpu

E, A = 8, 2


def _engine(seed=5, depth=False, **options):
    from megaverse_b200 import capi

    g = capi.Engine("Collect", E, A, 128, 72, num_threads=2, depth=depth)
    for k, v in options.items():
        g.set_option(k, v)
    g.seed(seed)
    return g


def _delta(g, call):
    n0 = g.kernel_launches()
    call()
    return g.kernel_launches() - n0


@pytest.mark.parametrize("overlap", [0, 1])
@pytest.mark.parametrize("sliced", [False, True], ids=["zero_copy", "slices4"])
def test_launches_and_kernel_times(overlap, sliced):
    import torch

    opts = {"overlap": overlap, "final_obs": 1}
    if sliced:
        opts.update(zero_copy=0, host_slices=4)
    g = _engine(**opts)
    try:
        raster = 4 if sliced else 1  # raster launches of a host-facing delivery: E = 8 envs in four slices of two
        rng = np.random.default_rng(3)
        acts = lambda t: helpers.purposeful_actions(rng, E * A, t).astype(np.int32)

        def times_split():  # both kernels timed on their own
            k, r = g.last_kernel_ms()
            assert k > 0 and r > 0, (k, r)

        assert _delta(g, g.reset) == 1 + raster
        k, r = g.last_kernel_ms()
        assert (k == -1.0 and r > 0) if overlap else (k > 0 and r > 0), (k, r)
        assert g.last_final_ms() == 0.0

        for t in range(3):
            assert _delta(g, lambda: g.step(acts(t))) == 1 + raster + 1
            k, r = g.last_kernel_ms()
            assert (k == -1.0 and r > 0) if overlap else (k > 0 and r > 0), (k, r)
            assert g.last_final_ms() > 0

        assert _delta(g, lambda: (g.step_begin(acts(3)), g.step_end())) == 1 + raster + 1
        k, r = g.last_kernel_ms()
        assert (k == -1.0 and r > 0) if overlap else (k > 0 and r > 0), (k, r)
        assert g.last_final_ms() > 0

        store = g.states_create(2)
        assert _delta(g, lambda: g.states_save(store, [0, 5], [0, 1])) == 1
        k, r = g.last_kernel_ms()
        assert k > 0 and r == 0.0, (k, r)

        assert _delta(g, lambda: g.states_load(store, [1, 0], [2, 5])) == 1 + raster
        times_split()

        assert _delta(g, lambda: g.reset_envs([1, 3])) == 1 + raster
        times_split()
        assert _delta(g, lambda: g.reset_envs([4], seeds=[11])) == 1 + raster
        times_split()

        assert _delta(g, lambda: g.draw_hires(256, 144)) == 1

        g.step(acts(4))  # a timed step right before the asynchronous ones
        before = g.last_kernel_ms()
        ends = torch.zeros(E, dtype=torch.uint8, device="cuda")
        ends[0] = 1  # env 0 has played five steps of its episode: the request is honoured
        torch.cuda.synchronize()
        # the asynchronous call draws into HBM in one launch whatever the host-facing delivery
        assert _delta(g, lambda: g.step_device(None, ends.data_ptr())) == 3
        g.sync()
        assert g.dones()[0] == 1
        if overlap:  # no events: the kernel times are still the last timed call's, and there is no terminal-frame time
            assert g.last_kernel_ms() == before
            assert g.last_final_ms() == 0.0
        else:
            times_split()
            assert g.last_final_ms() > 0
        assert _delta(g, lambda: g.step_device()) == 3
        g.sync()
        assert g.fault_word() == 0 and g.faults() == 0
    finally:
        g.close()


def test_raster_grid_cap_slices_and_hires():
    """a grid of 3 CTAs against the full grid, with the sliced download and the hi-res pass: the same bytes at every step"""
    ga = _engine(depth=True, zero_copy=0, host_slices=4)
    gb = _engine(depth=True, zero_copy=0, host_slices=4, raster_grid=3)
    try:
        rng = np.random.default_rng(9)
        for g in (ga, gb):
            g.reset()
        for t in range(12):
            a = helpers.purposeful_actions(rng, E * A, t).astype(np.int32)
            for g in (ga, gb):
                g.step(a)
            assert np.array_equal(ga.obs(), gb.obs()), "step %d: obs differ" % t
            assert np.array_equal(ga.depth().view(np.uint32), gb.depth().view(np.uint32)), "step %d: depth differs" % t
            assert np.array_equal(ga.rewards(), gb.rewards()) and np.array_equal(ga.dones(), gb.dones())
            if t % 4 == 0:
                assert np.array_equal(ga.draw_hires(768, 432), gb.draw_hires(768, 432)), "step %d: hi-res frames differ" % t
    finally:
        ga.close()
        gb.close()


def _device_of(ptr):
    cu = C.CDLL("libcuda.so.1")
    assert cu.cuInit(0) == 0
    dev = C.c_int(-1)
    assert cu.cuPointerGetAttribute(C.byref(dev), 9, C.c_uint64(ptr)) == 0  # CU_POINTER_ATTRIBUTE_DEVICE_ORDINAL
    return dev.value


def test_options_allocate_on_the_engine_device():
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from megaverse_b200 import capi

    found = {}

    def body():  # a new thread: its current device is 0
        try:
            g = capi.Engine("Collect", 4, 1, 128, 72, device=1)
            try:
                for k, v in (("depth", 1), ("segmentation", 1), ("level_slots", 4), ("static_cap", 64), ("tri_cap", 200)):
                    g.set_option(k, v)
                found["depth"] = _device_of(g.device_ptr("depth"))
                found["segmentation"] = _device_of(g.device_ptr("segmentation"))
            finally:
                g.close()
        except Exception as ex:  # reported by the assertion below
            found["error"] = repr(ex)

    th = threading.Thread(target=body)
    th.start()
    th.join()
    assert found == {"depth": 1, "segmentation": 1}
