"""Engine lifetime: closing an engine releases everything it holds, whatever it was used for -- device arrays, pinned mirrors, state
stores, events, streams and worker threads -- also while asynchronous steps are in flight or a level replacement is still being
generated.  Each cycle creates an engine of a few hundred MB, turns on every option and output that allocates, uses it and closes it."""
import gc
import os
import subprocess

import numpy as np
import pytest

import helpers

pytestmark = pytest.mark.gpu

SCENARIO, E, W, H = "HexExplore", 512, 128, 128  # HexExplore levels need hundreds of static boxes: static_cap 16 makes them grow the arrays
L = 16                                            # level-set engines: bank rows
FRAME = E * W * H * 4                             # one obs tensor: 33.5 MB.  An engine holds ~0.6 GB of HBM and ~0.36 GB of pinned memory
WARMUP, CYCLES = 4, 6
TOLERANCE = 3 * FRAME                             # a leaked obs tensor or mirror adds 2 * TOLERANCE over CYCLES
# One level worker per pool: every worker thread allocates from a malloc arena of its own, and with eight of them a new pool per cycle
# leaves the arenas growing by tens of MB over the first dozens of cycles (fragmentation, freed but held), which would mask a leak.  With
# one, the process's RSS still settles over the first few cycles: hence WARMUP
THREADS = 1


def _cycle(level_set):
    """one engine from create to close.  A level-slot engine is closed with two asynchronous steps in flight, a level-set engine with one
    in flight and a replacement requested just before (its worker may still be generating the level)"""
    import torch

    from megaverse_b200 import capi, rays

    rng = np.random.default_rng(1)
    g = capi.Engine(SCENARIO, E, 1, W, H, num_threads=THREADS, depth=True, segmentation=True)
    for k, v in (("final_obs", 1), ("state_tensors", 1), ("static_cap", 16)):
        g.set_option(k, v)
    if level_set:
        g.set_option("level_set_seed", 100)
        g.set_option("level_set", L)
    g.set_rays(rays.fan(8, 90.0), 20.0)
    g.raster_stats(enable=True, read=False)
    g.step_profile(enable=True, read=False)
    g.seed(5)
    g.reset()
    assert g.static_cap() > 16, "the first levels are meant to grow the static-box arrays"
    for t in range(3):
        g.step(helpers.purposeful_actions(rng, E, t))
    d_acts = torch.from_numpy(helpers.purposeful_actions(rng, E, 3)).cuda()
    for _ in range(3):
        g.step_device(d_acts.data_ptr())
    g.fetch_obs()

    # state stores: one destroyed here, one still alive at close
    envs = np.arange(E, dtype=np.int32)
    kept, dropped = g.states_create(E), g.states_create(E)
    g.states_save(dropped, envs, envs)
    g.step(helpers.purposeful_actions(rng, E, 4))
    g.states_load(dropped, envs, envs)
    g.states_destroy(dropped)
    g.states_save(kept, envs, envs)

    # spectator cameras, host and device, and the hi-res pass
    cams = np.arange(0, E, 64, dtype=np.int32)
    views = np.stack([g.view(int(e), 0) for e in cams])
    g.draw_cameras(cams, views, 256, 128, depth=True, seg=True)
    n = len(cams)
    d_cams, d_views = torch.from_numpy(cams).cuda(), torch.from_numpy(views).cuda()
    d_obs = torch.empty((n, 128, 256, 4), dtype=torch.uint8, device="cuda")
    d_depth = torch.empty((n, 128, 256), dtype=torch.float32, device="cuda")
    d_seg = torch.empty((n, 128, 256), dtype=torch.int16, device="cuda")
    torch.cuda.synchronize()
    g.draw_cameras_device(d_cams.data_ptr(), d_views.data_ptr(), n, 256, 128, d_obs.data_ptr(), d_depth.data_ptr(), d_seg.data_ptr())
    g.sync()
    g.draw_hires(256, 128)

    every = torch.ones(E, dtype=torch.uint8, device="cuda")
    if level_set:  # one replacement through to its rewrite: the row retires at the first call, the second rewrites it
        g.replace_levels([3], [9000])
        for _ in range(2):
            g.step_device(None, every.data_ptr())
            g.sync()
        seeds, retiring = g.level_rows()
        assert seeds[3] == 9000 and not retiring.any(), "the replacement was meant to be rewritten"
    assert g.faults() == 0 and g.fault_word() == 0

    if level_set:
        g.step_device(None, every.data_ptr())
        g.replace_levels([5], [9001])
    else:
        g.step_device(d_acts.data_ptr())
        g.step_device(d_acts.data_ptr())
    g.close()


def _settle():
    """give back what is freed but still held: Python's garbage, torch's cached blocks and the free pages of glibc's heaps"""
    import ctypes

    import torch

    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    ctypes.CDLL(None).malloc_trim(0)


def _host_rss():
    with open("/proc/self/status") as f:
        for line in f:
            if line.startswith("VmRSS:"):
                return int(line.split()[1]) * 1024
    raise AssertionError("no VmRSS in /proc/self/status")


def _device_used():
    """this process's device memory in bytes as nvidia-smi reports it, or None where the query is unavailable or does not list it"""
    try:
        out = subprocess.run(["nvidia-smi", "--query-compute-apps=pid,used_memory", "--format=csv,noheader,nounits"], capture_output=True,
                             text=True, timeout=60, check=True).stdout
    except (OSError, subprocess.SubprocessError):
        return None
    for line in out.splitlines():
        fields = [x.strip() for x in line.split(",")]
        if len(fields) == 2 and fields[0] == str(os.getpid()) and fields[1].isdigit():
            return int(fields[1]) << 20
    return None


@pytest.mark.parametrize("level_set", [False, True], ids=["steps_in_flight", "replacement_pending"])
def test_close_with_work_outstanding(built, level_set):
    """closing waits for the work it would free under: the next engine runs cleanly and the device reports no error"""
    import torch

    from megaverse_b200 import capi

    _cycle(level_set)
    torch.cuda.synchronize()
    g = capi.Engine("TowerBuilding", 4, 1)
    g.reset()
    g.step(np.zeros(4, dtype=np.int32))
    assert g.faults() == 0
    g.close()


def test_cycles_leave_memory_where_it_was(built):
    """after warm-up cycles of both kinds (lazily loaded kernels, the allocator's heaps, torch's cache), further cycles leave the
    process's host and device memory within TOLERANCE of where they were"""
    for c in range(WARMUP):
        _cycle(c % 2 == 1)
    _settle()
    host0, dev0 = _host_rss(), _device_used()
    for c in range(CYCLES):
        _cycle(c % 2 == 1)
    _settle()
    host1, dev1 = _host_rss(), _device_used()
    assert host1 - host0 < TOLERANCE, "host memory grew by %.1f MB over %d cycles" % ((host1 - host0) / 1e6, CYCLES)
    if dev0 is None or dev1 is None:
        pytest.skip("host memory held; nvidia-smi does not report this process's device memory here")
    assert dev1 - dev0 < TOLERANCE, "device memory grew by %.1f MB over %d cycles" % ((dev1 - dev0) / 1e6, CYCLES)
