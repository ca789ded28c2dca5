#!/usr/bin/env python
"""Spectator camera rates (mv_draw_cameras_device), Collect 1 024 x 4 at 128 x 72 unless stated.

1. mv_draw_cameras_device at 768 x 432 for 1, 16 and 64 overview cameras: ms per call (CUDA events around 20 calls on the engine stream)
   and the bytes its outputs take, against mv_draw_hires on a 16-env engine (every agent view at 768 x 432, HBM and pinned buffers);
2. one chase camera at 128 x 72 drawn after every mv_step_device: ms per step with and without it, alternated in one process (3 rounds);
3. all N agent views passed as cameras at 128 x 72 against the step's own raster launch (option overlap 0, CUDA events): the cost of the
   camera table lookup.
Prints the card's name and power limit with the numbers."""
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from megaverse_b200 import capi, cameras  # noqa: E402

E, A = 1024, 4
ROUNDS, STEPS, WARMUP = 3, 200, 20


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
        return out.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown card"


def engine(num_envs, overlap=True):
    g = capi.Engine("Collect", num_envs, A, 128, 72, num_threads=16, params={"episodeLengthSec": 600.0})
    g.set_option("overlap", int(overlap))
    for e in range(num_envs):
        g.seed_env(e, 42 + e)
    g.reset()
    return g


def event_ms(torch, stream, fn, n):
    s = torch.cuda.ExternalStream(stream)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    a.record(s)
    for _ in range(n):
        fn()
    b.record(s)
    b.synchronize()
    return a.elapsed_time(b) / n


def main():
    import torch

    print("card: %s" % card())
    rng = np.random.default_rng(4)
    g = engine(E)
    acts = torch.from_numpy((1 << rng.integers(0, 11, size=(64, E * A))).astype(np.int32)).cuda()
    for i in range(10):
        g.step_device(acts[i % 64].data_ptr())
    g.sync()
    bounds = g.level_bounds()

    # 1. overview cameras at 768 x 432
    for n in (1, 16, 64):
        envs = torch.arange(n, dtype=torch.int32, device="cuda")
        views = torch.from_numpy(cameras.overview_views(bounds[:n], 768, 432)).cuda()
        obs = torch.empty((n, 432, 768, 4), dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        ms = event_ms(torch, g.stream(), lambda: g.draw_cameras_device(envs.data_ptr(), views.data_ptr(), n, 768, 432, obs.data_ptr()), 20)
        print("overview x%d 768x432: %.3f ms per call, %.1f MB of frames" % (n, ms, obs.numel() / 1e6))
    h16 = engine(16)
    h16.draw_hires(768, 432)
    t0 = time.perf_counter()
    for _ in range(5):
        h16.draw_hires(768, 432)
    hires_ms = (time.perf_counter() - t0) * 1e3 / 5
    print("mv_draw_hires 16 envs x %d (%d frames) 768x432: %.3f ms per call (host clock, includes the download), %.1f MB HBM + %.1f MB pinned"
          % (A, 16 * A, hires_ms, 16 * A * 768 * 432 * 4 / 1e6, 16 * A * 768 * 432 * 4 / 1e6))
    h16.close()

    # 2. one chase camera after every step
    env0 = torch.zeros(1, dtype=torch.int32, device="cuda")
    chase = torch.empty(16, dtype=torch.float32, device="cuda")
    frame = torch.empty((1, 72, 128, 4), dtype=torch.uint8, device="cuda")
    d_views = torch.as_tensor(g.device_array("views"), device="cuda")
    shift = torch.from_numpy(cameras.chase_views(np.eye(4, dtype=np.float32).reshape(1, 16))[0].reshape(4, 4).T.copy()).cuda()

    def run(with_camera):
        s = torch.cuda.ExternalStream(g.stream())
        for i in range(WARMUP + STEPS):
            if i == WARMUP:
                g.sync()
                t0 = time.perf_counter()
            g.step_device(acts[i % 64].data_ptr())
            if with_camera:
                with torch.cuda.stream(s):  # the chase matrix from the agent's view in HBM, on the engine stream
                    chase.copy_((shift @ d_views[0].view(4, 4).T).T.reshape(16))
                g.draw_cameras_device(env0.data_ptr(), chase.data_ptr(), 1, 128, 72, frame.data_ptr())
        g.sync()
        return (time.perf_counter() - t0) * 1e3 / STEPS

    res = {False: [], True: []}
    for _ in range(ROUNDS):
        for flag in (False, True):
            res[flag].append(run(flag))
    print("mv_step_device ms per step: without camera %s, with one chase camera %s (medians %.3f / %.3f)"
          % (["%.3f" % x for x in res[False]], ["%.3f" % x for x in res[True]], np.median(res[False]), np.median(res[True])))
    g.close()

    # 3. every agent view as a camera against the step's own raster launch
    g = engine(E, overlap=False)
    raster = []
    for i in range(50):
        g.step_device(acts[i % 64].data_ptr())
        g.sync()
        raster.append(g.last_kernel_ms()[1])
    d_views = torch.as_tensor(g.device_array("views"), device="cuda").clone()
    envs = torch.arange(E, dtype=torch.int32, device="cuda").repeat_interleave(A)
    obs = torch.empty((E * A, 72, 128, 4), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    ms = event_ms(torch, g.stream(), lambda: g.draw_cameras_device(envs.data_ptr(), d_views.data_ptr(), E * A, 128, 72, obs.data_ptr()), 50)
    print("all %d agent views: step raster launch %.3f ms (median of 50), as cameras %.3f ms per call" % (E * A, float(np.median(raster)), ms))
    g.close()


if __name__ == "__main__":
    main()
