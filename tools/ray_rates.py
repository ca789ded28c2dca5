#!/usr/bin/env python
"""Ray sensor rates (mv_set_rays).

At the three bench.py workloads, with the rays off and with R = 16, 64 and 256 (a 180 degree fan), alternated in one process, three rounds:
1. mv_step_device: ms per call, host clock around 300 calls and a synchronise (the rays stay in HBM);
2. mv_step (host-facing; the rays come down in one copy on the step's stream): ms per call over 100 calls;
3. option overlap 0, a synchronise after every call: the ray launch's time (mv_last_rays_ms, CUDA events), median of 100 calls.
Episodes are long (episodeLengthSec 600).  Prints the card's name and power limit with the numbers."""
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from megaverse_b200 import capi, rays  # noqa: E402

WORKLOADS = [("Collect", 1024, 4, False), ("TowerBuilding", 256, 1, False), ("ObstaclesHard", 2048, 1, True)]
RAYS = [0, 16, 64, 256]
STEPS, HOST_STEPS, WARMUP, ROUNDS, TIMED = 300, 100, 30, 3, 100


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
        return out.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown card"


def engine(scenario, E, A, depth, R, overlap=1):
    g = capi.Engine(scenario, E, A, 128, 72, num_threads=16, params={"episodeLengthSec": 600.0}, depth=depth)
    g.set_option("overlap", overlap)
    if R:
        g.set_rays(rays.fan(R, 180.0), 60.0)
    for e in range(E):
        g.seed_env(e, 42 + e)
    g.reset()
    return g


def workload(scenario, E, A, depth):
    import torch

    rng = np.random.default_rng(2)
    host_acts = (1 << rng.integers(0, 11, size=(64, E * A))).astype(np.int32)
    acts = torch.from_numpy(host_acts).cuda()
    dev = {R: [] for R in RAYS}
    host = {R: [] for R in RAYS}
    kern = {R: [] for R in RAYS}
    for _ in range(ROUNDS):
        for R in RAYS:
            g = engine(scenario, E, A, depth, R)
            for i in range(WARMUP + STEPS):
                if i == WARMUP:
                    g.sync()
                    t0 = time.perf_counter()
                g.step_device(acts[i % len(acts)].data_ptr())
            g.sync()
            dev[R].append((time.perf_counter() - t0) * 1e3 / STEPS)
            for i in range(WARMUP + HOST_STEPS):
                if i == WARMUP:
                    t0 = time.perf_counter()
                g.step(host_acts[i % len(host_acts)])
            host[R].append((time.perf_counter() - t0) * 1e3 / HOST_STEPS)
            g.close()
            if R:
                g = engine(scenario, E, A, depth, R, overlap=0)
                ms = []
                for i in range(WARMUP + TIMED):
                    g.step(host_acts[i % len(host_acts)])
                    if i >= WARMUP:
                        ms.append(g.last_rays_ms())
                kern[R].append(float(np.median(ms)))
                g.close()
    base_d, base_h = float(np.median(dev[0])), float(np.median(host[0]))
    for R in RAYS:
        d, h = float(np.median(dev[R])), float(np.median(host[R]))
        k = ("%.3f" % float(np.median(kern[R]))) if R else "-"
        print("%-14s %5d x %d  R=%3d  step_device %.3f ms (+%.3f)  step %.3f ms (+%.3f)  ray kernel %s ms   [rounds: dev %s host %s]"
              % (scenario, E, A, R, d, d - base_d, h, h - base_h, k, " ".join("%.3f" % x for x in dev[R]), " ".join("%.3f" % x for x in host[R])),
              flush=True)


def main():
    print("card:", card(), flush=True)
    for w in WORKLOADS:
        workload(*w)


if __name__ == "__main__":
    main()
