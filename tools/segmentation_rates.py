#!/usr/bin/env python
"""Segmentation rates (option "segmentation"): the option off against on, alternated in one process, three rounds each.

For each workload (bench.py's three: Collect 1 024 x 4, TowerBuilding 256 x 1, ObstaclesHard 2 048 x 1 with depth):
1. The device-resident loop (mv_step_device): ms per step, host clock around 300 steps and a synchronise.
2. The host-facing mv_step (zero-copy delivery of obs, depth and segmentation into pinned memory): ms per step, host clock around 100
   steps, each of which returns with the tensors in host memory.
3. Option overlap 0, a synchronise after every mv_step_device: the raster kernel's time (mv_last_kernel_ms [1], CUDA events), median over
   100 steps.

Episodes run at the scenarios' own lengths.  Prints the card's name and power limit with the numbers."""
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from megaverse_b200 import capi  # noqa: E402

WORKLOADS = [("Collect", 1024, 4, False), ("TowerBuilding", 256, 1, False), ("ObstaclesHard", 2048, 1, True)]
STEPS, HOST_STEPS, WARMUP, ROUNDS, TIMED = 300, 100, 30, 3, 100


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
        return out.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown card"


def engine(scenario, E, A, depth, seg):
    g = capi.Engine(scenario, E, A, 128, 72, num_threads=16, depth=depth, segmentation=seg)
    for e in range(E):
        g.seed_env(e, 42 + e)
    g.reset()
    return g


def workload(scenario, E, A, depth):
    import torch

    engines = {"off": engine(scenario, E, A, depth, False), "on": engine(scenario, E, A, depth, True)}
    rng = np.random.default_rng(2)
    host_acts = (1 << rng.integers(0, 11, size=(64, E * A))).astype(np.int32)
    acts = torch.from_numpy(host_acts).cuda()
    torch.cuda.synchronize()
    step = {"off": 0, "on": 0}
    dev = {k: [] for k in engines}
    host = {k: [] for k in engines}
    for _ in range(ROUNDS):
        for name, g in engines.items():
            for i in range(WARMUP + STEPS):
                if i == WARMUP:
                    g.sync()
                    t0 = time.perf_counter()
                g.step_device(acts[step[name] % 64].data_ptr())
                step[name] += 1
            g.sync()
            dev[name].append((time.perf_counter() - t0) * 1e3 / STEPS)
        for name, g in engines.items():
            for i in range(WARMUP + HOST_STEPS):
                if i == WARMUP:
                    t0 = time.perf_counter()
                g.step(host_acts[step[name] % 64])
                step[name] += 1
            host[name].append((time.perf_counter() - t0) * 1e3 / HOST_STEPS)
    kern = {k: [] for k in engines}
    for g in engines.values():
        g.set_option("overlap", 0)
    for _ in range(ROUNDS):
        for name, g in engines.items():
            for i in range(WARMUP + TIMED // ROUNDS):
                g.step_device(acts[step[name] % 64].data_ptr())
                step[name] += 1
                g.sync()
                if i >= WARMUP:
                    kern[name].append(g.last_kernel_ms()[1])
    for name in engines:
        print("segmentation %-13s %4d x %d%s | %-3s | mv_step_device %.4f ms/step (rounds %s) | mv_step %.4f ms/step (rounds %s) | overlap 0: raster %.4f ms"
              % (scenario, E, A, " +depth" if depth else "", name, float(np.median(dev[name])), ", ".join("%.4f" % x for x in dev[name]),
                 float(np.median(host[name])), ", ".join("%.4f" % x for x in host[name]), float(np.median(kern[name]))))
    for g in engines.values():
        assert g.fault_word() == 0
        g.close()


def main():
    print("card:", card())
    for w in WORKLOADS:
        workload(*w)


if __name__ == "__main__":
    main()
