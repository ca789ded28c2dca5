#!/usr/bin/env python
"""Action-repeat rates (option "action_repeat" k = 1, 2, 4).

For each workload three engines, one per k, on bench.py's env seeds (42 + env) and action stream (one random action bit per agent per
call), with the scenarios' own episode lengths (natural ends only), alternated in one process, three rounds each:
1. The device-resident loop with option obs_to_host 0 (mv_step: frames stay in HBM, rewards and dones come back every call): ms per call,
   host clock around 300 calls; from it simulated env ticks per second (envs x k per call) and frames per second (views drawn per call).
   mv_step_device is not used: some levels of these seeds are solved at once and end within two calls at k >= 2, which the asynchronous
   call's three-call contract refuses (DESIGN.md section 2).
2. Option overlap 0: the step kernel (mv_last_kernel_ms [0]) and the raster kernel ([1]), CUDA events, medians over 90 calls.
Prints the card's name and power limit with the numbers."""
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from megaverse_b200 import capi  # noqa: E402

WORKLOADS = [("Collect", 1024, 4, False), ("TowerBuilding", 256, 1, False), ("ObstaclesHard", 2048, 1, True)]
REPEATS = (1, 2, 4)
STEPS, WARMUP, ROUNDS, TIMED = 300, 30, 3, 90


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
        return out.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown card"


def engine(scenario, E, A, depth, k):
    g = capi.Engine(scenario, E, A, 128, 72, num_threads=16, depth=depth)
    g.set_option("action_repeat", k)
    g.set_option("obs_to_host", 0)
    for e in range(E):
        g.seed_env(e, 42 + e)  # bench.py's seeds
    g.reset()
    return g


def workload(scenario, E, A, depth):
    engines = {k: engine(scenario, E, A, depth, k) for k in REPEATS}
    rng = np.random.default_rng(1)  # bench.py's action stream: one uniformly random action bit per agent per call
    acts = (1 << rng.integers(0, 11, size=(64, E * A))).astype(np.int32)
    step = {k: 0 for k in REPEATS}
    ms = {k: [] for k in REPEATS}
    for _ in range(ROUNDS):
        for k, g in engines.items():
            for i in range(WARMUP + STEPS):
                if i == WARMUP:
                    t0 = time.perf_counter()
                g.step(acts[step[k] % 64])
                step[k] += 1
            ms[k].append((time.perf_counter() - t0) * 1e3 / STEPS)
    kern = {k: [] for k in REPEATS}
    for g in engines.values():
        g.set_option("overlap", 0)
    for _ in range(ROUNDS):
        for k, g in engines.items():
            for i in range(WARMUP + TIMED // ROUNDS):
                g.step(acts[step[k] % 64])
                step[k] += 1
                if i >= WARMUP:
                    kern[k].append(g.last_kernel_ms())
    base = float(np.median(ms[1]))
    for k in REPEATS:
        m = float(np.median(ms[k]))
        kk = np.median(np.array(kern[k]), axis=0)
        print("action_repeat %-13s %4d x %d%s | k=%d | %.4f ms/call (rounds %s) | %.0f ticks/s (%.2fx k=1) | %.0f frames/s | overlap 0: step kernel %.4f ms, raster %.4f ms"
              % (scenario, E, A, " +depth" if depth else "", k, m, ", ".join("%.4f" % x for x in ms[k]), E * k * 1e3 / m, k * base / m,
                 E * A * 1e3 / m, kk[0], kk[1]))
    for g in engines.values():
        assert g.fault_word() == 0
        g.close()


def main():
    print("card:", card())
    for w in WORKLOADS:
        workload(*w)


if __name__ == "__main__":
    main()
