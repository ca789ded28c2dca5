#!/usr/bin/env python
"""Env state store rates (mv_states_save / mv_states_load of every env): bytes per row, wall time of a save and of a load, the copy
kernel's and the load's re-render kernel's time (CUDA events), the copy kernel's achieved bandwidth (bytes read + written) against the H100
SXM data sheet's 3.35 TB/s, and the host part of a save: its wall time less the copy kernel (level-generator and host-mirror copies, which
overlap the kernel, and the synchronisation).  A save is the same copy and host work as a load without the re-render.  Prints the card's
name and power limit with the numbers."""
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ.setdefault("BOXOBAN_LEVELS", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "boxoban"))
from megaverse_b200 import capi  # noqa: E402

CONFIGS = [("Collect", 1024, 4), ("TowerBuilding", 256, 1), ("HexExplore", 256, 1)]
HBM_PEAK_GBS = 3350.0  # NVIDIA H100 SXM data sheet (HBM3)
REPS = 20


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
        return out.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown card"


def main():
    print("card:", card())
    for scenario, E, A in CONFIGS:
        g = capi.Engine(scenario, E, A, 128, 72, num_threads=16)
        for e in range(E):
            g.seed_env(e, 42 + e)
        g.reset()
        rng = np.random.default_rng(1)
        for t in range(20):
            g.step((1 << rng.integers(0, 11, size=E * A)).astype(np.int32))
        row = g.state_row_bytes()
        store = g.states_create(E)
        envs = np.arange(E, dtype=np.int32)
        g.states_save(store, envs, envs)  # warm-up
        g.states_load(store, envs, envs)
        res = {"save": [], "save_copy": [], "load": [], "load_copy": [], "load_render": []}
        for _ in range(REPS):
            t0 = time.perf_counter()
            g.states_save(store, envs, envs)  # synchronous: returns after the copy finished
            res["save"].append((time.perf_counter() - t0) * 1e3)
            res["save_copy"].append(g.last_kernel_ms()[0])
            t0 = time.perf_counter()
            g.states_load(store, envs, envs)
            res["load"].append((time.perf_counter() - t0) * 1e3)
            copy_ms, render_ms = g.last_kernel_ms()
            res["load_copy"].append(copy_ms)
            res["load_render"].append(render_ms)
        med = {k: float(np.median(v)) for k, v in res.items()}
        moved = 2.0 * row * E  # bytes read + bytes written
        copy_ms = (med["save_copy"] + med["load_copy"]) / 2
        gbs = moved / (copy_ms * 1e-3) / 1e9
        print("%-13s %4d x %d: row %.1f KB (%.1f MB for all envs) | save %.3f ms (copy kernel %.3f ms, host part %.3f ms) | load %.3f ms "
              "(copy kernel %.3f ms, re-render kernel %.3f ms) | copy kernel %.0f GB/s = %.0f%% of %.0f GB/s | faults %d"
              % (scenario, E, A, row / 1024, row * E / 2**20, med["save"], med["save_copy"], med["save"] - med["save_copy"], med["load"],
                 med["load_copy"], med["load_render"], gbs, 100 * gbs / HBM_PEAK_GBS, HBM_PEAK_GBS, g.faults()))
        g.states_destroy(store)
        g.close()


if __name__ == "__main__":
    main()
