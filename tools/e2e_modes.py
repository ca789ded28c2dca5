#!/usr/bin/env python
"""End-to-end step time through host buffers (mv_set_actions + mv_step) under the delivery modes: zero-copy stores from the raster
kernel into the pinned host slab, one copy-engine download after the raster, and the raster in N slices whose downloads overlap the
next slice's kernels.   e2e_modes.py [scenario envs agents [depth]]"""
import os, sys, time
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from megaverse_b200 import capi

scenario = sys.argv[1] if len(sys.argv) > 1 else "TowerBuilding"
E = int(sys.argv[2]) if len(sys.argv) > 2 else 256
A = int(sys.argv[3]) if len(sys.argv) > 3 else 1
depth = len(sys.argv) > 4 and sys.argv[4] == "depth"
g = capi.Engine(scenario, E, A, 128, 72, num_threads=8, depth=depth)
for e in range(E):
    g.seed_env(e, 42 + e)
g.reset()
rng = np.random.default_rng(1)
K = 40
acts = (1 << rng.integers(0, 11, size=(K + 10, E * A))).astype(np.int32)
mb = E * A * 128 * 72 * (8 if depth else 4) / 1e6
for name, opts in [("zero-copy stores", {"zero_copy": 1}), ("one copy after the raster", {"zero_copy": 0, "host_slices": 1}), ("2 slices", {"zero_copy": 0, "host_slices": 2}),
                   ("4 slices", {"zero_copy": 0, "host_slices": 4}), ("8 slices", {"zero_copy": 0, "host_slices": 8}), ("16 slices", {"zero_copy": 0, "host_slices": 16}),
                   ("by size (default)", {"zero_copy": -1, "host_slices": 0}), ("no delivery (obs_to_host 0)", {"obs_to_host": 0})]:
    for k, v in opts.items():
        g.set_option(k, v)
    for t in range(5):
        g.step(acts[t])
    t0 = time.perf_counter()
    for t in range(5, 5 + K):
        g.step(acts[t])
    dt = (time.perf_counter() - t0) / K
    print("%-28s %8.1f us/step = %.2fM obs/s, %.1f GB/s of %.0f MB (faults %d)" % (name, dt * 1e6, E * A / dt / 1e6, mb / dt / 1e3, mb, g.faults()))
    g.set_option("obs_to_host", 1)
g.close()
