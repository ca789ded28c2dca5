#!/usr/bin/env python
"""Steps with an active set at the headline shape (Collect 1 024 envs x 4 agents, 128 x 72, bench.py's env seeds 42 + e and its random
one-bit action stream), against the full calls they reduce to.

1. mv_step_device_active at active fractions 100 %, 50 %, 10 %, 1 % and 0 % (seeded random masks) against mv_step_device: ms per call, host
   clock around STEPS calls that end in a device synchronise.
2. mv_step_envs against mv_step at the same fractions (synchronous, zero-copy delivery into the pinned host buffer).
3. Step kernel and raster kernel times with option overlap 0 (CUDA events, mv_last_kernel_ms) for both asynchronous calls.

The full and the subset call alternate at every fraction, in ROUNDS rounds.  Prints the card's name and power limit, read in the same run."""
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from megaverse_b200 import capi  # noqa: E402

SCENARIO, E, A = "Collect", 1024, 4
FRACTIONS = (1.0, 0.5, 0.1, 0.01, 0.0)
STEPS, WARMUP, ROUNDS, KERNEL_STEPS, MASKS = 200, 20, 2, 40, 16


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
        return out.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown card"


def main():
    import torch

    print("card:", card())
    g = capi.Engine(SCENARIO, E, A, 128, 72, num_threads=16)
    for e in range(E):
        g.seed_env(e, 42 + e)  # bench.py's seeds
    g.reset()
    acts_host = (1 << np.random.default_rng(1).integers(0, 11, size=(64, E * A))).astype(np.int32)  # bench.py's action stream
    acts = torch.from_numpy(acts_host).cuda()
    rng = np.random.default_rng(3)
    masks = {f: [(rng.random(E) < f).astype(np.uint8) for _ in range(MASKS)] for f in FRACTIONS}
    dmasks = {f: [torch.from_numpy(m).cuda() for m in ms] for f, ms in masks.items()}
    lists = {f: [np.flatnonzero(m).astype(np.int32) for m in ms] for f, ms in masks.items()}
    torch.cuda.synchronize()
    t = [0]

    def device(f):  # f None: the full call
        if f is None:
            g.step_device(acts[t[0] % 64].data_ptr())
        else:
            g.step_device_active(acts[t[0] % 64].data_ptr(), 0, dmasks[f][t[0] % MASKS].data_ptr())
        t[0] += 1

    def host(f):
        if f is None:
            g.step(acts_host[t[0] % 64])
        else:
            g.step_envs(acts_host[t[0] % 64], lists[f][t[0] % MASKS])
        t[0] += 1

    def timed(fn, f, steps):
        for _ in range(WARMUP):
            fn(f)
        g.sync()
        t0 = time.perf_counter()
        for _ in range(steps):
            fn(f)
        g.sync()
        return (time.perf_counter() - t0) * 1e3 / steps

    res = {}
    for r in range(ROUNDS):
        for f in FRACTIONS:
            for kind, fn in (("device", device), ("host", host)):
                res.setdefault((kind, "full", f), []).append(timed(fn, None, STEPS))
                res.setdefault((kind, "active", f), []).append(timed(fn, f, STEPS))
    g.set_option("overlap", 0)
    kern = {}
    for r in range(ROUNDS):
        for f in FRACTIONS:
            for which in (None, f):
                ks = []
                for i in range(WARMUP + KERNEL_STEPS):
                    device(which)
                    g.sync()
                    if i >= WARMUP:
                        ks.append(g.last_kernel_ms())
                kern.setdefault((which is not None, f), []).append(np.mean(np.array(ks), axis=0))
    g.set_option("overlap", 1)
    assert g.fault_word() == 0 and g.faults() == 0

    print("%s %d x %d, 128 x 72: ms per call (median of %d rounds; rounds in brackets)" % (SCENARIO, E, A, ROUNDS))
    print("| active | mv_step_device | mv_step_device_active | mv_step | mv_step_envs | step kernel full / active | raster kernel full / active |")
    print("|---|---|---|---|---|---|---|")

    def cell(key):
        v = res[key]
        return "%.3f (%s)" % (float(np.median(v)), ", ".join("%.3f" % x for x in v))

    for f in FRACTIONS:
        kf, ka = np.median(np.array(kern[(False, f)]), axis=0), np.median(np.array(kern[(True, f)]), axis=0)
        print("| %g %% | %s | %s | %s | %s | %.3f / %.3f | %.3f / %.3f |" % (
            f * 100, cell(("device", "full", f)), cell(("device", "active", f)), cell(("host", "full", f)), cell(("host", "active", f)),
            kf[0], ka[0], kf[1], ka[1]))
    g.close()


if __name__ == "__main__":
    main()
