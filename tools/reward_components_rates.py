#!/usr/bin/env python
"""Reward-component rates (option "reward_components").

At the three bench.py workloads, the option off and on alternated in one process, three rounds each:
1. mv_step_device: ms per call, host clock around 300 calls and a synchronise (the rows stay in HBM);
2. mv_step (host-facing; the step and episode rows come down with the rewards): ms per call over 100 calls;
3. option overlap 0, a synchronise after every call: the step kernel's time (mv_last_kernel_ms [0], CUDA events), median of 100 calls.
Episodes are 20 s (300 calls), so the timed windows cross episode ends.  --off-only times the option off alone: copied into a checkout
that predates the option, it gives that build's figures to set beside these.  Prints the card's name and power limit with the numbers."""
import argparse
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


def engine(scenario, E, A, depth, on):
    g = capi.Engine(scenario, E, A, 128, 72, num_threads=16, params={"episodeLengthSec": 20.0}, depth=depth)
    if on:
        g.set_option("reward_components", 1)
    for e in range(E):
        g.seed_env(e, 42 + e)
    g.reset()
    return g


def workload(scenario, E, A, depth, names):
    import torch

    rng = np.random.default_rng(2)
    host_acts = (1 << rng.integers(0, 11, size=(64, E * A))).astype(np.int32)
    acts = torch.from_numpy(host_acts).cuda()
    engines = {name: engine(scenario, E, A, depth, name == "on") for name in names}
    torch.cuda.synchronize()
    dev = {k: [] for k in engines}
    host = {k: [] for k in engines}
    for _ in range(ROUNDS):
        for name, g in engines.items():
            for i in range(WARMUP + STEPS):
                if i == WARMUP:
                    g.sync()
                    t0 = time.perf_counter()
                g.step_device(acts[i % 64].data_ptr())
            g.sync()
            dev[name].append((time.perf_counter() - t0) * 1e3 / STEPS)
        for name, g in engines.items():
            for i in range(WARMUP + HOST_STEPS):
                if i == WARMUP:
                    t0 = time.perf_counter()
                g.step(host_acts[i % 64])
            host[name].append((time.perf_counter() - t0) * 1e3 / HOST_STEPS)
    kern = {k: [] for k in engines}
    for g in engines.values():
        g.set_option("overlap", 0)
    for _ in range(ROUNDS):
        for name, g in engines.items():
            for i in range(WARMUP + TIMED // ROUNDS):
                g.step_device(acts[i % 64].data_ptr())
                g.sync()
                if i >= WARMUP:
                    kern[name].append(g.last_kernel_ms()[0])
    tag = "%s %d x %d%s" % (scenario, E, A, " +depth" if depth else "")
    for name in engines:
        k = np.array(kern[name])
        print("reward_components %-24s | %-3s | mv_step_device %.4f ms (rounds %s) | mv_step %.4f ms (rounds %s) | overlap 0: step kernel "
              "median %.4f ms, p10 %.4f, p90 %.4f" % (tag, name, float(np.median(dev[name])), ", ".join("%.4f" % x for x in dev[name]),
                                                      float(np.median(host[name])), ", ".join("%.4f" % x for x in host[name]), float(np.median(k)),
                                                      float(np.percentile(k, 10)), float(np.percentile(k, 90))))
    for g in engines.values():
        assert g.fault_word() == 0
        g.close()


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--off-only", action="store_true", help="time the option off only (a checkout without the option)")
    args = ap.parse_args()
    print("card:", card())
    print("library:", capi.LIB_PATH)
    for w in WORKLOADS:
        workload(*w, names=("off",) if args.off_only else ("off", "on"))


if __name__ == "__main__":
    main()
