#!/usr/bin/env python
"""Level refresh rates (mv_replace_levels): what a bank that is refreshed while the envs run costs against a static level set and against
the streams.

Workloads: Collect 1 024 x 4 and ObstaclesHard 2 048 x 1 with depth, mv_step_device_ends with 1 % and 10 % of the envs asked to end per
call.  Arms, alternated in one process, three rounds of 300 calls each (host clock around the calls and a synchronise):
  stream   the level streams, level_slots 2 (a host worker generates every ended env's next level);
  static   a level set of L = 1 024 levels per scenario;
  r=R      the same set with R rows replaced per call (fresh seeds, rows chosen among those not being replaced).
Then, with option overlap 0, the step kernel's time (mv_last_kernel_ms, CUDA events), median over 100 calls per arm.  Prints the card's
name and power limit with the numbers."""
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from megaverse_b200 import capi  # noqa: E402

WORKLOADS = [("Collect", 1024, 4, False), ("ObstaclesHard", 2048, 1, True)]
END_FRACTIONS = [0.01, 0.10]
ARMS = ["stream", "static", 1, 10, 50]
L, STEPS, WARMUP, ROUNDS, TIMED, THREADS = 1024, 300, 30, 3, 100, 16


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
        return out.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown card"


def engine(scenario, E, A, depth, arm):
    g = capi.Engine(scenario, E, A, 128, 72, num_threads=THREADS, depth=depth)
    if arm != "stream":
        g.set_option("level_set", L)
    for e in range(E):
        g.seed_env(e, 42 + e)
    g.reset()
    return g


class Refresher:
    """R rows per call, fresh seeds, rows taken in turn among those not being replaced"""

    def __init__(self, R):
        self.R, self.next_seed, self.cursor = R, 1 << 20, 0

    def __call__(self, g):
        if not self.R:
            return
        retiring = g.level_rows()[1]
        free = np.flatnonzero(~retiring)
        if free.size <= self.R:
            return
        rows = np.roll(free, -self.cursor)[:self.R]
        self.cursor = (self.cursor + self.R) % free.size
        g.replace_levels(rows, np.arange(self.next_seed, self.next_seed + self.R))
        self.next_seed += self.R


def run(g, acts, ends, refresh, n, timed_kernel=False):
    ms = []
    for i in range(n):
        refresh(g)
        g.step_device(acts[i % len(acts)].data_ptr(), ends[i % len(ends)].data_ptr())
        if timed_kernel:
            g.sync()
            ms.append(g.last_kernel_ms()[0])
    return ms


def workload(scenario, E, A, depth):
    import torch

    rng = np.random.default_rng(2)
    acts = torch.from_numpy((1 << rng.integers(0, 11, size=(64, E * A))).astype(np.int32)).cuda()
    engines = {arm: engine(scenario, E, A, depth, arm) for arm in ARMS}
    for frac in END_FRACTIONS:
        ends = [torch.from_numpy((rng.random(E) < frac).astype(np.uint8)).cuda() for _ in range(64)]
        calls = {arm: [] for arm in ARMS}
        kern = {}
        refresh = {arm: Refresher(arm if isinstance(arm, int) else 0) for arm in ARMS}
        for _ in range(ROUNDS):
            for arm in ARMS:
                g = engines[arm]
                try:
                    run(g, acts, ends, refresh[arm], WARMUP)
                    g.sync()
                    t0 = time.perf_counter()
                    run(g, acts, ends, refresh[arm], STEPS)
                    g.sync()
                    calls[arm].append((time.perf_counter() - t0) * 1e3 / STEPS)
                except capi.MegaverseError as err:  # the streams refuse episodes shorter than their pipeline
                    calls[arm].append(float("nan"))
                    print("  %s: %s" % (arm, err), flush=True)
                    engines[arm].close()
                    engines[arm] = engine(scenario, E, A, depth, arm)
        for arm in ARMS:
            g = engines[arm]
            try:
                g.set_option("overlap", 0)
                kern[arm] = float(np.median(run(g, acts, ends, refresh[arm], TIMED, timed_kernel=True)))
                g.set_option("overlap", 1)
            except capi.MegaverseError:
                kern[arm] = float("nan")
                engines[arm].close()
                engines[arm] = engine(scenario, E, A, depth, arm)
        for arm in ARMS:
            c = calls[arm]
            name = arm if isinstance(arm, str) else "r=%d" % arm
            print("%-14s %5d x %d  ends %4.1f %%  %-7s  %.3f ms per call  [rounds %s; spread %.3f]  step kernel %.3f ms  faults %d"
                  % (scenario, E, A, 100 * frac, name, float(np.median(c)), " ".join("%.3f" % x for x in c), float(np.max(c) - np.min(c)),
                     kern[arm], engines[arm].fault_word()), flush=True)
    for g in engines.values():
        g.close()


def main():
    print("card:", card(), flush=True)
    for w in WORKLOADS:
        workload(*w)


if __name__ == "__main__":
    main()
