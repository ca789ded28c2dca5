#!/usr/bin/env python
"""Terminal-frame rates (option "final_obs").

For each workload, four settings alternated in one process, three rounds each:
  off, 0 %  the option off, no episode ends in the window;
  off, 1 %  the option off, 1 % of the envs asked to end per step through d_ends (each env every 100 steps): the cost of the ends alone;
  on, 0 %   the option on, no ends (the terminal-frame launch finds no env to draw);
  on, 1 %   the option on, the same ends.
1. The device-resident loop (mv_step_device_ends): ms per step, host clock around 300 steps and a synchronise.
2. Option overlap 0, a synchronise after every step: the step kernel (mv_last_kernel_ms [0]), the step's own raster launch ([1]) and the
   terminal-frame launch (mv_last_final_ms), CUDA events, medians over 100 steps.

Episodes are long (episodeLengthSec 600), so the only ends are the requested ones.  Prints the card's name and power limit with the numbers."""
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from megaverse_b200 import capi  # noqa: E402

WORKLOADS = [("Collect", 1024, 4, False), ("TowerBuilding", 256, 1, False), ("ObstaclesHard", 2048, 1, True)]
STEPS, WARMUP, ROUNDS, TIMED = 300, 30, 3, 100


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
        return out.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown card"


def engine(scenario, E, A, depth, final):
    g = capi.Engine(scenario, E, A, 128, 72, num_threads=16, params={"episodeLengthSec": 600.0}, depth=depth)
    if final:
        g.set_option("final_obs", 1)
    for e in range(E):
        g.seed_env(e, 42 + e)
    g.reset()
    return g


def workload(scenario, E, A, depth):
    import torch

    off, on = engine(scenario, E, A, depth, False), engine(scenario, E, A, depth, True)
    rng = np.random.default_rng(2)
    acts = torch.from_numpy((1 << rng.integers(0, 11, size=(64, E * A))).astype(np.int32)).cuda()
    zeros = torch.zeros(E, dtype=torch.uint8, device="cuda")
    # env e is asked to end at every step t with (e + t) % 100 == 0: 1 % of the envs per step, each every 100 steps
    bank = torch.stack([torch.from_numpy(((np.arange(E) + t) % 100 == 0).astype(np.uint8)) for t in range(100)]).cuda()
    torch.cuda.synchronize()
    settings = {"off, 0 %": (off, lambda t: zeros.data_ptr()), "off, 1 %": (off, lambda t: bank[t % 100].data_ptr()),
                "on, 0 %": (on, lambda t: zeros.data_ptr()), "on, 1 %": (on, lambda t: bank[t % 100].data_ptr())}
    step = {"off": 0, "on": 0}
    ms = {k: [] for k in settings}
    for _ in range(ROUNDS):
        for name, (g, ends) in settings.items():
            key = name.split(",")[0]
            for i in range(WARMUP + STEPS):
                if i == WARMUP:
                    g.sync()
                    t0 = time.perf_counter()
                g.step_device(acts[step[key] % 64].data_ptr(), ends(step[key]))
                step[key] += 1
            g.sync()
            ms[name].append((time.perf_counter() - t0) * 1e3 / STEPS)
    kern = {k: [] for k in settings}
    for g in (off, on):
        g.set_option("overlap", 0)
    for _ in range(ROUNDS):
        for name, (g, ends) in settings.items():
            key = name.split(",")[0]
            for i in range(WARMUP + TIMED // ROUNDS):
                g.step_device(acts[step[key] % 64].data_ptr(), ends(step[key]))
                step[key] += 1
                g.sync()
                if i >= WARMUP:
                    kern[name].append(g.last_kernel_ms() + (g.last_final_ms(),))
    for name in settings:
        k = np.median(np.array(kern[name]), axis=0)
        print("final_obs %-13s %4d x %d%s | %-8s | %.4f ms/step (rounds %s) | overlap 0: step kernel %.4f ms, raster %.4f ms, terminal frames %.4f ms"
              % (scenario, E, A, " +depth" if depth else "", name, float(np.median(ms[name])), ", ".join("%.4f" % x for x in ms[name]), k[0], k[1], k[2]))
    for g in (off, on):
        assert g.fault_word() == 0
        g.close()


def main():
    print("card:", card())
    for w in WORKLOADS:
        workload(*w)


if __name__ == "__main__":
    main()
