#!/usr/bin/env python
"""Per-env episode control rates.

1. mv_reset_envs of 1, 64 and all envs, without and with seeds: wall time of the call, the reset kernel and the re-render kernel (CUDA
   events, mv_last_kernel_ms) and the host part (wall time less both kernels: the level generation of reseeded envs and of the levels after
   next, the uploads and the synchronisation).
2. The device-resident loop (mv_step_device_ends) at the headline shape, ms per step with d_ends = NULL, with an all-zero mask and with 1 %
   of the envs ending per step, the three settings alternated in one process, three rounds each.

Prints the card's name and power limit with the numbers."""
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from megaverse_b200 import capi  # noqa: E402

RESET_CONFIGS = [("Collect", 1024, 4), ("TowerBuilding", 256, 1)]
LOOP_CONFIG = ("Collect", 1024, 4)
REPS = 10
STEPS, WARMUP, ROUNDS = 300, 30, 3


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
        return out.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown card"


def engine(scenario, E, A):
    g = capi.Engine(scenario, E, A, 128, 72, num_threads=16)
    for e in range(E):
        g.seed_env(e, 42 + e)
    g.reset()
    return g


def reset_rates():
    rng = np.random.default_rng(1)
    for scenario, E, A in RESET_CONFIGS:
        g = engine(scenario, E, A)
        for _ in range(10):
            g.step((1 << rng.integers(0, 11, size=E * A)).astype(np.int32))
        for n in (1, 64, E):
            for seeded in (False, True):
                wall, kern, render = [], [], []
                for rep in range(REPS + 1):
                    envs = rng.choice(E, size=n, replace=False).astype(np.int32)
                    seeds = rng.integers(0, 1 << 30, size=n).astype(np.int32) if seeded else None
                    t0 = time.perf_counter()
                    g.reset_envs(envs, seeds)  # synchronous
                    ms = (time.perf_counter() - t0) * 1e3
                    if rep:  # the first call warms up
                        k, r = g.last_kernel_ms()
                        wall.append(ms); kern.append(k); render.append(r)
                med = [float(np.median(x)) for x in (wall, kern, render)]
                print("reset_envs %-13s %4d x %d: %4d envs %-9s | wall %.3f ms | reset kernel %.3f ms | re-render %.3f ms | host %.3f ms"
                      % (scenario, E, A, n, "reseeded" if seeded else "unseeded", med[0], med[1], med[2], med[0] - med[1] - med[2]))
        assert g.fault_word() == 0
        g.close()


def loop_rates():
    import torch

    scenario, E, A = LOOP_CONFIG
    g = engine(scenario, E, A)
    rng = np.random.default_rng(2)
    acts = torch.from_numpy((1 << rng.integers(0, 11, size=(64, E * A))).astype(np.int32)).cuda()
    zeros = torch.zeros(E, dtype=torch.uint8, device="cuda")
    # env e is asked to end at every step t with (e + t) % 100 == 0: 1 % of the envs per step, each every 100 steps
    bank = torch.stack([torch.from_numpy(((np.arange(E) + t) % 100 == 0).astype(np.uint8)) for t in range(100)]).cuda()
    torch.cuda.synchronize()
    settings = {"NULL": lambda t: 0, "all-zero": lambda t: zeros.data_ptr(), "1% end": lambda t: bank[t % 100].data_ptr()}
    res = {k: [] for k in settings}
    step = 0
    for _ in range(ROUNDS):
        for name, ends in settings.items():
            for i in range(WARMUP + STEPS):
                if i == WARMUP:
                    g.sync()
                    t0 = time.perf_counter()
                g.step_device(acts[step % 64].data_ptr(), ends(step))
                step += 1
            g.sync()
            res[name].append((time.perf_counter() - t0) * 1e3 / STEPS)
    for name, v in res.items():
        print("step_device_ends %-13s %4d x %d, d_ends %-8s: %.4f ms/step (rounds %s)" % (scenario, E, A, name, float(np.median(v)),
                                                                                        ", ".join("%.4f" % x for x in v)))
    assert g.fault_word() == 0
    g.close()


def main():
    print("card:", card())
    reset_rates()
    loop_rates()


if __name__ == "__main__":
    main()
