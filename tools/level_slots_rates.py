#!/usr/bin/env python
"""Level-slot rates (option "level_slots" 2 or 4).

1. Collect 1 024 x 4 on bench.py's env seeds (42 + env) and action stream (one random action bit per agent per call) at action_repeat
   k = 1, 2, 4: the asynchronous mv_step_device at level_slots 4 against mv_step with obs_to_host 0 at level_slots 2 (the arrangement the
   action-repeat measurements had to use, since level_slots 2 refuses the short episodes these seeds hold at k >= 2).  Alternated in one
   process, three rounds of 300 calls; ms per call (host clock around the calls, ending in a device synchronisation) and env ticks per second.
2. The cost of the deeper queue: mv_step_device at k = 1, level_slots 2 against 4, with 1 % of the envs asked to end per call
   (mv_step_device_ends), as in final_obs_rates.py.
3. First mv_reset wall time at level_slots 2 and 4, HBM and pinned bytes of the level arrays (from the code's layout), mv_state_row_bytes.
Prints the card's name and power limit with the numbers."""
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from megaverse_b200 import capi  # noqa: E402

E, A = 1024, 4
REPEATS = (1, 2, 4)
STEPS, WARMUP, ROUNDS = 300, 30, 3


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
        return out.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown card"


def engine(k, slots, timed_reset=False):
    g = capi.Engine("Collect", E, A, 128, 72, num_threads=16)
    g.set_option("action_repeat", k)
    g.set_option("level_slots", slots)
    g.set_option("obs_to_host", 0)
    for e in range(E):
        g.seed_env(e, 42 + e)  # bench.py's seeds
    t0 = time.perf_counter()
    g.reset()
    return (g, (time.perf_counter() - t0) * 1e3) if timed_reset else g


def main():
    import torch

    print("card:", card())
    rng = np.random.default_rng(1)  # bench.py's action stream
    acts = (1 << rng.integers(0, 11, size=(64, E * A))).astype(np.int32)
    dacts = torch.from_numpy(acts).cuda()
    ends_rng = np.random.default_rng(2)
    ends = torch.from_numpy((ends_rng.random((64, E)) < 0.01).astype(np.uint8)).cuda()
    torch.cuda.synchronize()
    step_bytes = E * A * 4

    # ---- 1. asynchronous at 4 slots against synchronous at 2 slots
    runs = {}
    for k in REPEATS:
        runs[(k, "device4")] = engine(k, 4)
        runs[(k, "host2")] = engine(k, 2)
    pos = {key: 0 for key in runs}
    ms = {key: [] for key in runs}

    def call(key, g):
        i = pos[key] % 64
        if key[1] == "host2":
            g.step(acts[i])
        elif key[1] == "ends":
            g.step_device(dacts.data_ptr() + i * step_bytes, ends[i].data_ptr())
        else:
            g.step_device(dacts.data_ptr() + i * step_bytes)
        pos[key] += 1

    for _ in range(ROUNDS):
        for key, g in runs.items():
            for i in range(WARMUP + STEPS):
                if i == WARMUP:
                    g.sync()
                    t0 = time.perf_counter()
                call(key, g)
            g.sync()
            ms[key].append((time.perf_counter() - t0) * 1e3 / STEPS)
    for k in REPEATS:
        for how, label in (("device4", "mv_step_device, level_slots 4"), ("host2", "mv_step obs_to_host 0, level_slots 2")):
            m = float(np.median(ms[(k, how)]))
            print("Collect %d x %d | k=%d | %-38s | %.4f ms/call (rounds %s) | %.0f env ticks/s"
                  % (E, A, k, label, m, ", ".join("%.4f" % x for x in ms[(k, how)]), E * k * 1e3 / m))
    for g in runs.values():
        assert g.fault_word() == 0
        g.close()

    # ---- 2. the deeper queue at k = 1 with 1 % requested ends per call
    runs = {(1, "ends", 2): engine(1, 2), (1, "ends", 4): engine(1, 4)}
    pos = {key: 0 for key in runs}
    ms = {key: [] for key in runs}
    for _ in range(ROUNDS):
        for key, g in runs.items():
            for i in range(WARMUP + STEPS):
                if i == WARMUP:
                    g.sync()
                    t0 = time.perf_counter()
                call(key, g)
            g.sync()
            ms[key].append((time.perf_counter() - t0) * 1e3 / STEPS)
    for key in runs:
        m = float(np.median(ms[key]))
        print("Collect %d x %d | k=1, 1%% of envs ending per call | mv_step_device_ends, level_slots %d | %.4f ms/call (rounds %s)"
              % (E, A, key[2], m, ", ".join("%.4f" % x for x in ms[key])))
    for g in runs.values():
        assert g.fault_word() == 0
        g.close()

    # ---- 3. reset time and memory
    for slots in (2, 4):
        times, rows = [], 0
        for _ in range(3):
            g, t = engine(1, slots, timed_reset=True)
            times.append(t)
            rows = g.state_row_bytes()
            g.close()
        print("Collect %d x %d | level_slots %d | first mv_reset %.0f ms (runs %s) | mv_state_row_bytes %d"
              % (E, A, slots, float(np.median(times)), ", ".join("%.0f" % x for x in times), rows))
    # the level arrays per env and slot, in HBM and again pinned: MvLevel, static boxes and rotations at the default static_cap, one
    # decoration, three bit planes of the Collect grid
    slot = 33248 + 768 * 40 + 80 + 12 * ((74 * 62 * 74 + 127) // 128 * 4)
    for slots in (2, 4):
        print("Collect %d envs | level_slots %d | level arrays %.0f MB in HBM and %.0f MB pinned" % (E, slots, E * slots * slot / 1e6, E * slots * slot / 1e6))


if __name__ == "__main__":
    main()
