#!/usr/bin/env python
"""Autoreset-mode rates (option "autoreset").

At the three bench.py workloads, each with a level set of L = 1024 levels, three arms alternated in one process, three rounds each:
  same-step            option autoreset 0 (the default);
  same-step + final    autoreset 0 with option final_obs (the terminal frame in a second buffer, drawn by a second launch);
  next-step            autoreset 1 (the terminal frame is the observation; the env's next call restarts it without a tick).
Each arm runs the device-resident loop (mv_step_device_ends) with 0 % and with 1 % of the envs asked to end per call (env e at every call
t with (e + t) % 100 == 0).  Episodes are long (episodeLengthSec 600), so the only ends are the requested ones.
1. ms per call: host clock around STEPS calls and a synchronise.  Env ticks per second: same-step arms tick every env in every call;
   next-step spends one tick-less call per episode, so at 1 % it ticks E - (envs that ended in the previous call) envs per call.
2. Option overlap 0, a synchronise after every call: the step kernel's time (mv_last_kernel_ms [0]), CUDA events, median over TIMED calls.
3. Memory: the device memory the engine holds after its first reset (cudaMemGetInfo before creation and after the reset), and the pinned
   host bytes the arm adds over same-step, computed from the buffers it allocates.
Prints the card's name and power limit with the numbers."""
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from megaverse_b200 import capi  # noqa: E402

WORKLOADS = [("Collect", 1024, 4, False), ("TowerBuilding", 256, 1, False), ("ObstaclesHard", 2048, 1, True)]
L, STEPS, ROUNDS, TIMED = 1024, 300, 3, 100
ARMS = {"same-step": (0, False), "same-step + final": (0, True), "next-step": (1, False)}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
        return out.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown card"


def engine(torch, scenario, E, A, depth, mode, final):
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    g = capi.Engine(scenario, E, A, 128, 72, num_threads=16, params={"episodeLengthSec": 600.0}, depth=depth)
    if final:
        g.set_option("final_obs", 1)
    if mode:
        g.set_option("autoreset", mode)
    g.set_option("level_set", L)
    for e in range(E):
        g.seed_env(e, 42 + e)
    g.reset()
    g.sync()
    hbm = free0 - torch.cuda.mem_get_info()[0]
    return g, hbm


def pinned_extra(E, N, depth, mode, final):
    """pinned host bytes the arm allocates beyond same-step: the final-frame buffers, or the awaiting flags and their three ring mirrors"""
    px = 128 * 72
    if final:
        return N * px * 4 + (N * px * 4 if depth else 0)
    return 4 * E if mode else 0


def workload(scenario, E, A, depth):
    import torch

    N = E * A
    engines = {}
    for name, (mode, final) in ARMS.items():
        engines[name] = engine(torch, scenario, E, A, depth, mode, final)
    rng = np.random.default_rng(2)
    acts = torch.from_numpy((1 << rng.integers(0, 11, size=(64, N))).astype(np.int32)).cuda()
    zeros = torch.zeros(E, dtype=torch.uint8, device="cuda")
    bank_np = np.stack([((np.arange(E) + t) % 100 == 0).astype(np.uint8) for t in range(100)])
    bank = torch.from_numpy(bank_np).cuda()
    torch.cuda.synchronize()
    rates = {"0 %": lambda t: zeros.data_ptr(), "1 %": lambda t: bank[t % 100].data_ptr()}
    ms = {(a, r): [] for a in ARMS for r in rates}
    kern = {(a, r): [] for a in ARMS for r in rates}
    step = {a: 0 for a in ARMS}
    for _ in range(ROUNDS):
        for arm in ARMS:
            g = engines[arm][0]
            for rate, ends in rates.items():
                g.set_option("overlap", 1)
                for _ in range(20):  # warm, and the previous setting's work drained
                    g.step_device(acts[step[arm] % 64].data_ptr(), ends(step[arm]))
                    step[arm] += 1
                g.sync()
                t0 = time.perf_counter()
                for _ in range(STEPS):
                    g.step_device(acts[step[arm] % 64].data_ptr(), ends(step[arm]))
                    step[arm] += 1
                g.sync()
                ms[(arm, rate)].append((time.perf_counter() - t0) * 1e3 / STEPS)
                g.set_option("overlap", 0)
                k = []
                for _ in range(TIMED):
                    g.step_device(acts[step[arm] % 64].data_ptr(), ends(step[arm]))
                    step[arm] += 1
                    g.sync()
                    k.append(g.last_kernel_ms()[0])
                kern[(arm, rate)].append(float(np.median(k)))
    tag = "%s %d x %d%s, level_set %d" % (scenario, E, A, " +depth" if depth else "", L)
    for (arm, rate), ts in ms.items():
        call_ms = float(np.median(ts))
        # next-step at 1 %: the envs that ended in the previous call run no tick in this one (every call, bank_np[t - 1].sum() of them)
        ticking = E - (float(bank_np.sum(1).mean()) if (arm == "next-step" and rate == "1 %") else 0.0)
        print("autoreset %-36s | %-18s | ends %-4s | %.4f ms per call | %.3f M env ticks/s | step kernel %.4f ms (rounds %s)"
              % (tag, arm, rate, call_ms, ticking / call_ms * 1e-3, float(np.median(kern[(arm, rate)])), ", ".join("%.4f" % x for x in ts)))
    for arm, (g, hbm) in engines.items():
        mode, final = ARMS[arm]
        print("autoreset %-36s | %-18s | engine HBM %.1f MB | pinned beyond same-step %.3f MB (computed)"
              % (tag, arm, hbm / 1e6, pinned_extra(E, N, depth, mode, final) / 1e6))
        assert g.fault_word() == 0
        g.close()


def main():
    print("card:", card())
    print("library:", capi.LIB_PATH)
    for w in WORKLOADS:
        workload(*w)


if __name__ == "__main__":
    main()
