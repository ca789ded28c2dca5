#!/usr/bin/env python
"""State-tensor rates (option "state_tensors").

At the three bench.py workloads, the option off and on alternated in one process, three rounds each:
1. mv_step_device: ms per call, host clock around 300 calls and a synchronise (the rows stay in HBM);
2. mv_step (host-facing; the rows come down in one copy on the copy stream): ms per call over 100 calls;
3. option overlap 0, a synchronise after every call: the step kernel's time (mv_last_kernel_ms [0], CUDA events), median of 100 calls;
4. the device loop again with option final_obs on as well and 1 % of the envs asked to end per call (terminal rows written).
Episodes are long (episodeLengthSec 600), so the only ends are the requested ones.  Prints the card's name and power limit with the numbers."""
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


def engine(scenario, E, A, depth, state, final=False):
    g = capi.Engine(scenario, E, A, 128, 72, num_threads=16, params={"episodeLengthSec": 600.0}, depth=depth)
    if state:
        g.set_option("state_tensors", 1)
    if final:
        g.set_option("final_obs", 1)
    for e in range(E):
        g.seed_env(e, 42 + e)
    g.reset()
    return g


def timed_device(g, acts, ends, n):
    for i in range(WARMUP + n):
        if i == WARMUP:
            g.sync()
            t0 = time.perf_counter()
        g.step_device(acts[i % len(acts)].data_ptr(), ends(i))
    g.sync()
    return (time.perf_counter() - t0) * 1e3 / n


def workload(scenario, E, A, depth):
    import torch

    rng = np.random.default_rng(2)
    host_acts = (1 << rng.integers(0, 11, size=(64, E * A))).astype(np.int32)
    acts = torch.from_numpy(host_acts).cuda()
    zeros = torch.zeros(E, dtype=torch.uint8, device="cuda")
    bank = torch.stack([torch.from_numpy(((np.arange(E) + t) % 100 == 0).astype(np.uint8)) for t in range(100)]).cuda()
    engines = {"off": engine(scenario, E, A, depth, False), "on": engine(scenario, E, A, depth, True),
               "off +final": engine(scenario, E, A, depth, False, True), "on +final": engine(scenario, E, A, depth, True, True)}
    torch.cuda.synchronize()
    dev = {k: [] for k in engines}
    host = {k: [] for k in ("off", "on")}
    for _ in range(ROUNDS):
        for name, g in engines.items():
            dev[name].append(timed_device(g, acts, (lambda t: bank[t % 100].data_ptr()) if "final" in name else (lambda t: zeros.data_ptr()), STEPS))
        for name in host:
            g = engines[name]
            for i in range(WARMUP + HOST_STEPS):
                if i == WARMUP:
                    t0 = time.perf_counter()
                g.step(host_acts[i % 64])
            host[name].append((time.perf_counter() - t0) * 1e3 / HOST_STEPS)
    kern = {k: [] for k in ("off", "on")}
    for name in kern:
        engines[name].set_option("overlap", 0)
    for _ in range(ROUNDS):
        for name in kern:
            g = engines[name]
            for i in range(WARMUP + TIMED // ROUNDS):
                g.step_device(acts[i % 64].data_ptr(), zeros.data_ptr())
                g.sync()
                if i >= WARMUP:
                    kern[name].append(g.last_kernel_ms()[0])
    tag = "%s %d x %d%s" % (scenario, E, A, " +depth" if depth else "")
    for name in ("off", "on"):
        print("state_tensors %-24s | %-3s | mv_step_device %.4f ms (rounds %s) | mv_step %.4f ms (rounds %s) | overlap 0: step kernel %.4f ms"
              % (tag, name, float(np.median(dev[name])), ", ".join("%.4f" % x for x in dev[name]), float(np.median(host[name])),
                 ", ".join("%.4f" % x for x in host[name]), float(np.median(kern[name]))))
    for name in ("off +final", "on +final"):
        print("state_tensors %-24s | %-10s 1 %% ends | mv_step_device_ends %.4f ms (rounds %s)"
              % (tag, name, float(np.median(dev[name])), ", ".join("%.4f" % x for x in dev[name])))
    for g in engines.values():
        assert g.fault_word() == 0
        g.close()


def main():
    print("card:", card())
    for w in WORKLOADS:
        workload(*w)


if __name__ == "__main__":
    main()
