#!/usr/bin/env python
"""Level-set rates: what an episode end costs when the next level is a row of a bank in HBM (option "level_set") instead of a level the
host generates (the stream engine at level_slots 2 and 4).  Collect 1 024 x 4, the arms alternated in one process.

1. The device-resident loop (mv_step_device_ends) with 0 %, 1 % and 10 % of the envs ending per call: ms per call, three rounds of 300
   calls, median and the rounds; then, in a separate pass with option overlap 0, the step and raster kernel times (CUDA events).
2. The same loop at action_repeat 4 with natural ends only.
3. mv_reset_envs of 1, 64 and 1 024 envs, unseeded and reseeded: wall, reset kernel, re-render, host.
4. The first mv_reset and the HBM the engine takes, at L = 64, 1 024 and 8 192 against the stream engine at level_slots 2 and 4.

Fails without a GPU.  Prints the card's name and power limit with the numbers."""
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from megaverse_b200 import capi  # noqa: E402

SCENARIO, E, A = "Collect", 1024, 4
STEPS, WARMUP, ROUNDS = 300, 30, 3
ARMS = {"stream D=2": {"level_slots": 2}, "stream D=4": {"level_slots": 4}, "level set L=1024": {"level_set": 1024}}


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
    return out.strip().splitlines()[0]


def engine(opts, reset=True):
    g = capi.Engine(SCENARIO, E, A, 128, 72, num_threads=16)
    for k, v in opts.items():
        g.set_option(k, v)
    for e in range(E):
        g.seed_env(e, 42 + e)
    if reset:
        g.reset()
    return g


def end_masks(percent):
    """env e is asked to end at every call t with (e + t) % period == 0; None: no mask"""
    import torch

    if not percent:
        return None
    period = 100 // percent
    return torch.stack([torch.from_numpy(((np.arange(E) + t) % period == 0).astype(np.uint8)) for t in range(period)]).cuda()


def loop_rates(k):
    import torch

    rng = np.random.default_rng(2)
    acts = torch.from_numpy((1 << rng.integers(0, 11, size=(64, E * A))).astype(np.int32)).cuda()
    rates = (0, 1, 10) if k == 1 else (0,)
    masks = {p: end_masks(p) for p in rates}
    engines = {name: engine(dict(opts, action_repeat=k)) for name, opts in ARMS.items()}
    torch.cuda.synchronize()
    res = {(name, p): [] for name in engines for p in rates}
    ends_seen = {key: 0 for key in res}
    step = 0

    def call(g, p):
        m = masks[p]
        g.step_device(acts[step % 64].data_ptr(), 0 if m is None else m[step % m.shape[0]].data_ptr())

    for _ in range(ROUNDS):
        for p in rates:
            for name, g in engines.items():
                for i in range(WARMUP + STEPS):
                    if i == WARMUP:
                        g.sync()
                        t0 = time.perf_counter()
                    call(g, p)
                    step += 1
                g.sync()
                res[(name, p)].append((time.perf_counter() - t0) * 1e3 / STEPS)
    for (name, p), v in res.items():
        print("loop k=%d %-17s %2d %% requested ends: %.4f ms/call (rounds %s)" % (k, name, p, float(np.median(v)), ", ".join("%.4f" % x for x in v)))
    # kernel times: the kernels one after the other (overlap 0), every call synchronised and read
    for g in engines.values():
        g.sync()
        g.set_option("overlap", 0)
    for p in rates:
        for name, g in engines.items():
            ks, kr, n_end = [], [], 0
            for i in range(20 + 100):
                call(g, p)
                step += 1
                g.sync()
                if i >= 20:
                    a, b = g.last_kernel_ms()
                    ks.append(a); kr.append(b)
                    n_end += int(np.array(g.dones()).sum())
            print("kernels k=%d %-17s %2d %% requested ends: step %.4f ms, raster %.4f ms (medians of 100 calls, %.1f ends per call)"
                  % (k, name, p, float(np.median(ks)), float(np.median(kr)), n_end / 100.0))
    for g in engines.values():
        assert g.fault_word() == 0
        g.close()


def reset_rates():
    rng = np.random.default_rng(1)
    for name in ("stream D=2", "level set L=1024"):
        g = engine(ARMS[name])
        for _ in range(10):
            g.step((1 << rng.integers(0, 11, size=E * A)).astype(np.int32))
        for n in (1, 64, E):
            for seeded in (False, True):
                wall, kern, render = [], [], []
                for rep in range(6):
                    envs = rng.choice(E, size=n, replace=False).astype(np.int32)
                    seeds = rng.integers(0, 1 << 30, size=n).astype(np.int32) if seeded else None
                    t0 = time.perf_counter()
                    g.reset_envs(envs, seeds)  # synchronous
                    ms = (time.perf_counter() - t0) * 1e3
                    if rep:  # the first call warms up
                        a, b = g.last_kernel_ms()
                        wall.append(ms); kern.append(a); render.append(b)
                med = [float(np.median(x)) for x in (wall, kern, render)]
                print("reset_envs %-17s %4d envs %-9s | wall %.3f ms | reset kernel %.3f ms | re-render %.3f ms | host %.3f ms"
                      % (name, n, "reseeded" if seeded else "unseeded", med[0], med[1], med[2], med[0] - med[1] - med[2]))
        assert g.fault_word() == 0
        g.close()


def first_reset():
    import torch

    arms = [("stream D=2", {"level_slots": 2}), ("stream D=4", {"level_slots": 4})] + [("level set L=%d" % L, {"level_set": L}) for L in (64, 1024, 8192)]
    for name, opts in arms:
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        g = engine(opts, reset=False)
        t0 = time.perf_counter()
        g.reset()
        ms = (time.perf_counter() - t0) * 1e3
        used = free0 - torch.cuda.mem_get_info()[0]
        print("first reset %-17s: %.1f ms, engine HBM %.1f MiB, static_cap %d, state row %d B" % (name, ms, used / 2**20, g.static_cap(), g.state_row_bytes()))
        g.close()


def main():
    import torch

    if not torch.cuda.is_available():
        sys.exit("level_set_rates needs a GPU")
    print("card:", card())
    first_reset()
    reset_rates()
    loop_rates(1)
    loop_rates(4)


if __name__ == "__main__":
    main()
