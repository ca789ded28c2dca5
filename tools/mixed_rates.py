#!/usr/bin/env python
"""Megaverse-8 mixed batch (BASELINE config 5's shape: 1 024 envs x 1 agent, 128x72, global env i runs MEGAVERSE8[i % 8], seeded 42 + i,
bench.py's action stream) in two arrangements:

  (a) eight single-scenario engines on eight streams rasterising into blocks of one obs tensor: bench.measure_mixed(gather=False)
  (b) one mixed-scenario engine (mv_create_mixed), one step kernel and one raster launch per step, driven by step_device

Timed: (a) and (b) alternately, REPS times each in one process, both as measure_mixed times it (events around K back-to-back steps) and
(b) also with the L2 flushed before every step (bench.py's timed_flushed).  Untimed, in a separate run: kernel launches per step, the step
and raster kernels' times with option overlap off (for (a) the eight engines' kernels summed, each engine stepped on its own), and an
exact output check -- both arrangements stepped CHECK_STEPS steps with every global env given the same mask, (b)'s obs tensor, rewards
and dones permuted into (a)'s per-scenario blocks must be byte-identical.  Prints one JSON line with the card's name and power limit."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("BOXOBAN_LEVELS", os.path.join(ROOT, "tests", "golden", "boxoban"))
import bench  # noqa: E402

MEGAVERSE8, W, H = bench.MEGAVERSE8, bench.W, bench.H
E = bench.MIXED_ENVS_PER_GPU
PER = E // len(MEGAVERSE8)
K, WARMUP, REPS, CHECK_STEPS, KERNEL_STEPS = 100, 10, 3, 200, 30


def block_index():
    """position of global env i (= e*8 + k, scenario k) in (a)'s per-scenario blocks: k*PER + e"""
    i = np.arange(E)
    return (i % len(MEGAVERSE8)) * PER + i // len(MEGAVERSE8)


def mixed_engine(cores):
    from megaverse_b200 import capi

    g = capi.Engine([MEGAVERSE8[i % len(MEGAVERSE8)] for i in range(E)], E, 1, W, H, num_threads=max(1, min(16, cores)))
    for i in range(E):
        g.seed_env(i, 42 + i)
    g.reset()
    return g


def single_engines(cores, obs):
    """measure_mixed's arrangement: engine k holds global envs e*8 + k and draws into obs[k*PER:(k+1)*PER]"""
    from megaverse_b200 import capi

    engines = []
    for k, scenario in enumerate(MEGAVERSE8):
        g = capi.Engine(scenario, PER, 1, W, H, num_threads=max(1, min(16, cores) // 2))
        g.set_obs_buffer(obs[k * PER:(k + 1) * PER].data_ptr())
        for e in range(PER):
            g.seed_env(e, 42 + e * len(MEGAVERSE8) + k)
        g.reset()
        engines.append(g)
    return engines


def time_mixed(hz, torch, cores, masks_b):
    """(b) timed as measure_mixed times (a): events around K back-to-back steps; then with the L2 flushed before every step"""
    g = mixed_engine(cores)
    stream = torch.cuda.ExternalStream(g.stream())
    ptr0 = masks_b.data_ptr()

    def step(t):
        g.step_device(ptr0 + (t % masks_b.shape[0]) * E * 4)

    for t in range(WARMUP):
        step(t)
    g.sync()
    ms_window = hz.timed(stream, step, K, WARMUP)
    g.sync()
    ms_flushed = hz.timed_flushed(stream, g.sync, step, K, WARMUP + K)
    faults = g.faults()
    g.close()
    return {"ms_per_step": ms_window / K, "value": E * K / (ms_window / 1e3), "ms_per_step_l2_flushed": ms_flushed / K,
            "value_l2_flushed": E * K / (ms_flushed / 1e3), "faults": int(faults)}


def check_and_count(torch, cores, masks_a, masks_b):
    """untimed: launches per step, kernel times with overlap off, and (b) against (a) byte for byte over CHECK_STEPS steps"""
    obs_a = torch.empty((E, H, W, 4), dtype=torch.uint8, device="cuda")
    engines = single_engines(cores, obs_a)
    g = mixed_engine(cores)
    pos = torch.from_numpy(block_index()).cuda()  # (b)'s row i goes to (a)'s row pos[i]
    torch.cuda.synchronize()
    la0, lb0 = sum(x.kernel_launches() for x in engines), g.kernel_launches()
    mismatches = []
    for t in range(CHECK_STEPS):
        for k, x in enumerate(engines):
            x.step_device(masks_a.data_ptr() + ((t % masks_a.shape[0]) * E + k * PER) * 4)
        g.step_device(masks_b.data_ptr() + (t % masks_b.shape[0]) * E * 4)
        for x in engines:
            x.sync()
        g.sync()
        obs_b = torch.as_tensor(g.device_array("obs"), device="cuda")
        rew_a = torch.cat([torch.as_tensor(x.device_array("rewards"), device="cuda") for x in engines])
        done_a = torch.cat([torch.as_tensor(x.device_array("dones"), device="cuda") for x in engines])
        rew_b = torch.empty_like(rew_a).index_copy_(0, pos, torch.as_tensor(g.device_array("rewards"), device="cuda"))
        done_b = torch.empty_like(done_a).index_copy_(0, pos, torch.as_tensor(g.device_array("dones"), device="cuda"))
        same_obs = torch.equal(torch.empty_like(obs_a).index_copy_(0, pos, obs_b), obs_a)
        same_rew = torch.equal(rew_a.view(torch.int32), rew_b.view(torch.int32))
        if not (same_obs and same_rew and torch.equal(done_a, done_b)):
            mismatches.append(t)
    launches_a = (sum(x.kernel_launches() for x in engines) - la0) / CHECK_STEPS
    launches_b = (g.kernel_launches() - lb0) / CHECK_STEPS
    # kernel times, kernels back to back (overlap off); (a): each engine stepped and waited for on its own, the eight summed
    for x in engines + [g]:
        x.set_option("overlap", 0)
    ka, kb = [], []
    for t in range(CHECK_STEPS, CHECK_STEPS + 4 + KERNEL_STEPS):
        s = r = 0.0
        for k, x in enumerate(engines):
            x.step_device(masks_a.data_ptr() + ((t % masks_a.shape[0]) * E + k * PER) * 4)
            x.sync()
            sm, rm = x.last_kernel_ms()
            s += sm; r += rm
        g.step_device(masks_b.data_ptr() + (t % masks_b.shape[0]) * E * 4)
        g.sync()
        if t >= CHECK_STEPS + 4:  # the first four settle the serialised mode
            ka.append((s, r)); kb.append(g.last_kernel_ms())
    faults = sum(x.faults() for x in engines) + g.faults()
    for x in engines + [g]:
        x.close()
    ka, kb = np.array(ka), np.array(kb)
    return {"launches_per_step": {"a": launches_a, "b": launches_b},
            "kernel_ms_overlap_off": {"a_step_sum_of_8": float(ka[:, 0].mean()), "a_raster_sum_of_8": float(ka[:, 1].mean()),
                                      "b_step": float(kb[:, 0].mean()), "b_raster": float(kb[:, 1].mean())},
            "outputs_identical": not mismatches, "mismatched_steps": mismatches[:10], "check_steps": CHECK_STEPS, "faults": int(faults)}


def main():
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("mixed_rates.py needs a CUDA device")
    torch.cuda.set_device(0)
    cores = os.cpu_count() or 1
    hz = bench.Harness(torch, None, 1, 0)
    # bench.measure_mixed's action stream: row t, position k*PER + e is global env e*8 + k; (b) takes the same masks in global order
    acts_a = bench.action_stream(64, E, 101)
    acts_b = np.empty_like(acts_a)
    acts_b[:, :] = acts_a[:, block_index()]
    masks_a, masks_b = torch.from_numpy(acts_a).cuda(), torch.from_numpy(acts_b).cuda()
    torch.cuda.synchronize()

    checked = check_and_count(torch, cores, masks_a, masks_b)
    runs = {"a": [], "b": []}
    for _ in range(REPS):
        runs["a"].append(bench.measure_mixed(hz, K, WARMUP, 0, cores, gather=False))
        runs["b"].append(time_mixed(hz, torch, cores, masks_b))
    summary = {}
    for arm, recs in runs.items():
        ms = [r["ms_per_step"] for r in recs]
        summary[arm] = {"ms_per_step": ms, "obs_per_s": [E / (m / 1e3) for m in ms], "median_ms": float(np.median(ms))}
    summary["b"]["ms_per_step_l2_flushed"] = [r["ms_per_step_l2_flushed"] for r in runs["b"]]
    print(json.dumps({"workload": "Megaverse-8 mixed, %d envs x 1 agent, 128x72 RGB, global env i runs MEGAVERSE8[i %% 8], seed 42 + i" % E,
                      "arrangements": {"a": "eight single-scenario engines on eight streams (bench.measure_mixed, gather=False)",
                                       "b": "one mv_create_mixed engine, step_device"},
                      "timing": "events around %d back-to-back steps after %d warm-up steps (measure_mixed's window); (a) and (b) alternated %d times" % (K, WARMUP, REPS),
                      "timed": summary, "untimed": checked,
                      "gpu": {"name": torch.cuda.get_device_name(0), "power_limit_w": bench.power_limit(0)}}))


if __name__ == "__main__":
    main()
