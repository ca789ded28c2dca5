#!/usr/bin/env python
"""Stream-step rates (mv_step_stream): what a CUDA graph gains over eager calls.

At the three bench.py workloads, each with a level set of L = 1024 levels, the arms alternated in one process, three rounds each, ms per
step from a host clock around STEPS steps and a device synchronise.  Every arm runs on a torch side stream, which the stream steps fork
from and join back to (a null handle would leave them unordered against the policy's kernels), and option overlap is set outside the
timed window:
1. device loop: mv_step_device on an engine that never takes a stream step (engine-owned actions);
2. eager mv_step_stream on the torch stream, option overlap 1 and 0;
3. replays of a graph of K = 32 stream steps, captured at overlap 1 and at overlap 0 (the two differ only if stream capture keeps the
   programmatic edge between the step kernel and its raster launch);
4. a small torch CNN policy on the obs in the loop: policy then mv_step_stream eagerly, against replays of one graph of 32 (policy, step)
   pairs.
Prints the card's name and power limit with the numbers."""
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from megaverse_b200 import capi  # noqa: E402

WORKLOADS = [("Collect", 1024, 4, False), ("TowerBuilding", 256, 1, False), ("ObstaclesHard", 2048, 1, True)]
L, K, STEPS, ROUNDS = 1024, 32, 320, 3


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
        return out.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown card"


def engine(scenario, E, A, depth):
    g = capi.Engine(scenario, E, A, 128, 72, num_threads=16, depth=depth)
    g.set_option("zero_copy", 0)  # the reset's frames in HBM too: the policy reads them
    g.set_option("level_set", L)
    for e in range(E):
        g.seed_env(e, 42 + e)
    g.reset()
    return g


class Policy:
    """obs uint8[N, 72, 128, 4] -> one action bit per agent: two small convolutions, a mean, a linear layer, the arg max"""

    def __init__(self, torch):
        nn = torch.nn
        torch.manual_seed(0)
        self.torch = torch
        self.net = nn.Sequential(nn.Conv2d(4, 8, 8, stride=8), nn.ReLU(), nn.Conv2d(8, 16, 3, stride=2), nn.ReLU(), nn.AdaptiveAvgPool2d(1),
                                 nn.Flatten(), nn.Linear(16, 11)).cuda().eval()

    def __call__(self, obs):
        with self.torch.no_grad():
            x = obs.permute(0, 3, 1, 2).float() * (1.0 / 255.0)
            i = self.net(x).argmax(1)
            return self.torch.bitwise_left_shift(self.torch.ones_like(i), i).to(self.torch.int32)


def workload(scenario, E, A, depth):
    import torch

    dev, st = engine(scenario, E, A, depth), engine(scenario, E, A, depth)
    policy = Policy(torch)
    obs = torch.as_tensor(st.device_array("obs"), device="cuda")
    masks = torch.zeros((K, st.N), dtype=torch.int32, device="cuda")
    pol_masks = torch.zeros((K, st.N), dtype=torch.int32, device="cuda")

    def eager_stream():
        s = torch.cuda.current_stream().cuda_stream
        for i in range(STEPS):
            st.step_stream(s, masks[i % K].data_ptr())

    def capture(body):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            s = torch.cuda.current_stream().cuda_stream
            for k in range(K):
                body(s, k)
        return g

    def step_k(s, k):
        st.step_stream(s, masks[k].data_ptr())

    def policy_k(s, k):
        pol_masks[k].copy_(policy(obs))
        st.step_stream(s, pol_masks[k].data_ptr())

    # warm-up: the first stream step (stream mode), the policy's kernels, then the graphs
    eager_stream()
    pol_masks[0].copy_(policy(obs))
    torch.cuda.synchronize()
    graphs = {}
    for ov in (1, 0):
        st.set_option("overlap", ov)
        graphs[ov] = capture(step_k)
    st.set_option("overlap", 1)
    graphs["policy"] = capture(policy_k)
    torch.cuda.synchronize()

    def policy_eager():
        s = torch.cuda.current_stream().cuda_stream
        for i in range(STEPS):
            pol_masks[i % K].copy_(policy(obs))
            st.step_stream(s, pol_masks[i % K].data_ptr())

    def replays(name):
        for _ in range(STEPS // K):
            graphs[name].replay()

    # name: (option overlap of the stream engine while the arm runs, the arm)
    arms = {
        "device loop (mv_step_device)": (1, lambda: [dev.step_device(None) for _ in range(STEPS)]),
        "eager mv_step_stream, overlap 1": (1, eager_stream),
        "eager mv_step_stream, overlap 0": (0, eager_stream),
        "graph of 32 stream steps, overlap 1": (1, lambda: replays(1)),
        "graph of 32 stream steps, overlap 0": (1, lambda: replays(0)),
        "CNN policy + mv_step_stream, eager": (1, policy_eager),
        "CNN policy + mv_step_stream, graph of 32": (1, lambda: replays("policy")),
    }
    times = {k: [] for k in arms}
    for _ in range(ROUNDS):
        for name, (ov, fn) in arms.items():
            st.set_option("overlap", ov)
            fn()  # one untimed pass: warm, and the previous arm's work drained
            dev.sync()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            if name.startswith("device loop"):
                dev.sync()
            torch.cuda.synchronize()
            times[name].append((time.perf_counter() - t0) * 1e3 / STEPS)
    tag = "%s %d x %d%s, level_set %d" % (scenario, E, A, " +depth" if depth else "", L)
    for name, ts in times.items():
        print("stream_steps %-40s | %-42s | %.4f ms per step (rounds %s)" % (tag, name, float(np.median(ts)), ", ".join("%.4f" % x for x in ts)))
    for g in (dev, st):
        assert g.fault_word() == 0
        g.close()


def main():
    print("card:", card())
    print("library:", capi.LIB_PATH)
    import torch

    with torch.cuda.stream(torch.cuda.Stream()):
        for w in WORKLOADS:
            workload(*w)


if __name__ == "__main__":
    main()
