#!/usr/bin/env python3
"""bench_region.py -- cost of a render region (vpt_set_render_region) on the headline frame, on one GPU.

    python tools/bench_region.py [--config C] [--steps K] [--warmup W] [--profile-frames P]

The workload is bench.py's (BASELINE.json configuration 2 by default: dragon.vdb 1920x1080 64 spp, ray_depth 100, sun + HDRI).  One
renderer runs steps of SPP passes, each a new frame at iteration 0 (where a region takes effect), under four regions, alternated: the
full frame, a 480x270 region on the dragon (the frame's centre), the same size in the empty sky of the top-left corner, and a 1x1 region.
CUDA events around each step, L2 flushed before each, median per step.  Then, with the "profile" option, P steps of each for the
per-kernel device time.  Prints ONE JSON line with both and the card name and power limit read in the same run.  Writes nothing to the tree.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np
import torch

import bench as B
from bench_adaptive import gpu_identity


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, default=2, help="BASELINE.json configuration (bench.py's workloads)")
    ap.add_argument("--steps", type=int, default=20, help="timed steps of each region")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile-frames", type=int, default=3)
    args = ap.parse_args()
    args.warmup = max(args.warmup, 1)
    torch.cuda.set_device(0)

    import vpt_b200 as V
    dev = "cuda:0"
    wl = B.build_workload(V, args.config, dev)
    scene, W, H, SPP = wl["scene"], wl["width"], wl["height"], wl["spp"]
    stream = torch.cuda.current_stream().cuda_stream
    flush_buf = torch.zeros(64 * 1024 * 1024, dtype=torch.float32, device=dev)
    sampler = B.ClockSampler(0)
    rw, rh = W // 4, H // 4
    regions = {"full": None, "dragon_480x270": ((W - rw) // 2, (H - rh) // 2, (W + rw) // 2, (H + rh) // 2),
               "sky_480x270": (0, 0, rw, rh), "1x1": (W // 2, H // 2, W // 2 + 1, H // 2 + 1)}

    r = V.Renderer(scene, W, H, kp=wl["kp"])

    def step(name):
        reg = regions[name]
        if reg is None: r.clear_region()
        else: r.set_region(*reg)
        r.kp.iteration = 0
        r.render(SPP, stream=stream)

    for _ in range(args.warmup):
        for name in regions: step(name)
    torch.cuda.synchronize()
    ms = {name: [] for name in regions}
    sampler.start()
    tw0 = time.time()
    for _ in range(args.steps):                                  # alternate: every region sees the same clocks and neighbours
        for name in regions:
            B.flush_l2(flush_buf)
            a = torch.cuda.Event(enable_timing=True); b = torch.cuda.Event(enable_timing=True)
            a.record(); step(name); b.record()
            b.synchronize()
            ms[name].append(a.elapsed_time(b))
    sampler.window(tw0, time.time())
    clocks = sampler.stop()

    # per-kernel device time per step, from the CUDA events of the "profile" option
    r.set_option("profile", 1); r.kernel_times()
    kernels = {name: [] for name in regions}
    for _ in range(args.profile_frames):
        for name in regions:
            step(name); torch.cuda.synchronize()
            kernels[name].append(r.kernel_times())
    r.set_option("profile", 0)
    per_kernel = {}
    for name, ks in kernels.items():
        per_kernel[name] = {k: float(np.median([kt[k]["ms"] for kt in ks])) for k in ks[0]}

    med = {name: float(np.median(v)) for name, v in ms.items()}
    line = {"metric": "ms per step under a render region", "value": med["dragon_480x270"], "unit": "ms/step", "higher_is_better": False,
            "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "gpu": gpu_identity(),
            "regions": {name: list(reg) if reg else None for name, reg in regions.items()},
            "ms_per_step": med, "ms_per_step_spread": {name: [float(min(v)), float(max(v))] for name, v in ms.items()},
            "kernel_ms_per_step": per_kernel, "profile_frames": args.profile_frames,
            "timing": "median of CUDA-event times per step, regions alternated, L2 flushed before each",
            "workload": wl["name"], "width": W, "height": H, "spp": SPP, "clocks": clocks}
    print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
