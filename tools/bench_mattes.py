#!/usr/bin/env python3
"""bench_mattes.py -- cost of the instance mattes (vpt_set_instance_mattes) on bench.py's workloads, on one GPU.

    python tools/bench_mattes.py [--config C] [--steps K] [--warmup W] [--profile-frames P] [--mattes 1,8]

The workload is bench.py's (BASELINE.json configuration 2 by default: dragon.vdb 1920x1080 64 spp; configuration 5 is the instanced
scene).  One renderer alternates frames with the mattes off and with K mattes for every K of --mattes (instance i in matte i mod K, the
sphere in matte 0; a buffer per K, registered before its frame; every frame starts at iteration 0, where a registration takes effect),
CUDA events around each frame, L2 flushed before each, median per frame.  Then, with the "profile" option, P frames of each, alternated,
for the generate / trace / resolve device time per frame.  Prints ONE JSON line with both, the trace kernel's rays per lane, the card
name and power limit read in the same run, and whether accum came out bit-identical with the mattes on.  Writes nothing to the tree.
"""
import argparse
import ctypes as C
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
    ap.add_argument("--steps", type=int, default=10, help="timed frames of each kind")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile-frames", type=int, default=3)
    ap.add_argument("--mattes", default="1,8", help="matte counts K to time against mattes off")
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

    r = V.Renderer(scene, W, H, kp=wl["kp"])
    n_inst = len(scene.instances)
    ks = [int(k) for k in args.mattes.split(",")]
    kinds = [0] + ks
    mattes = {k: torch.zeros(k, r.n_local, 4, dtype=torch.float32, device=dev) for k in ks}
    maps = {k: (C.c_int * n_inst)(*[i % k for i in range(n_inst)]) for k in ks}

    def use(k):
        if k == 0:
            V._native.check(V.lib.vpt_set_instance_mattes(r.ctx, None, 0, None, 0, -1), r.ctx, "vpt_set_instance_mattes")
        else:
            V._native.check(V.lib.vpt_set_instance_mattes(r.ctx, C.c_void_p(mattes[k].data_ptr()), k, maps[k], n_inst, 0), r.ctx,
                            "vpt_set_instance_mattes")

    def step(k):
        use(k)
        r.kp.iteration = 0
        r.render(SPP, stream=stream)

    for _ in range(args.warmup):
        for k in kinds: step(k)
    torch.cuda.synchronize()
    ms = {k: [] for k in kinds}
    sampler.start()
    tw0 = time.time()
    for _ in range(args.steps):                                  # alternate: every kind sees the same clocks and neighbours
        for k in kinds:
            B.flush_l2(flush_buf)
            a = torch.cuda.Event(enable_timing=True); b = torch.cuda.Event(enable_timing=True)
            a.record(); step(k); b.record()
            b.synchronize()
            ms[k].append(a.elapsed_time(b))
    sampler.window(tw0, time.time())
    clocks = sampler.stop()

    # generate / trace / resolve time per frame, from the per-kernel CUDA events of the "profile" option
    r.set_option("profile", 1); r.kernel_times()
    parts = ("generate", "trace", "resolve")
    prof = {k: {p: [] for p in parts} for k in kinds}
    for _ in range(args.profile_frames):
        for k in kinds:
            step(k); torch.cuda.synchronize()
            t = r.kernel_times()
            for p in parts: prof[k][p].append(t[p]["ms"])
    r.set_option("profile", 0)

    # accum with the mattes on is the very accum without them
    scene.reset_blue_noise(); r.buffers.zero_(); step(0); torch.cuda.synchronize()
    accum_off = r.buffers.accum.clone()
    same = True
    for k in ks:
        scene.reset_blue_noise(); step(k); torch.cuda.synchronize()
        same &= bool(torch.equal(accum_off, r.buffers.accum))

    med = {k: float(np.median(ms[k])) for k in kinds}
    name = lambda k: "off" if k == 0 else f"K={k}"
    line = {"metric": "ms per frame with instance mattes", "value": med[ks[-1]], "unit": "ms/frame", "higher_is_better": False, "n_gpus": 1,
            "steps": args.steps, "warmup": args.warmup, "gpu": gpu_identity(), "instances": n_inst,
            "ms_per_frame": {name(k): med[k] for k in kinds},
            "over_off": {f"K={k}": med[k] / med[0] for k in ks},
            "ms_per_frame_spread": {name(k): [float(min(ms[k])), float(max(ms[k]))] for k in kinds},
            "kernel_ms_per_frame": {name(k): {p: float(np.median(prof[k][p])) for p in parts} for k in kinds},
            "profile_frames": args.profile_frames, "accum_bitwise_equal": same,
            "timing": "median of CUDA-event times per frame, mattes off and each K alternated, L2 flushed before each",
            "workload": wl["name"], "width": W, "height": H, "spp": SPP, "clocks": clocks}
    print(json.dumps(line), flush=True)
    return 0 if same else 1


if __name__ == "__main__":
    sys.exit(main())
