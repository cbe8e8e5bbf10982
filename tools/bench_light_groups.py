#!/usr/bin/env python3
"""bench_light_groups.py -- cost of the light groups (vpt_set_light_group_buffers) on one GPU.

    python tools/bench_light_groups.py [--config C] [--steps K] [--warmup W] [--profile-frames P] [--generic-spp S]

Two workloads, each with the groups off and on:
  headline  bench.py's (BASELINE.json configuration 2 by default: dragon.vdb 1920x1080 64 spp, ray_depth 100, sun + HDRI).  The lean trace
            kernel is unchanged; with groups it writes wide sample records instead of compact ones and k_resolve<0, false, true> splits them.
  generic   the same dragon, camera and frame with two point lights and the sphere in view, so the generic trace kernel runs; with groups
            it is k_trace<0, false, 3, false, true>, which keeps the group sums in the sample scratch.
Per workload two renderers of the same frame, one with the groups registered and one without, alternate frames (one context toggling them
would reallocate its sample scratch at every switch, since groups change the lean kernel's record layout), CUDA events around each frame,
L2 flushed before each, median per frame.  Then, with
the "profile" option, P frames of each for the trace and resolve kernels' device time per frame.  Prints ONE JSON line with both
workloads, the card name and power limit read in the same run, and whether accum came out bit-identical with the groups on.  Writes
nothing to the tree.
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

LIGHTS = [((9.0, 6.0, 2.0), (1.0, 0.8, 0.6), 40.0), ((-2.0, 3.0, 8.0), (0.5, 0.7, 1.0), 25.0)]


def copy_kp(V, kp):
    out = V.default_kernel_params()
    C.memmove(C.addressof(out), bytes(kp), C.sizeof(kp))
    return out


def measure(V, scene, make, spp, steps, warmup, profile_frames, flush_buf, stream):
    """Two renderers of the same frame, one without and one with groups, so neither reallocates its sample scratch when the other runs
    (groups change the lean kernel's record layout: toggling them on one context would time cudaMalloc / cudaFree)."""
    rs = {False: make(), True: make()}
    rs[True].enable_light_groups()

    def step(on):
        r = rs[on]
        r.kp.iteration = 0
        r.render(spp, stream=stream)

    for _ in range(warmup):
        step(False); step(True)
    torch.cuda.synchronize()
    ms = {False: [], True: []}
    for _ in range(steps):                                       # alternate: both see the same clocks and neighbours
        for on in (False, True):
            B.flush_l2(flush_buf)
            a = torch.cuda.Event(enable_timing=True); b = torch.cuda.Event(enable_timing=True)
            a.record(); step(on); b.record()
            b.synchronize()
            ms[on].append(a.elapsed_time(b))

    kt = {False: {"trace": [], "resolve": []}, True: {"trace": [], "resolve": []}}
    for on in (False, True):
        rs[on].set_option("profile", 1); rs[on].kernel_times()
    for _ in range(profile_frames):
        for on in (False, True):
            step(on); torch.cuda.synchronize()
            t = rs[on].kernel_times()
            for k in ("trace", "resolve"): kt[on][k].append(t[k]["ms"])
    for on in (False, True):
        rs[on].set_option("profile", 0)

    acc = {}
    for on in (False, True):
        scene.reset_blue_noise(); rs[on].buffers.zero_(); step(on); torch.cuda.synchronize()
        acc[on] = rs[on].buffers.accum.clone()
    same = bool(torch.equal(acc[False], acc[True]))
    off, on = float(np.median(ms[False])), float(np.median(ms[True]))
    return {"ms_per_frame_off": off, "ms_per_frame_on": on, "on_over_off": on / off,
            "ms_per_frame_spread": {"off": [float(min(ms[False])), float(max(ms[False]))], "on": [float(min(ms[True])), float(max(ms[True]))]},
            "trace_ms_per_frame_off": float(np.median(kt[False]["trace"])), "trace_ms_per_frame_on": float(np.median(kt[True]["trace"])),
            "resolve_ms_per_frame_off": float(np.median(kt[False]["resolve"])), "resolve_ms_per_frame_on": float(np.median(kt[True]["resolve"])),
            "accum_bitwise_equal": same, "spp": spp}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, default=2, help="BASELINE.json configuration (bench.py's workloads)")
    ap.add_argument("--steps", type=int, default=10, help="timed frames of each kind, per workload")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile-frames", type=int, default=3)
    ap.add_argument("--generic-spp", type=int, default=16, help="passes per frame of the generic-kernel workload")
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

    sampler.start()
    tw0 = time.time()
    head = measure(V, scene, lambda: V.Renderer(scene, W, H, kp=copy_kp(V, wl["kp"])), SPP, args.steps, args.warmup, args.profile_frames,
                   flush_buf, stream)

    # the generic kernel: the headline's volume, camera and parameters plus two point lights and the sphere in view
    gscene = V.Scene(list(scene.instances), device=dev, env="Barce_Rooftop_C_3k.hdr", lights=LIGHTS)
    sp = gscene.h_sphere; sp.center = V.f3(4.0, 6.5, 3.0); sp.radius = 1.2; sp.roughness = 0.7; sp.color = V.f3(0.8, 0.6, 0.3)
    gscene.d_sphere.copy_(torch.frombuffer(bytearray(bytes(sp)), dtype=torch.uint8))
    gen = measure(V, gscene, lambda: V.Renderer(gscene, W, H, kp=copy_kp(V, wl["kp"])), args.generic_spp, args.steps, args.warmup, args.profile_frames, flush_buf, stream)
    sampler.window(tw0, time.time())
    clocks = sampler.stop()

    line = {"metric": "ms per frame with light groups", "value": head["ms_per_frame_on"], "unit": "ms/frame", "higher_is_better": False,
            "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "gpu": gpu_identity(),
            "headline": head, "generic": gen, "profile_frames": args.profile_frames,
            "timing": "median of CUDA-event times per frame, groups off and on alternated, L2 flushed before each",
            "workload": wl["name"], "width": W, "height": H, "clocks": clocks}
    print(json.dumps(line), flush=True)
    return 0 if head["accum_bitwise_equal"] and gen["accum_bitwise_equal"] else 1


if __name__ == "__main__":
    sys.exit(main())
