#!/usr/bin/env python3
"""bench_projection.py -- an equirectangular panorama (vpt_set_projection) from the headline camera position, with the miss cull on and off.

    python tools/bench_projection.py [--config C] [--width W] [--height H] [--steps K] [--warmup W] [--profile-frames P]

The scene and Kernel_params are bench.py's (BASELINE.json configuration 2 by default: dragon.vdb, 64 spp, ray_depth 100, sun + HDRI); the
frame is a 4096x2048 360x180-degree panorama from the headline camera's position and orientation.  Two renderers, option "miss_cull" 1
and 0, run steps of SPP passes, each a new frame at iteration 0, alternated.  CUDA events around each step, L2 flushed before each, median
per step.  Then, with the "profile" option, P steps of each for the per-kernel device time.  The culled fraction is the NumPy restatement's
(tests/projection_ref.py) for the same camera and root box.  Prints ONE JSON line with the card name and power limit read in the same
run.  Writes nothing to the tree.
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
    ap.add_argument("--width", type=int, default=4096)
    ap.add_argument("--height", type=int, default=2048)
    ap.add_argument("--steps", type=int, default=5, help="timed steps of each arm")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--profile-frames", type=int, default=2)
    args = ap.parse_args()
    args.warmup = max(args.warmup, 1)
    torch.cuda.set_device(0)

    import vpt_b200 as V
    import miss_cull_ref as M
    import projection_ref as P
    dev = "cuda:0"
    wl = B.build_workload(V, args.config, dev)
    scene, SPP = wl["scene"], wl["spp"]
    W, H = args.width, args.height
    stream = torch.cuda.current_stream().cuda_stream
    flush_buf = torch.zeros(64 * 1024 * 1024, dtype=torch.float32, device=dev)
    sampler = B.ClockSampler(0)

    rs = {}
    for name, cull in (("cull_on", 1), ("cull_off", 0)):
        r = V.Renderer(scene, W, H, kp=wl["kp"].__class__.from_buffer_copy(wl["kp"]), cam=scene.frame_camera(wl["width"], wl["height"]))
        r.set_option("miss_cull", cull)
        r.set_projection("equirect", hfov=360.0, vfov=180.0)
        rs[name] = r

    def step(name):
        r = rs[name]
        r.kp.iteration = 0
        r.render(SPP, stream=stream)

    for _ in range(args.warmup):
        for name in rs:
            scene.reset_blue_noise(); step(name)              # the same blue noise for both arms: their frames are compared below
    torch.cuda.synchronize()
    same = torch.equal(rs["cull_on"].buffers.accum.view(torch.int32), rs["cull_off"].buffers.accum.view(torch.int32))
    ms = {name: [] for name in rs}
    sampler.start()
    tw0 = time.time()
    for _ in range(args.steps):                                  # alternate: both arms see the same clocks and neighbours
        for name in rs:
            scene.reset_blue_noise(); B.flush_l2(flush_buf)
            a = torch.cuda.Event(enable_timing=True); b = torch.cuda.Event(enable_timing=True)
            a.record(); step(name); b.record()
            b.synchronize()
            ms[name].append(a.elapsed_time(b))
    sampler.window(tw0, time.time())
    clocks = sampler.stop()

    kernels = {name: [] for name in rs}
    for name, r in rs.items():
        r.set_option("profile", 1); r.kernel_times()
    for _ in range(args.profile_frames):
        for name, r in rs.items():
            step(name); torch.cuda.synchronize()
            kernels[name].append(r.kernel_times())
    per_kernel = {name: {k: float(np.median([kt[k]["ms"] for kt in ks])) for k in ks[0]} for name, ks in kernels.items()}

    # the culled fraction, from the restatement: the renderer's camera, the headline root box and sphere
    s = M.headline_setup()
    cam = rs["cull_on"].cam
    mask = P.cull_mask(P.camera_dict(cam), np.float32(np.deg2rad(360.0)), np.float32(np.deg2rad(180.0)), W, H, s["pmin"], s["pmax"],
                       s["sph_center"], s["sph_radius"])
    for r in rs.values(): r.close()

    med = {name: float(np.median(v)) for name, v in ms.items()}
    line = {"metric": "ms per step of an equirectangular panorama", "value": med["cull_on"], "unit": "ms/step", "higher_is_better": False,
            "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "gpu": gpu_identity(),
            "ms_per_step": med, "ms_per_step_spread": {name: [float(min(v)), float(max(v))] for name, v in ms.items()},
            "kernel_ms_per_step": per_kernel, "profile_frames": args.profile_frames,
            "culled_fraction": float(mask.mean()), "accum_bit_identical": bool(same),
            "timing": "median of CUDA-event times per step, cull on / off alternated, L2 flushed before each",
            "workload": wl["name"], "width": W, "height": H, "hfov": 360.0, "vfov": 180.0, "spp": SPP, "clocks": clocks}
    print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
