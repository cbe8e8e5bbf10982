#!/usr/bin/env python3
"""bench_ods.py -- an omni-directional stereo panorama (vpt_set_projection_ods, over-under) against the equirectangular panorama of the same
size, from the headline camera position.

    python tools/bench_ods.py [--config C] [--width W] [--height H] [--steps K] [--warmup W] [--profile-frames P]

The scene and Kernel_params are bench.py's (BASELINE.json configuration 2 by default: dragon.vdb, 64 spp, ray_depth 100, sun + HDRI); the
frame is 4096x2048, 360x180 degrees (per eye for ODS, ipd 5 % of the volume's size), from the headline camera's position and orientation.
Three arms: the equirectangular and the ODS frame with the miss cull (the default), and the ODS frame with option "miss_cull" 0.  They
run steps of SPP passes, each a new frame at iteration 0, alternated.  CUDA events around each step, L2 flushed before each, median per step.  Then, with the "profile"
option, P steps of each for the per-kernel device time (generate, trace, resolve).  Prints ONE JSON line with the card name and power limit
read in the same run, the culled fraction of the NumPy restatement (tests/ods_ref.py) and whether the ODS accum is the same with the cull
on and off.  Writes nothing to the tree.
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
    import ods_ref as O
    import projection_ref as P
    dev = "cuda:0"
    wl = B.build_workload(V, args.config, dev)
    scene, SPP = wl["scene"], wl["spp"]
    W, H = args.width, args.height
    lo, hi = scene.world_bounds()
    ipd = 0.05 * float(np.linalg.norm(hi - lo))
    stream = torch.cuda.current_stream().cuda_stream
    flush_buf = torch.zeros(64 * 1024 * 1024, dtype=torch.float32, device=dev)
    sampler = B.ClockSampler(0)

    rs = {}
    for name in ("equirect", "ods", "ods_cull_off"):
        r = V.Renderer(scene, W, H, kp=wl["kp"].__class__.from_buffer_copy(wl["kp"]), cam=scene.frame_camera(wl["width"], wl["height"]))
        if name == "equirect": r.set_projection("equirect", hfov=360.0, vfov=180.0)
        else: r.set_projection("ods", hfov=360.0, vfov=180.0, ipd=ipd, layout="over_under")
        r.set_option("miss_cull", 0 if name == "ods_cull_off" else 1)
        rs[name] = r

    def step(name):
        r = rs[name]
        r.kp.iteration = 0
        r.render(SPP, stream=stream)

    for _ in range(args.warmup):
        for name in rs:
            scene.reset_blue_noise(); step(name)
    torch.cuda.synchronize()
    same = torch.equal(rs["ods"].buffers.accum.view(torch.int32), rs["ods_cull_off"].buffers.accum.view(torch.int32))
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
    mask = O.cull_mask(P.camera_dict(rs["ods"].cam), O.params(360.0, 180.0, ipd=ipd), W, H, s["pmin"], s["pmax"], s["sph_center"],
                       s["sph_radius"])
    for r in rs.values(): r.close()

    med = {name: float(np.median(v)) for name, v in ms.items()}
    line = {"metric": "ms per step of an over-under ODS panorama", "value": med["ods"], "unit": "ms/step", "higher_is_better": False,
            "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "gpu": gpu_identity(),
            "ms_per_step": med, "ms_per_step_spread": {name: [float(min(v)), float(max(v))] for name, v in ms.items()},
            "kernel_ms_per_step": per_kernel, "profile_frames": args.profile_frames, "ipd": ipd,
            "culled_fraction": float(mask.mean()), "accum_bit_identical_cull_on_off": bool(same),
            "timing": "median of CUDA-event times per step, equirect / ODS / ODS without cull alternated, L2 flushed before each",
            "workload": wl["name"], "width": W, "height": H, "hfov": 360.0, "vfov": 180.0, "spp": SPP, "clocks": clocks}
    print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
