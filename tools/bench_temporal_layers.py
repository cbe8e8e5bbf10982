#!/usr/bin/env python3
"""bench_temporal_layers.py -- the cost of the layers of vpt_temporal_layers on one GPU, plane set by plane set.

    python tools/bench_temporal_layers.py [--launches N] [--warmup W]

Times the call at 1920x1080 on synthetic inputs with a history (fractional motion over 40 % coverage, the rest the environment's motion
of a camera moved sideways) and display words, adding planes as DESIGN.md section 8n's table does: none (vpt_temporal itself), + the
AOVs (alpha, volume), + the four light groups, + the collision AOVs (position, normal, albedo), + deep K = 8, + mattes K = 8.  Each
configuration is launched N times after W warm-up launches, the configurations alternated launch by launch, with CUDA events around every
launch, straight through the C ABI; the median is reported.  Algorithmic GB/s counts the beauty's 60 B per pixel (bench_temporal.py) and, per layer plane of c
channels, its current value, history and output once each (12 c B per pixel).  Prints ONE JSON line with the card name and power limit
read in the same run.  Writes nothing to the tree.
"""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np
import torch

import bench as B
from bench_denoise_layers import card
from bench_temporal import BYTES_PER_PIXEL

W, H = 1920, 1080
# name -> (channels, planes)
PLANES = {"alpha": (1, 1), "volume": (3, 1), **{g: (3, 1) for g in ("sun", "point", "emission", "environment")},
          "position": (4, 1), "normal": (3, 1), "albedo": (3, 1), "deep": (4, 8), "mattes": (4, 8)}
CONFIGS = {"none": [], "aovs": ["alpha", "volume"]}
CONFIGS["aovs+groups"] = CONFIGS["aovs"] + ["sun", "point", "emission", "environment"]
CONFIGS["aovs+groups+collision"] = CONFIGS["aovs+groups"] + ["position", "normal", "albedo"]
CONFIGS["aovs+groups+collision+deep8"] = CONFIGS["aovs+groups+collision"] + ["deep"]
CONFIGS["aovs+groups+collision+deep8+mattes8"] = CONFIGS["aovs+groups+collision+deep8"] + ["mattes"]


def layer_bytes(names, px):
    """each plane of c channels: current value, history and output, 4 c B per pixel each"""
    return sum(3 * 4 * PLANES[n][0] * PLANES[n][1] for n in names) * px


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    import vpt_b200 as V
    dev = "cuda:0"
    wl = B.build_workload(V, 2, dev)
    r = V.Renderer(wl["scene"], W, H)
    n = W * H
    g = torch.Generator(device=dev).manual_seed(1)
    rnd = lambda *s: torch.rand(*s, device=dev, generator=g)
    c, hist = rnd(n, 3) * 2, rnd(n, 3) * 2
    ln = torch.randint(1, 16, (n,), device=dev, generator=g).float()
    m = torch.zeros(n, 3, device=dev)
    m[:, 2] = (rnd(n) < 0.4).float()
    m[:, :2] = (rnd(n, 2) - 0.5) * 6 * m[:, 2:3]
    prev = V.camera.from_buffer_copy(bytes(r.cam))
    prev.origin = V._native.f3(prev.origin.x + 0.05, prev.origin.y, prev.origin.z)
    shape = lambda name: (PLANES[name][1], H, W, PLANES[name][0])
    src = {name: rnd(*shape(name)) for name in PLANES}
    lhist = {name: rnd(*shape(name)) for name in PLANES}
    out = {"beauty": torch.empty(n * 3, device=dev), "len": torch.empty(n, device=dev),
           **{name: torch.empty(shape(name), device=dev) for name in PLANES}}
    ref = r.temporal(prev, color=c, vectors=m, history=hist, history_len=ln, display=True)
    words = torch.empty(n, dtype=torch.int32, device=dev)
    opt = V._native.temporal_options(16, float("inf"))
    p = lambda t: C.c_void_p(t.data_ptr())
    # the calls are enqueued straight through the C ABI with their descriptors built beforehand, so the events time the kernel and not
    # the Python wrapper
    descs = {k: (V._native.temporal_layer * max(1, len(names)))(*[V._native.temporal_layer(src[nm].data_ptr(), lhist[nm].data_ptr(),
                                                                                            out[nm].data_ptr(), *PLANES[nm]) for nm in names])
             for k, names in CONFIGS.items()}
    times = {k: [] for k in CONFIGS}
    equal = {k: True for k in CONFIGS}
    for i in range(args.warmup + args.launches):
        for k, names in CONFIGS.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            rc = V.lib.vpt_temporal_layers(r.ctx, W, H, p(c), p(m), C.byref(r.cam), C.byref(prev), p(hist), p(ln), C.byref(opt), 1.0,
                                           p(out["beauty"]), p(out["len"]), p(words), descs[k], len(names), None)
            b.record()
            b.synchronize()
            assert rc == 0, V.lib.vpt_last_error(r.ctx)
            if i >= args.warmup:
                times[k].append(a.elapsed_time(b))
                equal[k] = equal[k] and torch.equal(out["beauty"].view(torch.int32), ref[0].reshape(-1).view(torch.int32)) and \
                    torch.equal(words, ref[2].reshape(-1))
    base = float(np.median(times["none"]))
    result = {"card": card(), "frame": f"{W}x{H}", "launches": args.launches, "configs": {}}
    for k, names in CONFIGS.items():
        ms = float(np.median(times[k]))
        planes = sum(PLANES[nm][1] for nm in names)
        byts = BYTES_PER_PIXEL * n + layer_bytes(names, n)
        result["configs"][k] = {"ms": round(ms, 4), "p10_ms": round(float(np.percentile(times[k], 10)), 4),
                                "p90_ms": round(float(np.percentile(times[k], 90)), 4), "planes": planes,
                                "channels": sum(PLANES[nm][0] * PLANES[nm][1] for nm in names), "bytes": byts,
                                "GB_per_s": round(byts / ms / 1e6, 1),
                                "ms_per_plane_over_none": round((ms - base) / planes, 4) if planes else None,
                                "beauty_equal_to_vpt_temporal": equal[k]}
    r.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
