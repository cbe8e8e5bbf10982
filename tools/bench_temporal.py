#!/usr/bin/env python3
"""bench_temporal.py -- the temporal filter (vpt_temporal) on one GPU: its time, and the sweep that fixes its defaults.

    python tools/bench_temporal.py [--launches N] [--frames F] [--passes P] [--ref-passes R]

1. k_temporal at 1920x1080 on synthetic inputs with a history (fractional motion, partial coverage), with the default clip and without:
   median of CUDA events around single launches (L2 flushed before each), and algorithmic GB/s from the bytes one call must move --
   C, M, H, L, out, L_out and the display word, 60 B per pixel.
2. A sweep of max_history x clip_sigma over a slow pan and an orbit of bench.py's headline scene (dragon, sun + HDRI) at 480x270, F frames
   of P passes each through Renderer.render_temporal: the last frame's RMSE against an R-pass frame of the last pose, its ratio to the
   unfiltered frame's RMSE, and the drift of the mean luminance against that frame.
Prints ONE JSON line with both and the card name and power limit read in the same run.  Writes nothing to the tree.
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
from bench_adaptive import gpu_identity

BYTES_PER_PIXEL = 12 + 12 + 12 + 4 + 12 + 4 + 4       # C, M, H, L read once; out, L_out, display written


def time_filter(V, scene, n_launches, dev):
    W, H = 1920, 1080
    n = W * H
    r = V.Renderer(scene, W, H)
    g = torch.Generator(device=dev).manual_seed(1)
    c = torch.rand(n, 3, device=dev, generator=g) * 2
    hist = torch.rand(n, 3, device=dev, generator=g) * 2
    ln = torch.randint(1, 16, (n,), device=dev, generator=g).float()
    m = torch.zeros(n, 3, device=dev)
    m[:, 2] = (torch.rand(n, device=dev, generator=g) < 0.4).float()
    m[:, :2] = (torch.rand(n, 2, device=dev, generator=g) - 0.5) * 6 * m[:, 2:3]
    prev = V.camera.from_buffer_copy(bytes(r.cam))
    prev.origin = V._native.f3(prev.origin.x + 0.05, prev.origin.y, prev.origin.z)
    out = torch.empty(n * 3, device=dev); out_len = torch.empty(n, device=dev)
    flush = torch.zeros(64 * 1024 * 1024, dtype=torch.float32, device=dev)
    res = {}
    for label, clip in (("default_clip", None), ("no_clip", float("inf"))):
        times = []
        for i in range(n_launches + 3):
            flush.add_(1.0)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            r.temporal(prev, color=c, vectors=m, history=hist, history_len=ln, clip_sigma=clip, display=True, out=out, out_len=out_len)
            b.record()
            b.synchronize()
            if i >= 3: times.append(a.elapsed_time(b))
        ms = float(np.median(times))
        res[label] = {"median_ms": round(ms, 4), "p10_ms": round(float(np.percentile(times, 10)), 4),
                      "p90_ms": round(float(np.percentile(times, 90)), 4), "algorithmic_GBps": round(BYTES_PER_PIXEL * n / (ms * 1e-3) / 1e9, 1)}
    r.close()
    res["bytes_per_pixel"] = BYTES_PER_PIXEL
    return res


def path_cameras(V, scene, w, h, kind, n):
    lo, hi = scene.world_bounds()
    centre = (hi + lo) / 2
    dist = float(np.linalg.norm(hi - lo))
    cams = []
    for i in range(n):
        if kind == "pan":                                 # the camera stays, the view turns by 0.25 degree per frame
            frm = centre + dist * np.array([1.0, 0.6, 1.0]) / np.sqrt(2.0)
            ang = np.radians(0.25 * i)
            fwd = centre - frm
            at = frm + np.array([np.cos(ang) * fwd[0] - np.sin(ang) * fwd[2], fwd[1], np.sin(ang) * fwd[0] + np.cos(ang) * fwd[2]])
        else:                                             # the camera circles the volume by 1 degree per frame
            ang = np.radians(45.0 + 1.0 * i)
            frm = centre + dist * np.array([np.cos(ang), 0.6, np.sin(ang)])
            at = centre
        cam = V.camera()
        V.lib.vpt_camera_look_at(C.byref(cam), V._native.fvec(np.float32(frm)), V._native.fvec(np.float32(at)), V._native.fvec((0, 1, 0)),
                                 30.0, w / h, 0.0)
        cams.append(cam)
    return cams


def luminance(x):
    return 0.2126 * x[..., 0] + 0.7152 * x[..., 1] + 0.0722 * x[..., 2]


def sweep(V, wl, frames, passes, ref_passes):
    scene, kp = wl["scene"], wl["kp"]
    w, h = 480, 270
    out = {}
    for kind in ("pan", "orbit"):
        cams = path_cameras(V, scene, w, h, kind, frames)
        ref = V.Renderer(scene, w, h, kp=kp, cam=V.camera.from_buffer_copy(bytes(cams[-1])))
        ref.set_sample_offset(1 << 24); ref.kp.iteration = 0; ref.render(ref_passes); torch.cuda.synchronize()
        want = ref.buffers.accum.reshape(h, w, 3).clone()
        ref.close()
        rmse = lambda x: float(torch.sqrt(((x - want) ** 2).mean()))
        drift = lambda x: float(luminance(x).mean() / luminance(want).mean() - 1.0)
        rows = []
        for mh in (4, 8, 16, 32):
            for clip in (1.0, 1.5, 2.0, 3.0, float("inf")):
                r = V.Renderer(scene, w, h, kp=kp, cam=V.camera.from_buffer_copy(bytes(cams[0])))
                r.enable_temporal(max_history=mh, clip_sigma=clip)
                scene.reset_blue_noise()
                for cam in cams:
                    res, ln = r.render_temporal(cam, passes)
                torch.cuda.synchronize()
                raw = r.buffers.accum.reshape(h, w, 3)
                rows.append({"max_history": mh, "clip_sigma": clip if np.isfinite(clip) else "inf", "rmse": round(rmse(res), 6),
                             "rmse_unfiltered": round(rmse(raw), 6), "gain": round(rmse(raw) / rmse(res), 3),
                             "mean_luminance_drift_pct": round(100 * drift(res), 3), "mean_L": round(float(ln.mean()), 2)})
                r.close()
        out[kind] = rows
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=100)
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--passes", type=int, default=2)
    ap.add_argument("--ref-passes", type=int, default=1024)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    import vpt_b200 as V
    dev = "cuda:0"
    wl = B.build_workload(V, 2, dev)
    result = {"gpu": gpu_identity(), "filter_1080p": time_filter(V, wl["scene"], args.launches, dev),
              "sweep": {"width": 480, "height": 270, "frames": args.frames, "passes_per_frame": args.passes, "ref_passes": args.ref_passes,
                        **sweep(V, wl, args.frames, args.passes, args.ref_passes)}}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
