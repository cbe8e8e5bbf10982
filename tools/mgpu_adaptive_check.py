#!/usr/bin/env python3
"""torchrun --nproc-per-node N tools/mgpu_adaptive_check.py : adaptive frames sharded over the peer-memory exchange
(DistributedRenderer.render_adaptive, real IPC peer mappings) must equal the single-GPU adaptive frame bit for bit -- full-frame
accumulators, display words, pass counts, error map and passes_run -- for two adaptive frames back to back (another threshold the second
time), then a fixed-count frame on the same exchange.  NCCL mode must refuse adaptive frames.  Prints BITWISE_OK on rank 0 when
everything matches."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch, torch.distributed as dist
import vpt_b200 as V
from vpt_b200.scene import synthetic_env
local = int(os.environ.get("LOCAL_RANK", "0")); torch.cuda.set_device(local)
dist.init_process_group(backend="nccl", device_id=torch.device(f"cuda:{local}"))
rank, world = dist.get_rank(), dist.get_world_size()
W, H, P, MIN, IV = 1920, 1080, 32, 8, 8
FRAMES = (("adaptive", 0.2), ("adaptive", 0.1), ("fixed", P))
vol = V.Volume.load_vdb(V.find_asset("dragon.vdb"))
scene = V.Scene([vol.instance()], device=f"cuda:{local}", env=synthetic_env(512, 256))
def kp():
    k = V.default_kernel_params(); k.environment_type = 1; k.ray_depth = 100; k.max_interactions = 1000; return k
bits = lambda t: t.contiguous().view(torch.int32) if t.dtype == torch.float32 else t.contiguous()
same = lambda a, b: tuple(a.shape) == tuple(b.shape) and torch.equal(bits(a), bits(b))

def single_gpu_frames(cam):
    """rank 0: the same sequence of frames on one GPU (one blue-noise state carried through, as on every rank)"""
    r = V.Renderer(scene, W, H, kp=kp(), cam=cam)
    scene.reset_blue_noise()
    out = []
    for kind, arg in FRAMES:
        r.kp.iteration = 0
        if kind == "adaptive":
            run, counts, err = r.render_adaptive(P, threshold=arg, min_passes=MIN, check_interval=IV, error_map=True)
        else:
            r.render(arg); run, counts, err = arg, None, None
        torch.cuda.synchronize()
        out.append((run, r.buffers.accum.clone(), r.buffers.display.clone(), None if counts is None else counts.clone(),
                    None if err is None else err.clone()))
    r.close()
    return out

ok = True
scene.reset_blue_noise()
dr = V.DistributedRenderer(scene, W, H, kp=kp(), stripe_rows=8, gather_display=True, exchange="p2p")
if dr.exchange != "p2p":
    print(f"[mgpu_adaptive_check] rank {rank}: peer-memory exchange unavailable ({getattr(dr, 'p2p_error', '?')})", flush=True); ok = False
got = []
for kind, arg in FRAMES:
    if not ok: break
    dr.r.kp.iteration = 0
    if kind == "adaptive":
        run, counts, err = dr.render_adaptive(P, threshold=arg, min_passes=MIN, check_interval=IV, error_map=True)
        torch.cuda.synchronize()
        got.append((run, dr.full_accum().reshape(-1, 3).clone(), dr.full_display.clone(), counts.clone(), err.clone()))
    else:
        dr.render(arg); torch.cuda.synchronize()
        got.append((arg, dr.full_accum().reshape(-1, 3).clone(), dr.full_display.clone(), None, None))
lost = dr.abandoned_waits() if ok else -1
cam = dr.r.cam
dist.barrier(); dr.close()

# NCCL exchange: adaptive frames are refused
dn = V.DistributedRenderer(scene, W, H, kp=kp(), cam=cam, stripe_rows=8, exchange="nccl")
try:
    dn.render_adaptive(P, threshold=0.1, min_passes=MIN, check_interval=IV); refused = False
except V.VptError:
    refused = True
dist.barrier(); dn.close()

if rank == 0:
    want = single_gpu_frames(cam)
    for i, ((kind, arg), g, w) in enumerate(zip(FRAMES, got, want)):
        checks = dict(passes_run=g[0] == w[0], accum=same(g[1], w[1]), display=same(g[2], w[2]))
        if kind == "adaptive":
            checks.update(counts=same(g[3], w[3]), err=same(g[4], w[4]), classes=len(torch.unique(w[3])))
        ok = ok and all(v for k, v in checks.items() if k != "classes")
        print(f"[mgpu_adaptive_check] world={world} frame {i} ({kind} {arg}): {checks}", flush=True)
    ok = ok and len(got) == len(FRAMES) and lost == 0 and refused
    print(f"[mgpu_adaptive_check] abandoned flag waits {lost}; NCCL mode refused: {refused}", flush=True)
    if ok: print("BITWISE_OK", flush=True)
dist.barrier(); dist.destroy_process_group()
sys.exit(0 if ok else 1)
