#!/usr/bin/env python3
"""torchrun --nproc-per-node N tools/mgpu_binned_check.py : DistributedRenderer(deep_slices=8, n_mattes=3) over real IPC peer mappings must
hold, on every rank, the single-GPU deep slices and instance mattes bit for bit next to the accumulators -- after a fixed-count frame with
a continued call and after an adaptive frame.  NCCL mode must refuse them.  Prints BITWISE_OK on rank 0 when every rank matches."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch, torch.distributed as dist
import vpt_b200 as V
from vpt_b200.scene import synthetic_env
local = int(os.environ.get("LOCAL_RANK", "0")); torch.cuda.set_device(local)
dist.init_process_group(backend="nccl", device_id=torch.device(f"cuda:{local}"))
rank, world = dist.get_rank(), dist.get_world_size()
W, H, P, K = 640, 360, 12, 8
vol = V.Volume.load_vdb(V.find_asset("dragon.vdb"))
scene = V.Scene([vol.instance(pos=(-20.0, 0.0, 0.0)), vol.instance(pos=(20.0, 0.0, 0.0))], device=f"cuda:{local}", env=synthetic_env(512, 256))
SETS, SPHERE = [[0], [1], []], 2
lo, hi = scene.world_bounds()
BOUNDS = [float(z) for z in np.linspace(0.0, 4.0 * float(np.linalg.norm(hi - lo)), K)] + [float("inf")]
def kp():
    k = V.default_kernel_params(); k.environment_type = 1; k.ray_depth = 3; k.max_interactions = 1000; return k
bits = lambda t: t.contiguous().view(torch.int32) if t.dtype == torch.float32 else t.contiguous()
same = lambda a, b: a.numel() == b.numel() and torch.equal(bits(a).reshape(-1), bits(b).reshape(-1))

ok = True
got = {}
scene.reset_blue_noise()
dr = V.DistributedRenderer(scene, W, H, kp=kp(), stripe_rows=8, gather_display=True, exchange="p2p", deep_slices=K, n_mattes=len(SETS))
if dr.exchange != "p2p":
    print(f"[mgpu_binned_check] rank {rank}: peer-memory exchange unavailable ({getattr(dr, 'p2p_error', '?')})", flush=True); ok = False
else:
    dr.enable_deep(BOUNDS); dr.enable_mattes(SETS, SPHERE)
    for adaptive in (False, True):
        dr.r.kp.iteration = 0
        if adaptive: dr.render_adaptive(P, threshold=0.05, min_passes=4, check_interval=4)
        else: dr.render(P); dr.render(P)
        torch.cuda.synchronize()
        got[adaptive] = (dr.full_accum().reshape(-1, 3).clone(), dr.full_deep().clone(), dr.full_mattes().clone())
lost = dr.abandoned_waits() if ok else -1
cam = dr.r.cam
dist.barrier(); dr.close()

dn = V.DistributedRenderer(scene, W, H, kp=kp(), cam=cam, stripe_rows=8, exchange="nccl", deep_slices=K, n_mattes=len(SETS))
refused = True
for fn in (dn.full_deep, dn.full_mattes):
    try:
        fn(); refused = False
    except V.VptError:
        pass
dist.barrier(); dn.close()

# every rank checks its own copy against its own single-GPU render of the same frames
r = V.Renderer(scene, W, H, kp=kp(), cam=cam)
r.enable_deep(BOUNDS); r.enable_mattes(SETS, SPHERE)
scene.reset_blue_noise()
for adaptive in (False, True):
    if not ok: break
    r.kp.iteration = 0
    if adaptive: r.render_adaptive(P, threshold=0.05, min_passes=4, check_interval=4)
    else: r.render(P); r.render(P)
    torch.cuda.synchronize()
    acc, deep, mattes = got[adaptive]
    checks = dict(accum=same(acc, r.buffers.accum), deep=same(deep, r.deep_image()), mattes=same(mattes, r.matte_image()),
                  signal=float(r.deep_image()[..., 3].max()) > 0 and float(r.matte_image()[1, ..., 3].max()) > 0)
    ok = ok and all(checks.values())
    print(f"[mgpu_binned_check] rank {rank}/{world} {'adaptive' if adaptive else 'fixed'}: {checks}", flush=True)
r.close()
ok = ok and lost == 0 and refused
flag = torch.tensor([1 if ok else 0], dtype=torch.int32, device=f"cuda:{local}")
dist.all_reduce(flag, op=dist.ReduceOp.MIN)
if rank == 0:
    print(f"[mgpu_binned_check] abandoned flag waits {lost}; NCCL mode refused the binned layers: {refused}", flush=True)
    if int(flag.item()) == 1: print("BITWISE_OK", flush=True)
dist.barrier(); dist.destroy_process_group()
sys.exit(0 if int(flag.item()) == 1 else 1)
