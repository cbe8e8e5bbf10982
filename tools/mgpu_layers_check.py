#!/usr/bin/env python3
"""torchrun --nproc-per-node N tools/mgpu_layers_check.py : DistributedRenderer(layers=all seven) over real IPC peer mappings must hold,
on every rank, the single-GPU depth, alpha, volume and light-group buffers bit for bit next to the accumulators -- after a fixed-count
frame with a continued call and after an adaptive frame -- and denoise() must equal Renderer.denoise of the single-GPU frame.  NCCL mode
must refuse the layers.  Prints BITWISE_OK on rank 0 when every rank matches."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch, torch.distributed as dist
import vpt_b200 as V
from vpt_b200.scene import synthetic_env
local = int(os.environ.get("LOCAL_RANK", "0")); torch.cuda.set_device(local)
dist.init_process_group(backend="nccl", device_id=torch.device(f"cuda:{local}"))
rank, world = dist.get_rank(), dist.get_world_size()
W, H, P = 640, 360, 12
LAYERS = tuple(V._native.LAYER_BITS)
LIGHTS = [((9.0, 6.0, 2.0), (1.0, 0.8, 0.6), 40.0), ((-2.0, 3.0, 8.0), (0.5, 0.7, 1.0), 25.0)]
vol = V.Volume.load_vdb(V.find_asset("dragon.vdb"))
scene = V.Scene([vol.instance()], device=f"cuda:{local}", env=synthetic_env(512, 256), lights=LIGHTS)
def kp():
    k = V.default_kernel_params(); k.environment_type = 1; k.ray_depth = 3; k.max_interactions = 1000; return k
bits = lambda t: t.contiguous().view(torch.int32) if t.dtype == torch.float32 else t.contiguous()
same = lambda a, b: a.numel() == b.numel() and torch.equal(bits(a).reshape(-1), bits(b).reshape(-1))

def layers_of(dr):
    return {n: (dr.full_depth() if n == "depth" else dr.full_alpha() if n == "alpha" else dr.full_volume() if n == "volume"
                else dr.full_light_group(n)).clone() for n in LAYERS}

ok = True
got = {}
scene.reset_blue_noise()
dr = V.DistributedRenderer(scene, W, H, kp=kp(), stripe_rows=8, gather_display=True, exchange="p2p", layers=LAYERS)
if dr.exchange != "p2p":
    print(f"[mgpu_layers_check] rank {rank}: peer-memory exchange unavailable ({getattr(dr, 'p2p_error', '?')})", flush=True); ok = False
else:
    dr.enable_aovs(); dr.enable_light_groups()
    for adaptive in (False, True):
        dr.r.kp.iteration = 0
        if adaptive: dr.render_adaptive(P, threshold=0.05, min_passes=4, check_interval=4)
        else: dr.render(P); dr.render(P)
        torch.cuda.synchronize()
        got[adaptive] = (dr.full_accum().reshape(-1, 3).clone(), dr.full_display.clone(), layers_of(dr), dr.denoise(display=True))
lost = dr.abandoned_waits() if ok else -1
cam = dr.r.cam
dist.barrier(); dr.close()

dn = V.DistributedRenderer(scene, W, H, kp=kp(), cam=cam, stripe_rows=8, exchange="nccl", layers=("depth",))
try:
    dn.full_depth(); refused = False
except V.VptError:
    refused = True
dist.barrier(); dn.close()

# every rank checks its own copy against its own single-GPU render of the same frames
r = V.Renderer(scene, W, H, kp=kp(), cam=cam)
r.enable_aovs(); r.enable_light_groups()
scene.reset_blue_noise()
for adaptive in (False, True):
    if not ok: break
    r.kp.iteration = 0
    err = r.render_adaptive(P, threshold=0.05, min_passes=4, check_interval=4, error_map=True)[2] if adaptive else (r.render(P), r.render(P))[0]
    torch.cuda.synchronize()
    b = r.buffers
    want = dict(depth=b.depth, alpha=b.alpha, volume=b.volume, **b.groups)
    acc, disp, lay, dn_got = got[adaptive]
    dn_want = r.denoise(rel_error=err, display=True)
    checks = dict(accum=same(acc, b.accum), display=same(disp, b.display), denoise=same(dn_got[0], dn_want[0]) and same(dn_got[1], dn_want[1]),
                  **{n: same(lay[n], want[n]) for n in LAYERS})
    ok = ok and all(checks.values())
    print(f"[mgpu_layers_check] rank {rank}/{world} {'adaptive' if adaptive else 'fixed'}: {checks}", flush=True)
r.close()
ok = ok and lost == 0 and refused
flag = torch.tensor([1 if ok else 0], dtype=torch.int32, device=f"cuda:{local}")
dist.all_reduce(flag, op=dist.ReduceOp.MIN)
if rank == 0:
    print(f"[mgpu_layers_check] abandoned flag waits {lost}; NCCL mode refused the layers: {refused}", flush=True)
    if int(flag.item()) == 1: print("BITWISE_OK", flush=True)
dist.barrier(); dist.destroy_process_group()
sys.exit(0 if int(flag.item()) == 1 else 1)
