"""Adaptive frames sharded over the peer-memory exchange (vpt_render_adaptive on a partitioned context).

R contexts on ONE GPU render the R shards of a frame and exchange through each other's blocks (same-process import), the way
test_peer_memory_exchange_with_three_shards_on_one_gpu runs the fixed-count exchange: one scene per shard (its own blue-noise replica),
each shard on its own stream.  Every convergence test waits for the peers, so each shard's call runs in its own Python thread (ctypes
releases the GIL), and the threads are joined with a timeout.

Pixels are independent, every RNG stream is keyed by the global pixel and the 3x3 rule is defined on the global frame, so the sharded
frame must equal the single-context adaptive frame of the same options bit for bit: passes_run, pass counts, error map, every buffer at
the rank's rows, every rank's full-frame planes and every blue-noise replica."""
import ctypes as C
import os
import subprocess
import sys
import threading

import numpy as np
import pytest
import torch

import vpt_b200 as V
from vpt_b200.renderer import _DeviceView, stripe_rows_of_rank
from vpt_b200.scene import synthetic_env
import adaptive_ref as A
from test_parity_gpu import make_kp

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLT_MAX = float(np.finfo(np.float32).max)
BUFFERS = ("accum", "depth", "cost", "raw", "display")
W, H = 333, 197                                    # ragged: neither a multiple of the 32x4 tile nor of any stripe height used here
chk = V._native.check


@pytest.fixture(scope="module")
def dragon():
    return V.Volume.load_vdb(V.find_asset("dragon.vdb"))


@pytest.fixture(scope="module")
def atmosphere():
    atm = V.Atmosphere()
    yield atm
    atm.destroy()


def bits(t):
    t = t.contiguous()
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def same(a, b):
    return tuple(a.shape) == tuple(b.shape) and torch.equal(bits(a), bits(b))


class Case:
    """Scene factory (one scene per shard plus one for the single context), camera and Kernel_params of one configuration."""

    def __init__(self, dragon, integrator=0, instances=1, atmosphere=None, w=W, h=H, cam=None):
        rng = np.random.RandomState(7)
        self.inst = [dragon.instance()]
        for _ in range(instances - 1):
            q = rng.randn(4); q /= np.linalg.norm(q)
            self.inst.append(dragon.instance(pos=tuple(rng.uniform(-6, 6, 3)), quat=tuple(q), scale=float(rng.uniform(0.7, 1.3))))
        self.integrator, self.atm, self.w, self.h = integrator, atmosphere, w, h
        self.cam = cam if cam is not None else self.scene().frame_camera(w, h)

    def scene(self):
        s = V.Scene(list(self.inst), env=synthetic_env(512, 256))
        if self.integrator: self.atm.apply(s.atmos)               # integrator 1 ends every path on the precomputed sky
        return s

    def kp(self):
        return make_kp(integrator=1, ray_depth=4) if self.integrator else make_kp(ray_depth=3, volume_depth=2)

    def single(self):
        scene = self.scene()
        return scene, V.Renderer(scene, self.w, self.h, kp=self.kp(), cam=self.cam)


class Shards:
    """R contexts of one frame on one GPU sharing one peer-memory exchange."""

    def __init__(self, case, R, stripe_rows):
        self.case, self.R, self.sr, self.w, self.h = case, R, stripe_rows, case.w, case.h
        self.scenes = [case.scene() for _ in range(R)]
        self.rs = [V.Renderer(self.scenes[k], self.w, self.h, kp=case.kp(), cam=case.cam, rank=k, n_ranks=R, stripe_rows=stripe_rows)
                   for k in range(R)]
        blocks = (C.c_uint64 * R)()
        for k, r in enumerate(self.rs):
            raw = (C.c_ubyte * 64)()
            chk(V.lib.vpt_comm_p2p_export(r.ctx, k, R, stripe_rows, self.w, self.h, 1, raw), r.ctx, "vpt_comm_p2p_export")
            b = C.c_uint64(0); chk(V.lib.vpt_comm_p2p_block(r.ctx, C.byref(b)), r.ctx, "vpt_comm_p2p_block"); blocks[k] = b.value
        self.frames = []
        for r in self.rs:
            chk(V.lib.vpt_comm_p2p_import_local(r.ctx, blocks), r.ctx, "vpt_comm_p2p_import_local")
            pa, pd, pc, pe = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
            chk(V.lib.vpt_comm_p2p_frame(r.ctx, C.byref(pa), C.byref(pd)), r.ctx, "vpt_comm_p2p_frame")
            chk(V.lib.vpt_comm_p2p_adaptive_frame(r.ctx, C.byref(pc), C.byref(pe)), r.ctx, "vpt_comm_p2p_adaptive_frame")
            view = lambda p, shape, t: torch.as_tensor(_DeviceView(p.value, shape, t), device="cuda")
            self.frames.append(dict(accum=view(pa, (self.w * self.h, 3), "<f4"), display=view(pd, (self.w * self.h,), "<i4"),
                                    counts=view(pc, (self.h, self.w), "<i4"), err=view(pe, (self.h, self.w), "<f4")))
        self.streams = [torch.cuda.Stream() for _ in range(R)]
        torch.cuda.synchronize()

    def run(self, fn):
        """fn(k, renderer, stream) for every shard, each in its own thread; returns the R results."""
        out, errs = [None] * self.R, [None] * self.R

        def body(k):
            try:
                out[k] = fn(k, self.rs[k], self.streams[k].cuda_stream)
            except BaseException as e:                           # re-raised on the main thread
                errs[k] = e
        ts = [threading.Thread(target=body, args=(k,), daemon=True) for k in range(self.R)]
        for t in ts: t.start()
        for t in ts: t.join(timeout=300)
        assert not any(t.is_alive() for t in ts), "a shard's call did not return"
        torch.cuda.synchronize()
        for e in errs:
            if e is not None: raise e
        return out

    def adaptive(self, max_passes, min_passes, interval, threshold):
        def fn(k, r, stream):
            r.kp.iteration = 0
            return r.render_adaptive(max_passes, threshold=threshold, min_passes=min_passes, check_interval=interval, error_map=True, stream=stream)
        return self.run(fn)

    def fixed(self, n_passes):
        def fn(k, r, stream):
            r.kp.iteration = 0
            r.render(n_passes, stream=stream)
        self.run(fn)

    def reset_blue_noise(self):
        for s in self.scenes: s.reset_blue_noise()

    def abandoned_waits(self):
        out = []
        for r in self.rs:
            n = C.c_uint64(0); chk(V.lib.vpt_comm_p2p_status(r.ctx, C.byref(n)), r.ctx, "vpt_comm_p2p_status"); out.append(int(n.value))
        return out

    def close(self):
        self.frames.clear()
        for r in self.rs: r.close()


def single_adaptive(scene, r, max_passes, min_passes, interval, threshold):
    r.kp.iteration = 0
    out = r.render_adaptive(max_passes, threshold=threshold, min_passes=min_passes, check_interval=interval, error_map=True)
    torch.cuda.synchronize()
    return out


def assert_sharded_equals_single(sh, shard_out, scene, ref, ref_out):
    run, counts, err = ref_out
    for k, (r, (run_k, counts_k, err_k)) in enumerate(zip(sh.rs, shard_out)):
        assert run_k == run, f"passes_run of shard {k}"
        rows = torch.as_tensor(stripe_rows_of_rank(sh.h, k, sh.R, sh.sr), device=counts.device)
        valid = rows < sh.h; g = rows[valid]
        assert counts_k.shape == (len(rows), sh.w)
        assert same(counts_k[valid], counts[g]), f"pass counts of shard {k}"
        assert bool((counts_k[~valid] == 0).all()), f"padding rows of shard {k}"
        assert same(err_k[valid], err[g]), f"error map of shard {k}"
        for name in BUFFERS:
            mine = getattr(r.buffers, name).view(len(rows), sh.w, -1)[valid]
            want = getattr(ref.buffers, name).view(sh.h, sh.w, -1)[g]
            assert same(mine, want), f"{name} of shard {k}"
        f = sh.frames[k]
        assert same(f["accum"], ref.buffers.accum), f"full-frame accum held by shard {k}"
        assert same(f["display"], ref.buffers.display), f"full-frame display held by shard {k}"
        assert same(f["counts"], counts), f"full-frame pass counts held by shard {k}"
        assert same(f["err"], err), f"full-frame error map held by shard {k}"
        assert torch.equal(sh.scenes[k].d_blue_noise, scene.d_blue_noise), f"blue-noise replica of shard {k}"


def splitting_threshold(scene, ref, max_passes, min_passes, interval, q=0.4):
    """A threshold that stops part of the frame at the first test: a quantile of the 3x3 maxima of the first test's errors."""
    scene.reset_blue_noise()
    _, _, first = single_adaptive(scene, ref, max_passes, min_passes, interval, FLT_MAX)
    scene.reset_blue_noise()
    return float(np.quantile(A.max3x3(first.cpu().numpy()), q))


# ranks, stripe_rows, integrator, instances: every (ranks, stripe_rows) pair once, both integrators, a scene of 8 instances
CONFIGS = [(2, 1, 0, 1), (3, 1, 1, 1), (2, 6, 0, 8), (3, 6, 0, 1), (2, 8, 1, 1), (3, 8, 0, 8)]


@pytest.mark.parametrize("R,stripe_rows,integrator,instances", CONFIGS)
def test_sharded_adaptive_equals_single_context(dragon, atmosphere, R, stripe_rows, integrator, instances):
    P, mn, iv = 24, 4, 4
    case = Case(dragon, integrator=integrator, instances=instances, atmosphere=atmosphere)
    scene, ref = case.single()
    thr = splitting_threshold(scene, ref, P, mn, iv)
    ref_out = single_adaptive(scene, ref, P, mn, iv, thr)
    classes = torch.unique(ref_out[1]).tolist()
    print(f"R={R} stripe_rows={stripe_rows} integrator={integrator} instances={instances}: threshold {thr:.4g}, "
          f"passes_run {ref_out[0]}, count classes {classes}")
    assert len(classes) >= 3
    sh = Shards(case, R, stripe_rows)
    out = sh.adaptive(P, mn, iv, thr)
    assert_sharded_equals_single(sh, out, scene, ref, ref_out)
    assert sh.abandoned_waits() == [0] * R
    sh.close(); ref.close()


def test_idle_rank_keeps_advancing_with_the_others(dragon):
    """The volume lies in one half of the frame and each of two ranks owns one half: all pixels of the idle rank stop at the first test
    while the other rank still samples, and the idle rank keeps issuing its blue-noise advances and barriers until the frame ends."""
    w, h, P, mn, iv = 320, 180, 24, 4, 4
    base = Case(dragon, w=w, h=h)
    lo, hi = base.scene().world_bounds()
    center = (hi + lo) / np.float32(2); dist = float(np.linalg.norm(hi - lo))
    up = np.array([-1.0, 2.0, -1.0], np.float32) / np.float32(np.sqrt(6.0))     # the camera's up vector for a view along -(1,1,1)
    lookat = (center + np.float32(0.54 * dist) * up).astype(np.float32)            # the scene's bounding sphere lands in one half
    lookfrom = (lookat + np.float32(4.0 * dist / np.sqrt(3.0))).astype(np.float32)
    cam = V._native.camera()
    V.lib.vpt_camera_look_at(C.byref(cam), V._native.fvec(lookfrom), V._native.fvec(lookat), V._native.fvec((0, 1, 0)), 30.0, w / h, 0.0)
    case = Case(dragon, w=w, h=h, cam=cam)
    scene, ref = case.single()
    stripe = (h + 1) // 2                                        # rank 0: rows [0, stripe), rank 1: the rest
    scene.reset_blue_noise()
    _, _, first = single_adaptive(scene, ref, P, mn, iv, FLT_MAX)
    scene.reset_blue_noise()
    m3 = A.max3x3(first.cpu().numpy())
    worst = [float(m3[:stripe].max()), float(m3[stripe:].max())]
    idle, busy = (0, 1) if worst[0] < worst[1] else (1, 0)
    print(f"largest 3x3 error at the first test per rank: {worst}")
    assert worst[busy] > 2 * worst[idle], "the volume should lie in one half of the frame"
    thr = 0.5 * (worst[0] + worst[1])
    ref_out = single_adaptive(scene, ref, P, mn, iv, thr)
    sh = Shards(case, 2, stripe)
    out = sh.adaptive(P, mn, iv, thr)
    run = out[0][0]
    assert run > mn and int(out[idle][1].max()) < run and int(out[busy][1].max()) == run
    assert_sharded_equals_single(sh, out, scene, ref, ref_out)
    assert sh.abandoned_waits() == [0, 0]
    sh.close(); ref.close()


def test_edge_thresholds(dragon):
    """Threshold 0: every pixel takes every pass, and the frame is the sharded fixed-count frame of that many passes.  FLT_MAX: every
    pixel stops at min_passes."""
    P, mn, iv = 12, 4, 4
    case = Case(dragon)
    scene, ref = case.single()
    sh = Shards(case, 3, 6)
    scene.reset_blue_noise(); sh.reset_blue_noise()
    out = sh.adaptive(P, mn, iv, 0.0)
    ref_out = single_adaptive(scene, ref, P, mn, iv, 0.0)
    assert ref_out[0] == P and bool((ref_out[1] == P).all())
    assert_sharded_equals_single(sh, out, scene, ref, ref_out)
    adaptive = [(f["accum"].clone(), f["display"].clone()) for f in sh.frames]
    sh.reset_blue_noise()
    sh.fixed(P)
    for k, f in enumerate(sh.frames):
        assert same(f["accum"], adaptive[k][0]) and same(f["display"], adaptive[k][1]), f"threshold 0 vs render({P}), shard {k}"
    scene.reset_blue_noise(); sh.reset_blue_noise()
    out = sh.adaptive(P, mn, iv, FLT_MAX)
    ref_out = single_adaptive(scene, ref, P, mn, iv, FLT_MAX)
    assert ref_out[0] == mn and bool((ref_out[1] == mn).all())
    assert_sharded_equals_single(sh, out, scene, ref, ref_out)
    assert sh.abandoned_waits() == [0, 0, 0]
    sh.close(); ref.close()


def test_sequence_of_adaptive_and_fixed_frames_on_one_exchange(dragon):
    """adaptive, adaptive (another threshold), fixed-count, adaptive on the same exchange: each frame equals its single-context counterpart,
    which takes both handshakes (ready / done of every call, the two barriers of every test) through several calls."""
    P, mn, iv = 20, 4, 4
    case = Case(dragon)
    scene, ref = case.single()
    thr1 = splitting_threshold(scene, ref, P, mn, iv, q=0.3)
    thr2 = splitting_threshold(scene, ref, P, mn, iv, q=0.7)
    sh = Shards(case, 2, 8)
    for step in ("a1", "a2", "fixed", "a1"):
        if step == "fixed":
            sh.fixed(P)
            ref.kp.iteration = 0; ref.render(P); torch.cuda.synchronize()
            for k, f in enumerate(sh.frames):
                assert same(f["accum"], ref.buffers.accum) and same(f["display"], ref.buffers.display), f"fixed frame, shard {k}"
                assert torch.equal(sh.scenes[k].d_blue_noise, scene.d_blue_noise)
            continue
        thr = thr1 if step == "a1" else thr2
        out = sh.adaptive(P, mn, iv, thr)
        ref_out = single_adaptive(scene, ref, P, mn, iv, thr)
        assert len(torch.unique(ref_out[1])) >= 2
        assert_sharded_equals_single(sh, out, scene, ref, ref_out)
    assert sh.abandoned_waits() == [0, 0]
    sh.close(); ref.close()


def test_sharded_refusals(dragon):
    case = Case(dragon)
    sh = Shards(case, 2, 8)
    r = sh.rs[0]
    chk(V.lib.vpt_comm_p2p_enable(r.ctx, 0), r.ctx, "vpt_comm_p2p_enable")
    with pytest.raises(V.VptError, match="partitioned"):                   # a suspended exchange
        r.render_adaptive(8, min_passes=4, check_interval=4)
    chk(V.lib.vpt_comm_p2p_enable(r.ctx, 1), r.ctx, "vpt_comm_p2p_enable")
    r.kp.resolution = V._native.u2(W - 1, H)                               # another frame size than the exported one
    opt = V._native.adaptive_options(4, 4, 0.01)
    counts = torch.empty(r.n_local, dtype=torch.int32, device="cuda")
    rc = V.lib.vpt_render_adaptive(r.ctx, r.params.array, 8, C.byref(opt), C.c_void_p(counts.data_ptr()), None, None, None)
    assert rc == -1 and b"another frame size" in V.lib.vpt_last_error(r.ctx)
    r.kp.resolution = V._native.u2(W, H)
    sh.close()
    lone = V.Renderer(case.scene(), W, H, kp=case.kp(), cam=case.cam)       # no exchange block
    pc = C.c_uint64(0)
    assert V.lib.vpt_comm_p2p_adaptive_frame(lone.ctx, C.byref(pc), None) == -1
    lone.close()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs on the box")
def test_two_rank_adaptive_exchange_is_bitwise_identical():
    """tools/mgpu_adaptive_check.py under torchrun on 2 GPUs: DistributedRenderer.render_adaptive over real IPC peer mappings, two adaptive
    frames and a fixed-count frame back to back, each equal to the single-GPU frame bit for bit; NCCL mode is refused."""
    env = dict(os.environ); env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29534", os.path.join(ROOT, "tools", "mgpu_adaptive_check.py")]
    out = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
    print(out.stdout[-2000:], out.stderr[-2000:])
    assert out.returncode == 0 and "BITWISE_OK" in out.stdout
