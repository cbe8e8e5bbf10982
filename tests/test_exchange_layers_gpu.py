"""Exchange layers (vpt_comm_p2p_export_layers): depth, the compositing AOVs and the light groups full-frame in every rank's block.

R contexts on ONE GPU render the R shards of a frame and exchange through each other's blocks (same-process import, one scene per shard
with its own blue-noise replica, each shard on its own stream and its own Python thread, as in test_adaptive_sharded_gpu.py).  Pixels are
independent and every RNG stream is keyed by the global pixel, so every layer plane of every rank's block must equal the single-context
buffer bit for bit, as the accumulators and display words do.  The DistributedRenderer of each shard is bound to its exchange with
DistributedRenderer.over_exchange (one process cannot hold several torch.distributed ranks)."""
import ctypes as C
import os
import subprocess
import sys
import threading

import numpy as np
import pytest
import torch

import vpt_b200 as V
from vpt_b200.scene import synthetic_env
import adaptive_ref as A
from test_parity_gpu import make_kp

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLT_MAX = float(np.finfo(np.float32).max)
W, H = 333, 197                                    # ragged: neither a multiple of the 32x4 tile nor of any stripe height used here
LAYERS = tuple(V._native.LAYER_BITS)               # depth, alpha, volume, sun, point, emission, environment
ALL = 0x7F
LIGHTS = [((9.0, 6.0, 2.0), (1.0, 0.8, 0.6), 40.0), ((-2.0, 3.0, 8.0), (0.5, 0.7, 1.0), 25.0)]
SENTINEL = -12345.5
chk = V._native.check


@pytest.fixture(scope="module")
def dragon():
    return V.Volume.load_vdb(V.find_asset("dragon.vdb"))


@pytest.fixture(scope="module")
def emissive():
    """A synthetic fireball: a soft ball of density with a hot core, so the emission walk has something to add."""
    n = 48
    z, y, x = np.mgrid[0:n, 0:n, 0:n].astype(np.float32)
    c = (n - 1) / 2.0
    r = np.sqrt((x - c) ** 2 + (y - c) ** 2 + (z - c) ** 2) / c
    density = (np.clip(1.1 - r, 0.0, None) ** 1.5).astype(np.float32)
    heat = (3.0 * np.clip(0.8 - r, 0.0, None)).astype(np.float32)
    return V.Volume.from_dense(density, bbox_min=(-c, -c, -c), emission=heat)


@pytest.fixture(scope="module")
def atmosphere():
    atm = V.Atmosphere()
    yield atm
    atm.destroy()


def bits(t):
    t = t.contiguous()
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def same(a, b):
    return a.numel() == b.numel() and torch.equal(bits(a).reshape(-1), bits(b).reshape(-1))


class Case:
    """Scene factory (one scene per shard plus one for the single context), camera and Kernel_params of one configuration:
    hdri        dragon, point lights, the HDRI environment, direct integrator (generic kernel)
    bruneton    dragon, the precomputed sky, direct integrator (k_resolve<1>)
    vol_emit    the fireball, point lights, emission, volumetric path integrator (ends on the precomputed sky: k_resolve<2>)"""

    def __init__(self, name, dragon, emissive, atmosphere):
        self.name, self.atm = name, atmosphere
        self.vol = emissive if name == "vol_emit" else dragon
        self.cam = self.scene().frame_camera(W, H)

    def scene(self):
        lights = None if self.name == "bruneton" else LIGHTS
        s = V.Scene([self.vol.instance()], env=synthetic_env(512, 256), lights=lights)
        if self.name != "hdri": self.atm.apply(s.atmos)
        return s

    def kp(self):
        if self.name == "hdri": return make_kp(ray_depth=3, volume_depth=2)
        if self.name == "bruneton": return make_kp(environment_type=0, elevation=25.0, ray_depth=3)
        return make_kp(integrator=1, ray_depth=4, volume_depth=3, emission_scale=1.0, emission_pivot=1.0)

    def renderer(self, scene, rank=0, n_ranks=1, stripe_rows=16):
        return V.Renderer(scene, W, H, kp=self.kp(), cam=self.cam, rank=rank, n_ranks=n_ranks, stripe_rows=stripe_rows)


class Shards:
    """R contexts of one frame on one GPU sharing one peer-memory exchange with layers, and the single context of the same frame."""

    def __init__(self, case, R, stripe_rows, masks=ALL):
        masks = masks if isinstance(masks, (list, tuple)) else [masks] * R
        self.case, self.R, self.sr = case, R, stripe_rows
        self.scenes = [case.scene() for _ in range(R)]
        self.rs = [case.renderer(self.scenes[k], k, R, stripe_rows) for k in range(R)]
        self.ref_scene = case.scene()
        self.ref = case.renderer(self.ref_scene)
        blocks = (C.c_uint64 * R)()
        for k, r in enumerate(self.rs):
            raw = (C.c_ubyte * 64)()
            chk(V.lib.vpt_comm_p2p_export_layers(r.ctx, k, R, stripe_rows, W, H, 1, masks[k], raw), r.ctx, "vpt_comm_p2p_export_layers")
            b = C.c_uint64(0); chk(V.lib.vpt_comm_p2p_block(r.ctx, C.byref(b)), r.ctx, "vpt_comm_p2p_block"); blocks[k] = b.value
        self.blocks, self.masks = blocks, masks
        self.d = []
        if len(set(masks)) == 1:
            names = [n for n in LAYERS if masks[0] & V._native.LAYER_BITS[n]]
            for r in self.rs:
                chk(V.lib.vpt_comm_p2p_import_local(r.ctx, blocks), r.ctx, "vpt_comm_p2p_import_local")
                self.d.append(V.DistributedRenderer.over_exchange(r, layers=names, gather_display=True))
        self.streams = [torch.cuda.Stream() for _ in range(R)]
        torch.cuda.synchronize()

    def all(self, fn):
        """fn(k, renderer, stream) for every shard, each in its own thread; fn(-1, ref, None) for the single context first."""
        fn(-1, self.ref, None)
        torch.cuda.synchronize()
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

    def each(self, fn):
        """fn(renderer) on the single context and on every shard (set-up calls that exchange nothing)."""
        for r in [self.ref] + self.rs: fn(r)

    def render(self, n, iteration=None):
        def fn(k, r, stream):
            if iteration is not None: r.kp.iteration = iteration
            r.render(n, stream=stream)
        self.all(fn)

    def ref_layer(self, name):
        b = self.ref.buffers
        if name == "depth": return b.depth
        if name in ("alpha", "volume"): return getattr(b, name)
        return b.groups[name]

    def prefill(self, value=SENTINEL):
        """Every rank-local buffer, every buffer of the single context and every plane of every block := value (display: int(value))."""
        for r in [self.ref] + self.rs:
            b = r.buffers
            for t in (b.accum, b.cost, b.depth, b.raw, b.alpha, b.volume, *(b.groups.values() if b.groups else ())):
                if t is not None: t.fill_(value)
            b.display.fill_(int(value))
        for d in self.d:
            d.full.fill_(value); d.full_display.fill_(int(value))
            for name in d.layers: d._layer(name, "prefill").fill_(value)
        torch.cuda.synchronize()

    def check(self, what, layers=None, untouched=()):
        """Every rank's accum, display and layer planes against the single context, bit for bit; planes in `untouched` hold SENTINEL."""
        for k, d in enumerate(self.d):
            assert same(d.full, self.ref.buffers.accum), f"{what}: full-frame accum held by shard {k}"
            assert same(d.full_display, self.ref.buffers.display), f"{what}: full-frame display held by shard {k}"
            for name in (layers if layers is not None else d.layers):
                plane = d._layer(name, "check")
                if name in untouched:
                    assert bool((plane == SENTINEL).all()), f"{what}: layer {name} of shard {k} was written"
                else:
                    assert same(plane, self.ref_layer(name)), f"{what}: layer {name} held by shard {k}"
            assert torch.equal(self.scenes[k].d_blue_noise, self.ref_scene.d_blue_noise), f"{what}: blue-noise replica of shard {k}"

    def abandoned_waits(self):
        out = []
        for r in self.rs:
            n = C.c_uint64(0); chk(V.lib.vpt_comm_p2p_status(r.ctx, C.byref(n)), r.ctx, "vpt_comm_p2p_status"); out.append(int(n.value))
        return out

    def close(self):
        self.d.clear()
        for r in self.rs: r.close()
        self.ref.close()


def enable_all(r):
    r.enable_aovs(); r.enable_light_groups()


def some_signal(sh):
    """The frame must exercise the layers: coverage somewhere, volume colour, and each light class that the scene has."""
    b = sh.ref.buffers
    assert float(b.alpha.max()) > 0 and float(b.depth.max()) > 0 and float(b.volume.max()) > 0
    assert float(b.groups["environment"].max()) > 0
    if sh.case.name == "vol_emit": assert float(b.groups["emission"].max()) > 0


# case, ranks, stripe rows: 1, 16 and an odd stripe height, both integrators, HDRI and the precomputed sky, lights and emission
FIXED = [("hdri", 2, 1), ("hdri", 3, 16), ("bruneton", 3, 7), ("vol_emit", 2, 7), ("vol_emit", 3, 1)]


@pytest.mark.parametrize("name,R,stripe_rows", FIXED)
def test_fixed_count_frames_carry_every_layer(dragon, emissive, atmosphere, name, R, stripe_rows):
    """A new frame, a continued call, a call with render == 0 and a call past max_interactions (the kernel tail), then the denoiser."""
    sh = Shards(Case(name, dragon, emissive, atmosphere), R, stripe_rows)
    sh.each(enable_all)
    sh.render(5, iteration=0); sh.check("iteration 0"); some_signal(sh)
    sh.render(4); sh.check("continued")
    sh.each(lambda r: setattr(r.kp, "render", 0))
    sh.render(2); sh.check("render == 0")
    sh.each(lambda r: (setattr(r.kp, "render", 1), setattr(r.kp, "max_interactions", r.kp.iteration)))
    sh.render(2); sh.check("iteration >= max_interactions")
    want = sh.ref.denoise(display=True)
    for k, d in enumerate(sh.d):
        got = d.denoise(display=True)
        assert same(got[0], want[0]) and same(got[1], want[1]), f"denoised frame of shard {k}"
    assert sh.abandoned_waits() == [0] * R
    sh.close()


def test_sharded_adaptive_frame_carries_every_layer_and_denoises_alike(dragon, emissive, atmosphere):
    P, mn, iv = 24, 4, 4
    sh = Shards(Case("hdri", dragon, emissive, atmosphere), 3, 5)
    sh.each(enable_all)
    sh.ref.kp.iteration = 0
    _, _, first = sh.ref.render_adaptive(P, threshold=FLT_MAX, min_passes=mn, check_interval=iv, error_map=True)
    thr = float(np.quantile(A.max3x3(first.cpu().numpy()), 0.4))        # stops part of the frame at the first test
    sh.ref_scene.reset_blue_noise()
    res = {}

    def fn(k, r, stream):
        r.kp.iteration = 0
        if k < 0:
            res["ref"] = r.render_adaptive(P, threshold=thr, min_passes=mn, check_interval=iv, error_map=True)
        else:
            return sh.d[k].render_adaptive(P, threshold=thr, min_passes=mn, check_interval=iv, error_map=True, stream=stream)
    out = sh.all(fn)
    run, counts, err = res["ref"]
    assert len(torch.unique(counts)) >= 2
    for k, (run_k, counts_k, err_k) in enumerate(out):
        assert run_k == run and same(counts_k, counts) and same(err_k, err), f"adaptive frame of shard {k}"
    sh.check("adaptive")
    want = sh.ref.denoise(rel_error=err)
    for k, d in enumerate(sh.d):
        assert same(d.denoise(), want), f"denoised adaptive frame of shard {k}"
    assert sh.abandoned_waits() == [0, 0, 0]
    sh.close()


def test_region_frame_stores_only_the_region(dragon, emissive, atmosphere):
    sh = Shards(Case("hdri", dragon, emissive, atmosphere), 2, 16)
    sh.each(enable_all)
    sh.prefill()
    sh.each(lambda r: r.set_region(37, 21, 301, 150))
    sh.render(5, iteration=0); sh.check("region frame")
    sh.render(3); sh.check("continued region frame")
    plane = sh.d[0].full_depth()
    assert bool((plane[:21] == SENTINEL).all()) and bool((plane[21:150, 37:301] != SENTINEL).any())
    sh.close()


def test_equirect_panorama_with_miss_cull(dragon, emissive, atmosphere):
    sh = Shards(Case("hdri", dragon, emissive, atmosphere), 3, 7)
    sh.each(enable_all)
    sh.each(lambda r: (r.set_projection("equirect", hfov=360.0, vfov=180.0), r.set_option("miss_cull", 1)))
    sh.render(6, iteration=0); sh.check("equirectangular frame")
    sh.close()


def test_depth_only_with_aovs_enabled(dragon, emissive, atmosphere):
    sh = Shards(Case("hdri", dragon, emissive, atmosphere), 2, 1, masks=V._native.LAYER_BITS["depth"])
    sh.each(enable_all)
    sh.render(5, iteration=0); sh.check("depth only", layers=("depth",))
    for d in sh.d:
        assert d.layers == ("depth",)
        p = C.c_uint64(0)
        assert V.lib.vpt_comm_p2p_layer(d.r.ctx, V._native.LAYER_BITS["alpha"], C.byref(p)) == -1
        assert b"exported without layer" in V.lib.vpt_last_error(d.r.ctx)
        with pytest.raises(V.VptError, match="not requested"):
            d.full_alpha()
        with pytest.raises(V.VptError, match="not requested"):
            d.full_light_group("sun")
    sh.close()


def test_exported_layer_that_is_not_active_keeps_its_plane(dragon, emissive, atmosphere):
    """No AOVs or groups on the first frame; then AOVs registered between two calls of a frame stay inactive until the next iteration-0
    call, and groups that were never registered stay off: their planes keep the sentinel while depth and accum follow the frame."""
    sh = Shards(Case("hdri", dragon, emissive, atmosphere), 2, 16)
    sh.render(3, iteration=0)
    sh.each(lambda r: r.enable_aovs())
    sh.prefill()
    sh.render(2, iteration=0)
    sh.each(lambda r: r.enable_light_groups())
    idle = ("sun", "point", "emission", "environment")
    sh.check("AOVs on, groups registered mid-frame", untouched=idle)
    sh.render(2); sh.check("continued", untouched=idle)
    sh.close()


def test_refusals(dragon, emissive, atmosphere):
    case = Case("hdri", dragon, emissive, atmosphere)
    r = case.renderer(case.scene(), 0, 2, 8)
    raw = (C.c_ubyte * 64)()
    assert V.lib.vpt_comm_p2p_export_layers(r.ctx, 0, 2, 8, W, H, 1, 0x80, raw) == -1
    assert b"unknown layer" in V.lib.vpt_last_error(r.ctx)
    chk(V.lib.vpt_comm_p2p_export_layers(r.ctx, 0, 2, 8, W, H, 1, 0x05, raw), r.ctx, "vpt_comm_p2p_export_layers")
    p = C.c_uint64(0)
    for bad in (0x02, 0x03, 0x80, 0):
        assert V.lib.vpt_comm_p2p_layer(r.ctx, bad, C.byref(p)) == -1, hex(bad)
    for good in (0x01, 0x04):
        chk(V.lib.vpt_comm_p2p_layer(r.ctx, good, C.byref(p)), r.ctx, "vpt_comm_p2p_layer"); assert p.value
    r.close()
    lone = case.renderer(case.scene())
    with pytest.raises(V.VptError, match="unknown layer"):
        V.DistributedRenderer.over_exchange(lone, layers=("depth", "normals"))
    lone.close()

    sh = Shards(case, 2, 8, masks=[0x01, 0x03])                           # mismatched masks: neither rank maps the other
    for k, r in enumerate(sh.rs):
        assert V.lib.vpt_comm_p2p_import_local(r.ctx, sh.blocks) == -1
        msg = V.lib.vpt_last_error(r.ctx).decode()
        assert f"rank {1 - k} exported" in msg and "layers 0x0" in msg, msg
        assert V.lib.vpt_comm_p2p_enable(r.ctx, 1) == -1                    # nothing was mapped
    sh.close()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs on the box")
def test_two_rank_layers_over_ipc_are_bitwise_identical():
    """tools/mgpu_layers_check.py under torchrun on 2 GPUs: DistributedRenderer(layers=all) over real IPC peer mappings, every plane equal
    to the single-GPU buffers bit for bit."""
    env = dict(os.environ); env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29537", os.path.join(ROOT, "tools", "mgpu_layers_check.py")]
    out = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
    print(out.stdout[-2000:], out.stderr[-2000:])
    assert out.returncode == 0 and "BITWISE_OK" in out.stdout
