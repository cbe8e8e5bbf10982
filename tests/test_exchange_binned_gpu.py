"""Binned exchange layers (vpt_comm_p2p_export_binned): the deep slices and the instance mattes full-frame in every rank's block.

R contexts on ONE GPU render the R shards of a frame and exchange through each other's blocks (same-process import, one scene per shard
with its own blue-noise replica, each shard on its own stream and its own Python thread, as in test_exchange_layers_gpu.py).  Pixels are
independent and every RNG stream is keyed by the global pixel, so every slice and matte of every rank's block must equal the single
context's deep_image() / matte_image() bit for bit, as the accumulators and display words do.  The DistributedRenderer of each shard is
bound to its exchange with DistributedRenderer.over_exchange."""
import ctypes as C
import os
import subprocess
import sys
import threading

import numpy as np
import pytest
import torch

import vpt_b200 as V
from vpt_b200 import deep as D
from vpt_b200.scene import synthetic_env
import adaptive_ref as A
from test_parity_gpu import make_kp

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLT_MAX = float(np.finfo(np.float32).max)
W, H = 333, 197                                    # ragged: neither a multiple of the 32x4 tile nor of any stripe height used here
LAYERS = tuple(V._native.LAYER_BITS)
ALL = 0x7F
LIGHTS = [((9.0, 6.0, 2.0), (1.0, 0.8, 0.6), 40.0), ((-2.0, 3.0, 8.0), (0.5, 0.7, 1.0), 25.0)]
SENTINEL = -12345.5
INF = float("inf")
chk = V._native.check
DEEP, MATTES = V._native.VPT_BINNED_DEEP, V._native.VPT_BINNED_MATTES


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
    vol_emit    the fireball, point lights, emission, volumetric path integrator (ends on the precomputed sky: k_resolve<2>)
    instances   two dragons side by side, point lights, the HDRI, direct integrator: a multi-instance scene for the mattes"""

    def __init__(self, name, dragon, emissive, atmosphere):
        self.name, self.atm, self.dragon = name, atmosphere, dragon
        self.vol = emissive if name == "vol_emit" else dragon
        s = self.scene()
        self.cam = s.frame_camera(W, H)
        self.n_instances = len(s.instances)
        lo, hi = s.world_bounds()
        o = np.array([self.cam.origin.x, self.cam.origin.y, self.cam.origin.z], dtype=np.float64)
        d, size = float(np.linalg.norm((hi + lo) / 2.0 - o)), float(np.linalg.norm(hi - lo))
        self.near, self.far = max(0.0, d - size), d + size

    def scene(self):
        lights = None if self.name == "bruneton" else LIGHTS
        if self.name == "instances":
            insts = [self.dragon.instance(pos=(-20.0, 0.0, 0.0)), self.dragon.instance(pos=(20.0, 0.0, 0.0))]
        else:
            insts = [self.vol.instance()]
        s = V.Scene(insts, env=synthetic_env(512, 256), lights=lights)
        if self.name in ("bruneton", "vol_emit"): self.atm.apply(s.atmos)
        return s

    def kp(self):
        if self.name == "bruneton": return make_kp(environment_type=0, elevation=25.0, ray_depth=3)
        if self.name == "vol_emit": return make_kp(integrator=1, ray_depth=4, volume_depth=3, emission_scale=1.0, emission_pivot=1.0)
        return make_kp(ray_depth=3, volume_depth=2)

    def renderer(self, scene, rank=0, n_ranks=1, stripe_rows=16):
        return V.Renderer(scene, W, H, kp=self.kp(), cam=self.cam, rank=rank, n_ranks=n_ranks, stripe_rows=stripe_rows)

    def bounds(self, k):
        """k slices: {0, inf} for k = 1, else k - 1 equal steps across the volume's depth range and an open last slice"""
        if k == 1: return [0.0, INF]
        return [float(z) for z in np.linspace(self.near, self.far, k)] + [INF]

    def sets(self, k):
        """k mattes: every instance in matte 0 for k = 1, else instance i in matte i and the sphere in the last matte"""
        if k == 1: return [list(range(self.n_instances))], 0
        sets = [[i] if i < self.n_instances else [] for i in range(k)]
        return sets, k - 1


class Shards:
    """R contexts of one frame on one GPU sharing one peer-memory exchange with binned layers, and the single context of the same frame."""

    def __init__(self, case, R, stripe_rows, mask=0, n_slices=0, n_mattes=0, counts=None):
        self.case, self.R, self.sr = case, R, stripe_rows
        counts = counts or [(n_slices, n_mattes)] * R
        self.scenes = [case.scene() for _ in range(R)]
        self.rs = [case.renderer(self.scenes[k], k, R, stripe_rows) for k in range(R)]
        self.ref_scene = case.scene()
        self.ref = case.renderer(self.ref_scene)
        blocks = (C.c_uint64 * R)()
        for k, r in enumerate(self.rs):
            raw = (C.c_ubyte * 64)()
            chk(V.lib.vpt_comm_p2p_export_binned(r.ctx, k, R, stripe_rows, W, H, 1, mask, counts[k][0], counts[k][1], raw), r.ctx,
                "vpt_comm_p2p_export_binned")
            b = C.c_uint64(0); chk(V.lib.vpt_comm_p2p_block(r.ctx, C.byref(b)), r.ctx, "vpt_comm_p2p_block"); blocks[k] = b.value
        self.blocks = blocks
        self.d = []
        if len(set(counts)) == 1:
            names = [n for n in LAYERS if mask & V._native.LAYER_BITS[n]]
            for r in self.rs:
                chk(V.lib.vpt_comm_p2p_import_local(r.ctx, blocks), r.ctx, "vpt_comm_p2p_import_local")
                self.d.append(V.DistributedRenderer.over_exchange(r, layers=names, gather_display=True, deep_slices=n_slices, n_mattes=n_mattes))
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

    def enable(self, deep=0, mattes=0, layers=False):
        bounds = self.case.bounds(deep) if deep else None
        sets, sphere = self.case.sets(mattes) if mattes else (None, None)

        def fn(r):
            if layers: r.enable_aovs(); r.enable_light_groups()
            if deep: r.enable_deep(bounds)
            if mattes: r.enable_mattes(sets, sphere)
        self.each(fn)

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
        """Every rank-local buffer, every buffer of the single context and every plane and array of every block := value."""
        for r in [self.ref] + self.rs:
            b = r.buffers
            for t in (b.accum, b.cost, b.depth, b.raw, b.alpha, b.volume, b.deep, b.mattes, *(b.groups.values() if b.groups else ())):
                if t is not None: t.fill_(value)
            b.display.fill_(int(value))
        for d in self.d:
            d.full.fill_(value); d.full_display.fill_(int(value))
            for name in d.layers: d._layer(name, "prefill").fill_(value)
            if d.deep_slices: d.full_deep().fill_(value)
            if d.n_mattes: d.full_mattes().fill_(value)
        torch.cuda.synchronize()

    def check(self, what, untouched=()):
        """Every rank's accum, display, layer planes and binned arrays against the single context, bit for bit; binned layers in
        `untouched` ("deep", "mattes") hold SENTINEL."""
        for k, d in enumerate(self.d):
            assert same(d.full, self.ref.buffers.accum), f"{what}: full-frame accum held by shard {k}"
            assert same(d.full_display, self.ref.buffers.display), f"{what}: full-frame display held by shard {k}"
            for name in d.layers:
                assert same(d._layer(name, "check"), self.ref_layer(name)), f"{what}: layer {name} held by shard {k}"
            for name, count, full, ref in (("deep", d.deep_slices, d.full_deep, self.ref.deep_image),
                                           ("mattes", d.n_mattes, d.full_mattes, self.ref.matte_image)):
                if not count: continue
                got = full()
                assert got.shape == (count, H, W, 4), f"{what}: {name} array of shard {k} is {tuple(got.shape)}"
                if name in untouched:
                    assert bool((got == SENTINEL).all()), f"{what}: {name} of shard {k} was written"
                else:
                    assert same(got, ref()), f"{what}: {name} held by shard {k}"
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


def some_signal(sh, deep=0, mattes=0):
    """The frame must exercise the binned layers: coverage in more than one slice of a frame of 8 slices or more, in every instance's
    matte."""
    if deep:
        cov = sh.ref.deep_image()[..., 3].flatten(1).amax(1)
        assert float(cov.max()) > 0 and (deep < 8 or int((cov > 0).sum()) >= 2), cov
    if mattes:
        cov = sh.ref.matte_image()[..., 3].flatten(1).amax(1)
        assert all(float(cov[i]) > 0 for i in range(min(mattes, sh.case.n_instances))), cov


# case, ranks, stripe rows, deep slices, mattes, with all seven layers: the three resolve kernels, K = 1 / 8 / 32 slices, one matte with
# everything mapped and three with a sphere matte, both together with every layer
FIXED = [("hdri", 2, 1, 1, 0, False), ("bruneton", 3, 7, 8, 1, False), ("vol_emit", 2, 16, 32, 1, False),
         ("instances", 3, 1, 0, 1, False), ("instances", 2, 7, 0, 3, False), ("instances", 3, 16, 8, 3, True)]


@pytest.mark.parametrize("name,R,stripe_rows,n_slices,n_mattes,layers", FIXED)
def test_fixed_count_frames_carry_the_binned_layers(dragon, emissive, atmosphere, name, R, stripe_rows, n_slices, n_mattes, layers):
    """A new frame, a continued call, a call with render == 0 and a call past max_interactions (the kernel tail)."""
    sh = Shards(Case(name, dragon, emissive, atmosphere), R, stripe_rows, ALL if layers else 0, n_slices, n_mattes)
    sh.enable(n_slices, n_mattes, layers)
    sh.render(5, iteration=0); sh.check("iteration 0"); some_signal(sh, n_slices, n_mattes)
    sh.render(4); sh.check("continued")
    sh.each(lambda r: setattr(r.kp, "render", 0))
    sh.render(2); sh.check("render == 0")
    sh.each(lambda r: (setattr(r.kp, "render", 1), setattr(r.kp, "max_interactions", r.kp.iteration)))
    sh.render(2); sh.check("iteration >= max_interactions")
    assert sh.abandoned_waits() == [0] * R
    sh.close()


def test_sharded_adaptive_frame_carries_the_binned_layers(dragon, emissive, atmosphere):
    P, mn, iv = 24, 4, 4
    sh = Shards(Case("instances", dragon, emissive, atmosphere), 3, 5, ALL, 8, 3)
    sh.enable(8, 3, layers=True)
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
    sh.check("adaptive"); some_signal(sh, 8, 3)
    assert sh.abandoned_waits() == [0, 0, 0]
    sh.close()


def test_region_frame_stores_only_the_region(dragon, emissive, atmosphere):
    sh = Shards(Case("instances", dragon, emissive, atmosphere), 2, 16, 0, 8, 3)
    sh.enable(8, 3)
    sh.prefill()
    sh.each(lambda r: r.set_region(37, 21, 301, 150))
    sh.render(5, iteration=0); sh.check("region frame")
    sh.render(3); sh.check("continued region frame")
    for full in (sh.d[0].full_deep(), sh.d[1].full_mattes()):
        inside = torch.zeros(H, W, dtype=torch.bool, device=full.device); inside[21:150, 37:301] = True
        assert bool((full[:, ~inside] == SENTINEL).all()) and bool((full[:, inside] != SENTINEL).all())
    sh.close()


def test_equirect_panorama_with_miss_cull(dragon, emissive, atmosphere):
    sh = Shards(Case("instances", dragon, emissive, atmosphere), 3, 7, 0, 8, 3)
    sh.enable(8, 3)
    sh.each(lambda r: (r.set_projection("equirect", hfov=360.0, vfov=180.0), r.set_option("miss_cull", 1)))
    sh.render(6, iteration=0); sh.check("equirectangular frame")
    sh.close()


def test_ods_panorama_with_miss_cull(dragon, emissive, atmosphere):
    sh = Shards(Case("hdri", dragon, emissive, atmosphere), 2, 16, 0, 8, 1)
    sh.enable(8, 1)
    sh.each(lambda r: (r.set_projection("ods", hfov=360.0, vfov=180.0, ipd=2.0, layout="left"), r.set_option("miss_cull", 1)))
    sh.render(6, iteration=0); sh.check("ODS frame")
    sh.close()


def test_exported_binned_layers_that_are_not_active_keep_their_arrays(dragon, emissive, atmosphere):
    """No slices or mattes on the first frame; then slices registered before an iteration-0 call take over, while mattes registered
    between two calls of a frame stay inactive until the next iteration-0 call: their arrays keep the sentinel meanwhile."""
    case = Case("instances", dragon, emissive, atmosphere)
    sh = Shards(case, 3, 7, 0, 4, 2)
    sh.render(3, iteration=0)
    sets, sphere = case.sets(2)
    sh.each(lambda r: r.enable_deep(case.bounds(4)))
    sh.prefill()
    sh.render(2, iteration=0)
    sh.each(lambda r: r.enable_mattes(sets, sphere))
    sh.check("slices on, mattes registered mid-frame", untouched=("mattes",))
    sh.render(2); sh.check("continued", untouched=("mattes",))
    sh.render(2, iteration=0); sh.check("mattes taken over"); some_signal(sh, 4, 2)
    sh.close()


def test_refusals(dragon, emissive, atmosphere):
    case = Case("instances", dragon, emissive, atmosphere)
    # counts out of range, and vpt_comm_p2p_binned on a block without the layer
    r = case.renderer(case.scene(), 0, 2, 8)
    raw = (C.c_ubyte * 64)()
    for ns, nm in ((33, 0), (0, 33)):
        assert V.lib.vpt_comm_p2p_export_binned(r.ctx, 0, 2, 8, W, H, 1, 0, ns, nm, raw) == -1
        assert b"must be 0 or 1..32" in V.lib.vpt_last_error(r.ctx)
    chk(V.lib.vpt_comm_p2p_export_binned(r.ctx, 0, 2, 8, W, H, 1, 0, 5, 0, raw), r.ctx, "vpt_comm_p2p_export_binned")
    p, k = C.c_uint64(0), C.c_uint(0)
    chk(V.lib.vpt_comm_p2p_binned(r.ctx, DEEP, C.byref(p), C.byref(k)), r.ctx, "vpt_comm_p2p_binned")
    assert p.value % 256 == 0 and k.value == 5
    assert V.lib.vpt_comm_p2p_binned(r.ctx, MATTES, C.byref(p), C.byref(k)) == -1
    assert b"exported without mattes" in V.lib.vpt_last_error(r.ctx)
    for bad in (0, 3):
        assert V.lib.vpt_comm_p2p_binned(r.ctx, bad, C.byref(p), C.byref(k)) == -1
    r.close()

    # mismatched counts: neither rank maps the other, and the message names the rank and both counts
    sh = Shards(case, 2, 8, 0, counts=[(8, 1), (4, 1)])
    for k, r in enumerate(sh.rs):
        assert V.lib.vpt_comm_p2p_import_local(r.ctx, sh.blocks) == -1
        msg = V.lib.vpt_last_error(r.ctx).decode()
        mine, theirs = (8, 4) if k == 0 else (4, 8)
        assert f"rank {1 - k} exported its block with {theirs} deep slices and 1 mattes" in msg, msg
        assert f"this rank ({k}) with {mine} deep slices" in msg, msg
        assert V.lib.vpt_comm_p2p_enable(r.ctx, 1) == -1                    # nothing was mapped
    sh.close()
    sh = Shards(case, 2, 8, 0x01, counts=[(0, 2), (0, 3)])
    for k, r in enumerate(sh.rs):
        assert V.lib.vpt_comm_p2p_import_local(r.ctx, sh.blocks) == -1
        assert "mattes" in V.lib.vpt_last_error(r.ctx).decode()
    sh.close()


def test_count_mismatch_at_render_time_enqueues_nothing(dragon, emissive, atmosphere):
    """Every rank with 4 active slices on an exchange of 8 is refused before it enqueues anything: no flag wait is abandoned, and the next
    call with 8 slices works on the same exchange.  Then the same for the mattes."""
    case = Case("instances", dragon, emissive, atmosphere)
    sh = Shards(case, 3, 7, 0, 8, 3)
    sh.enable(0, 3)
    for what, wrong, right in (("deep slices", lambda r: r.enable_deep(case.bounds(4)), lambda r: r.enable_deep(case.bounds(8))),
                               ("mattes", lambda r: r.enable_mattes([[0], [1]]), lambda r: r.enable_mattes(*case.sets(3)))):
        sh.each(wrong)
        errs = []

        def fn(k, r, stream):
            if k < 0: return
            r.kp.iteration = 0
            try:
                r.render(3, stream=stream)
            except V.VptError as e:
                errs.append(str(e))
        sh.all(fn)
        assert len(errs) == 3, errs
        for e in errs:
            assert f"exported with {8 if what == 'deep slices' else 3} {what}" in e and f"are {4 if what == 'deep slices' else 2}" in e, e
        assert sh.abandoned_waits() == [0, 0, 0]
        sh.each(right)
        sh.render(3, iteration=0); sh.check(f"after the refused {what}")
        assert sh.abandoned_waits() == [0, 0, 0]
    sh.close()


def test_python_full_frames_and_refusals(dragon, emissive, atmosphere, tmp_path):
    """over_exchange's full_deep() / full_mattes() on shards, deep.flatten / insert / exr_samples on full_deep(), the copies on one rank,
    and the VptError cases."""
    case = Case("instances", dragon, emissive, atmosphere)
    sh = Shards(case, 2, 7, 0, 8, 3)
    sh.enable(8, 3)
    sh.render(4, iteration=0); sh.check("python")
    bounds = sh.ref.deep_bounds
    want, got = sh.ref.deep_image(), sh.d[1].full_deep()
    z = 0.5 * (case.near + case.far)
    element = torch.rand(H, W, 4, device=want.device); element[..., :3] *= element[..., 3:]
    plate = torch.rand(H, W, 3, device=want.device)
    for a, b in zip(D.flatten(got, bounds), D.flatten(want, bounds)): assert same(a, b)
    for a, b in zip(D.flatten(got, bounds, z), D.flatten(want, bounds, z)): assert same(a, b)
    for a, b in zip(D.insert(got, bounds, z, element, plate), D.insert(want, bounds, z, element, plate)): assert same(a, b)
    for a, b in zip(D.exr_samples(got, bounds), D.exr_samples(want, bounds)): assert same(a, b)
    d = sh.d[0]
    with pytest.raises(V.VptError, match="4 deep slices, but the peer-memory exchange carries 8"):
        d.enable_deep(case.bounds(4))
    with pytest.raises(V.VptError, match="2 mattes, but the peer-memory exchange carries 3"):
        d.enable_mattes([[0], [1]])
    d.exchange = "nccl"                                                   # as after a fallback to the NCCL exchange
    with pytest.raises(V.VptError, match="does not carry deep slices"):
        d.full_deep()
    with pytest.raises(V.VptError, match="does not carry mattes"):
        d.full_mattes()
    d.exchange = "p2p"
    with pytest.raises(V.VptError, match="was exported with 8"):
        V.DistributedRenderer.over_exchange(sh.rs[0], deep_slices=4, n_mattes=3)
    sh.close()

    sh = Shards(case, 2, 7, 0, 8, 0)
    with pytest.raises(V.VptError, match="mattes were not requested"):
        sh.d[0].full_mattes()
    sh.close()

    # one rank: copies of the renderer's buffers
    import torch.distributed as dist
    own = not dist.is_initialized()
    if own: dist.init_process_group("gloo", init_method=f"file://{tmp_path}/pg", rank=0, world_size=1)
    try:
        one = V.DistributedRenderer(case.scene(), W, H, cam=case.cam, kp=case.kp(), deep_slices=8, n_mattes=3)
        one.enable_deep(case.bounds(8)); one.enable_mattes(*case.sets(3))
        one.render(3); torch.cuda.synchronize()
        for full, img in ((one.full_deep(), one.r.deep_image()), (one.full_mattes(), one.r.matte_image())):
            assert full.shape == (img.shape[0], H, W, 4) and same(full, img) and full.data_ptr() != img.data_ptr()
        one.close()
        none = V.DistributedRenderer(case.scene(), W, H, cam=case.cam, kp=case.kp())
        with pytest.raises(V.VptError, match="deep slices were not requested"):
            none.full_deep()
        none.close()
    finally:
        if own: dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs on the box")
def test_two_rank_binned_layers_over_ipc_are_bitwise_identical():
    """tools/mgpu_binned_check.py under torchrun on 2 GPUs: DistributedRenderer(deep_slices=8, n_mattes=3) over real IPC peer mappings,
    every slice and matte equal to the single-GPU buffers bit for bit."""
    env = dict(os.environ); env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29541", os.path.join(ROOT, "tools", "mgpu_binned_check.py")]
    out = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
    print(out.stdout[-2000:], out.stderr[-2000:])
    assert out.returncode == 0 and "BITWISE_OK" in out.stdout
