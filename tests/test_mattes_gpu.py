"""Instance mattes on the GPU (vpt_set_instance_mattes): the compositing AOVs split by the volume instance of each camera ray's first
collision (include/vpt_b200.h, DESIGN.md section 8l).

Cases: the headline frame (lean kernel, compact records), lights + sphere + thin lens, the volumetric path integrator on the tabulated
sky, the Bruneton sky, 120 instances, the NaN / Inf environment stripes on prefilled buffers, and the mixed scene S1 of
tests/mixed_scenes.py (different volumes, several per leaf).  Frames are 8 passes in chunks of 5 + 3 unless said otherwise."""
import ctypes as C

import numpy as np
import pytest
import torch

import vpt_b200 as V
import mixed_scenes as M
from vpt_b200.renderer import stripe_rows_of_rank
from vpt_b200.scene import synthetic_env
from test_aov_gpu import make_aov_case
from test_deep_gpu import bitwise, pattern
from test_parity_gpu import make_kp
from test_projection_gpu import headline_pano

pytestmark = pytest.mark.gpu
BUFFERS = ("accum", "depth", "cost", "raw", "display")
AOVS = ("alpha", "volume")
PASSES = 8
INF = float("inf")
SENTINEL = 0x7FBADBAD
NAMES = ["headline", "lights_sphere", "vol_sky_table", "sky", "instanced", "nan_prefilled", "mixed"]
GROUPS_TOO = ("lights_sphere", "vol_sky_table", "mixed")


@pytest.fixture(scope="module")
def dragon():
    return V.Volume.load_vdb(V.find_asset("dragon.vdb"))


@pytest.fixture(scope="module")
def vols():
    return M.Volumes()


@pytest.fixture(scope="module")
def cases(dragon, vols):
    cache = {}
    def get(name):
        if name not in cache:
            if name == "mixed":                                  # different volumes, up to four per leaf, lights and the sphere
                scene = M.build_s1(vols)
                cam = scene.frame_camera(256, 160)
                def mk():
                    r = V.Renderer(scene, 256, 160, kp=make_kp(ray_depth=3), cam=cam, options={"passes_per_chunk": 5})
                    r.enable_aovs()
                    return r
                cache[name] = (scene, mk, [])
            else:
                cache[name] = make_aov_case(name, dragon, None)
        return cache[name]
    return get


def run(scene, r, passes=PASSES, single=False, fill=None):
    """a new frame of `passes` passes from non-zero buffers (the case's prefill, the AOVs from a pattern; the mattes from their own
    pattern, or the words `fill`)"""
    scene.reset_blue_noise(); r.kp.iteration = 0; r.buffers.zero_()
    b, dev = r.buffers, r.buffers.accum.device
    if hasattr(r, "prefill"):
        r.prefill()
    if b.volume is not None:
        first = pattern(1, r.n_local, 0, dev)[0]
        b.volume.copy_(first[:, :3]); b.alpha.copy_(first[:, 3])
    if b.mattes is not None:
        if fill is not None: b.mattes.view(torch.int32).fill_(fill)
        else: b.mattes.copy_(pattern(b.mattes.shape[0], r.n_local, 0, dev))
    if b.deep is not None:
        b.deep.copy_(pattern(b.deep.shape[0], r.n_local, 0, dev))
    if single:
        for _ in range(passes): r.render_pass()
    else:
        r.render(passes)
    torch.cuda.synchronize()
    out = {k: getattr(b, k).clone() for k in BUFFERS + AOVS + ("deep", "mattes") if getattr(b, k) is not None}
    if b.groups: out.update({"group_" + g: t.clone() for g, t in b.groups.items()})
    out["blue_noise"] = scene.d_blue_noise.clone()
    return out


def everything(scene):
    return [list(range(len(scene.instances)))]


@pytest.mark.parametrize("name", NAMES)
def test_mattes_interfere_with_nothing_and_one_matte_is_the_aovs(cases, name):
    """(1) accum, depth, cost, raw, display, the blue noise, the AOVs, the light groups and the deep slices are bit-identical with the
    mattes off and on; (2) K = 1 with every instance and the sphere mapped is (volume, alpha) bit for bit; the fused 5 + 3 chunks give
    the mattes of 8 single-pass calls."""
    scene, mk, _ = cases(name)
    groups = name in GROUPS_TOO

    def make(mattes):
        r = mk()
        if groups: r.enable_light_groups()
        r.enable_deep([0.0, 30.0, INF])
        if mattes: r.enable_mattes(everything(scene), sphere=0)
        return r

    off_r, r = make(False), make(True)
    off, on = run(scene, off_r), run(scene, r)
    assert r.stats()[0] - off_r.stats()[0] == 2, "one more resolve kernel per chunk (5 + 3) with the mattes on"
    for k in off:
        assert bitwise(on[k], off[k]), f"{name}: {k} changes when the mattes are on"
    assert 0.0 < float(on["alpha"].mean()) < 1.0, "the frame must show volume and background"
    m = on["mattes"][0]
    assert bitwise(m[:, :3], on["volume"]), f"{name}: the colour of the one matte is not the volume AOV"
    assert bitwise(m[:, 3], on["alpha"]), f"{name}: the coverage of the one matte is not alpha"
    single = run(scene, make(True), single=True)
    assert bitwise(single["mattes"], on["mattes"]), f"{name}: 8 single passes differ from the fused 5 + 3 chunks"


@pytest.mark.parametrize("name", ["instanced", "mixed", "lights_sphere"])
def test_each_matte_is_its_own_frame_and_they_sum_to_the_aovs(cases, name):
    """(2) each matte of K = 4 is bit for bit the single matte of a K = 1 frame whose map selects the same set; with every id mapped the
    mattes sum to (volume, alpha) within the rounding of the separate means (the bound of test_deep_gpu.test_slices_sum_to_the_aovs)."""
    scene, mk, _ = cases(name)
    n = len(scene.instances)
    sets = [[i for i in range(n) if i % 3 == k] for k in range(3)] + [[]]
    r = mk(); r.enable_mattes(sets, sphere=3)
    f = run(scene, r)
    if n > 1:
        assert sum(float(f["mattes"][k][:, 3].sum()) > 0.0 for k in range(3)) >= 2, "at least two instance mattes must be covered"
    one = mk()
    for k in range(4):
        one.enable_mattes([sets[k]], sphere=0 if k == 3 else None)
        g = run(scene, one)
        assert bitwise(g["mattes"][0], f["mattes"][k]), f"{name}: matte {k} differs from the frame of its own set"
    K, eps = 4, 2.0 ** -24
    s = f["mattes"].double()
    aov = torch.cat([f["volume"], f["alpha"][:, None]], 1).double()
    scale = torch.maximum(aov.abs(), s.abs().amax(0))
    err = (s.sum(0) - aov).abs()
    assert bool((err <= (K + 2) * 4 * PASSES * PASSES * eps * scale).all()), f"{name}: the mattes do not sum to the AOVs"


def ray_hits_box(o, d, lo, hi):
    """float64 slab test of the rays o + t d (t >= 0) against the box [lo, hi]: (n,) bool"""
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = 1.0 / d
        t0, t1 = (lo - o) * inv, (hi - o) * inv
    tn = np.nanmax(np.minimum(t0, t1), axis=1)
    tf = np.nanmin(np.maximum(t0, t1), axis=1)
    return (tf >= np.maximum(tn, 0.0))


def test_disjoint_instances(dragon):
    """(3) two instances side by side, the sphere out of view, one pass: for a pixel whose camera ray (vpt_debug_camera_rays) meets
    instance i's bounds (vpt_volume_bounds, grown by 1 %) and misses the other's, matte i is (volume, alpha) bit for bit and the other
    matte is 0 -- so matte i is instance i's.  Both instances are seen."""
    W, H = 320, 160
    scene = V.Scene([dragon.instance(pos=(-120.0, 0.0, 0.0)), dragon.instance(pos=(120.0, 0.0, 0.0))], env=synthetic_env(512, 256))
    sp = scene.h_sphere; sp.center = V.f3(0.0, 1e6, 0.0); sp.radius = 1.0        # far out of view
    scene.d_sphere.copy_(torch.frombuffer(bytearray(bytes(sp)), dtype=torch.uint8))
    r = V.Renderer(scene, W, H, kp=make_kp(ray_depth=4), cam=scene.frame_camera(W, H))
    r.enable_aovs(); r.enable_mattes([[0], [1]])
    scene.reset_blue_noise(); r.kp.iteration = 0; r.buffers.zero_()
    b0 = r.camera_rays()[:, :3].double().cpu().numpy()                   # the first pass's rays, before the pass
    f = run(scene, r, 1)
    o = np.array([r.cam.origin.x, r.cam.origin.y, r.cam.origin.z], np.float64)
    d = b0 / np.linalg.norm(b0, axis=1, keepdims=True)
    hit = []
    for i in range(2):
        b = (C.c_float * 6)()
        V.lib.vpt_volume_bounds(C.byref(scene.h_volumes[i]), b)
        lo, hi = np.array(b[:3], np.float64), np.array(b[3:], np.float64)
        pad = 0.01 * (hi - lo)
        hit.append(ray_hits_box(o, d, lo - pad, hi + pad))
    m = f["mattes"].cpu()
    alpha, vol = f["alpha"].cpu(), f["volume"].cpu()
    for i in range(2):
        only = torch.from_numpy(hit[i] & ~hit[1 - i])
        assert bool((alpha[only] > 0).any()), f"instance {i} must be seen"
        assert bitwise(m[i][only, 3], alpha[only]) and bitwise(m[i][only, :3], vol[only]), f"matte {i} is not the AOVs on instance {i}'s rays"
        assert bool((m[1 - i][only] == 0).all()), f"matte {1 - i} is not 0 on the rays that meet only instance {i}"
        assert bool((m[i][torch.from_numpy(~hit[i])] == 0).all()), f"matte {i} is covered on rays that miss instance {i}'s bounds"


def test_twins_split_the_coverage(dragon):
    """(4) two instances of one grid with one transform: each takes a collision with probability 1/2, so each twin's collision count is
    half the twins' within 5 sigma of a binomial, and the two together give alpha within rounding.  (A denser block off to the side lifts
    the root majorant above the twins' summed density, so every collision test is a probability; it and the sphere go to matte 2.)"""
    W, H, P = 480, 240, 32
    dmax = float(dragon.rec.vdb_info.max_density)
    block = V.Volume.from_dense(np.full((8, 8, 8), 2.0 * dmax + 1.0, np.float32))
    scene = V.Scene([dragon.instance(), dragon.instance(), block.instance(pos=(-60.0, 0.0, 0.0))], env=synthetic_env(512, 256), keep=[block])
    r = V.Renderer(scene, W, H, kp=make_kp(ray_depth=4, density_mult=50.0), cam=scene.frame_camera(W, H))
    r.enable_aovs(); r.enable_mattes([[0], [1], [2]], sphere=2)
    f = run(scene, r, P)
    counts = torch.round(f["mattes"][:2, :, 3].double() * P)           # collision samples per pixel and twin
    N = float(counts.sum())
    assert N > 2000
    for k in (0, 1):
        assert abs(float(counts[k].sum()) - N / 2) <= 5 * (N / 4) ** 0.5, f"twin {k}: {float(counts[k].sum())} of {N} collisions"
    free = f["mattes"][2][:, 3] == 0
    total = torch.round(f["alpha"].double() * P)
    assert bool((counts.sum(0)[free] == total[free]).all())
    s = f["mattes"][:2].double().sum(0)[free]
    assert torch.allclose(s[:, 3], f["alpha"][free].double(), atol=1e-6)
    assert torch.allclose(s[:, :3], f["volume"][free].double(), rtol=1e-5, atol=1e-6)


def test_sphere_matte(cases):
    """(5) the sphere in view (lights_sphere): where no instance matte is covered, the sphere matte is (volume, alpha) bit for bit, and
    it is covered somewhere."""
    scene, mk, _ = cases("lights_sphere")
    r = mk(); r.enable_mattes([list(range(len(scene.instances))), []], sphere=1)
    f = run(scene, r)
    m = f["mattes"]
    assert float(m[1][:, 3].max()) > 0.0, "the sphere must be seen"
    px = m[0][:, 3] == 0
    assert bitwise(m[1][px, 3], f["alpha"][px]) and bitwise(m[1][px, :3], f["volume"][px])


def test_adaptive_frame_mattes_equal_the_fixed_count_frames(cases):
    """(6) every pixel's mattes equal those of a fixed-count frame of its own pass count"""
    scene, mk, _ = cases("instanced")
    sets = [list(range(0, 60)), list(range(60, 120))]
    r, f = mk(), mk()
    r.enable_mattes(sets); f.enable_mattes(sets)
    scene.reset_blue_noise(); r.kp.iteration = 0; r.buffers.zero_()
    run_, counts = r.render_adaptive(32, threshold=0.12, min_passes=8, check_interval=8)
    torch.cuda.synchronize()
    got = r.buffers.mattes.clone()
    flat = counts.reshape(-1)
    classes = [int(c) for c in torch.unique(flat).tolist()]
    assert len(classes) >= 2
    for c in classes:
        f.reset(); f.render(c); torch.cuda.synchronize()
        m = flat == c
        assert bitwise(got[:, m], f.buffers.mattes[:, m]), f"the mattes differ on the {int(m.sum())} pixels of {c} passes"


def test_region_writes_no_matte_outside_it(cases):
    """(6) with a render region R the mattes inside R equal the full frame's; a sentinel outside R survives."""
    scene, mk, _ = cases("mixed")
    sets = [[0, 1], [2, 3]]
    full_r = mk(); full_r.enable_mattes(sets)
    full = run(scene, full_r)
    r = mk(); r.enable_mattes(sets)
    x0, y0, x1, y1 = 37, 21, 201, 133
    r.set_region(x0, y0, x1, y1)
    got = run(scene, r, fill=SENTINEL)
    H, W = r.height, r.width
    g, w = got["mattes"].view(2, H, W, 4), full["mattes"].view(2, H, W, 4)
    assert bitwise(g[:, y0:y1, x0:x1], w[:, y0:y1, x0:x1])
    inside = torch.zeros(H, W, dtype=torch.bool, device=g.device); inside[y0:y1, x0:x1] = True
    assert bool((g.view(torch.int32)[:, ~inside] == SENTINEL).all()), "a matte was written outside the region"


def test_equirect_mattes_with_and_without_the_miss_cull(dragon):
    """(6) an equirectangular panorama: the one matte is (volume, alpha), and the mattes are the same with and without the cull"""
    scene, mk = headline_pano(dragon, 512, 256, aovs=True)
    culled, kept = mk(1), mk(0)
    culled.enable_mattes([[0]], sphere=0); kept.enable_mattes([[0]], sphere=0)
    a, c = run(scene, culled), run(scene, kept)
    assert bitwise(a["mattes"][0][:, :3], a["volume"]) and bitwise(a["mattes"][0][:, 3], a["alpha"])
    for k in ("mattes", "accum", "alpha", "volume"):
        assert bitwise(a[k], c[k]), k


def test_ods_mattes_with_and_without_the_miss_cull(dragon):
    """(6) an ODS panorama: the one matte is (volume, alpha), and the mattes are the same with and without the cull"""
    from test_ods_gpu import headline_ods
    got = {}
    for cull in (1, 0):
        scene, mk, _, _ = headline_ods(dragon, 512, 256, aovs=True, cull=cull)
        r = mk(); r.enable_mattes([[0]], sphere=0)
        got[cull] = run(scene, r)
        r.close()
    a, c = got[1], got[0]
    assert 0.0 < float((a["alpha"] > 0).float().mean()) < 0.5, "the volume should cover part of the panorama"
    assert bitwise(a["mattes"][0][:, :3], a["volume"]) and bitwise(a["mattes"][0][:, 3], a["alpha"])
    for k in ("mattes", "accum", "alpha", "volume"):
        assert bitwise(a[k], c[k]), k


def test_distributed_renderer_mattes(dragon, tmp_path):
    """DistributedRenderer.enable_mattes / matte_image / disable_mattes act on the rank's renderer: on one rank its mattes are those of a
    Renderer of the same frame"""
    import torch.distributed as dist
    W, H = 256, 128
    scene = V.Scene([dragon.instance(pos=(-20.0, 0.0, 0.0)), dragon.instance(pos=(20.0, 0.0, 0.0))], env=synthetic_env(512, 256))
    cam = scene.frame_camera(W, H)
    ref = V.Renderer(scene, W, H, kp=make_kp(ray_depth=4), cam=cam)
    ref.enable_mattes([[1], [0]])
    want = run(scene, ref, 3)["mattes"].view(2, H, W, 4)
    own = not dist.is_initialized()
    if own: dist.init_process_group("gloo", init_method=f"file://{tmp_path}/pg", rank=0, world_size=1)
    try:
        d = V.DistributedRenderer(scene, W, H, cam=cam, kp=make_kp(ray_depth=4))
        d.enable_mattes([[1], [0]])
        scene.reset_blue_noise(); d.render(3); torch.cuda.synchronize()
        assert bitwise(d.matte_image(), want)
        d.disable_mattes()
        d.r.buffers.mattes.fill_(7.0)
        d.r.kp.iteration = 0; d.render(1); torch.cuda.synchronize()
        assert bool((d.matte_image() == 7.0).all())
        d.close()
    finally:
        if own: dist.destroy_process_group()


def test_partitioned_contexts_keep_rank_local_mattes(dragon):
    """(6) three shards on one GPU: each shard's rank-local matte rows equal the single-context rows."""
    W, H, R, SR = 320, 200, 3, 8
    scene = V.Scene([dragon.instance(pos=(-20.0, 0.0, 0.0)), dragon.instance(pos=(20.0, 0.0, 0.0))], env=synthetic_env(512, 256))
    cam = scene.frame_camera(W, H)
    one = V.Renderer(scene, W, H, kp=make_kp(ray_depth=4), cam=cam)
    one.enable_mattes([[1], [0]])
    full = run(scene, one, 3)["mattes"].view(2, H, W, 4)
    assert float(full[..., 3].sum()) > 0.0
    for rank in range(R):
        r = V.Renderer(scene, W, H, kp=make_kp(ray_depth=4), cam=cam, rank=rank, n_ranks=R, stripe_rows=SR)
        r.enable_mattes([[1], [0]])
        run(scene, r, 3)
        rows = stripe_rows_of_rank(H, rank, R, SR)
        own = torch.as_tensor(np.nonzero(rows < H)[0], device=full.device)
        glob = torch.as_tensor(rows[rows < H], device=full.device)
        assert bitwise(r.matte_image()[:, own], full[:, glob]), f"rank {rank}"
        r.close()


def test_activation_and_refusals(dragon):
    """(7) mattes enabled mid-frame stay untouched until the next iteration-0 call; a NULL buffer stops at once; every bad argument is
    refused when set and changes nothing; a map of another instance count, overlaps and brick mode are refused at render time."""
    W, H = 160, 100
    scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
    cam = scene.frame_camera(W, H)
    mk = lambda: V.Renderer(scene, W, H, kp=make_kp(ray_depth=4), cam=cam)
    ref = mk(); ref.enable_mattes([[0]])
    want = run(scene, ref, 3)

    r = mk()
    with pytest.raises(V.VptError, match="not enabled"):
        r.matte_image()
    scene.reset_blue_noise(); r.render(2)
    r.enable_mattes([[0]])
    r.buffers.mattes.fill_(7.0)
    r.render(2); torch.cuda.synchronize()                                      # iteration 2: not active yet
    assert bool((r.buffers.mattes == 7.0).all())
    got = run(scene, r, 3)                                                     # iteration 0: active from here on
    assert bitwise(got["mattes"], want["mattes"]) and r.matte_image().shape == (1, H, W, 4)
    r.disable_mattes()
    r.buffers.mattes.fill_(7.0)
    r.kp.iteration = 0
    r.render(1); torch.cuda.synchronize()
    assert bool((r.buffers.mattes == 7.0).all()), "a NULL buffer turns the mattes off"

    # refused when set; a refused call leaves the registered mattes as they were
    z = mk(); z.enable_mattes([[0]])
    buf = torch.zeros(33 * W * H * 4 + 4, dtype=torch.float32, device=z.buffers.accum.device)
    p = C.c_void_p(buf.data_ptr())
    m0, m2, mneg = (C.c_int * 1)(0), (C.c_int * 1)(2), (C.c_int * 1)(-2)
    bad = [(p, 0, m0, 1, -1), (p, 33, m0, 1, -1), (p, 1, None, 1, -1), (p, 2, m2, 1, -1), (p, 2, mneg, 1, -1), (p, 2, m0, 1, 2),
           (C.c_void_p(buf.data_ptr() + 4), 1, m0, 1, -1)]
    for args in bad:
        assert V.lib.vpt_set_instance_mattes(z.ctx, *args) == -1, args
        assert V.lib.vpt_last_error(z.ctx).startswith(b"vpt_set_instance_mattes")
    with pytest.raises(V.VptError, match="in set 0 and set 1"):
        z.enable_mattes([[0], [0]])
    assert bitwise(run(scene, z, 3)["mattes"], want["mattes"])

    # refused at render time: another instance count, overlaps naming the buffer, brick mode
    o = mk()
    free = torch.zeros(W * H, 4, dtype=torch.float32, device=o.buffers.accum.device)
    m = (C.c_int * 2)(0, 0)
    V._native.check(V.lib.vpt_set_instance_mattes(o.ctx, C.c_void_p(free.data_ptr()), 1, m, 2, -1), o.ctx, "vpt_set_instance_mattes")
    o.kp.iteration = 0
    with pytest.raises(V.VptError, match="covers 2 instances, the scene has 1"):
        o.render(1)
    o.enable_deep([0.0, INF])
    V._native.check(V.lib.vpt_set_instance_mattes(o.ctx, C.c_void_p(o.buffers.deep.data_ptr()), 1, m, 1, -1), o.ctx, "vpt_set_instance_mattes")
    o.kp.iteration = 0
    with pytest.raises(V.VptError, match="matte buffer overlaps the deep slice buffer"):
        o.render(1)
    V._native.check(V.lib.vpt_set_instance_mattes(o.ctx, C.c_void_p(o.buffers.accum.data_ptr()), 1, m, 1, -1), o.ctx, "vpt_set_instance_mattes")
    o.kp.iteration = 0
    with pytest.raises(V.VptError, match="matte buffer overlaps Kernel_params.accum_buffer"):
        o.render(1)

    perlin = V.Volume.procedural((48, 40, 36), scale=0.1, seed=3)
    perlin.build_bricks()
    ps = V.Scene([perlin.instance()], env=synthetic_env(512, 256), keep=[perlin])
    b = V.Renderer(ps, 64, 36, kp=make_kp(ray_depth=2), cam=ps.frame_camera(64, 36))
    b.set_brick_volume(perlin)
    b.enable_mattes([[0]])
    with pytest.raises(V.VptError, match="brick or cell mode"):
        b.render(1)
