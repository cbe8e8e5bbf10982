"""Motion vectors (vpt_set_motion_vectors; DESIGN.md section 8o) on the GPU.

1. Vectors on and off leave accum, depth, cost, raw, display, the blue noise, the AOVs, light groups, deep slices and mattes bit for bit
   as they are: the lean HDRI kernel (compact records), the generic kernel with point lights and the sphere (wide records), the volumetric
   path integrator on the precomputed sky and brick mode, across a chunk boundary and a continued call.
2. With the target equal to the frame camera x and y are exactly +0 everywhere and z is the alpha AOV bit for bit (also in an adaptive
   frame and in a region); n fused passes equal n single-pass calls bit for bit.
3. One pass at iteration 0 against the float64 restatement (tests/motion_vectors_ref.py), pinhole, thin lens and camera motion.
4. The running mean from prefilled buffers at a continued iteration.
5. Adaptive frames, regions, four partitioned contexts and three peer-exchange shards carrying VPT_LAYER_MOTION.
6. Refusals, activation at iteration 0 and the launch count."""
import ctypes as C

import numpy as np
import pytest
import torch

import vpt_b200 as V
from vpt_b200 import _native as N
from vpt_b200.scene import synthetic_env
from test_parity_gpu import make_kp
from test_aov_gpu import make_aov_case
from test_exchange_layers_gpu import Case as LayerCase, Shards as LayerShards, enable_all, FLT_MAX, ALL
import adaptive_ref as A
import motion_ref as MR
import motion_vectors_ref as M

pytestmark = pytest.mark.gpu
BUFFERS = ("accum", "depth", "cost", "raw", "display")
SENTINEL = -7.25


@pytest.fixture(scope="module")
def dragon():
    return V.Volume.load_vdb(V.find_asset("dragon.vdb"))


@pytest.fixture(scope="module")
def perlin():
    vol = V.Volume.procedural((96, 80, 72), scale=0.1, seed=123)
    vol.build_bricks()
    return vol


@pytest.fixture(scope="module")
def emissive():
    n = 48
    z, y, x = np.mgrid[0:n, 0:n, 0:n].astype(np.float32)
    c = (n - 1) / 2.0
    r = np.sqrt((x - c) ** 2 + (y - c) ** 2 + (z - c) ** 2) / c
    return V.Volume.from_dense((np.clip(1.1 - r, 0.0, None) ** 1.5).astype(np.float32), bbox_min=(-c, -c, -c),
                               emission=(3.0 * np.clip(0.8 - r, 0.0, None)).astype(np.float32))


@pytest.fixture(scope="module")
def atmosphere():
    atm = V.Atmosphere()
    yield atm
    atm.destroy()


def bits(t):
    t = t.contiguous()
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def same(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


def copy_cam(cam):
    return N.camera.from_buffer_copy(bytes(cam))


def moved(cam, scale):
    """cam translated sideways and turned: origin moves by 0.06 scale along x and -0.04 scale along z, the view point by 0.03 scale up."""
    c = copy_cam(cam)
    def add(v, d): return N.f3(*[float(np.float32(getattr(v, a)) + np.float32(x)) for a, x in zip("xyz", d)])
    c.origin = add(cam.origin, (0.06 * scale, 0.0, -0.04 * scale))
    c.lower_left_corner = add(cam.lower_left_corner, (0.06 * scale, 0.03 * scale, -0.04 * scale))
    return c


def scale_of(scene):
    lo, hi = scene.world_bounds()
    return float(np.linalg.norm(hi - lo))


def outputs(scene, r):
    b = r.buffers
    out = {k: getattr(b, k).clone() for k in BUFFERS}
    for k in ("alpha", "volume", "deep", "mattes"):
        if getattr(b, k) is not None: out[k] = getattr(b, k).clone()
    for g, t in (b.groups or {}).items(): out["group_" + g] = t.clone()
    out["blue_noise"] = scene.d_blue_noise.clone()
    return out


def sequence(scene, r, pass_by_pass=False):
    """8 passes in chunks of 5 + 3 from iteration 0, then a continued call of 3 passes."""
    scene.reset_blue_noise(); r.kp.iteration = 0; r.buffers.zero_()
    if pass_by_pass:
        for _ in range(11): r.render_pass()
    else:
        r.render(8); r.render(3)
    torch.cuda.synchronize()
    return outputs(scene, r)


# ---- 1, 2: nothing else moves; identities --------------------------------------------------------------------------------------------------
NAMES = ["headline", "lights_sphere", "vol_sky_table", "brick"]


@pytest.mark.parametrize("name", NAMES)
def test_nothing_else_moves_and_the_identities_hold(dragon, perlin, name):
    scene, mk, keep = make_aov_case(name, dragon, perlin)

    def renderer(target):
        r = mk()
        r.enable_deep([0.0, float("inf")])
        if name != "brick":
            r.enable_mattes([range(len(scene.instances))], sphere=0)
        if name in ("lights_sphere", "vol_sky_table"):
            r.enable_light_groups()
        if target is not None:
            r.enable_motion_vectors(target)
        return r

    r0 = renderer(None)
    off = sequence(scene, r0)
    r = renderer(moved(r0.cam, scale_of(scene)))
    on = sequence(scene, r)
    for k in off:
        assert same(on[k], off[k]), f"{name}: {k} changes when the motion vectors are on"
    mv = r.buffers.motion
    assert same(mv[:, 2], on["alpha"]), f"{name}: z is not the alpha AOV"
    assert float(mv[:, :2].abs().max()) > 0.5, f"{name}: the target must move the volume on the film"
    single = sequence(scene, r, pass_by_pass=True)
    assert same(single["accum"], on["accum"])
    assert same(r.buffers.motion, mv), f"{name}: 11 single passes differ from the fused 5 + 3 + 3"

    ident = renderer(copy_cam(r.cam))
    out = sequence(scene, ident)
    m = ident.buffers.motion
    assert bool((bits(m[:, :2]) == 0).all()), f"{name}: target == frame camera must give +0 in x and y"
    assert same(m[:, 2], out["alpha"]) and float(out["alpha"].max()) > 0


# ---- 3: one pass against the restatement ---------------------------------------------------------------------------------------------------
W1, H1 = 192, 96
U24 = 2.0 ** -24


def tolerance(cam, P, W, H, depth):
    """Per-pixel bound of |vector - restatement| in pixels.  The kernel rounds P = org + depth dir in float32 (org and depth exact, dir from
    a normalize whose fast rsqrt is good to about 2^-22 relative), and the projection rounds d, k, q, s, t and the products by W, H in
    float32 with fast divisions (a few ulps each): an error of a few 2^-24 relative in P moves the film position by f |P - o| / z_cam
    times that, and the projection's own rounding adds a few ulps of |s W| + |t H|.  64 ulps of each, for both cameras, bounds that with
    a wide margin."""
    f = M.fields(cam)
    fpx = W / np.linalg.norm(f["horizontal"])                      # pixels per unit of film at focus distance 1
    o = f["origin"]
    dist = np.linalg.norm(P - o, axis=-1)
    zc = np.abs((P - o) @ (np.cross(f["horizontal"], f["vertical"]) / np.linalg.norm(np.cross(f["horizontal"], f["vertical"]))))
    return 64 * U24 * (2 * (W + H) + 2 * fpx * (np.linalg.norm(o) + depth + dist) / np.maximum(zc, 1e-6))


def one_pass_case(dragon, lens):
    scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
    cam = scene.frame_camera(W1, H1)
    if lens == "thin":
        cam.lens_radius = np.float32(0.02 * scale_of(scene))
    r = V.Renderer(scene, W1, H1, kp=make_kp(ray_depth=2), cam=cam)
    target = moved(cam, scale_of(scene))
    r.enable_motion_vectors(target)
    if lens == "motion":
        r.set_camera_motion(moved(cam, 0.5 * scale_of(scene)))
    return scene, r, target


@pytest.mark.parametrize("lens", ["pinhole", "thin", "motion"])
def test_one_pass_against_the_restatement(dragon, lens):
    scene, r, target = one_pass_case(dragon, lens)
    W, H = W1, H1
    scene.reset_blue_noise(); r.kp.iteration = 0; r.buffers.zero_()
    bn = scene.d_blue_noise.clone().cpu().numpy().reshape(-1, 3)
    cams = r.motion_cameras().cpu().numpy().reshape(-1, 20) if lens == "motion" else None
    b0 = r.camera_rays().cpu().numpy()[:, :3].astype(np.float64) if lens != "motion" else None
    r.render(1); torch.cuda.synchronize()
    depth = r.buffers.depth.cpu().numpy().astype(np.float64)
    mv = r.buffers.motion.cpu().numpy()
    hit = depth > 0
    assert np.array_equal(mv[:, 2].view(np.int32), hit.astype(np.float32).view(np.int32)), "coverage must be [depth > 0] bit for bit"
    assert hit.sum() > 200
    idx = np.nonzero(hit)[0]
    ys, xs = idx // W, idx % W
    cam = M.fields(r.cam)
    if lens == "pinhole":
        org = np.broadcast_to(cam["origin"], (len(idx), 3))
        d = b0[idx]
    elif lens == "thin":
        lib, acc, t2, t3 = MR.oracle_lib(), MR.accept_table(), MR.vdc_table(2), MR.vdc_table(3)
        lr = float(np.float32(r.cam.lens_radius))
        uu = np.array([getattr(r.cam.u, a) for a in "xyz"], np.float64); vv = np.array([getattr(r.cam.v, a) for a in "xyz"], np.float64)
        pts = np.array([M.lens_point(MR.Stream(lib, int(y) * W + int(x), 0), acc, t2, t3) for y, x in zip(ys, xs)])
        off = lr * pts[:, :1] * uu + lr * pts[:, 1:] * vv
        org = cam["origin"] + off
        d = b0[idx] - off
    else:
        c = cams[idx].astype(np.float64)
        o, llc, h, v = c[:, 1:4], c[:, 4:7], c[:, 7:10], c[:, 10:13]
        j = bn[(ys % 256) * 256 + xs % 256].astype(np.float64)
        s = ((xs + j[:, 0]) / W)[:, None]; t = ((ys + j[:, 1]) / H)[:, None]
        org, d = o, llc + s * h + t * v - o
    d = d / np.linalg.norm(d, axis=1, keepdims=True)
    P = org + depth[idx, None] * d
    want = M.sample_vectors(r.cam, target, P, np.ones(len(idx), bool), W, H)
    err = np.abs(mv[idx, :2].astype(np.float64) - want).max(axis=1)
    tol = tolerance(r.cam, P, W, H, depth[idx]) + tolerance(target, P, W, H, depth[idx])
    assert (err <= tol).all(), f"{lens}: worst {err.max():.3g} px against a bound of {tol[np.argmax(err - tol)]:.3g}"
    assert np.abs(want).max() > 8.0, "the target must move the silhouette by several pixels"
    assert np.array_equal(mv[~hit, :2], np.zeros((int((~hit).sum()), 2), np.float32))
    r.close()


# ---- 4: the running mean -------------------------------------------------------------------------------------------------------------------
def test_running_mean_from_prefilled_buffers(dragon):
    scene, r, target = one_pass_case(dragon, "pinhole")
    W, H = W1, H1
    r.enable_aovs()
    it = 5
    scene.reset_blue_noise(); r.kp.iteration = 0; r.buffers.zero_(); r.render(1)       # activates the vectors and the AOVs
    rng = np.random.default_rng(3)
    X = torch.tensor(rng.uniform(-4, 4, (r.n_local, 3)).astype(np.float32), device=r.buffers.accum.device)
    X[:, 2] = torch.tensor(rng.uniform(0, 1, r.n_local).astype(np.float32))
    r.buffers.motion.copy_(X); r.buffers.alpha.copy_(X[:, 2]); r.buffers.depth.zero_()
    scene.reset_blue_noise(); r.kp.iteration = it
    b0 = r.camera_rays().cpu().numpy()[:, :3].astype(np.float64)
    r.render(1); torch.cuda.synchronize()
    mv = r.buffers.motion.cpu().numpy().astype(np.float64)
    assert same(r.buffers.motion[:, 2], r.buffers.alpha), "z must be the alpha AOV at a continued iteration"
    depth = r.buffers.depth.cpu().numpy().astype(np.float64) * (it + 1)        # the sample's depth, from 0 + (d - 0) / (it + 1)
    hit = depth > 0
    assert hit.sum() > 200
    d = b0 / np.linalg.norm(b0, axis=1, keepdims=True)
    P = M.fields(r.cam)["origin"] + depth[:, None] * d
    S = M.sample_vectors(r.cam, target, P, hit, W, H)
    want = M.running_mean(X.cpu().numpy()[:, :2], S, it, r.kp.max_interactions)
    tol = 1e-5 * (1 + np.abs(want)) + np.where(hit, tolerance(r.cam, P, W, H, depth) + tolerance(target, P, W, H, depth), 0)[:, None]
    assert (np.abs(mv[:, :2] - want) <= tol).all()
    r.close()


# ---- 5: composition ------------------------------------------------------------------------------------------------------------------------
def small_case(dragon, **kw):
    scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
    cam = scene.frame_camera(160, 96)
    def mk(**k2):
        r = V.Renderer(scene, 160, 96, kp=make_kp(ray_depth=2), cam=copy_cam(cam), **{**kw, **k2})
        r.set_option("passes_per_chunk", 5)
        return r
    return scene, mk, moved(cam, scale_of(scene))


def test_adaptive_pixels_equal_the_fixed_count_frame_of_their_count(dragon):
    scene, mk, target = small_case(dragon)
    r = mk(); r.enable_aovs(); r.enable_motion_vectors(target)
    P, mn, iv = 16, 4, 4
    scene.reset_blue_noise(); r.kp.iteration = 0
    _, _, first = r.render_adaptive(P, threshold=FLT_MAX, min_passes=mn, check_interval=iv, error_map=True)
    thr = float(np.quantile(A.max3x3(first.cpu().numpy()), 0.5))
    scene.reset_blue_noise(); r.kp.iteration = 0
    _, counts = r.render_adaptive(P, threshold=thr, min_passes=mn, check_interval=iv)
    torch.cuda.synchronize()
    got = r.buffers.motion.clone()
    assert same(got[:, 2], r.buffers.alpha), "z must be the alpha AOV in an adaptive frame"
    counts = counts.reshape(-1)
    assert len(torch.unique(counts)) >= 2
    f = mk(); f.enable_motion_vectors(target)
    for n in torch.unique(counts).tolist():
        scene.reset_blue_noise(); f.kp.iteration = 0; f.render(int(n)); torch.cuda.synchronize()
        sel = counts == n
        assert same(got[sel], f.buffers.motion[sel]), f"pixels that took {n} passes"


def test_region_equals_the_full_frame_inside_and_writes_nothing_outside(dragon):
    scene, mk, target = small_case(dragon)
    full = mk(); full.enable_aovs(); full.enable_motion_vectors(target)
    scene.reset_blue_noise(); full.kp.iteration = 0; full.render(8); torch.cuda.synchronize()
    r = mk(); r.enable_aovs(); r.enable_motion_vectors(target)
    x0, y0, x1, y1 = 37, 11, 121, 70
    r.set_region(x0, y0, x1, y1)
    r.buffers.motion.fill_(SENTINEL)
    scene.reset_blue_noise(); r.kp.iteration = 0; r.render(8); torch.cuda.synchronize()
    got, want = r.buffers.motion.view(96, 160, 3), full.buffers.motion.view(96, 160, 3)
    inside = torch.zeros(96, 160, dtype=torch.bool, device=got.device); inside[y0:y1, x0:x1] = True
    assert same(got[inside], want[inside])
    assert bool((got[~inside] == SENTINEL).all())
    assert same(r.buffers.motion.view(96, 160, 3)[inside][:, 2], r.buffers.alpha.view(96, 160)[inside])


def test_four_partitioned_contexts_equal_the_single_context(dragon):
    scene, mk, target = small_case(dragon)
    one = mk(); one.enable_motion_vectors(target)
    scene.reset_blue_noise(); one.kp.iteration = 0; one.render(6); torch.cuda.synchronize()
    want = one.buffers.motion.view(96, 160, 3)
    for k in range(4):
        sc = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
        r = V.Renderer(sc, 160, 96, kp=make_kp(ray_depth=2), cam=copy_cam(one.cam), rank=k, n_ranks=4, stripe_rows=8)
        r.set_option("passes_per_chunk", 5)
        r.enable_motion_vectors(target)
        r.kp.iteration = 0; r.render(6); torch.cuda.synchronize()
        rows = V.stripe_rows_of_rank(96, k, 4, 8)
        loc = r.buffers.motion.view(-1, 160, 3)
        ok = rows < 96
        assert same(loc[torch.as_tensor(np.nonzero(ok)[0], device=loc.device)], want[torch.as_tensor(rows[ok], device=loc.device)]), f"rank {k}"
        r.close()


def test_three_shards_carry_the_motion_layer(dragon, emissive, atmosphere):
    case = LayerCase("hdri", dragon, emissive, atmosphere)
    target = moved(case.cam, scale_of(case.scene()))
    sh = LayerShards(case, 3, 7, masks=ALL | N.VPT_LAYER_MOTION)
    try:
        sh.each(enable_all)
        sh.each(lambda r: r.enable_motion_vectors(target))
        H, W = sh.ref.height, sh.ref.width

        def planes():
            out = []
            for r in sh.rs:
                p = C.c_uint64(0)
                N.check(V.lib.vpt_comm_p2p_layer(r.ctx, N.VPT_LAYER_MOTION, C.byref(p)), r.ctx, "vpt_comm_p2p_layer")
                out.append(torch.as_tensor(V.renderer._DeviceView(p.value, (H * W, 3), "<f4"), device=r.buffers.accum.device))
            return out
        sh.ref_scene.reset_blue_noise()
        for s in sh.scenes: s.reset_blue_noise()
        sh.render(5, iteration=0); sh.check("frame")
        for k, pl in enumerate(planes()):
            assert same(pl, sh.ref.buffers.motion), f"motion plane held by shard {k}"
        assert float(sh.ref.buffers.motion[:, 2].max()) > 0
        sh.render(4); sh.check("continued")
        for k, pl in enumerate(planes()):
            assert same(pl, sh.ref.buffers.motion), f"continued: motion plane held by shard {k}"
        assert sh.abandoned_waits() == [0, 0, 0]
    finally:
        sh.close()


# ---- 6: contract ---------------------------------------------------------------------------------------------------------------------------
def test_refusals_activation_and_launch_count(dragon):
    scene, mk, target = small_case(dragon)
    r = mk()
    bad = copy_cam(target); bad.vertical = N.f3(0.0, float("nan"), 0.0)
    buf = torch.zeros(r.n_local, 3, dtype=torch.float32, device=r.buffers.accum.device)
    assert V.lib.vpt_set_motion_vectors(r.ctx, C.c_void_p(buf.data_ptr()), C.byref(bad)) == -1
    assert b"target.vertical is not finite" in V.lib.vpt_last_error(r.ctx)
    assert V.lib.vpt_set_motion_vectors(r.ctx, C.c_void_p(buf.data_ptr()), None) == -1

    # a buffer registered mid-frame is not touched before the next iteration-0 call
    scene.reset_blue_noise(); r.kp.iteration = 0; r.render(3)
    r.enable_motion_vectors(target); r.buffers.motion.fill_(SENTINEL)
    r.render(2); torch.cuda.synchronize()
    assert bool((r.buffers.motion == SENTINEL).all())
    before = r.stats()[0]
    scene.reset_blue_noise(); r.kp.iteration = 0; r.render(8); torch.cuda.synchronize()
    assert float(r.buffers.motion[:, 2].max()) > 0.0
    with_vec = r.stats()[0] - before
    r.disable_motion_vectors()
    before = r.stats()[0]
    scene.reset_blue_noise(); r.kp.iteration = 0; r.render(8); torch.cuda.synchronize()
    without = r.stats()[0] - before
    assert with_vec - without == 2, "one vector launch per chunk (5 + 3)"

    # overlapping buffers, named
    for name, t in (("Kernel_params.accum_buffer", r.buffers.accum), ("the alpha AOV buffer", None)):
        if t is None:
            r.enable_aovs(); t = r.buffers.alpha
        N.check(V.lib.vpt_set_motion_vectors(r.ctx, C.c_void_p(t.data_ptr()), C.byref(target)), r.ctx, "vpt_set_motion_vectors")
        r.kp.iteration = 0
        with pytest.raises(V.VptError, match=name):
            r.render(1)
    r.disable_motion_vectors(); r.disable_aovs()

    # panoramas
    for kind in ("equirect", "ods"):
        p = mk(); p.set_projection(kind); p.enable_motion_vectors(target)
        p.kp.iteration = 0
        with pytest.raises(V.VptError, match=r"\(-3\).*motion vectors"):
            p.render(1)
        p.close()
    r.close()
