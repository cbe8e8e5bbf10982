"""Camera motion (vpt_set_camera_motion): each sample's shutter draw places its camera between the shutter-open and shutter-close poses.

* Reference path: for about 100 pixels -- the volume, its silhouette and a random rest -- the reference kernel renders one pass with the
  reference camera set to the pixel's camera from vpt_debug_motion_cameras (lens, focus and viz_dof of the open pose), at the same
  resolution, iteration and blue-noise state, and the pixel must match the library's motion frame by the rule a perspective frame meets
  (cost bit-equal; accum, depth and raw.xyz within 1e-5 + 1e-4 |ref|; raw.w within 1e-5; display within 1 LSB; at least 90 % of the
  accum values bit-equal), at iteration 0 and at a continued iteration from identical prefilled buffers.  The camera both translates and
  turns.  The compared reference pixels are stored under tests/golden/oracle/, so a run without oracle/_ref replays them.
* The draw: vpt_debug_motion_cameras' xi equals the restatement on the oracle's Philox (tests/motion_ref.py) for every pixel, the poses
  the float64 lerp within 1 ulp, and components that do not move keep the open pose's bits.
* shutter_close == the open camera is the static frame (miss cull on) bit for bit on every output.
* Adaptive frames, regions and three peer-exchange shards with exchange layers; the blur itself; activation, clearing and refusals."""
import ctypes as C

import numpy as np
import pytest
import torch

import vpt_b200 as V
from vpt_b200 import _native as N
from vpt_b200.scene import synthetic_env
from test_parity_gpu import make_kp
from test_adaptive_gpu import _sky_power_table
from test_exchange_layers_gpu import Case as LayerCase, Shards as LayerShards, enable_all, FLT_MAX
import adaptive_ref as A
import motion_ref as M
import oracle_ref

pytestmark = pytest.mark.gpu
BUFFERS = ("accum", "depth", "cost", "raw", "display")
PASSES = 8                                   # passes_per_chunk 5: chunks of 5 + 3
SENTINEL_F = 0x7FBADBAD
SENTINEL_D = 0x13572468


@pytest.fixture(scope="module")
def dragon():
    return V.Volume.load_vdb(V.find_asset("dragon.vdb"))


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


def tensors(r):
    out = {k: getattr(r.buffers, k) for k in BUFFERS}
    for k in ("alpha", "volume", "deep"):
        if getattr(r.buffers, k) is not None: out[k] = getattr(r.buffers, k)
    if r.buffers.groups is not None:
        out.update({"group_" + g: t for g, t in r.buffers.groups.items()})
    return out


def snapshot(scene, r):
    out = {k: t.clone() for k, t in tensors(r).items()}
    out["blue_noise"] = scene.d_blue_noise.clone()
    return out


def assert_same(a, b, what=""):
    assert a.keys() == b.keys()
    for k in a:
        assert torch.equal(bits(a[k]), bits(b[k])), f"{what}: {k} differs"


def look_at(lookfrom, lookat, fov=30.0, aspect=2.0, aperture=0.0):
    cam = N.camera()
    V.lib.vpt_camera_look_at(C.byref(cam), N.fvec(lookfrom), N.fvec(lookat), N.fvec((0, 1, 0)), float(fov), float(aspect), float(aperture))
    return cam


def copy_cam(cam):
    return N.camera.from_buffer_copy(bytes(cam))


def translated(cam, d):
    """cam moved by d (origin and lower_left_corner; the basis keeps its bits)."""
    c = copy_cam(cam)
    c.origin = N.f3(*[float(np.float32(getattr(cam.origin, a)) + np.float32(v)) for a, v in zip("xyz", d)])
    c.lower_left_corner = N.f3(*[float(np.float32(getattr(cam.lower_left_corner, a)) + np.float32(v)) for a, v in zip("xyz", d)])
    return c


def poses(scene, W, H, aperture=0.0):
    """(open, close): the headline framing, and a pose translated sideways and turned, far enough that the silhouette moves by several
    pixels."""
    lo, hi = scene.world_bounds()
    centre = (hi + lo) / np.float32(2)
    d = np.float32(float(np.linalg.norm(hi - lo)))
    eye = centre + d
    open_ = look_at(eye, centre, aspect=W / H, aperture=aperture)
    close = look_at(eye + d * np.float32([0.06, 0.0, -0.06]), centre + d * np.float32([0.0, 0.03, 0.0]), aspect=W / H, aperture=aperture)
    return open_, close


def fresh(scene, r, iteration=0, prefill=False):
    scene.reset_blue_noise(); r.kp.iteration = iteration
    if prefill:
        for k, t in tensors(r).items(): bits(t).fill_(SENTINEL_D if k == "display" else SENTINEL_F)
    else:
        r.buffers.zero_()


def frame(scene, r, passes=PASSES, prefill=False):
    fresh(scene, r, prefill=prefill)
    r.render(passes); torch.cuda.synchronize()
    return snapshot(scene, r)


# ---- the reference path ---------------------------------------------------------------------------------------------------------------
W1, H1 = 256, 128


def ref_case(dragon, case):
    scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
    keep = []
    if case == "bruneton_vol":
        atm = V.Atmosphere(); atm.apply(scene.atmos)
        tables = V.EnvTables(_sky_power_table())
        keep += [atm, tables]

        def mkr(cam):
            r = V.Renderer(scene, W1, H1, kp=make_kp(integrator=1, environment_type=0, ray_depth=6), cam=cam)
            tables.apply(r.kp)
            return r
    else:
        mkr = lambda cam: V.Renderer(scene, W1, H1, kp=make_kp(ray_depth=100), cam=cam)
    return scene, mkr, keep


def pick_pixels(depth, cams, bn, rng):
    """~100 pixels: the volume (depth > 0), its silhouette (a miss next to a hit) and a random rest; none whose b0 (float64, from the
    pixel's camera and jitter) has a component near 0."""
    H, W = depth.shape
    vol = depth > 0
    sil = ~vol & (np.roll(vol, 1, 0) | np.roll(vol, -1, 0) | np.roll(vol, 1, 1) | np.roll(vol, -1, 1))
    picks = []
    for m in (vol, sil):
        ys, xs = np.nonzero(m)
        assert len(ys) >= 10
        sel = rng.choice(len(ys), min(40, len(ys)), replace=False)
        picks += list(zip(ys[sel], xs[sel]))
    picks += [(rng.randint(H), rng.randint(W)) for _ in range(25)]

    def b0_clear(y, x):
        f = cams[y, x, 1:19].astype(np.float64).reshape(6, 3)
        j = bn[(y % 256) * 256 + x % 256]
        b0 = f[1] + (x + float(j[0])) / W * f[2] + (y + float(j[1])) / H * f[3] - f[0]
        return bool(np.all(np.abs(b0) > 1e-6 * np.linalg.norm(b0)))
    return sorted({(int(y), int(x)) for y, x in picks if b0_clear(int(y), int(x))})


@pytest.mark.parametrize("case", ["hdri_pinhole", "hdri_lens", "bruneton_vol"])
def test_one_pass_equals_the_reference_kernel_per_pixel(dragon, case):
    if not oracle_ref.usable():
        pytest.skip("neither oracle/_ref nor stored oracle outputs")
    scene, mkr, keep = ref_case(dragon, case)
    open_, close = poses(scene, W1, H1, aperture=0.2 if case == "hdri_lens" else 0.0)
    mot = mkr(open_)
    mot.set_camera_motion(close)
    ref = mkr(copy_cam(open_))
    cam_bytes = bytes(open_)
    rs = np.random.RandomState(5)
    start = {k: torch.from_numpy(rs.rand(*t.shape).astype(np.float32)).cuda() for k, t in tensors(mot).items() if k != "display"}

    def prefill(r, it):
        scene.reset_blue_noise(); r.kp.iteration = it
        for k, t in tensors(r).items():
            if k == "display": t.fill_(7)
            else: t.copy_(start[k])

    oracle = oracle_ref.RefOracle()
    rng = np.random.RandomState(3)
    checked, ulps, exact = 0, dict(accum=0, depth=0, raw=0), dict(accum=0, depth=0, raw=0, display=0)
    for it in (0, 5):
        prefill(mot, it)
        bn0 = scene.d_blue_noise.clone()
        cams = mot.motion_cameras().cpu().numpy()
        assert torch.equal(bn0, scene.d_blue_noise), "vpt_debug_motion_cameras moved the blue noise"
        mot.render(1); torch.cuda.synchronize()
        got = {k: bits(t).view(H1, W1, -1).cpu().numpy() for k, t in tensors(mot).items()}
        if it == 0:
            pix = pick_pixels(got["depth"].view(np.float32)[..., 0], cams, bn0.view(-1, 3).cpu().numpy(), rng)
            assert len(pix) >= 70
        ys, xs = np.array([p[0] for p in pix]), np.array([p[1] for p in pix])
        key = oracle_ref._key("pixels")
        digest = oracle_ref._digest(case, it, W1, H1, ys.tobytes(), xs.tobytes(), cams[ys, xs].tobytes(), cam_bytes,
                                    oracle_ref._kp_scalars(ref.kp), bytes(scene.h_sphere),
                                    oracle_ref._volumes_digest(scene.h_volumes, len(scene.instances)),
                                    *[start[k].view(H1, W1, -1)[torch.from_numpy(ys).cuda(), torch.from_numpy(xs).cuda()].cpu().numpy().tobytes()
                                      for k in sorted(start)])
        if oracle.replay:
            z = oracle_ref._load(key, digest)
            want = {k: z[k] for k in BUFFERS}
        else:
            want = {k: [] for k in BUFFERS}
            for (y, x) in pix:
                f = cams[y, x, 1:19].reshape(6, 3)
                for n, name in enumerate(M.FIELDS):
                    setattr(ref.cam, name, N.f3(*[float(v) for v in f[n]]))
                prefill(ref, it)
                oracle.launch(ref.params.array, W1, H1, oracle.NOBN)
                oracle.bn_advance(ref.kp)
                torch.cuda.synchronize()
                for k, t in tensors(ref).items():
                    want[k].append(bits(t).view(H1, W1, -1)[y, x].cpu().numpy())
            want = {k: np.stack(v) for k, v in want.items()}
            oracle_ref._store(key, dict(digest=np.array(digest), **want))
        for n, (y, x) in enumerate(pix):
            what = f"{case}, iteration {it}, pixel ({x}, {y})"
            assert np.array_equal(got["cost"][y, x], want["cost"][n]), f"{what}: cost"
            for k, sl in (("accum", slice(None)), ("depth", slice(None)), ("raw", slice(0, 3))):
                g = got[k][y, x, sl].view(np.float32).astype(np.float64); w = want[k][n, sl].view(np.float32).astype(np.float64)
                assert np.array_equal(np.isnan(g), np.isnan(w)), f"{what}: {k} NaN in other places"
                assert (np.isnan(w) | (np.abs(g - w) <= 1e-5 + 1e-4 * np.abs(w))).all(), f"{what}: {k} {g} against {w}"
                d = int(np.abs(got[k][y, x, sl].astype(np.int64) - want[k][n, sl].astype(np.int64)).max())
                ulps[k] = max(ulps[k], d)
                exact[k] += d == 0
            gw, ww = float(got["raw"][y, x, 3:].view(np.float32)[0]), float(want["raw"][n, 3:].view(np.float32)[0])
            assert abs(gw - ww) <= 1e-5, f"{what}: raw.w"
            gd, wd = got["display"][y, x].view(np.uint8), want["display"][n].view(np.uint8)
            assert np.abs(gd.astype(int) - wd.astype(int)).max() <= 1, f"{what}: display {gd} against {wd}"
            exact["display"] += int(np.array_equal(gd, wd))
            checked += 1
    assert float(np.abs(got["accum"].view(np.float32)).mean()) > 1e-4
    print(f"\n{case}: {checked} pixel passes against the reference kernel ({'replayed' if oracle.replay else 'live'}): cost bit-equal; "
          f"bit-equal pixels {exact}; largest difference in ulp {ulps}")
    assert exact["accum"] >= 0.9 * checked, exact
    mot.close(); ref.close()


# ---- the draw ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lens", [0.0, 0.2], ids=["pinhole", "thin_lens"])
def test_motion_cameras_are_the_restated_draw_and_lerp(dragon, lens):
    W, H = 64, 32
    scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
    open_, turned = poses(scene, W, H, aperture=lens)
    lib = M.oracle_lib()
    for close, it in ((turned, 0), (turned, 7), (translated(open_, (0.5, -0.25, 1.0)), 3)):
        r = V.Renderer(scene, W, H, kp=make_kp(), cam=open_)
        r.set_camera_motion(close)
        if it:                                                   # the pose becomes current at iteration 0
            r.render(it); torch.cuda.synchronize()
        assert r.kp.iteration == it
        cams = r.motion_cameras().cpu().numpy()
        xi = cams[..., 0]
        assert np.array_equal(xi, M.shutter_draws(W, H, it, lib=lib)), f"shutter draws at iteration {it}"
        assert (cams[..., 19] == 0).all()
        o, c = M.camera_fields(open_), M.camera_fields(close)
        got = cams[..., 1:19].reshape(H, W, 6, 3)
        want = M.lerp64(o, c, xi)
        ulp = np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
        assert (np.abs(got.astype(np.float64) - want) <= ulp).all(), "poses beyond 1 ulp of the float64 lerp"
        still = (o == c)
        assert np.array_equal(got.view(np.int32)[:, :, still], np.broadcast_to(o.view(np.int32)[still], (H, W, int(still.sum()))))
        if close is not turned:
            assert still[2:].all()                               # a pure translation keeps the basis bits
        r.close()


# ---- close == open is the static frame ---------------------------------------------------------------------------------------------------
SETUPS = ["hdri_compact", "hdri_wide_layers", "bruneton", "vol_integrator"]


def static_case(name, dragon, atmosphere, W=160, H=96):
    scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
    if name in ("bruneton", "vol_integrator"): atmosphere.apply(scene.atmos)
    kp = {"hdri_compact": dict(ray_depth=100), "hdri_wide_layers": dict(ray_depth=3, volume_depth=2),
          "bruneton": dict(environment_type=0, elevation=25.0, ray_depth=3), "vol_integrator": dict(integrator=1, ray_depth=4)}[name]

    def mk(cam):
        r = V.Renderer(scene, W, H, kp=make_kp(**kp), cam=cam)
        r.set_option("passes_per_chunk", 5)
        if name == "hdri_wide_layers":
            r.enable_aovs(); r.enable_light_groups(); r.enable_deep([0.0, 2.0, 4.0, float("inf")])
        return r
    return scene, mk


def sequence(scene, r):
    """A new frame across a chunk boundary, a continued call, render == 0 and iteration >= max_interactions (both kernel tails)."""
    out = []
    fresh(scene, r); r.kp.render = 1; r.kp.max_interactions = 1000
    r.render(PASSES); torch.cuda.synchronize(); out.append(snapshot(scene, r))
    r.render(3); torch.cuda.synchronize(); out.append(snapshot(scene, r))
    r.kp.render = 0; r.render(2); torch.cuda.synchronize(); out.append(snapshot(scene, r))
    r.kp.render = 1; r.kp.max_interactions = r.kp.iteration; r.render(2); torch.cuda.synchronize(); out.append(snapshot(scene, r))
    return out


@pytest.mark.parametrize("setup", SETUPS)
@pytest.mark.parametrize("lens", [0.0, 0.15], ids=["pinhole", "thin_lens"])
def test_close_equal_to_open_is_the_static_frame(dragon, atmosphere, setup, lens):
    scene, mk = static_case(setup, dragon, atmosphere)
    cam = scene.frame_camera(160, 96, aperture=lens)
    static = mk(cam)
    static.set_option("miss_cull", 1)
    want = sequence(scene, static)
    mot = mk(cam)
    mot.set_camera_motion(copy_cam(cam))
    got = sequence(scene, mot)
    for n, (a, b) in enumerate(zip(want, got)):
        assert_same(a, b, f"{setup}, lens {lens}, step {n}")
    assert float(want[0]["depth"].max()) > 0
    static.close(); mot.close()


# ---- with the other features ---------------------------------------------------------------------------------------------------------------
def test_adaptive_pixels_equal_the_fixed_count_motion_frame_of_their_count(dragon):
    scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
    open_, close = poses(scene, 192, 96)
    r, f = (V.Renderer(scene, 192, 96, kp=make_kp(ray_depth=3, volume_depth=2), cam=open_) for _ in range(2))
    for x in (r, f):
        x.set_option("passes_per_chunk", 5); x.set_camera_motion(close)
    fresh(scene, r)
    run, counts, err = r.render_adaptive(32, threshold=0.2, min_passes=8, check_interval=8, error_map=True)
    torch.cuda.synchronize()
    got = snapshot(scene, r)
    classes = torch.unique(counts).tolist()
    assert len(classes) >= 2, classes
    for n in classes:
        fixed = frame(scene, f, passes=n)
        sel = counts.view(-1) == n
        for k in BUFFERS:
            assert torch.equal(bits(got[k]).view(sel.numel(), -1)[sel], bits(fixed[k]).view(sel.numel(), -1)[sel]), f"{k} on the pixels of {n} passes"
    r.close(); f.close()


def test_region_equals_the_full_motion_frame_inside_and_writes_nothing_outside(dragon):
    W, H = 192, 96
    scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
    open_, close = poses(scene, W, H)
    r = V.Renderer(scene, W, H, kp=make_kp(ray_depth=3, volume_depth=2), cam=open_)
    r.set_option("passes_per_chunk", 5); r.set_camera_motion(close); r.enable_aovs(); r.enable_light_groups()
    full = frame(scene, r, prefill=True)
    for reg in [(0, 0, 61, 33), (W // 3 + 1, H // 4 + 1, 2 * W // 3 + 3, 3 * H // 4 - 1)]:
        r.set_region(*reg)
        got = frame(scene, r, prefill=True)
        m = torch.zeros(H, W, dtype=torch.bool, device="cuda"); m[reg[1]:reg[3], reg[0]:reg[2]] = True
        m = m.view(-1)
        assert torch.equal(full["blue_noise"], got["blue_noise"])
        for k in full:
            if k == "blue_noise": continue
            a, b = bits(full[k]).view(m.numel(), -1), bits(got[k]).view(m.numel(), -1)
            assert torch.equal(a[m], b[m]), f"{k} inside {reg}"
            assert bool((b[~m] == (SENTINEL_D if k == "display" else SENTINEL_F)).all()), f"{k} written outside {reg}"
    r.close()


def test_three_shards_with_exchange_layers_equal_the_single_context(dragon, emissive, atmosphere):
    case = LayerCase("hdri", dragon, emissive, atmosphere)
    close = translated(case.cam, (0.4, 0.1, -0.3))
    sh = LayerShards(case, 3, 7)
    try:
        sh.each(enable_all)
        sh.each(lambda r: r.set_camera_motion(close))
        # The adaptive frame goes first: it sizes every shard's sample scratch for its 24 passes, so no later call reallocates it.  A call
        # that grows the scratch frees the old buffers (cudaFree waits for the device), and on one GPU that wait can fall behind a peer's
        # spinning flag wait until the wait gives up.
        P, mn, iv = 24, 4, 4
        sh.ref.kp.iteration = 0
        _, _, first = sh.ref.render_adaptive(P, threshold=FLT_MAX, min_passes=mn, check_interval=iv, error_map=True)
        thr = float(np.quantile(A.max3x3(first.cpu().numpy()), 0.4))
        sh.ref_scene.reset_blue_noise()
        res = {}

        def fn(k, r, stream):
            r.kp.iteration = 0
            if k < 0:
                res["ref"] = r.render_adaptive(P, threshold=thr, min_passes=mn, check_interval=iv, error_map=True)
            else:
                return sh.d[k].render_adaptive(P, threshold=thr, min_passes=mn, check_interval=iv, error_map=True, stream=stream)
        for s in sh.scenes: s.reset_blue_noise()
        out = sh.all(fn)
        run, counts, err = res["ref"]
        assert len(torch.unique(counts)) >= 2
        for k, (run_k, counts_k, err_k) in enumerate(out):
            assert run_k == run and torch.equal(counts_k, counts) and torch.equal(bits(err_k), bits(err)), f"adaptive motion frame of shard {k}"
        sh.check("adaptive motion frame")
        sh.ref_scene.reset_blue_noise()
        for s in sh.scenes: s.reset_blue_noise()
        sh.render(5, iteration=0); sh.check("motion frame")
        sh.render(4); sh.check("continued motion frame")
        assert sh.abandoned_waits() == [0, 0, 0]
    finally:
        sh.close()


# ---- it blurs -------------------------------------------------------------------------------------------------------------------------------
def test_a_pan_widens_the_partial_coverage_band():
    """Sanity, not parity: a 64-pass frame whose view pans by about 20 px over the shutter has a clearly wider band of partial coverage
    (0 < alpha < 1) at the silhouette than the static frame at the open pose.  The volume is an opaque ball, so partial coverage is the
    silhouette's alone (the dragon is partly transparent inside, which would mix its interior into the count)."""
    W, H = 256, 128
    n = 48
    z, y, x = np.mgrid[0:n, 0:n, 0:n].astype(np.float32)
    c = (n - 1) / 2.0
    ball = V.Volume.from_dense(np.where(np.sqrt((x - c) ** 2 + (y - c) ** 2 + (z - c) ** 2) < c, 50.0, 0.0).astype(np.float32),
                               bbox_min=(-c, -c, -c))
    scene = V.Scene([ball.instance()], env=synthetic_env(512, 256), keep=[ball])
    cam = scene.frame_camera(W, H)
    pan = copy_cam(cam)
    pan.lower_left_corner = N.f3(*[float(np.float32(getattr(cam.lower_left_corner, a)) + np.float32(20.0 / W) * np.float32(getattr(cam.horizontal, a)))
                                   for a in "xyz"])
    band = {}
    for moving in (False, True):
        r = V.Renderer(scene, W, H, kp=make_kp(ray_depth=3, volume_depth=2), cam=cam)
        r.enable_aovs()
        if moving: r.set_camera_motion(pan)
        frame(scene, r, passes=64)
        a = r.alpha_image()
        band[moving] = int(((a > 0.05) & (a < 0.95)).sum())
        r.close()
    print(f"\npartial-coverage pixels: static {band[False]}, 20 px pan {band[True]}")
    assert band[False] > 0 and band[True] > 3 * band[False], band


# ---- activation, clearing, refusals ---------------------------------------------------------------------------------------------------------
def test_activation_clearing_and_refusals(dragon):
    W, H = 128, 64
    scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
    open_, close = poses(scene, W, H)
    never = V.Renderer(scene, W, H, kp=make_kp(ray_depth=3, volume_depth=2), cam=open_)
    static = frame(scene, never)
    r = V.Renderer(scene, W, H, kp=make_kp(ray_depth=3, volume_depth=2), cam=open_)
    r.set_camera_motion(close)
    moving = frame(scene, r)
    assert not torch.equal(bits(moving["accum"]), bits(static["accum"]))
    # set or cleared mid-frame: the frame goes on with the pose it started with
    fresh(scene, r); r.render(3); r.clear_camera_motion(); r.render(5); torch.cuda.synchronize()
    assert_same(moving, snapshot(scene, r), "cleared at iteration 3")
    assert_same(static, frame(scene, r), "cleared: the static frame")
    fresh(scene, r); r.render(3); r.set_camera_motion(close); r.render(5); torch.cuda.synchronize()
    assert_same(static, snapshot(scene, r), "set at iteration 3")
    assert_same(moving, frame(scene, r), "set: the motion frame")
    # refused when set, changing nothing
    for field in M.FIELDS:
        for bad in (float("nan"), float("inf")):
            c = copy_cam(close)
            f = getattr(c, field); f.y = bad; setattr(c, field, f)
            assert V.lib.vpt_set_camera_motion(r.ctx, C.byref(c)) == -1, (field, bad)
            assert field.encode() in V.lib.vpt_last_error(r.ctx)
    assert_same(moving, frame(scene, r), "after refused poses")
    # w, time0, time1 and the lens fields of the close pose are not read
    c = copy_cam(close); c.w = N.f3(float("nan"), 0.0, 0.0); c.time0 = 5.0; c.time1 = float("inf"); c.lens_radius = 3.0; c.focus_dist = -1.0
    r.set_camera_motion(c)
    assert_same(moving, frame(scene, r), "fields that are not read")
    # vpt_debug_camera_rays refuses a motion frame; vpt_debug_motion_cameras a static one
    r.kp.iteration = 0
    with pytest.raises(V.VptError, match="vpt_debug_motion_cameras"):
        r.camera_rays()
    with pytest.raises(V.VptError):
        never.motion_cameras()
    # motion with the equirectangular projection is refused at render time
    r.set_projection("equirect"); r.kp.iteration = 0
    assert V.lib.vpt_render_passes(r.ctx, r.params.array, 2, None) == -3
    assert b"equirectangular" in V.lib.vpt_last_error(r.ctx)
    r.set_projection("perspective")
    assert_same(moving, frame(scene, r), "after the refused panorama")
    r.close(); never.close()
