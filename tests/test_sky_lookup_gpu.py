"""The run-time Bruneton sky look-up (vpt_atmosphere.cuh) against the reference kernel, across altitude, the horizon, space, the sun disc
and twilight.  Both kernels read this library's own tables (V.Atmosphere), so the look-up alone is compared.

  A  miss-only frames (tests/sky_cases.py: the instance and the sphere behind the camera, so every pixel is the look-up at the camera
     origin plus the running mean): every case under integrator 0 (k_resolve<1>) and integrator 1 (the k_resolve<2> tail), and through
     level (A).  Bar: accum, depth and display bit-equal to the reference on every pixel; depth holds the miss value everywhere.
     The frames listed in NOT_BIT_EQUAL are held to the project tolerance and to their measured count of differing pixels.
  B  luminance modes 1 and 2 (white balance off, exposure 2.5) on the horizon, space and sun-disc frames.  Same bar.
  C  in-path look-ups at altitude: the dragon at y = 300 m, 5 km and 25 km and straddling y = 0, framed as Scene.frame_camera frames it, under
     integrator 1 (environment_type 0, the frame's own sky table) with the sun at 30 and -15 degrees, and integrator 0 at 5 and 25 km.
     These frames track through the volume, so the bar is the project tolerance: at most 0.1 % of the pixels outside 1e-5 + 1e-4 |ref|.

Every case also shows that its frame depends on what it exercises: the reference frame is not constant; in the sun-disc frames every
pixel inside the disc differs from every pixel of the ring around it; in a frame wholly past the atmosphere every pixel off the disc
holds the reference's zero-radiance value.  Stored reference outputs under tests/golden/oracle/ replay the comparisons where
oracle/_ref is not built."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import vpt_b200 as V
from vpt_b200 import _native as N
from vpt_b200.scene import synthetic_env
import oracle_ref
import sky_cases as S
from test_parity_gpu import MAX_FLIPPED, flipped_fraction, make_kp, needs_ref
from test_scale_gpu import LEVEL_A, _launch_candidate

pytestmark = pytest.mark.gpu
needs_level_a = pytest.mark.skipif(not os.path.exists(LEVEL_A), reason="volume_rt_kernel_b200.cubin not built")
PASSES = 2
LUMINANCE = {"luminance1": dict(luminance=1, white_balance=False, exposure=2.5), "luminance2": dict(luminance=2, white_balance=False, exposure=2.5)}


@pytest.fixture(scope="module")
def dragon():
    return V.Volume.load_vdb(V.find_asset("dragon.vdb"))


@pytest.fixture(scope="module")
def atmospheres():
    cache = {}

    def get(name="default"):
        if name not in cache:
            cache[name] = V.Atmosphere(**LUMINANCE.get(name, {}))
        return cache[name]
    yield get
    for a in cache.values(): a.destroy()


def volume_bounds(g):
    b6 = (C.c_float * 6)()
    N.lib.vpt_volume_bounds(C.byref(g), b6)
    return np.array(list(b6), dtype=np.float32)


def miss_scene(dragon, g, atmosphere):
    """The one-instance scene of a miss-only geometry: the dragon's box and the reference sphere behind the camera plane."""
    pos, centre = S.placement(g)
    scene = V.Scene([dragon.instance(pos=pos)], env=synthetic_env(512, 256))
    assert np.array_equal(volume_bounds(scene.instances[0]), S.instance_bounds(pos)), "the CPU proof of the miss is about another box"
    sp = scene.h_sphere; sp.center = V.f3(*centre); sp.radius = S.SPHERE_RADIUS
    scene.d_sphere.copy_(torch.frombuffer(bytearray(bytes(sp)), dtype=torch.uint8))
    atmosphere.apply(scene.atmos)
    return scene


class Runs:
    """One scene and camera, rendered by the reference kernel, this library and level (A) from the same iteration and blue noise."""

    def __init__(self, scene, cam, W, H, passes):
        self.scene, self.cam, self.W, self.H, self.P = scene, cam, W, H, passes
        self.orc = oracle_ref.RefOracle()
        self.root = self.orc.build_octree(scene.h_volumes, len(scene.instances))
        self.tables = []

    def _renderer(self, kw):
        r = V.Renderer(self.scene, self.W, self.H, kp=make_kp(**kw), cam=self.cam)
        if r.kp.integrator == 1:
            # the reference's create_cdf tabulates the sky of the frame's own azimuth, elevation and sky_color
            t = V.EnvTables(V.sky_power_table(r.kp.azimuth, r.kp.elevation, (r.kp.sky_color.x, r.kp.sky_color.y, r.kp.sky_color.z)))
            t.apply(r.kp); self.tables.append(t)
        return r

    def _out(self, r):
        torch.cuda.synchronize()
        b = r.buffers
        return dict(accum=b.accum.cpu().numpy(), depth=b.depth.cpu().numpy(), display=b.display.cpu().numpy().view(np.uint32))

    def reference(self, **kw):
        r = self._renderer(kw)
        r.params.p_oct.value = self.root
        self.scene.reset_blue_noise(); self.orc.render(r, self.P)
        return self._out(r)

    def library(self, **kw):
        r = self._renderer(kw)
        self.scene.reset_blue_noise(); r.render(self.P)
        return self._out(r)

    def level_a(self, **kw):
        self.orc.load_kernels(); self.orc.load_candidate(LEVEL_A)
        r = self._renderer(kw)
        r.params.p_oct.value = self.root
        self.scene.reset_blue_noise(); _launch_candidate(self.orc, r, self.P)
        return self._out(r)

    def close(self):
        for t in self.tables: t.destroy()
        self.tables.clear()


def bit_equal_fraction(got, want):
    return float((got["accum"].view(np.int32) == want["accum"].view(np.int32)).all(axis=1).mean())


def max_abs(got, want):
    return float(np.nanmax(np.abs(got["accum"].astype(np.float64) - want["accum"])))


def differing_pixels(got, want):
    a, b = got["accum"].view(np.uint32), want["accum"].view(np.uint32)
    return int((a != b).any(axis=1).sum())


def check_bit_equal(got, want, what, known=0):
    """The bar of a miss-only frame: accum, depth and display bit-equal to the reference on every pixel.  A frame listed in
    NOT_BIT_EQUAL (`known` > 0 differing pixels measured) is held to the project tolerance and to at most that many differing pixels,
    and its display words to 1 LSB on at most MAX_FLIPPED of the pixels.  Returns the failures as text, so that a case reports every variant before it fails."""
    n = differing_pixels(got, want)
    print(f"{what}: bit-equal accum on {100 * bit_equal_fraction(got, want):.2f} % of the pixels ({n} differ), max |d| {max_abs(got, want):.3g}")
    bad = []
    if not np.isfinite(want["accum"]).all(): bad.append(f"{what}: the reference frame is not finite")
    if n > known: bad.append(f"{what}: accum differs on {n} pixels (known: {known})")
    if flipped_fraction(got["accum"], want["accum"]) > MAX_FLIPPED: bad.append(f"{what}: accum outside the tolerance")
    if not np.array_equal(got["depth"].view(np.uint32), want["depth"].view(np.uint32)): bad.append(f"{what}: depth differs")
    dm = got["display"].view(np.uint8).reshape(-1, 4).astype(int); dr = want["display"].view(np.uint8).reshape(-1, 4).astype(int)
    moved = np.abs(dm - dr).max(axis=1) > 0
    if (known == 0 and moved.any()) or np.abs(dm - dr).max() > 1 or moved.mean() > MAX_FLIPPED:
        bad.append(f"{what}: display differs on {int(moved.sum())} pixels")
    # a miss writes one depth value: every pixel holds it in both kernels
    d = want["depth"].view(np.uint32)
    if not (d == d[0]).all(): bad.append(f"{what}: the depth buffer is not the miss value everywhere")
    return bad


def assert_depends(want, g, sun_index, what):
    """Non-vacuity of a miss-only frame (the module text)."""
    acc = want["accum"].reshape(g.size[1], g.size[0], 3)
    claims = S.claims_of(g, sun_index)
    if "all_past" in claims:
        off = S.off_disc(g, sun_index)
        zero = acc[off]
        print(f"{what}: {int(off.sum())} pixels off the disc hold {zero[0]}")
        assert off.sum() > 0 and (zero.view(np.uint32) == zero[0].view(np.uint32)).all() and np.abs(zero[0]).max() <= 1e-6, \
            f"{what}: a pixel off the disc is not the zero-radiance value"
    if "disc" in claims:
        inside, ring = S.disc_masks(g, sun_index)
        a, b = acc[inside].sum(axis=1), acc[ring].sum(axis=1)
        print(f"{what}: disc {int(inside.sum())} pixels in [{a.min():.6g}, {a.max():.6g}], ring {int(ring.sum())} pixels in [{b.min():.6g}, {b.max():.6g}]")
        assert inside.sum() > 0 and ring.sum() > 0 and a.min() > b.max(), f"{what}: the sun disc does not stand out of the ring around it"
    if "all_past" not in claims and "mu_s-" not in claims:
        flat = acc.reshape(-1, 3)
        print(f"{what}: {100 * (flat != flat[0]).any(axis=1).mean():.2f} % of the pixels differ from the first")
        assert (flat != flat[0]).any(), f"{what}: the reference frame is constant"


def test_sky_case_constants_match_the_parameter_block(atmospheres):
    p = atmospheres().params
    assert (p.bottom_radius, p.top_radius) == (S.RG, S.RT)
    assert float(np.float32(p.sun_angular_radius)) == S.SUN_ANGULAR_RADIUS
    assert float(np.float32(p.mu_s_min)) == S.MU_S_MIN


# Miss-only frames whose accum is not bit-equal to the reference's: (case, [luminance mode,] integrator[, "A" for level (A)]) -> the
# number of differing pixels measured on an H100 (sm_90a), out of 3072, each off by 1-2 ulp (max |d| 3.1e-6).  They are frames in which
# the sun lights some ground point seen from 10 m or higher; this library and level (A) differ on the same pixels.  The operation is a
# sun-lit ground-branch term not yet pinned (DESIGN §5).  Every frame not listed must be bit-equal on every pixel.
NOT_BIT_EQUAL = {
    ('ground_up-az200-el45', 0): 1,
    ('ground_up-az200-el45', 1): 1,
    ('ground_up-az90-el3', 0): 1,
    ('ground_up-az90-el3', 1): 1,
    ('horizon_10m-az75-el3', 0): 79,
    ('horizon_10m-az75-el3', 1): 79,
    ('horizon_2000m-az75-el3', 0): 25,
    ('horizon_2000m-az75-el3', 1): 25,
    ('horizon_12000m-az75-el3', 0): 13,
    ('horizon_12000m-az75-el3', 1): 13,
    ('horizon_12000m-az75-el-0.5', 0): 4,
    ('horizon_12000m-az75-el-0.5', 1): 4,
    ('horizon_45000m-az75-el3', 0): 11,
    ('horizon_45000m-az75-el3', 1): 11,
    ('horizon_45000m-az75-el-0.5', 0): 6,
    ('horizon_45000m-az75-el-0.5', 1): 6,
    ('altitude_500m-az120-el30', 0): 49,
    ('altitude_500m-az120-el30', 1): 49,
    ('altitude_5000m-az120-el30', 0): 166,
    ('altitude_5000m-az120-el30', 1): 166,
    ('altitude_20000m-az120-el30', 0): 458,
    ('altitude_20000m-az120-el30', 1): 458,
    ('altitude_40000m-az120-el30', 0): 318,
    ('altitude_40000m-az120-el30', 1): 318,
    ('altitude_59900m-az120-el30', 0): 578,
    ('altitude_59900m-az120-el30', 1): 578,
    ('top_inside-az10-el45', 0): 464,
    ('top_inside-az10-el45', 1): 464,
    ('top_outside-az10-el45', 0): 106,
    ('top_outside-az10-el45', 1): 106,
    ('space_down_150km-az120-el30', 0): 594,
    ('space_down_150km-az120-el30', 1): 594,
    ('space_down_150km-az180-el3', 0): 44,
    ('space_down_150km-az180-el3', 1): 44,
    ('limb_1500km-az45-el30', 0): 37,
    ('limb_1500km-az45-el30', 1): 37,
    ('offset_40km-az120-el30', 0): 785,
    ('offset_40km-az120-el30', 1): 785,
    ('ground_up-az200-el45', 0, 'A'): 1,
    ('ground_up-az200-el45', 1, 'A'): 1,
    ('ground_up-az90-el3', 0, 'A'): 1,
    ('ground_up-az90-el3', 1, 'A'): 1,
    ('horizon_10m-az75-el3', 0, 'A'): 79,
    ('horizon_10m-az75-el3', 1, 'A'): 79,
    ('horizon_2000m-az75-el3', 0, 'A'): 25,
    ('horizon_2000m-az75-el3', 1, 'A'): 25,
    ('horizon_12000m-az75-el3', 0, 'A'): 13,
    ('horizon_12000m-az75-el3', 1, 'A'): 13,
    ('horizon_12000m-az75-el-0.5', 0, 'A'): 4,
    ('horizon_12000m-az75-el-0.5', 1, 'A'): 4,
    ('horizon_45000m-az75-el3', 0, 'A'): 11,
    ('horizon_45000m-az75-el3', 1, 'A'): 11,
    ('horizon_45000m-az75-el-0.5', 0, 'A'): 6,
    ('horizon_45000m-az75-el-0.5', 1, 'A'): 6,
    ('altitude_500m-az120-el30', 0, 'A'): 49,
    ('altitude_500m-az120-el30', 1, 'A'): 49,
    ('altitude_5000m-az120-el30', 0, 'A'): 166,
    ('altitude_5000m-az120-el30', 1, 'A'): 166,
    ('altitude_20000m-az120-el30', 0, 'A'): 458,
    ('altitude_20000m-az120-el30', 1, 'A'): 458,
    ('altitude_40000m-az120-el30', 0, 'A'): 318,
    ('altitude_40000m-az120-el30', 1, 'A'): 318,
    ('altitude_59900m-az120-el30', 0, 'A'): 578,
    ('altitude_59900m-az120-el30', 1, 'A'): 578,
    ('top_inside-az10-el45', 0, 'A'): 464,
    ('top_inside-az10-el45', 1, 'A'): 464,
    ('top_outside-az10-el45', 0, 'A'): 106,
    ('top_outside-az10-el45', 1, 'A'): 106,
    ('space_down_150km-az120-el30', 0, 'A'): 594,
    ('space_down_150km-az120-el30', 1, 'A'): 594,
    ('space_down_150km-az180-el3', 0, 'A'): 44,
    ('space_down_150km-az180-el3', 1, 'A'): 44,
    ('limb_1500km-az45-el30', 0, 'A'): 37,
    ('limb_1500km-az45-el30', 1, 'A'): 37,
    ('offset_40km-az120-el30', 0, 'A'): 785,
    ('offset_40km-az120-el30', 1, 'A'): 785,
    ('horizon_2000m-az75-el3', 'luminance1', 0): 25,
    ('horizon_2000m-az75-el3', 'luminance1', 1): 25,
    ('space_down_150km-az120-el30', 'luminance1', 0): 798,
    ('space_down_150km-az120-el30', 'luminance1', 1): 798,
    ('limb_1500km-az45-el30', 'luminance1', 0): 77,
    ('limb_1500km-az45-el30', 'luminance1', 1): 77,
}


# ---- A: miss-only frames, both integrators, this library and level (A) -------------------------------------------------------------
def miss_kw(sun, integrator):
    return dict(integrator=integrator, environment_type=0, azimuth=sun.azimuth, elevation=sun.elevation, ray_depth=2 if integrator == 0 else 6)


def run_miss_case(dragon, atmospheres, case, variant):
    """Both integrators of one miss-only case: the reference frame, its non-vacuity, and `variant` ("library" or "level_a") against it."""
    g, i = S.GEOMETRY[case[0]], case[1]
    sun = g.suns[i]
    scene = miss_scene(dragon, g, atmospheres())
    f = Runs(scene, S.camera(g), g.size[0], g.size[1], PASSES)
    bad = []
    try:
        for integrator in (0, 1):
            kw = miss_kw(sun, integrator)
            what = f"{S.case_id(case)} integrator {integrator}" + (" level A" if variant == "level_a" else "")
            want = f.reference(**kw)
            assert_depends(want, g, i, what)
            if "mu_s-" in S.claims_of(g, i):
                # the sun more than 30 degrees down: u_mu_s is clamped and the frame is one value; it is not the frame of a -15 degree sun
                above = f.reference(**dict(kw, elevation=-15.0))
                assert (want["accum"] == want["accum"][0]).all() and (above["accum"] != want["accum"]).any(axis=1).mean() > 0.25, what
            key = (S.case_id(case), integrator) + (("A",) if variant == "level_a" else ())
            bad += check_bit_equal(getattr(f, variant)(**kw), want, what, NOT_BIT_EQUAL.get(key, 0))
    finally:
        f.close(); scene.destroy()
    assert not bad, bad


@needs_ref
@pytest.mark.parametrize("case", S.CASES, ids=S.case_id)
def test_miss_only_frame_bit_equal(dragon, atmospheres, case):
    run_miss_case(dragon, atmospheres, case, "library")


@needs_ref
@needs_level_a
@pytest.mark.parametrize("case", S.CASES, ids=S.case_id)
def test_miss_only_frame_level_a_bit_equal(dragon, atmospheres, case):
    run_miss_case(dragon, atmospheres, case, "level_a")


# ---- B: luminance modes ---------------------------------------------------------------------------------------------------------------
B_CASES = [("horizon_2000m", 0), ("horizon_2000m", 1), ("space_down_150km", 0), ("limb_1500km", 0), ("disc_2m_sun30", 0), ("disc_150km_sun30", 0)]


# Luminance mode 2 with white balance off leaves every sky pixel off the sun disc at one value in both kernels, so only its sun-disc frames
# can show a difference
B_PARAMS = [(m, c) for m in LUMINANCE for c in B_CASES if m == "luminance1" or c[0].startswith("disc")]


@needs_ref
@pytest.mark.parametrize("mode,case", B_PARAMS, ids=[f"{S.case_id(c)}-{m}" for m, c in B_PARAMS])
def test_luminance_modes_bit_equal(dragon, atmospheres, mode, case):
    g, i = S.GEOMETRY[case[0]], case[1]
    sun = g.suns[i]
    scene = miss_scene(dragon, g, atmospheres(mode))
    f = Runs(scene, S.camera(g), g.size[0], g.size[1], PASSES)
    bad = []
    try:
        for integrator in (0, 1):
            kw = dict(integrator=integrator, environment_type=0, azimuth=sun.azimuth, elevation=sun.elevation, ray_depth=2 if integrator == 0 else 6)
            what = f"{S.case_id(case)} {mode} integrator {integrator}"
            want = f.reference(**kw)
            assert_depends(want, g, i, what)
            bad += check_bit_equal(f.library(**kw), want, what, NOT_BIT_EQUAL.get((S.case_id(case), mode, integrator), 0))
    finally:
        f.close(); scene.destroy()
    assert not bad, bad


# ---- C: in-path look-ups at altitude -----------------------------------------------------------------------------------------------------
C_W, C_H = 160, 96
C_CASES = [(alt, 1, el) for alt in (300.0, 5000.0, 25000.0, "straddle") for el in (30.0, -15.0)] + [(5000.0, 0, 30.0), (25000.0, 0, 30.0)]


def frame_instance(scene, width, height, fov=30.0):
    """Scene.frame_camera's framing (from the box centre plus the box diagonal's length on every axis, looking back at the centre) of the
    instance's own box: frame_camera's box also holds the world origin, which would put a volume 25 km up at the edge of its frame."""
    b = volume_bounds(scene.instances[0])
    lo, hi = b[:3], b[3:]
    centre = (hi + lo) / np.float32(2)
    lookfrom = centre + np.float32(float(np.linalg.norm(hi - lo)))
    cam = N.camera()
    N.lib.vpt_camera_look_at(C.byref(cam), N.fvec(lookfrom), N.fvec(centre), N.fvec((0, 1, 0)), float(fov), float(width) / float(height), 0.0)
    return cam


def _c_id(c):
    alt, integrator, el = c
    return f"{alt if isinstance(alt, str) else f'{alt:g}m'}-integrator{integrator}-el{el:g}"


@needs_ref
@pytest.mark.parametrize("case", C_CASES, ids=_c_id)
def test_in_path_lookups_at_altitude(dragon, atmospheres, case):
    alt, integrator, el = case
    if alt == "straddle":                                   # the box's centre at y = 0: scatter points above and below the ground sphere
        b = S.instance_bounds((0.0, 0.0, 0.0))
        y = -float(b[1] + b[4]) / 2
    else:
        y = alt
    scene = V.Scene([dragon.instance(pos=(0.0, y, 0.0))], env=synthetic_env(512, 256))
    atmospheres().apply(scene.atmos)
    lo, hi = volume_bounds(scene.instances[0])[1::3]
    if alt == "straddle": assert lo < 0 < hi
    f = Runs(scene, frame_instance(scene, C_W, C_H), C_W, C_H, PASSES)
    try:
        kw = dict(integrator=integrator, environment_type=0, azimuth=120.0, elevation=el, ray_depth=6 if integrator == 1 else 3)
        what = f"in path {_c_id(case)}"
        want = f.reference(**kw)
        got = f.library(**kw)
        frac = flipped_fraction(got["accum"], want["accum"])
        print(f"{what}: bit-equal accum on {100 * bit_equal_fraction(got, want):.2f} % of the pixels, max |d| {max_abs(got, want):.3g}, "
              f"flipped {frac:.3g}")
        flat = want["accum"]
        assert np.isfinite(flat).all() and (flat != flat[0]).any(), f"{what}: the reference frame is constant"
        assert frac <= MAX_FLIPPED, what
        assert flipped_fraction(got["depth"][:, None], want["depth"][:, None]) <= MAX_FLIPPED, f"{what}: depth"
    finally:
        f.close(); scene.destroy()
