"""The tail of the reference kernel (render_kernel.cu:2262-2316) against that kernel, from buffers that are not empty: the NaN / Inf guard,
the viz_dof tint, the running means of accum, depth and cost, ACES, exposure, gamma, the BGRA pack and raw.  Here that tail is
resolve_pixel of vpt_kernels.cu (k_resolve, k_resolve_adaptive) and of vpt_level_a.cu; every reference comparison runs on the wavefront
path (Renderer.render) and on level (A) through the reference loader.

  A  nothing sampled (iteration = max_interactions): chosen values re-tonemapped at five exposures -- no randomness, the tonemap alone;
  B  a frame continued from random buffers by passes that sample and passes that only re-tonemap, thin lens with viz_dof, per resolve
     variant (compact and wide HDRI records, k_resolve<1>, k_resolve<2>, level (A)), and across a chunk boundary;
  C  render == 0 from prefilled buffers: WHITE enters the mean, depth and cost decay;
  D  the guard from prefilled buffers: an environment with NaN and +Inf stripes, and a NaN sky_color that makes every sample non-finite.

Tolerances: accum and depth as everywhere (1e-5 + 1e-4 |ref| on >= 99.9 % of the pixels); cost, blue noise and iteration exact; raw.w
within 1e-5; raw.xyz NaN in the same places and within 1e-5 + 1e-4 |ref| elsewhere, on every pixel; display bit-equal on every pixel.
Measured on an H100: display 0 LSB everywhere; raw.xyz of level (A) within 0-4 ulp, of the wavefront path within 12 ulp in A and up to
655 ulp (values near 0 after the output matrix's cancellation) in B and D, because k_resolve rounds another product of the ACES input
matrix on its own than the reference (DESIGN.md section 5).
"""
import os

import numpy as np
import pytest
import torch

import vpt_b200 as V
from vpt_b200.scene import synthetic_env
import denoise_ref as D
import oracle_ref
from test_parity_gpu import flipped_fraction, make_kp, MAX_FLIPPED, needs_ref, _sky_power_table
from test_scale_gpu import LEVEL_A, _launch_candidate

pytestmark = [pytest.mark.gpu, needs_ref,
              pytest.mark.skipif(not os.path.exists(LEVEL_A), reason="volume_rt_kernel_b200.cubin not built")]


@pytest.fixture(scope="module")
def dragon():
    return V.Volume.load_vdb(V.find_asset("dragon.vdb"))


def prefill(b, seed):
    """Positive accum and depth and non-zero cost, from `seed` (multiples of 1/1024: exact in float32, and they store small); raw and
    display get junk, which every kernel must overwrite."""
    rng = np.random.RandomState(seed)
    n = b.accum.shape[0]
    b.accum.copy_(torch.from_numpy(rng.randint(1, 4096, (n, 3)).astype(np.float32) / 1024))
    b.depth.copy_(torch.from_numpy(rng.randint(1, 40 * 1024, n).astype(np.float32) / 1024))
    b.cost.copy_(torch.from_numpy(rng.randint(1, 4096, (n, 3)).astype(np.float32) / 1024))
    b.raw.fill_(-3.0); b.display.fill_(0x12345678)


def outputs(r, scene):
    torch.cuda.synchronize()
    b = r.buffers
    return dict(accum=b.accum.cpu().numpy(), depth=b.depth.cpu().numpy(), cost=b.cost.cpu().numpy(), raw=b.raw.cpu().numpy(),
                display=b.display.cpu().numpy().view(np.uint32), bn=scene.d_blue_noise.cpu().numpy(), iteration=int(r.kp.iteration))


def run_all(scene, mk, passes, fill, variants=(("wavefront", {}),), level_a=True):
    """The reference kernel, each wavefront variant (renderer options) and level (A), each from the buffers `fill` leaves and the initial
    blue noise -> (reference outputs, {label: outputs})."""
    orc = oracle_ref.RefOracle(); orc.load_kernels(); orc.load_candidate(LEVEL_A)
    root = orc.build_octree(scene.h_volumes, len(scene.instances))
    ref = mk(); ref.params.p_oct.value = root; fill(ref.buffers)
    scene.reset_blue_noise(); orc.render(ref, passes, full=True)
    want = outputs(ref, scene)
    got = {}
    for label, opts in variants:
        r = mk()
        for k, v in opts.items(): r.set_option(k, v)
        fill(r.buffers)
        scene.reset_blue_noise(); r.render(passes)
        got[label] = outputs(r, scene)
    if level_a:
        a = mk(); a.params.p_oct.value = root; fill(a.buffers)
        scene.reset_blue_noise(); _launch_candidate(orc, a, passes)
        got["level A"] = outputs(a, scene)
    return want, got


def ulps(a, b):
    """Largest |a - b| in float32 units in the last place, over the pairs where neither is NaN."""
    def ordered(x):
        i = np.ascontiguousarray(x, np.float32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7fffffff), i)
    d = np.abs(ordered(a) - ordered(b))
    d[np.isnan(a) | np.isnan(b)] = 0
    return int(d.max()) if d.size else 0


def lsbs(a, b):
    """Largest per-channel difference of two arrays of display words."""
    return int(np.abs(a.view(np.uint8).reshape(-1, 4).astype(int) - b.view(np.uint8).reshape(-1, 4).astype(int)).max())


def assert_tail(got, want, what):
    """Every output of one run against the reference kernel's; returns (raw.xyz ulps, display LSBs) for the record."""
    assert flipped_fraction(got["accum"], want["accum"]) <= MAX_FLIPPED, f"{what}: accum"
    assert flipped_fraction(got["depth"][:, None], want["depth"][:, None]) <= MAX_FLIPPED, f"{what}: depth"
    assert np.array_equal(got["cost"].view(np.int32), want["cost"].view(np.int32)), f"{what}: cost must be bit-equal"
    assert np.abs(got["raw"][:, 3] - want["raw"][:, 3]).max() <= 1e-5, f"{what}: raw.w"
    g, w = got["raw"][:, :3].astype(np.float64), want["raw"][:, :3].astype(np.float64)
    assert np.array_equal(np.isnan(g), np.isnan(w)), f"{what}: raw.xyz NaN in other places"
    with np.errstate(invalid="ignore"):
        ok = (g == w) | (np.abs(g - w) <= 1e-5 + 1e-4 * np.abs(w))
    bad = ~ok & ~np.isnan(w)
    assert not bad.any(), f"{what}: raw.xyz off on {int(bad.any(axis=1).sum())} pixels"
    d = lsbs(got["display"], want["display"])
    assert d == 0, f"{what}: display off by {d} LSB"
    assert np.array_equal(got["bn"], want["bn"]), f"{what}: blue-noise state"
    assert got["iteration"] == want["iteration"], f"{what}: iteration"
    u = ulps(got["raw"][:, :3], want["raw"][:, :3])
    print(f"{what}: raw.xyz within {u} ulp, display within {d} LSB, accum flipped {flipped_fraction(got['accum'], want['accum']):.3g}")
    return u, d


# ---- A: the re-tonemap table ---------------------------------------------------------------------------------------------------------
# ACES: after the input matrix (rows sum to 1) a grey x is v ~ x, and the fit's v * (v + 0.0245786) overflows float32 from v ~ 1.844e19:
# inf / inf is NaN there, which the gamma's fmaxf turns black.
TABLE = np.array([0.0, -0.0, 1e-40, 1e-8, 1e-3, 0.18, 1.0, 4.0, 65504.0, 1.7e19, 1.83e19, 1.845e19, 1.86e19, 2e19, 1e30, -1.0,
                  np.inf, np.nan], np.float32)


def table_fill(seed):
    def fill(b):
        prefill(b, seed)
        rng = np.random.RandomState(seed)
        vals = np.resize(TABLE, b.accum.numel())
        b.accum.copy_(torch.from_numpy(rng.permutation(vals).reshape(-1, 3)))
    return fill


@pytest.mark.parametrize("exposure", [1.0, 0.37, 4.0, 0.0, -1.0])
def test_retonemap_table_against_the_reference(dragon, exposure):
    """iteration = max_interactions: no pass samples, so accum, depth and cost stay as they were and raw / display are the tonemap of the
    chosen values alone."""
    W, H = 64, 48
    scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
    cam = scene.frame_camera(W, H)
    mk = lambda: V.Renderer(scene, W, H, kp=make_kp(ray_depth=2, iteration=4, max_interactions=4, exposure_scale=exposure), cam=cam)
    fill = table_fill(5)
    want, got = run_all(scene, mk, 2, fill)
    start = mk(); fill(start.buffers); start = outputs(start, scene)
    for k in ("accum", "depth", "cost"):
        assert np.array_equal(want[k].view(np.int32), start[k].view(np.int32)), f"the reference moved {k}"
    assert (want["raw"][:, 3] == 0).all()
    nan = np.isnan(want["raw"][:, :3]).any(axis=1)
    assert 0 < nan.sum() < W * H, "the table must give both finite and NaN raw colours"
    # the restatement on the rows of finite values below the overflow, where float32 rounding cannot decide between a colour and NaN
    rows = (np.abs(start["accum"]) < 1e19).all(axis=1)
    words = D.display_words(start["accum"][rows], exposure)
    for what, out in got.items():
        for k in ("accum", "depth", "cost"):
            assert np.array_equal(out[k].view(np.int32), start[k].view(np.int32)), f"{what} moved {k}"
        assert_tail(out, want, f"A exposure {exposure} {what}")
        print(f"A exposure {exposure} {what}: display within {lsbs(out['display'][rows], words)} LSB of denoise_ref.display_words")
        assert lsbs(out["display"][rows], words) <= 1


# ---- B: a frame continued, one case per resolve variant ------------------------------------------------------------------------------
def tint_classes(scene, mk):
    """Pixels of one pass at iteration 0 whose depth sample gets each viz_dof tint (red: behind the focus band, blue: in front of it,
    green: inside it), as the tail decides."""
    r = mk(); r.kp.iteration = 0; r.buffers.zero_()
    scene.reset_blue_noise(); r.render(1); torch.cuda.synchronize()
    d = r.buffers.depth.cpu().numpy()
    f, aof = np.float32(r.cam.focus_dist), np.float32(1) / np.float32(r.cam.lens_radius)
    return dict(red=int((d > f + aof).sum()), blue=int((d < f - aof).sum()), green=int(((d > f - aof) & (d < f + aof)).sum()))


def continued_case(name, dragon):
    """-> (scene, mk, keep-alive objects): 128x96, thin lens (aperture 2: a focus band 1 world unit either side of the dragon's centre)
    with viz_dof, iteration 5 of max_interactions 8, exposure 0.37"""
    W, H = 128, 96
    scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
    cam = scene.frame_camera(W, H, aperture=2.0)
    cam.viz_dof = 1
    kw = dict(ray_depth=3, iteration=5, max_interactions=8, exposure_scale=0.37)
    keep = []
    if name in ("sky", "vol_sky_table"):
        atm = V.Atmosphere(); atm.apply(scene.atmos); keep.append(atm)
        kw.update(environment_type=0, elevation=30.0)
    if name == "vol_sky_table":
        tables = V.EnvTables(_sky_power_table()); keep.append(tables)
        kw.update(integrator=1)
    def mk():
        r = V.Renderer(scene, W, H, kp=make_kp(**kw), cam=cam)
        if name == "vol_sky_table": tables.apply(r.kp)
        return r
    return scene, mk, keep


@pytest.mark.parametrize("name", ["hdri", "sky", "vol_sky_table"])
def test_continued_frame_against_the_reference(dragon, name):
    """5 passes from iteration 5 of 8: three sample, two only re-tonemap.  HDRI: the lean kernel's compact records, the generic kernel's
    wide records and level (A); the precomputed sky with the direct integrator (k_resolve<1>); the volumetric path integrator on the
    tabulated sky (k_resolve<2>).  The wavefront variants also run with a chunk boundary inside the call (passes_per_chunk = 2)."""
    scene, mk, keep = continued_case(name, dragon)
    tints = tint_classes(scene, mk)
    print(f"B {name}: tints {tints}")
    assert min(tints.values()) > 0, f"every viz_dof tint must occur: {tints}"
    variants = [("wavefront", {}), ("wavefront, chunks of 2", dict(passes_per_chunk=2))]
    if name == "hdri":
        variants += [("generic kernel", dict(generic_kernel=1)), ("generic kernel, chunks of 2", dict(generic_kernel=1, passes_per_chunk=2))]
    want, got = run_all(scene, mk, 5, lambda b: prefill(b, 17), variants=variants, level_a=name == "hdri")
    assert want["iteration"] == 10 and float(np.abs(want["cost"]).max()) > 0
    start = mk(); prefill(start.buffers, 17); start = outputs(start, scene)
    assert not np.array_equal(want["cost"], start["cost"]), "the cost must decay"
    for what, out in got.items():
        assert_tail(out, want, f"B {name} {what}")


# ---- C: render == 0 ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("iteration", [0, 3])
def test_render_off_against_the_reference(dragon, iteration):
    """render == 0 samples nothing: WHITE enters the mean (at iteration 0 it replaces accum), depth and cost decay towards 0."""
    W, H = 64, 48
    scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
    cam = scene.frame_camera(W, H)
    mk = lambda: V.Renderer(scene, W, H, kp=make_kp(ray_depth=2, render=0, iteration=iteration), cam=cam)
    want, got = run_all(scene, mk, 2, lambda b: prefill(b, 23))
    if iteration == 0:
        assert (want["accum"] == 1.0).all() and (want["depth"] == 0).all() and (want["cost"] == 0).all()
    else:
        assert (want["depth"] > 0).all() and (want["cost"] > 0).all()
    for what, out in got.items():
        assert_tail(out, want, f"C iteration {iteration} {what}")


# ---- D: the NaN / Inf guard ----------------------------------------------------------------------------------------------------------
def striped_env():
    """The synthetic sky with NaN stripes and +Inf stripes (12 texels wide each) around the whole horizon."""
    env = synthetic_env(512, 256)
    x = np.arange(512) % 64
    env[:, x < 12, :3] = np.nan
    env[:, (x >= 32) & (x < 44), :3] = np.inf
    return env


@pytest.mark.parametrize("iteration,passes", [(0, 1), (0, 4), (3, 2)])
@pytest.mark.parametrize("env", ["stripes", "nan_sky_color"])
def test_guard_against_the_reference(dragon, env, iteration, passes):
    """A non-finite sample becomes accum_buffer[idx]: at iteration 0 the buffer's previous content, later the running mean.  With a NaN
    sky_color every sample is non-finite, so accum keeps the prefill bit for bit."""
    W, H = 96, 64
    scene = V.Scene([dragon.instance()], env=striped_env() if env == "stripes" else synthetic_env(512, 256))
    cam = scene.frame_camera(W, H)
    kw = dict(ray_depth=2, iteration=iteration)
    if env == "nan_sky_color": kw["sky_color"] = V.f3(float("nan"), float("nan"), float("nan"))
    mk = lambda: V.Renderer(scene, W, H, kp=make_kp(**kw), cam=cam)
    want, got = run_all(scene, mk, passes, lambda b: prefill(b, 29))
    start = mk(); prefill(start.buffers, 29); start = outputs(start, scene)
    kept = (want["accum"] == start["accum"]).all(axis=1)
    print(f"D {env} iteration {iteration} x{passes}: {100 * kept.mean():.1f} % of the pixels keep their prefill")
    if env == "nan_sky_color":
        assert np.array_equal(want["accum"].view(np.int32), start["accum"].view(np.int32))
        moved = [what for what, out in got.items() if not np.array_equal(out["accum"].view(np.int32), start["accum"].view(np.int32))]
        assert not moved, f"{moved}: accum must keep the prefill"
    else:
        assert 0.001 < kept.mean() < 0.999, "the stripes must cover some pixels and not all"
    for what, out in got.items():
        assert_tail(out, want, f"D {env} iteration {iteration} x{passes} {what}")
