"""Adaptive sampling on the GPU (vpt_render_adaptive): every pixel of an adaptive frame holds, bit for bit, what a fixed-count frame of
its own pass count holds; the stopping rule is the one tests/adaptive_ref.py restates; the edge cases and refusals are those
include/vpt_b200.h documents.

The thresholds of the parity cases were picked once on an H100 so that each frame has at least three pass-count classes, at least 5 %
of its pixels stopped at min_passes and some pixels at max_passes; assert_spread checks that, so no case can pass vacuously."""
import numpy as np
import pytest
import torch

import vpt_b200 as V
from vpt_b200.scene import synthetic_env
import adaptive_ref as A
import oracle_ref
from test_parity_gpu import flipped_fraction, make_kp, MAX_FLIPPED

pytestmark = pytest.mark.gpu
FLT_MAX = float(np.finfo(np.float32).max)
BUFFERS = ("accum", "depth", "cost", "raw", "display")


@pytest.fixture(scope="module")
def dragon():
    return V.Volume.load_vdb(V.find_asset("dragon.vdb"))


@pytest.fixture(scope="module")
def perlin():
    vol = V.Volume.procedural((96, 80, 72), scale=0.1, seed=123)
    vol.build_bricks()
    return vol


def _sky_power_table(res=180, sun_az=2.0, sun_el=1.0):
    el = (np.arange(res, dtype=np.float32) / (res - 1) * np.pi)[:, None]
    az = (np.arange(res, dtype=np.float32) / (res - 1) * 2 * np.pi)[None, :]
    return (0.05 + np.sin(el) * (1.2 + np.cos(az - sun_az)) * (0.3 + np.exp(-4.0 * (el - sun_el) ** 2))).astype(np.float32)


def _instances(dragon, n=120, seed=11):
    rng = np.random.RandomState(seed)
    inst = []
    for _ in range(n):
        q = rng.randn(4); q /= np.linalg.norm(q)
        inst.append(dragon.instance(pos=tuple(rng.uniform(-25, 25, 3)), quat=tuple(q), scale=float(rng.uniform(0.7, 1.3))))
    return inst


# name -> (W, H, max_passes, min_passes, check_interval, threshold)
CASES = {
    "headline":      (1920, 1080, 64, 16, 8, 0.3),
    "vol_sky_table": (200, 120, 32, 8, 8, 0.12),
    "lights_sphere": (256, 160, 32, 8, 8, 0.08),
    "instanced":     (256, 144, 32, 8, 8, 0.12),
    "brick":         (320, 200, 32, 8, 8, 0.2),
    "nan_prefilled": (256, 160, 32, 8, 8, 0.1),
}


def make_case(name, dragon, perlin):
    """-> (scene, make_renderer(), keep-alive objects)"""
    W, H = CASES[name][:2]
    env = synthetic_env(512, 256)
    if name == "headline":                                       # BASELINE config 2: ray_depth 100, sun + HDRI environment
        scene = V.Scene([dragon.instance()], env=env)
        cam = scene.frame_camera(W, H)
        return scene, (lambda: V.Renderer(scene, W, H, kp=make_kp(ray_depth=100), cam=cam)), []
    if name == "vol_sky_table":                                  # volumetric path integrator, tabulated sky (environment_type 0)
        scene = V.Scene([dragon.instance()], env=env)
        atm = V.Atmosphere(); atm.apply(scene.atmos)
        tables = V.EnvTables(_sky_power_table())
        cam = scene.frame_camera(W, H)
        def mk():
            r = V.Renderer(scene, W, H, kp=make_kp(integrator=1, environment_type=0, ray_depth=6), cam=cam)
            tables.apply(r.kp)
            return r
        return scene, mk, [atm, tables]
    if name == "lights_sphere":                                  # point lights, the sphere in view, thin lens
        lights = [((9.0, 6.0, 2.0), (1.0, 0.8, 0.6), 40.0), ((-2.0, 3.0, 8.0), (0.5, 0.7, 1.0), 25.0)]
        scene = V.Scene([dragon.instance()], env=env, lights=lights)
        sp = scene.h_sphere; sp.center = V.f3(4.0, 6.5, 3.0); sp.radius = 1.2; sp.roughness = 0.7; sp.color = V.f3(0.8, 0.6, 0.3)
        scene.d_sphere.copy_(torch.frombuffer(bytearray(bytes(sp)), dtype=torch.uint8))
        cam = scene.frame_camera(W, H, aperture=0.15)
        return scene, (lambda: V.Renderer(scene, W, H, kp=make_kp(ray_depth=3, volume_depth=2), cam=cam)), []
    if name == "instanced":                                      # 120 instances: the 2-rays-per-lane trace kernel
        scene = V.Scene(_instances(dragon), env=env)
        cam = scene.frame_camera(W, H)
        return scene, (lambda: V.Renderer(scene, W, H, kp=make_kp(ray_depth=2), cam=cam)), []
    if name == "nan_prefilled":                                  # NaN / +Inf environment stripes, a frame started on prefilled buffers
        from test_resolve_tail_gpu import prefill, striped_env
        scene = V.Scene([dragon.instance()], env=striped_env())
        cam = scene.frame_camera(W, H)
        def mk():
            r = V.Renderer(scene, W, H, kp=make_kp(ray_depth=4), cam=cam)
            r.prefill = lambda: prefill(r.buffers, 31)
            return r
        return scene, mk, []
    if name == "brick":                                          # brick mode on the procedural grid
        scene = V.Scene([perlin.instance()], env=env, keep=[perlin])
        cam = scene.frame_camera(W, H)
        def mk():
            r = V.Renderer(scene, W, H, kp=make_kp(ray_depth=2), cam=cam)
            r.set_brick_volume(perlin)
            return r
        return scene, mk, []
    raise KeyError(name)


def restart(scene, r):
    """A new frame: iteration 0, the initial blue noise, and zeroed buffers or the case's prefilled ones."""
    scene.reset_blue_noise(); r.kp.iteration = 0; r.buffers.zero_()
    if hasattr(r, "prefill"): r.prefill()


def adaptive_frame(scene, r, max_passes, min_passes, interval, thr, error_map=False):
    restart(scene, r)
    out = r.render_adaptive(max_passes, threshold=thr, min_passes=min_passes, check_interval=interval, error_map=error_map)
    torch.cuda.synchronize()
    return out


def assert_matches_fixed_frames(scene, r, f, counts, run):
    """Every count class c of the adaptive frame in r against a fresh render(c) in f, bitwise; blue noise against render(run)."""
    bufs = {k: getattr(r.buffers, k).clone() for k in BUFFERS}
    bn = scene.d_blue_noise.clone()
    flat = counts.reshape(-1)
    classes = [int(c) for c in torch.unique(flat).tolist()]
    assert run == max(classes)
    for c in classes:
        restart(scene, f); f.render(c); torch.cuda.synchronize()
        m = flat == c
        for k in BUFFERS:
            assert torch.equal(bufs[k][m], getattr(f.buffers, k)[m]), f"{k} differs on the {int(m.sum())} pixels of {c} passes"
        if c == run:
            assert torch.equal(bn, scene.d_blue_noise), "blue-noise state differs from `passes_run` fixed passes"
    return classes


def assert_spread(counts, min_passes, max_passes):
    flat = counts.reshape(-1)
    classes = torch.unique(flat).tolist()
    at_min = float((flat == min_passes).float().mean())
    print(f"classes {classes}, {100 * at_min:.1f} % at min_passes, {int((flat == max_passes).sum())} pixels at max_passes")
    assert len(classes) >= 3 and at_min >= 0.05 and bool((flat == max_passes).any())


@pytest.mark.parametrize("name", list(CASES))
def test_every_pixel_equals_the_fixed_count_frame_of_its_count(dragon, perlin, name):
    W, H, mx, mn, iv, thr = CASES[name]
    scene, mk, keep = make_case(name, dragon, perlin)
    r, f = mk(), mk()
    run, counts = adaptive_frame(scene, r, mx, mn, iv, thr)
    assert counts.shape == (H, W) and int(counts.min()) >= min(mn, mx) and int(counts.max()) <= mx
    assert float(r.buffers.accum.mean()) > 1e-3 and bool(torch.isfinite(r.buffers.accum).all())
    assert_spread(counts, mn, mx)
    assert_matches_fixed_frames(scene, r, f, counts, run)


@pytest.fixture(scope="module")
def small(dragon):
    scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
    cam = scene.frame_camera(320, 200)
    return scene, (lambda **kw: V.Renderer(scene, 320, 200, kp=make_kp(ray_depth=100, **kw), cam=cam))


def test_threshold_flt_max_stops_every_pixel_at_the_first_test(small):
    scene, mk = small
    r, f = mk(), mk()
    run, counts = adaptive_frame(scene, r, 32, 8, 4, FLT_MAX)
    assert run == 8 and bool((counts == 8).all())
    assert_matches_fixed_frames(scene, r, f, counts, run)


def test_threshold_zero_never_stops(small):
    scene, mk = small
    r, f = mk(), mk()
    run, counts = adaptive_frame(scene, r, 24, 8, 4, 0.0)
    assert run == 24 and bool((counts == 24).all())
    assert_matches_fixed_frames(scene, r, f, counts, run)


def test_budget_below_min_passes_is_a_fixed_count_frame(small):
    scene, mk = small
    r, f = mk(), mk()
    run, counts = adaptive_frame(scene, r, 5, 16, 16, FLT_MAX)
    assert run == 5 and bool((counts == 5).all())
    assert_matches_fixed_frames(scene, r, f, counts, run)


def test_max_interactions_caps_the_pass_count(small):
    scene, mk = small
    r, f = mk(max_interactions=12), mk(max_interactions=12)
    run, counts = adaptive_frame(scene, r, 40, 8, 8, 0.0)
    assert run == 12 and bool((counts == 12).all())
    assert_matches_fixed_frames(scene, r, f, counts, run)


def test_stopping_rule_against_the_numpy_restatement(dragon):
    """Pass by pass into a zeroed accumulator, pass k leaves sample_k / (k + 1): the per-pass samples, rebuilt in float64, go through
    adaptive_ref.  Counts must agree except next to a pixel whose simulated err at some test lies within 1e-3 (relative) of the
    threshold; the error map must agree to 1e-4 relative (plus 1e-6 absolute for pixels whose samples are nearly constant)."""
    W, H, P, mn, iv = 160, 100, 48, 8, 8
    scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
    r = V.Renderer(scene, W, H, kp=make_kp(ray_depth=100))
    scene.reset_blue_noise()
    samples = np.empty((P, H, W, 3), np.float64)
    for k in range(P):
        r.buffers.accum.zero_()
        r.render_pass(); torch.cuda.synchronize()
        samples[k] = r.buffers.accum.cpu().numpy().astype(np.float64).reshape(H, W, 3) * (k + 1)
    first = A.simulate(samples, mn, iv, FLT_MAX)["tests"][0]["err"]
    thr = float(np.quantile(A.max3x3(first), 0.4))                # a threshold that splits the frame
    sim = A.simulate(samples, mn, iv, thr)
    run, counts, err = adaptive_frame(scene, V.Renderer(scene, W, H, kp=make_kp(ray_depth=100), cam=r.cam), P, mn, iv, thr, error_map=True)
    counts = counts.cpu().numpy(); err = err.cpu().numpy()
    near = np.zeros((H, W), bool)
    for t in sim["tests"]:
        near |= np.abs(t["err"].astype(np.float64) - thr) <= 1e-3 * thr
    excluded = A.max3x3(near.astype(np.float32)) > 0
    print(f"threshold {thr:.4g}: {len(np.unique(sim['counts']))} count classes, {100 * excluded.mean():.2f} % of the pixels excluded, "
          f"{int(((counts != sim['counts']) & ~excluded).sum())} mismatches")
    assert excluded.mean() < 0.05
    assert len(np.unique(sim["counts"])) >= 3
    assert np.array_equal(counts[~excluded], sim["counts"][~excluded])
    assert run == sim["passes_run"]
    e_sim = sim["err"].astype(np.float64)[~excluded]; e_dev = err.astype(np.float64)[~excluded]
    assert np.isfinite(e_dev).all()
    assert (np.abs(e_dev - e_sim) <= 1e-4 * np.abs(e_sim) + 1e-6).all(), float(np.max(np.abs(e_dev - e_sim) / np.maximum(e_sim, 1e-12)))


def test_two_adaptive_frames_are_bitwise_identical(small):
    scene, mk = small
    a, b = mk(), mk()
    ra, ca, ea = adaptive_frame(scene, a, 48, 8, 8, 0.05, error_map=True); bn_a = scene.d_blue_noise.clone()
    rb, cb, eb = adaptive_frame(scene, b, 48, 8, 8, 0.05, error_map=True)
    assert ra == rb and torch.equal(ca, cb) and torch.equal(ea, eb) and torch.equal(bn_a, scene.d_blue_noise)
    for k in BUFFERS:
        assert torch.equal(getattr(a.buffers, k), getattr(b.buffers, k)), k
    assert len(torch.unique(ca)) >= 2


def test_refusals_say_why(small, dragon):
    scene, mk = small
    r = mk()
    r.kp.iteration = 3
    with pytest.raises(V.VptError, match="iteration must be 0"):
        r.render_adaptive(16)
    r.kp.iteration = 0
    with pytest.raises(V.VptError, match="render is 0"):
        mk(render=0).render_adaptive(16)
    with pytest.raises(V.VptError, match="min_passes must be >= 2"):
        r.render_adaptive(16, min_passes=1)
    with pytest.raises(V.VptError, match="check_interval must be >= 1"):
        r.render_adaptive(16, check_interval=0)
    with pytest.raises(V.VptError, match="max_interactions must be >= 2"):
        mk(max_interactions=1).render_adaptive(16)
    import ctypes as C
    opt = V._native.adaptive_options(16, 16, 0.01)
    rc = V.lib.vpt_render_adaptive(r.ctx, r.params.array, 16, C.byref(opt), None, None, None, None)
    assert rc == -1 and b"d_pass_count is required" in V.lib.vpt_last_error(r.ctx)
    part = V.Renderer(scene, 320, 200, kp=make_kp(ray_depth=2), cam=r.cam, rank=0, n_ranks=2, stripe_rows=8)
    with pytest.raises(V.VptError, match="partitioned"):
        part.render_adaptive(16)
    # an adaptive frame is final: continuing it is refused, a new frame on the same buffers is not
    adaptive_frame(scene, r, 16, 8, 8, 0.05)
    assert r.kp.iteration > 0
    with pytest.raises(V.VptError, match="finished adaptive frame"):
        r.render(1)
    r.kp.iteration = 0; scene.reset_blue_noise()
    r.render(2); r.render(2); torch.cuda.synchronize()          # iteration 0 clears the mark; the frame then continues as usual
    f = mk(); scene.reset_blue_noise(); f.render(4); torch.cuda.synchronize()
    assert torch.equal(r.buffers.accum, f.buffers.accum)


@pytest.mark.skipif(not oracle_ref.available(), reason="needs the live reference build (oracle/_ref)")
def test_full_count_pixels_of_the_headline_frame_against_the_reference_kernel(dragon, perlin):
    W, H, mx, mn, iv, thr = CASES["headline"]
    scene, mk, keep = make_case("headline", dragon, perlin)
    r = mk()
    run, counts = adaptive_frame(scene, r, mx, mn, iv, thr)
    ref = mk()
    orc = oracle_ref.RefOracle()
    ref.params.p_oct.value = orc.build_octree(scene.h_volumes, 1)
    scene.reset_blue_noise(); orc.render(ref, mx); torch.cuda.synchronize()
    full = counts.reshape(-1) == mx
    assert int(full.sum()) > 0
    assert flipped_fraction(r.buffers.accum[full].cpu().numpy(), ref.buffers.accum[full].cpu().numpy()) <= MAX_FLIPPED
