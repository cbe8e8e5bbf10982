"""The adaptive stopping rule on the GPU, bit for bit against the exact float32 mode of tests/adaptive_ref.py.

vpt_debug_adapt_rule runs vpt_render_adaptive's schedule of chunks and tests, its Welford arithmetic, tile lists and convergence-test
kernels on caller-given samples, so counts, the error map at every test and the final error map can be compared with the restatement
exactly, with no exclusion band, on random, constant, two-valued, huge, tiny, subnormal, negative, overflowing and non-finite samples,
over the option grid, odd frame shapes and render regions.  Frame-level tests then check what the synthetic ones cannot: that an
adaptive frame's counts, error map and beauty do not move when a layer is switched on (each layer selects other resolve
instantiations, and with compact records other trace kernels), and that a NaN error holds its 3x3 neighbourhood running on one
context, under a region and across the stripes of a sharded frame."""
import ctypes as C
import itertools
import zlib

import numpy as np
import pytest
import torch

import vpt_b200 as V
from vpt_b200.renderer import stripe_rows_of_rank
from vpt_b200.scene import synthetic_env
import adaptive_ref as A
from test_adaptive_gpu import BUFFERS, adaptive_frame, make_case, restart
from test_adaptive_sharded_gpu import Case, Shards, single_adaptive
from test_light_groups_gpu import make_group_case
from test_motion_vectors_gpu import moved, scale_of
from test_parity_gpu import make_kp

pytestmark = pytest.mark.gpu
F32 = np.float32
FLT_MAX = float(np.finfo(np.float32).max)
INF = float("inf")
SENTINEL_COUNT = 0x7EADBEEF
SENTINEL_ERR = -7.25


@pytest.fixture(scope="module")
def dragon():
    return V.Volume.load_vdb(V.find_asset("dragon.vdb"))


def u32(a):
    """float32 bits, every NaN as one pattern (the device and NumPy produce different NaN payloads; the rule does not read them)"""
    a = np.asarray(a, np.float32)
    return np.where(np.isnan(a), np.uint32(0x7FFFFFFF), a.view(np.uint32))


def device_rule(samples, mn, iv, thr, region=None):
    """-> dict(counts, err, tests (list of [H][W] err maps), passes_run) from vpt_debug_adapt_rule on samples (P, H, W, 3) float32"""
    P, H, W, _ = samples.shape
    d = torch.from_numpy(np.ascontiguousarray(samples, np.float32)).cuda()
    counts = torch.full((H, W), SENTINEL_COUNT, dtype=torch.int32, device="cuda")
    err = torch.full((H, W), SENTINEL_ERR, dtype=torch.float32, device="cuda")
    T = max(1, -(-(P - mn) // iv)) if mn < P else 1
    tests = torch.full((T, H, W), SENTINEL_ERR, dtype=torch.float32, device="cuda")
    opt = V._native.adaptive_options(mn, iv, thr)
    reg = (C.c_uint * 4)(*region) if region is not None else None
    run, nt = C.c_uint(0), C.c_uint(0)
    V._native.check(V.lib.vpt_debug_adapt_rule(d.data_ptr(), W, H, P, C.byref(opt), reg, counts.data_ptr(), err.data_ptr(),
                                               tests.data_ptr(), T, C.byref(run), C.byref(nt)), None, "vpt_debug_adapt_rule")
    assert nt.value <= T
    return dict(counts=counts.cpu().numpy(), err=err.cpu().numpy(), tests=list(tests[:nt.value].cpu().numpy()), passes_run=run.value)


def assert_rule_matches(samples, mn, iv, thr, region=None, what=""):
    """Device against the exact restatement of the region's pixels (the whole frame without one), bit for bit; pixels outside the
    region keep the caller's counts and error map and read NaN in the per-test maps (no state: a test that read one would hold its
    neighbours running)."""
    P, H, W, _ = samples.shape
    x0, y0, x1, y1 = region if region is not None else (0, 0, W, H)
    dev = device_rule(samples, mn, iv, thr, region)
    sim = A.simulate(samples[:, y0:y1, x0:x1], mn, iv, thr, exact=True)
    tag = f"{what} P={P} min_passes={mn} interval={iv} threshold={thr!r} region={region}"
    assert dev["passes_run"] == sim["passes_run"], tag
    assert len(dev["tests"]) == len(sim["tests"]), tag
    c = dev["counts"][y0:y1, x0:x1]
    assert np.array_equal(c, sim["counts"]), f"{tag}: {int((c != sim['counts']).sum())} counts differ"
    assert np.array_equal(u32(dev["err"][y0:y1, x0:x1]), u32(sim["err"])), f"{tag}: final error map"
    for k, (dt, st) in enumerate(zip(dev["tests"], sim["tests"])):
        assert np.array_equal(u32(dt[y0:y1, x0:x1]), u32(st["err"])), f"{tag}: error map at test {k} ({st['passes']} passes)"
    outside = np.ones((H, W), bool); outside[y0:y1, x0:x1] = False
    assert (dev["counts"][outside] == SENTINEL_COUNT).all() and (dev["err"][outside] == SENTINEL_ERR).all(), tag
    for dt in dev["tests"]:
        assert np.isnan(dt[outside]).all(), tag
    return sim


def make_samples(kind, P, H, W, seed):
    """(P, H, W, 3) float32 samples of one kind"""
    rng = np.random.default_rng(seed)
    shape = (P, H, W, 3)
    level = rng.uniform(0.2, 3.0, (1, H, W, 1))
    sigma = rng.choice([0.0, 0.01, 0.1, 0.4, 1.0], (1, H, W, 1))
    s = level * (1 + sigma * rng.standard_normal(shape))
    if kind == "random":
        pass
    elif kind == "constant_two":                                 # err 0, two-valued, and random pixels side by side
        sel = rng.integers(0, 3, (1, H, W, 1))
        two = np.where(rng.integers(0, 2, shape) == 1, level, level * 1.5)
        s = np.where(sel == 0, level + 0 * s, np.where(sel == 1, two, s))
    elif kind == "huge":                                         # luminance near 1.7e38: d d overflows, errors are +Inf or NaN
        s = 1.7e38 * (1 + rng.choice([0.0, 1e-7, 0.05], (1, H, W, 1)) * rng.standard_normal(shape))
        s = np.minimum(s, 3.4e38)
    elif kind == "tiny":                                         # normal, barely normal and subnormal samples (flushed to 0)
        s = s * rng.choice([1e-30, 2e-38, 1e-39, 1e-42], (1, H, W, 1))
    elif kind == "negative":                                     # negative and near-zero means take the 1e-3 floor
        s = -s * rng.choice([1.0, 1e-3, 1e-4], (1, H, W, 1))
    elif kind == "mixed_overflow":                               # opposite signs of large magnitude: Y - mean overflows
        s = rng.choice([-1.0, 1.0], shape) * rng.uniform(1e38, 3.4e38, shape)
        s = np.where(rng.integers(0, 4, (1, H, W, 1)) == 0, s, level * (1 + sigma * rng.standard_normal(shape)))
    elif kind == "nonfinite":                                    # NaN and +-Inf at chosen passes of some pixels
        for p in sorted({0, 1, min(2, P - 1), P // 2, P - 1}):
            m = rng.random((H, W)) < 0.04
            s[p][m] = rng.choice([np.nan, np.inf, -np.inf], (int(m.sum()), 3))
            c = rng.random((H, W)) < 0.02                        # one channel only
            s[p][c, rng.integers(0, 3)] = rng.choice([np.nan, np.inf, -np.inf])
    else:
        raise KeyError(kind)
    with np.errstate(over="ignore", invalid="ignore"):
        return s.astype(np.float32)


KINDS = ["random", "constant_two", "huge", "tiny", "negative", "mixed_overflow", "nonfinite"]
FRAMES = [(1, 1), (1, 37), (41, 1), (33, 31), (257, 3)]         # (W, H): one pixel, a column, a row, tile edges, a wide strip


def thresholds(samples, mn):
    """0, a quantile of the first test's 3x3 maxima that splits the frame, FLT_MAX and +Inf"""
    out = [0.0, FLT_MAX, INF]
    first = A.simulate(samples[:mn + 1], mn, 1, FLT_MAX, exact=True)["tests"]
    if first:
        m = A.max3x3(first[0]["err"])
        q = float(F32(np.quantile(np.where(np.isfinite(m), m, FLT_MAX), 0.45)))
        if 0 < q < FLT_MAX: out.insert(1, q)
    return out


@pytest.mark.parametrize("W,H", FRAMES)
@pytest.mark.parametrize("kind", KINDS)
def test_rule_against_the_exact_restatement(kind, W, H):
    samples = make_samples(kind, 64, H, W, seed=zlib.crc32(f"{kind} {W} {H}".encode()))
    spread = set()
    for mn, iv, P in itertools.product((2, 3, 16), (1, 5, 16), (2, 17, 64)):
        for thr in thresholds(samples[:P], mn):
            sim = assert_rule_matches(samples[:P], mn, iv, thr, what=f"{kind} {W}x{H}")
            spread |= set(np.unique(sim["counts"]).tolist())
    print(f"{kind} {W}x{H}: pass counts seen {sorted(spread)}")
    if W * H > 1 and kind in ("random", "constant_two", "nonfinite"):
        assert len(spread) >= 4


REGIONS = [(0, 0, 1, 1), (32, 30, 33, 31), (17, 9, 18, 10), (0, 0, 33, 4), (29, 0, 33, 31), (0, 27, 33, 31), (0, 5, 1, 20),
           (3, 5, 20, 17), (31, 3, 33, 9)]


@pytest.mark.parametrize("region", REGIONS)
@pytest.mark.parametrize("kind", ["random", "nonfinite", "constant_two"])
def test_rule_under_a_region(kind, region):
    samples = make_samples(kind, 64, 31, 33, seed=17)
    x0, y0, x1, y1 = region
    for mn, iv, P in [(2, 1, 17), (3, 5, 64), (16, 16, 64), (3, 1, 2)]:
        for thr in thresholds(samples[:P, y0:y1, x0:x1], mn):
            assert_rule_matches(samples[:P], mn, iv, thr, region=region, what=kind)


@pytest.mark.parametrize("k", [-5, -2, 3, 40])
def test_scale_invariance_on_the_device(k):
    """Samples times 2^k: identical counts and err bits at every test while means stay above the floor and M2 finite."""
    H, W, P, mn, iv = 31, 33, 40, 4, 3
    s = np.abs(make_samples("random", P, H, W, 29)) + F32(0.05)
    Y = A.luminance_exact(s).astype(np.float64) * 2.0 ** k            # the claim's conditions on the scaled samples
    assert (np.cumsum(Y, axis=0) / np.arange(1, P + 1)[:, None, None])[mn - 1:].min() > 2e-3 and (Y ** 2).sum(axis=0).max() < 1e37
    base = device_rule(s, mn, iv, FLT_MAX)
    thr = float(F32(np.quantile(A.max3x3(base["tests"][0]), 0.5)))
    ref = device_rule(s, mn, iv, thr)
    assert len(np.unique(ref["counts"])) >= 3
    got = device_rule((s * F32(2.0 ** k)).astype(np.float32), mn, iv, thr)
    assert np.array_equal(got["counts"], ref["counts"]) and got["passes_run"] == ref["passes_run"]
    assert np.array_equal(u32(got["err"]), u32(ref["err"]))
    for a, b in zip(got["tests"], ref["tests"]):
        assert np.array_equal(u32(a), u32(b))


def test_past_overflow_a_scaled_pixel_never_stops_earlier():
    H, W, P, mn, iv = 31, 33, 40, 4, 3
    s = np.abs(make_samples("random", P, H, W, 29)) + F32(0.05)
    base = device_rule(s, mn, iv, FLT_MAX)
    thr = float(F32(np.quantile(A.max3x3(base["tests"][0]), 0.5)))
    ref = device_rule(s, mn, iv, thr)
    for k in (100, 120, 126):
        with np.errstate(over="ignore"):
            big = (s * F32(2.0 ** k)).astype(np.float32)
        got = device_rule(big, mn, iv, thr)
        assert (got["counts"] >= ref["counts"]).all(), k
        e0, r0 = got["tests"][0], ref["tests"][0]
        assert ((u32(e0) == u32(r0)) | np.isinf(e0) | np.isnan(e0)).all(), k
        if k == 126:
            assert (np.isinf(e0) | np.isnan(e0)).mean() > 0.5 and (got["counts"] == P).mean() > 0.5


def nan_counts_want(H, W, nan_px, P, mn, region=None):
    x0, y0, x1, y1 = region if region is not None else (0, 0, W, H)
    want = np.full((H, W), mn); m = np.zeros((H, W), bool)
    for (y, x) in nan_px: m[max(y - 1, 0):y + 2, max(x - 1, 0):x + 2] = True
    want[m] = P
    out = np.full((H, W), SENTINEL_COUNT); out[y0:y1, x0:x1] = want[y0:y1, x0:x1]
    return out


def test_nan_error_holds_its_neighbourhood_synthetic():
    """Constant samples (err 0) and a NaN at the first pass of a few pixels: those pixels and their 8 neighbours take every pass,
    every other pixel stops at the first test, on the whole frame and under a region whose corner is a NaN pixel."""
    H, W, P, mn, iv = 12, 20, 17, 2, 3
    s = np.ones((P, H, W, 3), np.float32)
    nan_px = [(0, 0), (5, 7), (11, 19), (3, 12)]
    for y, x in nan_px: s[0, y, x, 1] = np.nan
    for thr in (0.5, FLT_MAX, INF):
        dev = device_rule(s, mn, iv, thr)
        assert np.array_equal(dev["counts"], nan_counts_want(H, W, nan_px, P, mn)), thr
        assert all(np.isnan(dev["err"][y, x]) for y, x in nan_px)
        reg = (12, 3, 18, 9)                                     # (3, 12) is its top-left corner
        dev = device_rule(s, mn, iv, thr, region=reg)
        assert np.array_equal(dev["counts"], nan_counts_want(H, W, nan_px, P, mn, reg)), thr


# ---- real frames ---------------------------------------------------------------------------------------------------------------
def nan_sky(kp):
    kp.sky_color = V.f3(float("nan"), float("nan"), float("nan"))  # every sample is non-finite: the guard feeds it the prefill
    return kp


def prefill_constant(r, nan_lps):
    """accum 0.5 everywhere (every sample then equals it: err 0), NaN at the local pixels nan_lps"""
    r.buffers.zero_(); r.buffers.accum.fill_(0.5)
    for lp in nan_lps: r.buffers.accum[lp, 1] = float("nan")


def test_nan_error_holds_its_neighbourhood_in_a_frame(dragon):
    """A NaN sky colour makes every sample the prefilled accum: constant pixels (err 0) and, where the prefill is NaN, a NaN err.
    One context, then the same frame under a render region."""
    W, H, P, mn, iv = 96, 64, 12, 4, 4
    scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
    cam = scene.frame_camera(W, H)
    nan_px = [(0, 0), (20, 33), (63, 95), (40, 10)]
    for region in (None, (10, 18, 60, 50)):
        r = V.Renderer(scene, W, H, kp=nan_sky(make_kp(ray_depth=2)), cam=cam)
        if region is not None: r.set_region(*region)
        scene.reset_blue_noise(); r.kp.iteration = 0
        prefill_constant(r, [y * W + x for y, x in nan_px])
        run, counts, err = r.render_adaptive(P, threshold=0.5, min_passes=mn, check_interval=iv, error_map=True)
        torch.cuda.synchronize()
        counts = counts.cpu().numpy(); err = err.cpu().numpy()
        want = nan_counts_want(H, W, nan_px, P, mn, region)
        inside = want != SENTINEL_COUNT
        assert np.array_equal(counts[inside], want[inside]), region
        assert run == P
        r.close()


def test_nan_error_on_a_stripe_boundary_holds_the_other_ranks_pixels(dragon):
    """Three shards on one GPU, stripes of 6 rows: the NaN pixel on global row 6 (rank 1's first row) keeps rank 0's pixels of row 5
    running through the halo; the sharded frame equals the single-context one."""
    class NanCase(Case):
        def kp(self):
            return nan_sky(super().kp())
    P, mn, iv, R, sr = 12, 4, 4, 3, 6
    case = NanCase(dragon)
    w, h = case.w, case.h
    nan_px = [(6, 40), (17, 200), (23, 0)]                        # rows 6 (first of stripe 1), 17 (last of stripe 2), 23 (last of stripe 3)
    scene, ref = case.single()
    scene.reset_blue_noise(); ref.kp.iteration = 0
    prefill_constant(ref, [y * w + x for y, x in nan_px])
    ref_out = single_adaptive(scene, ref, P, mn, iv, 0.5)
    want = nan_counts_want(h, w, nan_px, P, mn)
    assert np.array_equal(ref_out[1].cpu().numpy(), want)
    sh = Shards(case, R, sr)
    try:
        sh.reset_blue_noise()
        for k, r in enumerate(sh.rs):
            rows = stripe_rows_of_rank(h, k, R, sr)
            mine = [lr * w + x for lr, g in enumerate(rows) for (y, x) in nan_px if g == y]
            prefill_constant(r, mine)
        out = sh.adaptive(P, mn, iv, 0.5)
        for k, (run_k, counts_k, err_k) in enumerate(out):
            rows = np.asarray(stripe_rows_of_rank(h, k, R, sr)); valid = rows < h
            assert run_k == ref_out[0]
            assert np.array_equal(counts_k.cpu().numpy()[valid], want[rows[valid]]), f"pass counts of shard {k}"
            assert np.array_equal(u32(err_k.cpu().numpy()[valid]), u32(ref_out[2].cpu().numpy()[rows[valid]])), f"errors of shard {k}"
    finally:
        sh.close()


# layer -> enable(renderer, scene)
LAYERS = {
    "aovs": lambda r, s: r.enable_aovs(),
    "light_groups": lambda r, s: r.enable_light_groups(),
    "deep": lambda r, s: r.enable_deep([0.0, 30.0, INF]),
    "mattes": lambda r, s: r.enable_mattes([[0]], sphere=0),
    "collision_aovs": lambda r, s: r.enable_collision_aovs(),
    "motion_vectors": lambda r, s: r.enable_motion_vectors(moved(r.cam, scale_of(s))),
    "cryptomatte": lambda r, s: r.enable_cryptomatte(3),
}


def layer_case(name, dragon):
    """-> (scene, make_renderer) of one frame kind"""
    if name in ("headline", "headline_no_cull", "lights_sphere", "vol_sky_table"):
        scene, mk, _ = make_case(name.replace("_no_cull", ""), dragon, None)
        if name == "headline_no_cull":
            def mk_nc(mk=mk):
                r = mk(); r.set_option("miss_cull", 0); return r
            return scene, mk_nc
        return scene, mk
    if name == "sky":
        info = make_group_case("sky", dragon, None, None)
        layer_case.keep.append(info["keep"])
        return info["scene"], info["mk0"]
    scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
    W, H = 256, 144
    cam = scene.frame_camera(W, H)
    def mk():
        r = V.Renderer(scene, W, H, kp=make_kp(ray_depth=3), cam=cam)
        if name == "equirect": r.set_projection("equirect", hfov=300.0, vfov=150.0)
        elif name == "ods": r.set_projection("ods")
        elif name == "camera_motion": r.set_camera_motion(moved(cam, scale_of(scene)))
        else: raise KeyError(name)
        return r
    return scene, mk


layer_case.keep = []
LAYER_CASES = ["headline", "headline_no_cull", "lights_sphere", "sky", "vol_sky_table", "equirect", "ods", "camera_motion"]


@pytest.mark.parametrize("name", LAYER_CASES)
def test_layers_do_not_move_the_counts_or_the_error_map(dragon, name):
    scene, mk = layer_case(name, dragon)
    P, mn, iv = 32, 8, 4
    base = mk()
    _, _, first = adaptive_frame(scene, base, P, mn, mn, FLT_MAX, error_map=True)
    thr = float(F32(np.quantile(A.max3x3(first.cpu().numpy()), 0.4)))
    run, counts, err = adaptive_frame(scene, base, P, mn, iv, thr, error_map=True)
    classes = torch.unique(counts).tolist()
    print(f"{name}: threshold {thr:.4g}, count classes {classes}")
    assert len(classes) >= 3
    bufs = {k: getattr(base.buffers, k).clone() for k in BUFFERS}
    base.close()
    for layer, enable in LAYERS.items():
        if layer in ("collision_aovs", "motion_vectors") and name in ("equirect", "ods"):
            continue                                             # refused with a panorama (include/vpt_b200.h)
        r = mk()
        enable(r, scene)
        run_l, counts_l, err_l = adaptive_frame(scene, r, P, mn, iv, thr, error_map=True)
        assert run_l == run, f"{name} + {layer}: passes_run"
        assert torch.equal(counts_l, counts), f"{name} + {layer}: {int((counts_l != counts).sum())} pass counts differ"
        assert torch.equal(err_l.view(torch.int32), err.view(torch.int32)), f"{name} + {layer}: error map"
        for k in BUFFERS:
            a, b = getattr(r.buffers, k), bufs[k]
            assert torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a, b.view(torch.int32) if b.dtype == torch.float32 else b), \
                f"{name} + {layer}: {k}"
        r.close()


def test_prefilled_non_finite_accum_runs_its_neighbourhood_to_the_end(dragon):
    """The striped environment's NaN / +Inf samples at iteration 0 take the prefilled accum: where that is NaN or +Inf the pixel's
    err is NaN, so it and its neighbours take every pass; every pixel still equals the fixed-count frame of its count."""
    W, H = 256, 160
    P, mn, iv, thr = 32, 8, 8, 0.1
    scene, mk, _ = make_case("nan_prefilled", dragon, None)
    probe = mk()
    restart(scene, probe)
    probe.buffers.accum.fill_(float("nan"))
    probe.render(1); torch.cuda.synchronize()
    first_bad = ~torch.isfinite(probe.buffers.accum).all(dim=1)          # pixels whose first sample is non-finite
    rng = np.random.default_rng(4)
    cand = torch.nonzero(first_bad).flatten().cpu().numpy()
    assert len(cand) > 100
    chosen = rng.choice(cand, 40, replace=False)
    probe.close()

    def with_non_finite(r):
        base = r.prefill
        def fill():
            base()
            for i, lp in enumerate(chosen): r.buffers.accum[int(lp)] = float("nan") if i % 2 == 0 else float("inf")
        r.prefill = fill
        return r
    r, f = with_non_finite(mk()), with_non_finite(mk())
    run, counts = adaptive_frame(scene, r, P, mn, iv, thr)
    m = np.zeros((H, W), bool)
    for lp in chosen:
        y, x = divmod(int(lp), W); m[max(y - 1, 0):y + 2, max(x - 1, 0):x + 2] = True
    c = counts.cpu().numpy()
    assert (c[m] == P).all(), f"{int((c[m] != P).sum())} pixels next to a non-finite accum stopped early"
    assert (c[~m] < P).any()
    # every count class against a fixed-count frame, bitwise (NaN accumulators included)
    bufs = {k: getattr(r.buffers, k).clone() for k in BUFFERS}
    flat = counts.reshape(-1)
    for cls in torch.unique(flat).tolist():
        restart(scene, f); f.render(cls); torch.cuda.synchronize()
        sel = flat == cls
        for k in BUFFERS:
            a, b = bufs[k][sel], getattr(f.buffers, k)[sel]
            if a.dtype == torch.float32: a, b = a.view(torch.int32), b.view(torch.int32)
            assert torch.equal(a, b), f"{k} differs on the {int(sel.sum())} pixels of {cls} passes"


def test_subnormal_threshold_is_refused(dragon):
    scene = V.Scene([dragon.instance()], env=synthetic_env(512, 256))
    r = V.Renderer(scene, 64, 32, kp=make_kp(ray_depth=2))
    for thr in (1e-45, 1e-39, float(np.nextafter(F32(np.finfo(np.float32).tiny), F32(0)))):
        with pytest.raises(V.VptError, match="subnormal"):
            r.render_adaptive(8, threshold=thr, min_passes=2, check_interval=2)
    r.render_adaptive(8, threshold=float(np.finfo(np.float32).tiny), min_passes=2, check_interval=2)
    torch.cuda.synchronize()
    s = np.ones((4, 2, 2, 3), np.float32)
    with pytest.raises(V.VptError, match="refused"):
        device_rule(s, 2, 1, 1e-40)
