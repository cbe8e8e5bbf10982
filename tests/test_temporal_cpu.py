"""Temporal accumulation without a GPU: the restatement of vpt_temporal (tests/temporal_ref.py) against closed forms -- the environment's
motion under a pan and a translation, zero motion, integer shifts, the frame edge, the clip and the history cap -- the still-camera
guarantee in accum's float32 arithmetic, and the refusals that need no device."""
import ctypes as C

import numpy as np
import pytest

import vpt_b200 as V
from vpt_b200 import _native as N
import denoise_ref as D
import temporal_ref as T
import temporal_layers_ref as TL

W, H = 641, 361                                   # odd: pixel (320, 180)'s centre is the image centre


def camera(origin, yaw=0.0, vfov_deg=40.0, w=W, h=H):
    """A pinhole camera in the reference's construction (focus distance 1): forward -w, right u, up v, turned by `yaw` about +y."""
    c, s = np.cos(yaw), np.sin(yaw)
    u = np.array([c, 0.0, -s]); v = np.array([0.0, 1.0, 0.0]); ww = np.array([s, 0.0, c])
    half_h = np.tan(np.radians(vfov_deg) / 2); half_w = w / h * half_h
    o = np.asarray(origin, np.float64)
    return {"origin": o, "lower_left_corner": o - half_w * u - half_h * v - ww, "horizontal": 2 * half_w * u, "vertical": 2 * half_h * v,
            "f": w / (2 * half_w)}


def uncovered(n, z=0.0):
    return np.tile(np.array([0.0, 0.0, z], np.float32), (n, 1))


def test_a_pan_by_theta_moves_the_image_centre_environment_by_f_tan_theta():
    a = camera((0, 0, 0))
    centre = 180 * W + 320
    for theta in (0.01, 0.1, -0.3):
        v, ok = T.pixel_motion(W, H, uncovered(W * H), a, camera((0, 0, 0), yaw=theta))
        assert ok[centre]
        assert abs(abs(v[centre, 0]) - a["f"] * abs(np.tan(theta))) < 1e-4 * a["f"] and abs(v[centre, 1]) < 1e-3, theta
        assert np.sign(v[centre, 0]) == np.sign(theta)


def test_a_pure_translation_leaves_the_environment_where_it_is():
    a = camera((0, 0, 0))
    for delta in ((0.5, 0, 0), (0, -2.0, 0), (1.0, 1.0, 3.0)):
        v, ok = T.pixel_motion(W, H, uncovered(W * H), a, camera(delta))
        assert ok.all() and np.abs(v).max() < 1e-3, delta


def test_the_same_camera_gives_plus_zero():
    a = camera((0.3, -0.2, 5.0), yaw=0.4)
    rng = np.random.default_rng(1)
    m = np.zeros((W * H, 3), np.float32)
    m[:, 2] = rng.choice([0.0, 0.25, 0.5, 1.0], W * H).astype(np.float32)
    v, ok = T.pixel_motion(W, H, m, a, a, dt=np.float32)
    assert ok.all() and (v == 0).all() and not np.signbit(v).any()


def _frame(rng, w, h):
    return rng.uniform(0.0, 2.0, (w * h, 3)).astype(np.float32)


def test_an_integer_pixel_shift_reads_the_shifted_history_bit_for_bit():
    w, h = 37, 23
    rng = np.random.default_rng(2)
    hist, c, cam = _frame(rng, w, h), _frame(rng, w, h), camera((0, 0, 0), w=w, h=h)
    for k, m in ((3, -2), (-5, 4), (0, 0), (1, 0)):
        vec = np.tile(np.array([k, m, 1.0], np.float32), (w * h, 1))
        r = T.temporal(w, h, c, vec, cam, cam, hist, np.full(w * h, 4, np.float32), dt=np.float32)
        y, x = np.divmod(np.arange(w * h), w)
        inside = (x + k >= 0) & (x + k < w) & (y + m >= 0) & (y + m < h)
        assert np.array_equal(r["used"], inside)
        src = ((y + m) * w + x + k)[inside]
        assert np.array_equal(r["h"][inside], hist[src]), (k, m)
        assert (r["L"][inside] == 5).all() and (r["L"][~inside] == 1).all()
        assert np.array_equal(r["out"][~inside], c[~inside])


def test_a_fractional_shift_is_the_bilinear_mean_of_the_four_taps():
    w, h = 9, 7
    rng = np.random.default_rng(3)
    hist, c, cam = _frame(rng, w, h), _frame(rng, w, h), camera((0, 0, 0), w=w, h=h)
    vec = np.tile(np.array([0.25, 0.5, 1.0], np.float32), (w * h, 1))
    r = T.temporal(w, h, c, vec, cam, cam, hist, np.ones(w * h, np.float32))
    hh = hist.reshape(h, w, 3).astype(np.float64)
    want = 0.375 * hh[3, 4] + 0.125 * hh[3, 5] + 0.375 * hh[4, 4] + 0.125 * hh[4, 5]
    assert np.allclose(r["h"][3 * w + 4], want, rtol=1e-12)
    # the last column's right taps lie outside the frame: the left ones alone, renormalised
    assert np.allclose(r["h"][3 * w + 8], 0.5 * hh[3, 8] + 0.5 * hh[4, 8], rtol=1e-12)


def test_q_off_the_frame_or_behind_b_gives_no_history():
    w, h = 16, 8
    rng = np.random.default_rng(4)
    hist, c, cam = _frame(rng, w, h), _frame(rng, w, h), camera((0, 0, 0), w=w, h=h)
    vec = np.tile(np.array([-0.6, 0.0, 1.0], np.float32), (w * h, 1))   # q.x = x - 0.1 < 0 in column 0 only
    r = T.temporal(w, h, c, vec, cam, cam, hist, np.ones(w * h, np.float32))
    col0 = np.arange(w * h) % w == 0
    assert not r["used"][col0].any() and r["used"][~col0].all()
    assert np.array_equal(r["out"][col0], c[col0].astype(np.float64)) and (r["L"][col0] == 1).all()
    back = camera((0, 0, 0), yaw=np.pi, w=w, h=h)                       # every environment direction of A lies behind B: k <= 0
    for z, used in ((0.0, False), (0.5, False), (1.0, True)):
        r = T.temporal(w, h, c, uncovered(w * h, z), cam, back, hist, np.ones(w * h, np.float32))
        assert (r["used"] == used).all(), z
    vec = np.tile(np.array([np.nan, 0.0, 1.0], np.float32), (w * h, 1))
    assert not T.temporal(w, h, c, vec, cam, cam, hist, np.ones(w * h, np.float32))["used"].any()


def test_the_clip_bounds_the_history_to_mu_plus_minus_gamma_sigma():
    w, h = 3, 3
    c = np.zeros((9, 3), np.float32)
    c[:, 0] = [0, 1, 2, 3, 4, 5, 6, 7, 8]
    c[:, 1] = 1.0
    mu, sigma = 4.0, np.sqrt(np.mean((np.arange(9) - 4.0) ** 2))
    cam = camera((0, 0, 0), w=w, h=h)
    hist = np.tile(np.array([100.0, 5.0, -0.5], np.float32), (9, 1))
    for gamma in (0.5, 1.0, 2.0):                                       # the window statistics in float64
        r = T.temporal(w, h, c, uncovered(9, 1.0), cam, cam, hist, np.ones(9, np.float32), clip_sigma=gamma, clip32=False)
        assert np.allclose(r["hc"][4], [mu + gamma * sigma, 1.0, 0.0], rtol=1e-12, atol=0)
    r = T.temporal(w, h, c, uncovered(9, 1.0), cam, cam, hist, np.ones(9, np.float32))
    assert np.array_equal(r["hc"][4], hist[4].astype(np.float64))       # clip_sigma = inf: no clip
    c[0] = np.inf                                                       # a non-finite neighbour drops out of the window
    r = T.temporal(w, h, c, uncovered(9, 1.0), cam, cam, hist, np.ones(9, np.float32), clip_sigma=1.0, clip32=False)
    m8 = np.arange(1, 9, dtype=np.float64)
    assert np.isclose(r["hc"][4, 0], m8.mean() + m8.std())


def test_the_history_length_saturates_at_max_history():
    w, h = 5, 4
    rng = np.random.default_rng(6)
    hist, c, cam = _frame(rng, w, h), _frame(rng, w, h), camera((0, 0, 0), w=w, h=h)
    lens = np.array([1, 2, 7, 8, 9, 100, 3, 8] * 2 + [1] * 4, np.float32)
    r = T.temporal(w, h, c, uncovered(w * h, 1.0), cam, cam, hist, lens, max_history=8)
    assert np.array_equal(r["L"], np.minimum(lens + 1, 8))
    r = T.temporal(w, h, c, uncovered(w * h, 1.0), cam, cam, hist, lens, max_history=1)
    assert (r["L"] == 1).all()


def test_a_still_camera_blend_is_accums_running_mean_bit_for_bit():
    w, h, F = 12, 9, 8
    rng = np.random.default_rng(7)
    cam = camera((0.1, 0.2, 3.0), yaw=0.2, w=w, h=h)
    m = np.zeros((w * h, 3), np.float32)
    m[:, 2] = rng.choice([0.0, 0.5, 1.0], w * h).astype(np.float32)
    frames = [rng.uniform(0.0, 3.0, (w * h, 3)).astype(np.float32) for _ in range(F)]
    acc = frames[0].copy()
    r = T.temporal(w, h, frames[0], m, cam, cam, dt=np.float32)
    out, L = r["out"], r["L"]
    for f in range(1, F):
        acc = T.accum_step(acc, frames[f], f + 1)
        r = T.temporal(w, h, frames[f], m, cam, cam, out, L, max_history=F, dt=np.float32)
        out, L = r["out"], r["L"]
        assert r["used"].all() and np.array_equal(out, acc) and (L == f + 1).all(), f


def test_refusals_that_need_no_device():
    cam = N.camera()
    assert V.lib.vpt_set_sample_offset(None, 3) == -1
    assert b"null context" in V.lib.vpt_last_error(None)
    assert V.lib.vpt_temporal(None, 4, 4, None, None, C.byref(cam), C.byref(cam), None, None, None, 1.0, None, None, None, None) == -1
    assert b"null context" in V.lib.vpt_last_error(None)
    assert N.temporal_defaults()[0] >= 1 and N.temporal_defaults()[1] > 0
    r = V.Renderer.__new__(V.Renderer)
    with pytest.raises(V.VptError, match="not enabled"):
        r.render_temporal(cam, 1)


# ---- the vectorised restatement, its float32 decisions and the pass rule ---------------------------------------------------------------
def hostile(w, h, seed):
    """Colours, vectors, histories and lengths with every rule of the filter in play: fractional, integer and far motions, NaN / +-inf
    colours and histories, negative and denormal values, and lengths that are NaN, +-inf, 0, negative, fractional or huge."""
    rng = np.random.default_rng(seed)
    n = w * h
    c = rng.uniform(-1.0, 2.0, (n, 3)).astype(np.float32)
    hist = rng.uniform(-1.0, 2.0, (n, 3)).astype(np.float32)
    ln = rng.choice(np.array([1, 2, 5, 11, np.nan, np.inf, -np.inf, 0, -1, -0.5, 2.5, 2 ** 24, 2 ** 25], np.float32), n)
    m = np.zeros((n, 3), np.float32)
    m[:, 2] = rng.choice([0.0, 0.5, 1.0, np.nan], n)
    m[:, :2] = np.where(rng.random((n, 1)) < 0.5, rng.uniform(-3, 3, (n, 2)), rng.integers(-3, 4, (n, 2)))
    m[rng.random(n) < 0.05, :2] = 1e30
    c[rng.random(n) < 0.05, rng.integers(0, 3)] = np.nan
    c[rng.random(n) < 0.03, 1] = -np.inf
    hist[rng.random(n) < 0.05, 2] = np.inf
    c[rng.random(n) < 0.03] = 1e-40
    return c, m, hist, ln


@pytest.mark.parametrize("wh", [(1, 1), (2, 1), (1, 2), (9, 7), (23, 17)])
def test_the_vectorised_restatement_equals_the_loop(wh):
    w, h = wh
    a = camera((0.0, 0.0, 0.0), w=w, h=h)
    b = camera((0.05, 0.01, 0.02), yaw=0.03, w=w, h=h)
    c, m, hist, ln = hostile(w, h, w * 31 + h)
    for mh, clip, fdt in ((16, np.inf, None), (3, 1.5, np.float32), (1 << 24, 0.25, None), (1, 64.0, np.float32)):
        want = T.temporal_loop(w, h, c, m, a, b, hist, ln, max_history=mh, clip_sigma=clip, footprint_dt=fdt)
        got = T.temporal(w, h, c, m, a, b, hist, ln, max_history=mh, clip_sigma=clip, footprint_dt=fdt, diff32=False, clip32=False,
                         ftz=False)
        for k in ("used", "L", "h", "hc", "out"):
            assert np.array_equal(got[k], want[k], equal_nan=True), (wh, mh, clip, k)


def edge_vectors(w, h, motions):
    """Vectors with M.z = 1 and the motion v of the given pixels: motions = {(x, y): (vx, vy)}"""
    m = np.zeros((w * h, 3), np.float32)
    m[:, 2] = 1.0
    for (x, y), v in motions.items():
        m[y * w + x, :2] = v
    return m


def test_the_float32_footprint_at_the_frame_edge():
    w, h = 6, 4
    f32 = np.float32
    up, down = lambda v: np.nextafter(f32(v), f32(np.inf)), lambda v: np.nextafter(f32(v), f32(-np.inf))
    mv = {(0, 0): (-0.5, 0), (5, 0): (0.5, 0), (1, 0): (0, -0.5), (1, 3): (0, 0.5),                  # q on 0, W, 0 and H
          (0, 1): (down(-0.5), 0), (5, 1): (up(6) - f32(5.5), 0), (2, 0): (0, down(-0.5)), (3, 3): (0, up(4) - f32(3.5)),   # a step out
          (0, 2): (up(-0.5), 0), (5, 2): (down(6) - f32(5.5), 0), (2, 3): (0, down(4) - f32(3.5)),   # a step in
          (4, 1): (1, -1)}                                                                              # integer px
    m = edge_vectors(w, h, mv)
    q = lambda x, y: (f32(x + 0.5) + m[y * w + x, 0], f32(y + 0.5) + m[y * w + x, 1])
    assert q(0, 1)[0] == -f32(2.0 ** -24) and q(5, 1)[0] == up(6) and q(2, 0)[1] == -f32(2.0 ** -24) and q(3, 3)[1] == up(4)
    assert q(0, 2)[0] == f32(2.0 ** -25) and q(5, 2)[0] == down(6) and q(2, 3)[1] == down(4)
    inside, x0, y0, fx, fy = T.footprint(w, h, m[:, :2], np.float32)
    at = lambda x, y: y * w + x
    # q = 0: px = -1/2 floors to -1 (truncation would give 0), fx = 1/2; q = W: x0 = W - 1; the same along y
    assert inside[at(0, 0)] and (x0[at(0, 0)], fx[at(0, 0)], y0[at(0, 0)], fy[at(0, 0)]) == (-1, 0.5, 0, 0)
    assert inside[at(5, 0)] and (x0[at(5, 0)], fx[at(5, 0)]) == (5, 0.5)
    assert inside[at(1, 0)] and (y0[at(1, 0)], fy[at(1, 0)]) == (-1, 0.5) and inside[at(1, 3)] and (y0[at(1, 3)], fy[at(1, 3)]) == (3, 0.5)
    # one float32 step outside 0, W and H: no history; one step inside: px rounds in float32
    assert not inside[[at(0, 1), at(5, 1), at(2, 0), at(3, 3)]].any()
    assert inside[at(0, 2)] and x0[at(0, 2)] == -1 and fx[at(0, 2)] == 0.5          # px = 2^-25 - 1/2 rounds to -1/2 + 2^-25, fx ties to 1/2
    assert inside[at(5, 2)] and x0[at(5, 2)] == 5 and fx[at(5, 2)] == down(6) - f32(6) + f32(0.5)
    assert inside[at(2, 3)] and y0[at(2, 3)] == 3 and fy[at(2, 3)] == f32(0.5) - f32(2.0 ** -22)
    assert inside[at(4, 1)] and (x0[at(4, 1)], y0[at(4, 1)], fx[at(4, 1)], fy[at(4, 1)]) == (5, 0, 0, 0)
    c = np.ones((w * h, 3), np.float32)
    hist = np.arange(3 * w * h, dtype=np.float32).reshape(-1, 3)
    bt = T.beauty_taps(w, h, c, m, None, None, hist, np.ones(w * h, np.float32), footprint_dt=np.float32)
    # q = 0 keeps (0, 0) alone, renormalised; q = W keeps (W - 1, 0) alone; an integer px reads its texel with weight 1, the three
    # weight-0 taps dropped
    assert list(bt["taps"][at(0, 0)]) == [-1, 0, -1, -1] and bt["sw"][at(0, 0)] == 0.5 and np.array_equal(bt["h"][at(0, 0)], hist[0])
    assert list(bt["taps"][at(5, 0)]) == [at(5, 0), -1, -1, -1] and np.array_equal(bt["h"][at(5, 0)], hist[at(5, 0)])
    assert list(bt["taps"][at(1, 3)]) == [at(1, 3), -1, -1, -1] and bt["sw"][at(1, 3)] == 0.5
    assert list(bt["taps"][at(4, 1)]) == [at(5, 0), -1, -1, -1] and np.array_equal(bt["h"][at(4, 1)], hist[at(5, 0)])
    assert not bt["used"][[at(0, 1), at(5, 1), at(2, 0), at(3, 3)]].any()
    assert bt["used"][[at(0, 2), at(5, 2), at(2, 3)]].all()


def test_float32_rounding_decides_q_on_the_frame_edge():
    """x + 1/2 + v rounds onto W in float32 where its float64 value lies just past it: the device keeps the pixel's history"""
    w, h = 1000, 1
    m = np.zeros((w, 3), np.float32)
    m[:, 2] = 1.0
    m[w - 1, 0] = np.nextafter(np.float32(0.5), np.float32(1))
    c, hist = np.ones((w, 3), np.float32), np.full((w, 3), 2.0, np.float32)
    args = (w, h, c, m, None, None, hist, np.ones(w, np.float32))
    assert T.beauty_taps(*args, footprint_dt=np.float32)["used"][w - 1]
    assert not T.beauty_taps(*args)["used"][w - 1]
    assert T.temporal(*args, footprint_dt=np.float32)["L"][w - 1] == 2


def test_a_nan_length_is_ignored_by_the_min():
    w, h = 4, 1
    m = np.tile(np.array([0.5, 0.0, 1.0], np.float32), (4, 1))           # taps (x, 0) and (x + 1, 0), each of weight 1/2
    c, hist = np.ones((4, 3), np.float32), np.full((4, 3), 3.0, np.float32)
    nan = np.nan
    for lens, mh, want in (([nan, 2, 2, 2], 16, [3, 3, 3, 3]), ([2, nan, 2, 2], 16, [3, 3, 3, 3]), ([nan, nan, 5, nan], 16, [16, 6, 6, 16]),
                           ([nan] * 4, 7, [7] * 4), ([np.inf, 1, -np.inf, 0], 8, [2, -np.inf, -np.inf, 1]),
                           ([-1, -0.5, 2.5, 2 ** 25], 1 << 24, [0, 0.5, 3.5, 1 << 24]), ([2 ** 24, 2 ** 24, 2 ** 24, nan], 1 << 24, [1 << 24] * 4)):
        ln = np.array(lens, np.float32)
        for fn in (T.temporal, T.temporal_loop):
            r = fn(w, h, c, m, None, None, hist, ln, max_history=mh)
            assert r["used"].all() and np.array_equal(r["L"], np.array(want, np.float64)), (lens, fn.__name__, r["L"])
        r = T.temporal(w, h, c, m, None, None, hist, ln, max_history=mh)
        L = r["L"]
        with np.errstate(all="ignore"):
            assert np.array_equal(r["out"][:, 0], 3.0 + (1.0 - 3.0) / L), lens                   # L = 0: -inf; L = -inf: h
    assert np.isfinite(T.temporal(w, h, c, m, None, None, hist, np.array([nan, 2, 2, 2], np.float32))["out"]).all()


def still(n, z=1.0):
    return uncovered(n, z)


def test_c_minus_h_overflows_in_float32():
    """C = 3e38 against h' = -3e38 with L_new = 2: float64 gives 0, the device's float32 difference +inf"""
    c, hist = np.full((1, 3), 3e38, np.float32), np.full((1, 3), -3e38, np.float32)
    args = (1, 1, c, still(1), None, None, hist, np.ones(1, np.float32))
    assert (T.temporal(*args)["out"] == np.inf).all()
    assert (T.temporal(*args, diff32=False)["out"] == 0).all()
    bt = T.beauty_taps(*args)
    assert (TL.blend_layer(bt, c[:, :1], hist[:, :1], 1) == np.inf).all()


def test_an_overflowing_window_sum_leaves_the_history_unclipped():
    """Three 3e38 neighbours sum past FLT_MAX in float32: mu = inf, mu - r NaN, and fmaxf / fminf drop the NaN"""
    w, h = 3, 1
    c = np.full((3, 3), 3e38, np.float32)
    c[:, 1:] = 1.0
    hist = np.full((3, 3), 1.0, np.float32)
    args = (w, h, c, still(3), None, None, hist, np.ones(3, np.float32))
    r = T.temporal(*args, clip_sigma=1.5)
    assert r["hc"][1, 0] == 1.0 and r["hc"][1, 1] == 1.0
    assert T.temporal(*args, clip_sigma=1.5, clip32=False)["hc"][1, 0] == np.float64(np.float32(3e38))
    lo, hi, _ = T.clip_bounds(w, h, c, 1.5)
    assert np.isnan(lo[1, 0]) and hi[1, 0] == np.inf


def test_denormals_flush_in_arithmetic_but_not_in_copies():
    """L_new = 0 divides C - h: with C = 2e-40 and h = 1e-40 flushed that is 0 / 0 = NaN on the device, +inf in exact arithmetic; a
    pixel without history keeps its denormal colour"""
    w, h = 2, 1
    c = np.full((2, 3), 2e-40, np.float32)
    hist = np.full((2, 3), 1e-40, np.float32)
    m = still(2)
    m[1, :2] = 1e30                                                     # no history
    ln = np.full(2, -1.0, np.float32)
    r = T.temporal(w, h, c, m, None, None, hist, ln)
    assert np.isnan(r["out"][0]).all() and r["L"][0] == 0
    assert (T.temporal(w, h, c, m, None, None, hist, ln, ftz=False)["out"][0] == np.inf).all()
    assert np.array_equal(r["out"][1].astype(np.float32).view(np.uint32), c[1].view(np.uint32))
    x = np.full((2, 1), 1e-40, np.float32)
    out = TL.blend_layer(T.beauty_taps(w, h, c, m, None, None, hist, np.ones(2, np.float32)), x, x, 1)
    assert out[0, 0, 0] == 0 and np.float32(out[0, 1, 0]).view(np.uint32) == x[1, 0].view(np.uint32)


def test_compare_rejects_a_moved_copy_and_a_wrong_value():
    rng = np.random.default_rng(9)
    src = rng.uniform(-2, 2, (50, 3)).astype(np.float32)
    want = src.astype(np.float64) * 0.5
    copied = np.zeros(50, bool)
    copied[:10] = True
    want[:10] = src[:10]
    want[10, 0], want[11, 1] = np.nan, -np.inf
    M = np.abs(src).max(1).astype(np.float64)
    got = want.astype(np.float32)
    assert T.compare(got, want, src, copied, M)[0] == []
    bad = got.copy(); bad[3, 1] = np.nextafter(bad[3, 1], np.float32(9))
    assert T.compare(bad, want, src, copied, M)[0]                      # one ulp off in a copy
    bad = got.copy(); bad[20, 2] += np.float32(3 * T.tolerance(M[20]))
    assert T.compare(bad, want, src, copied, M)[0]                      # a wrong finite value
    bad = got.copy(); bad[20, 2] += np.float32(0.3 * T.tolerance(M[20]))
    assert T.compare(bad, want, src, copied, M)[0] == []                # within the bound
    bad = got.copy(); bad[10, 0] = np.inf
    assert T.compare(bad, want, src, copied, M)[0]                      # NaN against +inf
    bad = got.copy(); bad[11, 1] = -3e38
    assert T.compare(bad, want, src, copied, M)[0]                      # -inf against a finite value


def test_display_words_follow_the_devices_nan_rules():
    w = T.display_words(np.array([[np.nan, np.inf, -np.inf], [0.5, 0.5, 0.5], [3e38, 3e38, 3e38]], np.float32))
    assert w[0] >> 24 == 0xff and (w[2] & 0xffffff) == 0                # ACES of 3e38 is inf / inf = NaN: 0
    assert w[1] == D.display_words(np.array([0.5, 0.5, 0.5], np.float32))
