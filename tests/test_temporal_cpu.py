"""Temporal accumulation without a GPU: the restatement of vpt_temporal (tests/temporal_ref.py) against closed forms -- the environment's
motion under a pan and a translation, zero motion, integer shifts, the frame edge, the clip and the history cap -- the still-camera
guarantee in accum's float32 arithmetic, and the refusals that need no device."""
import ctypes as C

import numpy as np
import pytest

import vpt_b200 as V
from vpt_b200 import _native as N
import temporal_ref as T

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
    for gamma in (0.5, 1.0, 2.0):
        r = T.temporal(w, h, c, uncovered(9, 1.0), cam, cam, hist, np.ones(9, np.float32), clip_sigma=gamma)
        assert np.allclose(r["hc"][4], [mu + gamma * sigma, 1.0, 0.0], rtol=1e-12, atol=0)
    r = T.temporal(w, h, c, uncovered(9, 1.0), cam, cam, hist, np.ones(9, np.float32))
    assert np.array_equal(r["hc"][4], hist[4].astype(np.float64))       # clip_sigma = inf: no clip
    c[0] = np.inf                                                       # a non-finite neighbour drops out of the window
    r = T.temporal(w, h, c, uncovered(9, 1.0), cam, cam, hist, np.ones(9, np.float32), clip_sigma=1.0)
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
