"""Temporal layers without a GPU: the restatement of vpt_temporal_layers (tests/temporal_layers_ref.py) against closed forms -- the colour
as a layer is temporal_ref's beauty, the blend is linear, a tap dropped for a non-finite beauty history drops the layer's finite value, a
pixel without history keeps the layer's value -- the ctypes layout of vpt_temporal_layer, and the refusals that need no device."""
import ctypes as C

import numpy as np
import pytest

import vpt_b200 as V
from vpt_b200 import _native as N
import temporal_ref as T
import temporal_layers_ref as TL
from test_temporal_cpu import camera

W, H = 23, 17


def case(seed, fractional=True):
    rng = np.random.default_rng(seed)
    n = W * H
    a = camera((0.0, 0.0, 0.0), w=W, h=H)
    b = camera((0.02, 0.0, 0.01), yaw=0.01, w=W, h=H)
    c = rng.uniform(0.0, 2.0, (n, 3)).astype(np.float32)
    hist = rng.uniform(0.0, 2.0, (n, 3)).astype(np.float32)
    ln = rng.integers(1, 12, n).astype(np.float32)
    m = np.zeros((n, 3), np.float32)
    m[:, 2] = rng.choice([0.0, 0.5, 1.0], n)
    m[:, :2] = (rng.uniform(-2.5, 2.5, (n, 2)) if fractional else rng.integers(-2, 3, (n, 2))) * m[:, 2:3]
    return a, b, c, m, hist, ln


def test_the_colour_as_a_layer_is_the_beauty():
    a, b, c, m, hist, ln = case(1)
    ref = T.temporal(W, H, c, m, a, b, hist, ln, max_history=8)
    bt = TL.beauty_taps(W, H, c, m, a, b, hist, ln, max_history=8)
    assert np.array_equal(bt["used"], ref["used"]) and np.array_equal(bt["L"], ref["L"])
    assert bt["used"].any() and (~bt["used"]).any()
    out = TL.blend_layer(bt, c, hist, 3)[0]
    assert np.array_equal(out, ref["out"])
    for ch in range(3):                                        # each channel as a 1-channel layer
        assert np.array_equal(TL.blend_layer(bt, c[:, ch].copy(), hist[:, ch].copy(), 1)[0, :, 0], ref["out"][:, ch])


def test_the_blend_is_linear_in_float64():
    a, b, c, m, hist, ln = case(2)
    rng = np.random.default_rng(3)
    n = W * H
    X, HX = rng.uniform(-1, 1, (2, n, 4)), rng.uniform(-1, 1, (2, n, 4))
    Y, HY = rng.uniform(-1, 1, (2, n, 4)), rng.uniform(-1, 1, (2, n, 4))
    X, HX, Y, HY = (t.astype(np.float32) for t in (X, HX, Y, HY))
    bt = TL.beauty_taps(W, H, c, m, a, b, hist, ln)
    ka, kb = 0.75, -1.5
    f64 = lambda t: t.astype(np.float64)
    Z, HZ = ka * f64(X) + kb * f64(Y), ka * f64(HX) + kb * f64(HY)
    # blend_layer reads float32 planes, so the combination (not float32) is blended here with the same taps
    out_x, out_y = TL.blend_layer(bt, X, HX, 4, 2, diff32=False), TL.blend_layer(bt, Y, HY, 4, 2, diff32=False)
    used = bt["used"]
    fma, _ = T._ops(np.float64)
    out_z = Z.copy()
    for p in np.flatnonzero(used):
        s = np.zeros((2, 4))
        for k in range(4):
            if bt["taps"][p, k] >= 0:
                s = fma(bt["w"][p, k], HZ[:, bt["taps"][p, k]], s)
        h = s / bt["sw"][p]
        out_z[:, p] = h + (Z[:, p] - h) / bt["L"][p]
    assert np.allclose(ka * out_x + kb * out_y, out_z, rtol=0, atol=1e-12)
    assert used.any()


def test_a_tap_dropped_for_a_non_finite_beauty_history_drops_the_layers_value():
    w, h = 4, 3
    cam = camera((0.0, 0.0, 0.0), w=w, h=h)
    n = w * h
    c = np.ones((n, 3), np.float32)
    m = np.zeros((n, 3), np.float32)
    m[:, 2] = 1.0
    m[:, 0] = 0.5                                               # halfway between two columns: taps (x, y) and (x + 1, y)
    hist = np.full((n, 3), 2.0, np.float32)
    hist[1 * w + 2] = np.nan                                    # pixel (2, 1)'s beauty history
    ln = np.full(n, 3.0, np.float32)
    layer, lh = np.zeros(n, np.float32), np.arange(n, dtype=np.float32)
    bt = TL.beauty_taps(w, h, c, m, cam, cam, hist, ln, dt=np.float32)
    out = TL.blend_layer(bt, layer, lh, 1, dt=np.float32)[0, :, 0]
    p = 1 * w + 1                                               # taps (1, 1) and (2, 1); (2, 1) is dropped
    assert bt["used"][p] and list(bt["taps"][p]) == [p, -1, -1, -1]
    assert out[p] == np.float32(lh[p] + (0.0 - lh[p]) / 4.0)
    q = 1 * w + 2                                               # taps (2, 1) dropped, (3, 1) kept
    assert list(bt["taps"][q]) == [-1, q + 1, -1, -1] and out[q] == np.float32(lh[q + 1] * 0.75)


def test_a_pixel_without_history_keeps_the_layers_value():
    a, b, c, m, hist, ln = case(4)
    n = W * H
    c[::7] = np.nan                                            # non-finite C
    m[1::11, :2] = 1e4; m[1::11, 2] = 1.0                      # q off the frame
    layer = np.random.default_rng(5).uniform(-3, 3, (n, 2)).astype(np.float32)
    lh = np.zeros((n, 2), np.float32)
    bt = TL.beauty_taps(W, H, c, m, a, b, hist, ln)
    out = TL.blend_layer(bt, layer, lh, 2)[0]
    free = ~bt["used"]
    assert free[::7].all() and free[1::11].all()
    assert np.array_equal(out[free], layer[free].astype(np.float64))
    none = TL.blend_layer(TL.beauty_taps(W, H, c, m, a, b, None, None), layer, None, 2)[0]   # no history buffers
    assert np.array_equal(none, layer.astype(np.float64))


def test_the_layer_struct_matches_the_header():
    assert C.sizeof(N.temporal_layer) == 32
    assert [getattr(N.temporal_layer, f).offset for f in ("src", "history", "dst", "channels", "count")] == [0, 8, 16, 24, 28]
    assert N.VPT_TEMPORAL_MAX_LAYERS == 16


def test_refusals_that_need_no_device():
    cam = N.camera()
    lay = (N.temporal_layer * 1)(N.temporal_layer(128, None, 256, 1, 1))
    assert V.lib.vpt_temporal_layers(None, 4, 4, None, None, C.byref(cam), C.byref(cam), None, None, None, 1.0, None, None, None,
                                     lay, 1, None) == -1
    assert b"vpt_temporal_layers" in V.lib.vpt_last_error(None) and b"null context" in V.lib.vpt_last_error(None)
    r = V.Renderer.__new__(V.Renderer)
    with pytest.raises(V.VptError, match="not enabled"):
        r.temporal_layer_images()


@pytest.mark.parametrize("wh", [(1, 1), (2, 1), (1, 2), (23, 17)])
def test_the_vectorised_blend_equals_the_loop(wh):
    from test_temporal_cpu import hostile
    w, h = wh
    n = w * h
    a, b = camera((0.0, 0.0, 0.0), w=w, h=h), camera((0.02, 0.0, 0.01), yaw=0.01, w=w, h=h)
    c, m, hist, ln = hostile(w, h, 3 * w + h)
    rng = np.random.default_rng(w + h)
    for fdt in (None, np.float32):
        bt = TL.beauty_taps(w, h, c, m, a, b, hist, ln, max_history=5, footprint_dt=fdt)
        for ch, k in ((1, 1), (2, 3), (4, 2)):
            src, lh = (rng.uniform(-3, 3, (k, n, ch)).astype(np.float32) for _ in range(2))
            lh[rng.random((k, n, ch)) < 0.05] = np.nan
            want = TL.blend_layer_loop(bt, src, lh, ch, k)
            assert np.array_equal(TL.blend_layer(bt, src, lh, ch, k, diff32=False, ftz=False), want, equal_nan=True), (wh, ch, k)


def test_the_layer_reach_is_the_src_and_the_used_taps():
    w, h = 4, 1
    m = np.tile(np.array([0.5, 0.0, 1.0], np.float32), (4, 1))
    c, hist = np.ones((4, 3), np.float32), np.ones((4, 3), np.float32)
    hist[2] = np.nan                                             # pixel 2's tap dropped for every layer
    bt = TL.beauty_taps(w, h, c, m, None, None, hist, np.ones(4, np.float32))
    src = np.array([[1, -2], [0, 0], [0.5, 0], [7, np.inf]], np.float32)
    lh = np.array([[3, 0], [-4, 1], [100, 0], [0, -6]], np.float32)
    M = TL.layer_reach(bt, src, lh, 2)[0]
    assert list(M) == [4, 4, 6, 7]                               # taps (0, 1), (1, -), (-, 3), (3, -)
