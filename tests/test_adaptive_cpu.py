"""Adaptive sampling without a GPU: the NumPy restatement of the statistic and of the 3x3 stopping rule (tests/adaptive_ref.py) on
synthetic sample stacks, and the host-only parts of the C entry points."""
import ctypes as C

import numpy as np
import pytest

import adaptive_ref as A

FLT_MAX = float(np.finfo(np.float32).max)


def noisy_stack(P, H, W, seed=0, level=1.0, sigma=0.5):
    return (level + sigma * np.random.RandomState(seed).randn(P, H, W)).astype(np.float32)


def test_constant_pixels_stop_at_min_passes():
    Y = np.full((48, 9, 11), 0.7, np.float32)
    out = A.simulate(Y, min_passes=16, check_interval=8, threshold=0.01)
    assert out["passes_run"] == 16
    assert (out["counts"] == 16).all()
    assert (out["err"] == 0).all()


def test_one_noisy_pixel_keeps_its_neighbours_running():
    P, H, W = 40, 7, 9
    Y = np.full((P, H, W), 0.5, np.float32)
    Y[:, 3, 4] = noisy_stack(P, 1, 1, seed=1)[:, 0, 0]
    out = A.simulate(Y, min_passes=8, check_interval=8, threshold=0.05)
    want = np.full((H, W), 8)
    want[2:5, 3:6] = P                                           # the noisy pixel and its 8 neighbours never pass the test
    assert np.array_equal(out["counts"], want)
    assert out["passes_run"] == P
    assert len(out["tests"]) == 4                                # at 8, 16, 24, 32; the frame ends at 40
    # the stopped neighbours' neighbours kept the err they stopped with: zero
    assert (out["err"][want == 8] == 0).all() and out["err"][3, 4] > 0.05


def test_err_matches_a_hand_computation():
    Y = np.array([1.0, 2.0, 3.0, 4.0, 6.0], np.float32).reshape(5, 1, 1)
    out = A.simulate(Y, min_passes=16, check_interval=16, threshold=0.01)      # no test within 5 passes
    m = 16.0 / 5
    var = sum((y - m) ** 2 for y in (1, 2, 3, 4, 6)) / 4                        # unbiased sample variance
    assert out["counts"][0, 0] == 5 and out["passes_run"] == 5
    assert abs(float(out["err"][0, 0]) - np.sqrt(var / 5) / m) <= 1e-6 * np.sqrt(var / 5) / m + 1e-7
    # the mean floor: a dark pixel is judged on its absolute error
    dark = np.array([0.0, 1e-4, 0.0, 1e-4], np.float32).reshape(4, 1, 1)
    e = float(A.simulate(dark, 8, 8, 0.01)["err"][0, 0])
    assert abs(e - np.sqrt(np.var([0, 1e-4, 0, 1e-4], ddof=1) / 4) / A.MEAN_FLOOR) < 1e-7
    # one sample has no error estimate
    assert np.isinf(A.rel_error(np.float32([1]), np.float32([1]), np.float32([0]))[0])


def test_threshold_zero_never_stops_and_flt_max_always_stops():
    Y = noisy_stack(32, 6, 5, seed=2)
    Y[:, :, :2] = 0.25                                           # constant columns: err exactly 0, still not < 0
    never = A.simulate(Y, min_passes=8, check_interval=4, threshold=0.0)
    assert (never["counts"] == 32).all() and never["passes_run"] == 32
    always = A.simulate(Y, min_passes=8, check_interval=4, threshold=FLT_MAX)
    assert (always["counts"] == 8).all() and always["passes_run"] == 8


def test_budget_below_min_passes_is_a_fixed_count_frame():
    out = A.simulate(noisy_stack(6, 4, 4), min_passes=16, check_interval=16, threshold=FLT_MAX)
    assert (out["counts"] == 6).all() and out["passes_run"] == 6 and out["tests"] == []


def test_rgb_samples_are_reduced_to_luminance():
    rgb = np.random.RandomState(4).rand(10, 3, 3, 3).astype(np.float32)
    a = A.simulate(rgb, 4, 2, 0.05)
    b = A.simulate(A.luminance(rgb), 4, 2, 0.05)
    assert np.array_equal(a["counts"], b["counts"]) and np.array_equal(a["err"], b["err"])


def test_options_defaults_and_null_context_fail_loudly():
    from vpt_b200 import _native as N
    o = N.adaptive_options(0, 0, 0.0)
    N.lib.vpt_adaptive_options_defaults(C.byref(o))
    assert (o.min_passes, o.check_interval) == (16, 16) and abs(o.threshold - 0.01) < 1e-9
    assert C.sizeof(N.adaptive_options) == 12
    run = C.c_uint(7)
    rc = N.lib.vpt_render_adaptive(None, None, 64, C.byref(o), None, None, C.byref(run), None)
    assert rc == -1                                              # VPT_ERR_INVALID
    assert b"vpt_render_adaptive" in N.lib.vpt_last_error(None)
    assert run.value == 7                                        # nothing was written
