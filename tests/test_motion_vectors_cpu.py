"""Motion vectors without a GPU: the restatement's film projection (tests/motion_vectors_ref.py) against closed forms for a pinhole
camera, the running mean, the exchange block with the motion plane, and the refusals that need no device."""
import ctypes as C

import numpy as np
import pytest

import vpt_b200 as V
from vpt_b200 import _native as N
from vpt_b200 import renderer as R
import motion_vectors_ref as M

W, H = 640, 360


def camera(origin, yaw=0.0, vfov_deg=40.0):
    """A pinhole camera in the reference's construction (focus distance 1): forward -w, right u, up v, turned by `yaw` about +y."""
    c, s = np.cos(yaw), np.sin(yaw)
    u = np.array([c, 0.0, -s]); v = np.array([0.0, 1.0, 0.0]); w = np.array([s, 0.0, c])
    half_h = np.tan(np.radians(vfov_deg) / 2); half_w = W / H * half_h
    o = np.asarray(origin, np.float64)
    return {"origin": o, "lower_left_corner": o - half_w * u - half_h * v - w, "horizontal": 2 * half_w * u, "vertical": 2 * half_h * v,
            "f": W / (2 * half_w)}


def test_a_pan_by_theta_moves_the_image_centre_by_f_tan_theta():
    a = camera((0, 0, 0))
    P = np.array([0.0, 0.0, -7.0])                            # on the optical axis: the image centre
    st, ok = M.project(a, P, W, H)
    assert ok and np.allclose(st, (W / 2, H / 2), atol=1e-9)
    for theta in (0.01, 0.1, -0.3):
        b = camera((0, 0, 0), yaw=theta)
        v = M.sample_vectors(a, b, P, True, W, H)
        assert abs(abs(v[0]) - a["f"] * abs(np.tan(theta))) < 1e-9 * a["f"] and abs(v[1]) < 1e-9, theta
        assert np.sign(v[0]) == np.sign(theta)                   # turning left (+yaw about y) moves the scene right on the film


def test_a_sideways_translation_moves_a_point_at_depth_z_by_f_delta_over_z():
    a = camera((0, 0, 0))
    for z, delta in ((2.0, 0.1), (10.0, 0.5), (3.0, -0.2)):
        b = camera((delta, 0, 0))
        P = np.array([[0.3, -0.2, -z], [-1.0, 0.5, -z]])
        v = M.sample_vectors(a, b, P, [True, True], W, H)
        assert np.allclose(v[:, 0], -a["f"] * delta / z, rtol=1e-12, atol=1e-9) and np.allclose(v[:, 1], 0.0, atol=1e-9), (z, delta)


def test_a_point_on_the_ray_through_a_film_position_projects_back_to_it():
    rng = np.random.default_rng(5)
    cam = N.camera()
    V.lib.vpt_camera_look_at(C.byref(cam), N.fvec((3, 2, 9)), N.fvec((0.2, 0.1, 0)), N.fvec((0, 1, 0)), 35.0, W / H, 0.0)
    x, y = rng.integers(0, W, 200), rng.integers(0, H, 200)
    jx, jy = rng.random(200), rng.random(200)
    P = M.film_point(cam, x, y, jx, jy, W, H, dist=rng.uniform(0.5, 40.0, 200))
    st, ok = M.project(cam, P, W, H)
    assert ok.all() and np.allclose(st, np.stack([x + jx, y + jy], -1), atol=1e-6)
    assert np.array_equal(M.sample_vectors(cam, cam, P, np.ones(200, bool), W, H), np.zeros((200, 2)))


def test_points_behind_the_camera_and_misses_give_zero():
    a, b = camera((0, 0, 0)), camera((0.3, 0, 0))
    P = np.array([[0.0, 0.0, 5.0], [0.0, 0.0, -5.0], [0.0, 0.0, -5.0]])
    v = M.sample_vectors(a, b, P, [True, False, True], W, H)
    assert np.array_equal(v[:2], np.zeros((2, 2))) and v[2, 0] != 0.0
    c = camera((0, 0, -10.0))                                  # the point lies behind B only
    assert np.array_equal(M.sample_vectors(a, c, P[1:2], [True], W, H), np.zeros((1, 2)))


def test_running_mean_is_accums_rule():
    assert M.running_mean(3.0, 5.0, 0, 10) == 5.0
    assert M.running_mean(3.0, 5.0, 3, 10) == 3.0 + (5.0 - 3.0) / 4
    assert M.running_mean(3.0, 5.0, 10, 10) == 3.0


def test_exchange_block_carries_the_motion_plane_after_the_seven_layers():
    def block(mask):
        out = C.c_size_t(0)
        assert V.lib.vpt_comm_p2p_block_bytes(333, 197, 1, mask, C.byref(out)) == 0, V.lib.vpt_last_error(None)
        return out.value
    plane = (12 * 333 * 197 + 255) // 256 * 256
    for mask in (0x01, 0x7F, 0x44):
        assert block(mask | N.VPT_LAYER_MOTION) == block(mask) + plane
    base = block(0)
    assert block(N.VPT_LAYER_MOTION) == (base + 255) // 256 * 256 + plane
    out = C.c_size_t(0)
    assert V.lib.vpt_comm_p2p_block_bytes(64, 64, 1, 0x80, C.byref(out)) == -1       # bit 7 stays unknown
    assert V.lib.vpt_comm_p2p_block_bytes(64, 64, 1, 0x200, C.byref(out)) == -1


def test_refusals_that_need_no_device():
    cam = N.camera()
    assert V.lib.vpt_set_motion_vectors(None, None, C.byref(cam)) == -1
    assert b"null context" in V.lib.vpt_last_error(None)
    assert R._layer_names(("motion", "depth")) == ("depth", "motion")
    assert R._layer_mask(("motion", "alpha")) == N.VPT_LAYER_MOTION | N.LAYER_BITS["alpha"]
    with pytest.raises(V.VptError, match="unknown layer"):
        R._layer_names(("motion", "vectors"))
    r = V.Renderer.__new__(V.Renderer)
    r.buffers = V.FrameBuffers.__new__(V.FrameBuffers); r.buffers.motion = None
    with pytest.raises(V.VptError, match="not enabled"):
        r.motion_vector_image()


def test_unpremultiply():
    import torch
    m = torch.tensor([[2.0, -1.0, 0.5], [0.0, 0.0, 0.0], [3.0, 3.0, 1.0]])
    v, z = R.unpremultiply_vectors(m)
    assert torch.equal(v, torch.tensor([[4.0, -2.0], [0.0, 0.0], [3.0, 3.0]])) and torch.equal(z, m[:, 2])
