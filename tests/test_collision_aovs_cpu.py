"""The collision-AOV restatement (tests/collision_aovs_ref.py) against closed forms, and the refusals that need no device."""
import ctypes as C

import numpy as np
import pytest

import collision_aovs_ref as R
import texfilter_ref as T

F32 = np.float32


def one_volume(grid, bmin=(0.0, 0.0, 0.0), colors=None):
    nz, ny, nx = grid.shape
    X = np.eye(4)
    rec = R.volume_rec(X, bmin, (nx, ny, nz))
    return R.Scene([rec], [grid.astype(F32)], colors=[colors] if colors is not None else None)


def interior_points(n, lo, hi, seed=0):
    rng = np.random.default_rng(seed)
    return rng.uniform(lo, hi, (n, 3)).astype(F32)


def test_volume_coord_of_the_identity_is_the_index_over_dims():
    rec = R.volume_rec(np.eye(4), (0.0, 0.0, 0.0), (64, 32, 16))
    P = np.array([[0, 0, 0], [32, 16, 8], [64, 32, 16], [65, 1, 1]], F32)
    uvw, inside = R.volume_coord(rec, P)
    assert np.array_equal(uvw[:3], np.array([[0, 0, 0], [0.5, 0.5, 0.5], [1, 1, 1]], F32))
    assert inside.tolist() == [True, True, True, False]


def test_volume_coord_of_a_translated_scaled_instance():
    X = np.diag([2.0, 2.0, 2.0, 1.0]); X[:3, 3] = (8.0, -4.0, 2.0)          # world = 2 index + t
    rec = R.volume_rec(X, (0.0, 0.0, 0.0), (32, 32, 32))
    P = np.array([[8 + 2 * 16, -4 + 2 * 8, 2 + 2 * 4]], F32)
    uvw, inside = R.volume_coord(rec, P)
    assert np.array_equal(uvw[0], np.array([0.5, 0.25, 0.125], F32)) and inside[0]


def test_a_linear_ramp_has_a_constant_gradient_within_one_weight_step():
    """rho = a x + b y + c z over texel centres: inside the grid the filter's 8-bit weights make rho piecewise linear with steps of
    1/256 of a texel, so each central difference over h is the slope within (1/256 texel * slope) * 2 / (2h) = slope / (256 h)."""
    n = 64
    z, y, x = np.mgrid[0:n, 0:n, 0:n].astype(np.float64)
    a, b, c = 0.02, -0.01, 0.005
    grid = (1.0 + a * x + b * y + c * z).astype(F32)
    sc = one_volume(grid)
    P = interior_points(2000, 8.0, n - 8.0)
    h = 1.0
    g, _ = R.gradient(sc, P, h)
    slope = np.array([a, b, c])
    step = np.abs(slope) / (256 * h) + 2 * np.spacing(F32(3.0)) / (2 * h)
    assert (np.abs(g - slope) <= step).all()
    nrm = R.normal_of_gradient(g)
    want = -slope / np.linalg.norm(slope)
    assert np.abs(nrm - want).max() < 0.05


def test_a_radial_grid_gives_radial_normals():
    """rho = max(0, 1 - r / R) about the grid centre: n = -grad rho / |grad rho| points away from the centre."""
    n = 64
    z, y, x = np.mgrid[0:n, 0:n, 0:n].astype(np.float64)
    c = 32.0                                                            # texel centres sit at index i + 1/2
    r = np.sqrt((x + 0.5 - c) ** 2 + (y + 0.5 - c) ** 2 + (z + 0.5 - c) ** 2)
    grid = np.clip(1.0 - r / 30.0, 0.0, None).astype(F32)
    sc = one_volume(grid)
    rng = np.random.default_rng(1)
    d = rng.normal(size=(1500, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
    P = (c + d * rng.uniform(6.0, 24.0, (1500, 1))).astype(F32)
    g, _ = R.gradient(sc, P, 1.0)
    nrm = R.normal_of_gradient(g)
    radial = (P - c) / np.linalg.norm(P - c, axis=1, keepdims=True)
    assert (np.einsum("ij,ij->i", nrm, radial) > 0.99).mean() > 0.99
    assert (np.einsum("ij,ij->i", nrm, radial) > 0.95).all()


def test_a_flat_grid_has_no_normal():
    sc = one_volume(np.full((16, 16, 16), 0.5, F32))
    g, _ = R.gradient(sc, interior_points(100, 3.0, 13.0), 1.0)
    assert np.array_equal(g, np.zeros_like(g))
    assert np.array_equal(R.normal_of_gradient(g), np.zeros_like(g))
    assert np.array_equal(R.normal_of_gradient(np.array([[np.inf, 0, 0], [np.nan, 1, 0]])), np.zeros((2, 3)))


def test_the_sphere_gives_p_minus_c_over_r():
    rng = np.random.default_rng(2)
    centre, radius = np.array([1.0, -2.0, 3.0]), 2.5
    d = rng.normal(size=(100, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
    org = centre + 10.0 * d + rng.normal(size=(100, 3))
    dirs = centre - org; dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    t = R.ray_sphere(org, dirs, centre, radius)
    P = org + t[:, None] * dirs
    assert np.allclose(np.linalg.norm(P - centre, axis=1), radius)
    assert np.allclose(R.sphere_normal(P, centre), (P - centre) / radius)


def test_a_coloured_grid_and_lut_give_the_expected_albedo():
    """Cd constant (0.2, 0.4, 0.8) inside, rho = 0.5 everywhere, max_extinction 1, pivot 1: index floor(0.5 * 255) = 127, and the albedo
    is albedo * Cd * lut[127] / extinction * energy_inject."""
    n = 16
    rgb = np.zeros((n, n, n, 3), F32); rgb[...] = (0.2, 0.4, 0.8)
    sc = one_volume(np.full((n, n, n), 0.5, F32), colors=rgb)
    P = interior_points(50, 2.0, 14.0)
    rho, _ = sc.density(P)
    assert np.array_equal(rho, np.full(50, 0.5, F32))
    idx = R.lut_index(R.lut_argument(rho, 1.0, 1.0))
    assert (idx == 127).all()
    lut = np.linspace(0, 1, 256 * 3).reshape(256, 3).astype(F32)
    Cd = sc.color(P)
    assert np.allclose(Cd, [0.2, 0.4, 0.8], rtol=1e-6)
    a = R.volume_albedo([0.9, 0.8, 0.7], Cd, lut, idx, [2.0, 2.0, 4.0], 1.5)
    want = np.array([0.9, 0.8, 0.7]) * np.array([0.2, 0.4, 0.8]) * lut[127].astype(np.float64) / np.array([2.0, 2.0, 4.0]) * 1.5
    assert np.allclose(a, want, rtol=1e-6)
    # outside every leaf / box: rho 0 -> index 0, Cd 0 -> albedo 0
    out = np.array([[-5.0, -5.0, -5.0]], F32)
    assert sc.density(out)[0][0] == 0 and np.array_equal(sc.color(out), np.zeros((1, 3), F32))
    assert R.lut_index(np.array([np.nan, -3.0, 1e9])).tolist() == [0, 0, 255]


def test_brick_and_cell_copies_give_the_restated_value():
    """The samplers of brick and cell mode read the grid's brick pool / cell table with the same filter: at any uvw the value is
    texfilter_ref.sample's (texfilter_ref's own tests check the device samplers against it bit for bit)."""
    grid = T.grid_values((16, 8, 8), "signed", seed=4).astype(F32)
    sc = one_volume(grid)
    P = interior_points(300, 0.0, 8.0, seed=5)
    uvw, inside = R.volume_coord(sc.recs[0], P)
    assert inside.all()
    assert np.array_equal(sc.density(P)[0], T.sample(grid, uvw)["value"])


def test_the_running_mean_is_accums_rule():
    assert R.running_mean(3.0, 5.0, 0, 10) == 5.0
    assert R.running_mean(3.0, 5.0, 3, 10) == 3.0 + (5.0 - 3.0) / 4
    assert R.running_mean(3.0, 5.0, 10, 10) == 3.0
    # a sample without coverage adds exact zeros: the mean of c P is the mean of P over the covered passes times their share
    xs = [R.running_mean(0.0, 0.0, 0, 100)]
    for i, s in enumerate([2.0, 0.0, 4.0], start=1):
        xs.append(R.running_mean(xs[-1], s, i, 100))
    assert np.isclose(xs[-1], (2.0 + 4.0) / 4)


def test_leaf_lists_sum_the_volumes_of_the_leaf_containing_the_point():
    """Two overlapping unit grids of value 1 and 2 under one fake octree whose root splits at x = 4: the left leaf lists volume 0, the
    right both, so rho is 1 left of the plane and 3 right of it (inside both boxes)."""
    class Box:
        def __init__(self, lo, hi):
            self.pmin = type("p", (), dict(x=lo[0], y=lo[1], z=lo[2]))(); self.pmax = type("p", (), dict(x=hi[0], y=hi[1], z=hi[2]))()
    class Node:
        def __init__(self, lo, hi, n=1):
            self.bbox = Box(lo, hi); self.num_volumes = n
    lo, hi, half = (0.0, 0.0, 0.0), (8.0, 8.0, 8.0), (4.0, 4.0, 4.0)
    nodes = {}
    def fill(j, lo, hi, depth, kid_base):
        nodes[j] = Node(lo, hi)
        if depth == 3:
            return
        h = [(a + b) / 2 for a, b in zip(lo, hi)]
        for c in range(8):
            clo = (h[0] if c & 1 else lo[0], lo[1] if c & 2 else h[1], h[2] if c & 4 else lo[2])
            chi = (hi[0] if c & 1 else h[0], h[1] if c & 2 else hi[1], hi[2] if c & 4 else h[2])
            kid = 1 + c if j == 0 else (9 + (j - 1) * 8 + c if j < 9 else 73 + (j - 9) * 8 + c)
            fill(kid, clo, chi, depth + 1, None)
    fill(0, lo, hi, 0, None)
    lists = [[0] if ((l >> 6) & 1) == 0 else [0, 1] for l in range(512)]
    oct_ = R.Octree(nodes, lists)
    recs = [R.volume_rec(np.eye(4), (0.0, 0.0, 0.0), (8, 8, 8)), R.volume_rec(np.eye(4), (0.0, 0.0, 0.0), (8, 8, 8))]
    sc = R.Scene(recs, [np.ones((8, 8, 8), F32), np.full((8, 8, 8), 2.0, F32)], octree=oct_)
    P = np.array([[2.0, 2.0, 2.0], [6.0, 2.0, 2.0], [9.0, 2.0, 2.0]], F32)
    assert oct_.leaf(P)[2] == -1
    assert sc.density(P)[0].tolist() == [1.0, 3.0, 0.0]
    assert half == (4.0, 4.0, 4.0)


# ---- refusals that need no device ----------------------------------------------------------------------------------------------------------
def native():
    import vpt_b200 as V
    return V


def test_a_null_context_is_refused():
    """(A context needs a device; the step and overlap refusals are checked in test_collision_aovs_gpu.py.)"""
    V = native()
    assert V.lib.vpt_set_collision_aovs(None, None, None, None, 1.0) == -1
    assert V.lib.vpt_set_collision_aovs(None, None, C.c_void_p(0x1000), None, float("nan")) == -1
