"""The restatement of the texture unit's filter (tests/texfilter_ref.py) against what the unit returned, and against the CPU oracle's filter.

  * every stored fetch of tests/golden/tex_unit_corner_weights.npz (eight one-hot 2x2x2 textures: the eight corner weights of 20 000
    points) and tests/golden/tex_unit_coordinates.npz (0/1 ramps of 49, 96, 1000 and 2047 texels along one axis: 5 x 20 000 coordinates)
    is reproduced exactly, with no allowance;
  * where the CPU oracle library is built, its orc_tex3d equals the restatement bit for bit on the grids and point categories the device
    samplers are tested on (tests/test_texfilter_gpu.py).
"""
import ctypes as C
import os

import numpy as np
import pytest

import texfilter_ref as R
import oracle_cpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_restatement_reproduces_every_captured_corner_weight():
    z = np.load(os.path.join(GOLD, "tex_unit_corner_weights.npz"))
    pts, w = z["pts"], z["w"]
    assert pts.shape == (20000, 3) and w.shape == (8, 20000)
    for c in range(8):
        got = R.sample(R.grid_values((2, 2, 2), f"onehot{c}"), pts)["value"]
        bad = np.nonzero(got != w[c].astype(np.float32))[0]
        assert len(bad) == 0, f"corner {c}: {len(bad)} of {len(pts)} weights differ, first at {pts[bad[0]]}"
    # and the weights themselves: eight integers summing to 256 on every point, clamped axes folded onto their edge texel
    ref = R.sample(R.grid_values((2, 2, 2), "onehot0"), pts)
    assert (ref["corners"].sum(1) == 256).all()


def test_restatement_reproduces_every_captured_coordinate():
    z = np.load(os.path.join(GOLD, "tex_unit_coordinates.npz"))
    keys = sorted(k for k in z.files if k.startswith("u_"))
    assert len(keys) == 5
    for key in keys:
        N, ax = [int(v) for v in key[2:].split("_")]
        dims = [2, 2, 2]; dims[ax] = N
        p = np.full((len(z[key]), 3), 0.25, dtype=np.float32)       # the other two axes sit on a texel centre: weights 0 and 256
        p[:, ax] = z[key]
        got = R.sample(R.grid_values(tuple(dims), f"ramp{ax}"), p)["value"]
        hw = z["hw_" + key[2:]]
        assert len(got) == 20000
        bad = np.nonzero(got != hw)[0]
        assert len(bad) == 0, f"N = {N}, axis {ax}: {len(bad)} of {len(got)} differ, first u = {p[bad[0], ax]!r}"
    # the exact u * N - 0.5 the rule replaces is NOT what the unit computes: it misses at N = 2047 (one weight step high)
    u = z["u_2047_0"]
    naive = np.floor((u.astype(np.float64) * 2047 - 0.5) % 1.0 * 256 + 0.5)
    _, A = R.axis(u, 2047)
    assert (naive % 256 != A).mean() > 0.05


def test_corner_weights_sum_to_256_and_split_z_then_x_then_y():
    A, B, C = [g.ravel() for g in np.meshgrid(np.arange(256), np.arange(256), np.arange(0, 256, 5), indexing="ij")]
    w = R.corner_weights(A, B, C)
    assert (w >= 0).all() and (w.sum(1) == 256).all()
    assert (w[:, 4:].sum(1) == C).all()                                      # z first: the upper half gets exactly C
    # the worked clamp case: T = 200, A = 128, B = 1 puts weight 0 on y = 1, while A = 0 (what a clamped axis gets) puts 1 there
    assert R.corner_weights(128, 1, 56)[[2, 3]].sum() == 0 and R.corner_weights(0, 1, 56)[[2, 3]].sum() == 1


needs_oracle = pytest.mark.skipif(not os.path.exists(oracle_cpu.LIB), reason="oracle/liboracle_cpu.so not built")


@needs_oracle
@pytest.mark.parametrize("dims", R.SHAPES, ids=lambda d: "x".join(map(str, d)))
def test_oracle_filter_equals_restatement(dims):
    lib = C.CDLL(oracle_cpu.LIB)
    lib.orc_tex3d.argtypes = [C.POINTER(C.c_float), C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float]
    lib.orc_tex3d.restype = C.c_float
    pts = R.points(dims, n_random=4096)
    for kind in ("signed", "spread"):
        g = R.grid_values(dims, kind)
        gp = g.ctypes.data_as(C.POINTER(C.c_float))
        for cat, p in pts.items():
            want = R.sample(g, p)["value"]
            got = np.array([lib.orc_tex3d(gp, dims[0], dims[1], dims[2], float(a), float(b), float(c)) for a, b, c in p], dtype=np.float32)
            bad = np.nonzero(got.view(np.uint32) != want.view(np.uint32))[0]
            assert len(bad) == 0, f"{kind} {cat}: {len(bad)} of {len(p)} differ, first at {p[bad[0]]!r}: {got[bad[0]]!r} vs {want[bad[0]]!r}"
