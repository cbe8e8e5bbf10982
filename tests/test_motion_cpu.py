"""Camera motion without a GPU: the draw-index logic of tests/motion_ref.py, which the GPU tests compare vpt_debug_motion_cameras' shutter
draws against, and the float64 restatement of the pose lerp."""
import ctypes as C

import numpy as np
import pytest

import motion_ref as M

f32 = np.float32


@pytest.fixture(scope="module")
def lib():
    lib = M.oracle_lib()
    lib.orc_stream_draw.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32]; lib.orc_stream_draw.restype = C.c_float
    return lib


def test_tables_are_the_radical_inverses():
    for base in (2, 3):
        t = M.vdc_table(base)
        for n in range(101):
            want, d, m = 0.0, 1.0, n
            while m:
                d *= base; want += (m % base) / d; m //= base
            assert abs(float(t[n]) - want) <= 2e-7, (base, n)
    assert M.vdc_table(2)[1] == f32(0.5) and M.vdc_table(3)[1] == f32(1 / 3)


def test_acceptance_does_not_depend_on_the_last_bits_of_the_tables():
    """The kernels divide with __fdividef, the restatement with IEEE division: a trial's fate must not hang on that.  Moving every
    table entry by up to two ulp either way leaves every one of the 101 x 101 decisions as it is, and the decisions are those of the
    unit disc away from its rim."""
    t2, t3 = M.vdc_table(2), M.vdc_table(3)
    acc = M.accept_table(t2, t3)
    for s in (-2, -1, 1, 2):
        step = lambda t: np.array([v if v == 0 else np.float32(v + s * np.spacing(v)) for v in t], dtype=np.float32)
        assert np.array_equal(M.accept_table(step(t2), step(t3)), acc), s
    px, py = 2.0 * t2.astype(np.float64) - 1.0, 2.0 * t3.astype(np.float64) - 1.0
    r2 = px[:, None] ** 2 + py[None, :] ** 2
    far = np.abs(r2 - 1.0) > 1e-6
    assert np.array_equal(acc[far], (r2 < 1.0)[far])
    assert 0.6 < acc.mean() < 0.9


def test_stream_is_the_oracles_stream(lib):
    rs = np.random.RandomState(11)
    for idx, it in [(0, 0), (5, 3), (2073599, 63), (77, 4194304)] + [(int(rs.randint(0, 2 ** 21)), int(rs.randint(0, 5000))) for _ in range(8)]:
        s = M.Stream(lib, idx, it)
        for k in range(11):
            assert s.next() == f32(lib.orc_stream_draw(idx, it, k)), (idx, it, k)


def test_the_shutter_draw_follows_the_lens_loop(lib):
    """xi is the draw right after the accepted trial: draw 2 t for a loop of t trials, and the trial counts follow the table's
    acceptance rate."""
    acc = M.accept_table()
    trials = []
    for idx in range(0, 4000, 7):
        xi, k = M.shutter_draw(M.Stream(lib, idx, 9), acc)
        assert k % 2 == 0 and k >= 2
        assert xi == f32(lib.orc_stream_draw(idx, 9, k))
        # the trials before the last were rejected, the last accepted
        s = M.Stream(lib, idx, 9)
        pairs = [(int(f32(s.next() * f32(100))), int(f32(s.next() * f32(100)))) for _ in range(k // 2)]
        assert all(not acc[p] for p in pairs[:-1]) and acc[pairs[-1]]
        trials.append(k // 2)
    p1 = np.mean(np.array(trials) == 1)
    assert abs(p1 - acc.mean()) < 0.06, (p1, acc.mean())
    assert 0.0 < xi <= 1.0


def test_lerp_restatement_ends():
    o = np.arange(18, dtype=np.float32).reshape(6, 3)
    c = o + np.float32(3)
    np.testing.assert_array_equal(M.lerp64(o, c, 0.0), o)
    np.testing.assert_array_equal(M.lerp64(o, c, 1.0), c)
    np.testing.assert_allclose(M.lerp64(o, c, np.array([0.25, 0.5])), [o + 0.75, o + 1.5])
