"""The omni-directional stereo camera without a GPU: the restatement in tests/ods_ref.py (which tests/test_ods_gpu.py holds the kernels'
diagnostic to) has the ODS geometry -- every ray tangent to its eye's viewing circle, the eyes on opposite sides, the pole merge and the
over-under layout as vpt_b200.h states them."""
import numpy as np
import pytest

import ods_ref as O
import projection_ref as P

f32 = np.float32


@pytest.fixture(scope="module")
def headline():
    return P.headline_pano_setup()


def random_pixels(W, H, n, seed):
    rs = np.random.RandomState(seed)
    return rs.randint(0, W, n), rs.randint(0, H, n), rs.rand(n).astype(f32), rs.rand(n).astype(f32)


@pytest.mark.parametrize("ipd", [0.064, 2.0])
def test_every_ray_is_tangent_to_its_eyes_circle(headline, ipd):
    cam = headline["cam"]
    W, H = 4096, 2048
    od = O.params(ipd=ipd)
    x, y, jx, jy = random_pixels(W, H, 20000, 1)
    org, llc, e, k = O.ods_camera(cam, od, W, H, x, y, jx, jy)
    o = np.asarray(cam["origin"], np.float64)
    d = org.astype(np.float64) - o                                   # s r, in float64
    ray = llc.astype(np.float64) - org.astype(np.float64)
    ray /= np.linalg.norm(ray, axis=-1, keepdims=True)
    s = e.astype(np.float64) * float(od["half_ipd"]) * k
    # |s r| is |s| up to the basis' rounding, and what is left of s r along the ray and along v is rounding: of origin' (an ulp of the
    # origin's size per component) and of the float basis, b0 and llc' - origin'
    tol = 8 * float(np.spacing(f32(np.abs(o).max()))) / np.maximum(np.abs(s), 1e-30) + 1e-5
    np.testing.assert_allclose(np.linalg.norm(d, axis=-1), np.abs(s), rtol=0, atol=4 * float(np.spacing(f32(np.abs(o).max()))) + 1e-6 * ipd)
    live = np.abs(s) > 0
    v = np.asarray(cam["v"], np.float64)
    assert (np.abs((d @ v)[live]) / np.abs(s[live]) <= tol[live]).all()
    assert (np.abs(np.sum(d * ray, -1)[live]) / np.abs(s[live]) <= tol[live]).all()
    # the left eye sits to the left of the viewing direction (d x ray points down the up axis), the right eye to the right
    side = np.cross(d, ray) @ v
    assert (np.sign(side[live]) == e[live]).all()
    assert abs(live.mean() - 150 / 180) < 0.02                       # rows with |theta| >= 75 degrees merge fully


def test_both_eyes_at_the_same_distance_on_opposite_sides(headline):
    cam = headline["cam"]
    W, H = 1024, 512
    x, y, jx, jy = random_pixels(W, H // 2, 2000, 2)
    o = np.asarray(cam["origin"], np.float64)
    left, _, el, kl = O.ods_camera(cam, O.params(ipd=0.5, layout=O.LEFT), W, H // 2, x, y, jx, jy)
    right, _, er, kr = O.ods_camera(cam, O.params(ipd=0.5, layout=O.RIGHT), W, H // 2, x, y, jx, jy)
    assert (el == -1).all() and (er == 1).all() and np.array_equal(kl, kr)
    dl, dr = left.astype(np.float64) - o, right.astype(np.float64) - o
    ulp = float(np.spacing(f32(np.abs(o).max())))
    np.testing.assert_allclose(dl, -dr, rtol=0, atol=2 * ulp)


def test_pole_merge_is_one_linear_and_zero_where_stated():
    od = O.params(merge=(60.0, 75.0))
    deg = np.linspace(-90, 90, 3601)
    th = (deg * np.pi / 180).astype(f32)
    k = O.pole_merge(od, th).astype(np.float64)
    a = np.abs(th.astype(np.float64)) * 180 / np.pi
    assert (k[a <= 59.999] == 1).all() and (k[a >= 75.001] == 0).all()
    mid = (a > 60.001) & (a < 74.999)
    np.testing.assert_allclose(k[mid], (75 - a[mid]) / 15, atol=2e-6)
    assert (np.diff(k[deg >= 0]) <= 0).all()                         # never grows towards the pole
    step = O.pole_merge(O.params(merge=(70.0, 70.0)), th)
    assert set(np.unique(step)) == {0.0, 1.0}
    assert (step[a < 69.999] == 1).all() and (step[a > 70.001] == 0).all()
    assert (O.pole_merge(O.params(merge=(90.0, 90.0)), th) == 1).all()
    assert (O.pole_merge(O.params(merge=(0.0, 0.0)), th[np.abs(th) > 0]) == 0).all()


def test_over_under_layout_has_the_left_eye_on_top(headline):
    cam = headline["cam"]
    W, H = 64, 32
    y = np.arange(H)
    e, ye, He = O.eye_rows(O.OVER_UNDER, H, y)
    assert He == H // 2
    assert (e[H // 2:] == -1).all() and (e[:H // 2] == 1).all()
    assert np.array_equal(ye[H // 2:], np.arange(H // 2)) and np.array_equal(ye[:H // 2], np.arange(H // 2))
    # each half is the single-eye frame of half the height
    xs, ys = np.meshgrid(np.arange(W), np.arange(H))
    jx = jy = np.full(xs.shape, f32(0.37))
    ou = O.ods_camera(cam, O.params(), W, H, xs, ys, jx, jy)
    for lay, rows in ((O.LEFT, slice(H // 2, H)), (O.RIGHT, slice(0, H // 2))):
        one = O.ods_camera(cam, O.params(layout=lay), W, H // 2, xs[:H // 2], ys[:H // 2], jx[:H // 2], jy[:H // 2])
        for a, b in zip(ou, one):
            assert np.array_equal(a[rows], b), lay
    # and the top row of the frame looks up, the bottom row down, in both eyes
    _, llc, _, _ = ou
    d = llc.astype(np.float64) - ou[0].astype(np.float64)
    up = (d / np.linalg.norm(d, axis=-1, keepdims=True)) @ np.asarray(cam["v"], np.float64)
    for r in (0, H // 2):
        assert (up[r] < -0.99).all()
    for r in (H // 2 - 1, H - 1):
        assert (up[r] > 0.99).all()


# ---- the miss cull -----------------------------------------------------------------------------------------------------------------------
SPP = 64
CULL_FRAMES = {"full_4096x2048": (4096, 2048, 360.0, 180.0), "partial_90x60": (1536, 1024, 90.0, 60.0)}


def _sphere_hits(c, r, o, d):
    """test_miss_cull_cpu.sphere_hits (the oracle's sphere_intersect in float32) with a per-ray origin."""
    oc = [(o[k] - f32(c[k])).astype(f32) for k in range(3)]
    A = ((d[0] * d[0]).astype(f32) + (d[1] * d[1]).astype(f32) + (d[2] * d[2]).astype(f32)).astype(f32)
    B = (f32(2) * ((d[0] * oc[0]).astype(f32) + (d[1] * oc[1]).astype(f32) + (d[2] * oc[2]).astype(f32)).astype(f32)).astype(f32)
    C = (sum((v.astype(np.float64) * v.astype(np.float64)) for v in oc) - float(f32(r) * f32(r))).astype(f32)
    discr = ((B * B).astype(f32) - (f32(4) * A * C).astype(f32)).astype(f32)
    sq = np.sqrt(np.maximum(discr, 0)).astype(f32)
    q = np.where(B < 0, f32(-0.5) * (B - sq), f32(-0.5) * (B + sq)).astype(f32)
    with np.errstate(divide="ignore", invalid="ignore"):
        x1 = (q / A).astype(f32); x2 = (C / q).astype(f32)
    return (discr >= 0) & ((np.minimum(x1, x2) >= 0) | (np.maximum(x1, x2) >= 0))


@pytest.fixture(scope="module", params=[(f, ipd) for f in sorted(CULL_FRAMES) for ipd in ("0.064", "5pct")], ids=lambda p: f"{p[0]}-{p[1]}")
def ods_pano(request):
    name, ipd = request.param
    W, H, hf, vf = CULL_FRAMES[name]
    s = P.headline_pano_setup(W, H, hf, vf)
    size = float(np.linalg.norm(s["pmax"].astype(np.float64) - s["pmin"]))
    s["od"] = O.params(hf, vf, ipd=0.064 if ipd == "0.064" else 0.05 * size)
    s["mask"] = O.cull_mask(s["cam"], s["od"], W, H, s["pmin"], s["pmax"], s["sph_center"], s["sph_radius"])
    s["name"] = f"{name}, ipd {ipd}"
    return s


def test_ods_culled_fraction(ods_pano):
    m = ods_pano["mask"]
    print(f"\nODS {ods_pano['name']}: {int(m.sum())} of {m.size} pixels culled ({100 * m.mean():.2f} %)")
    assert m.mean() > 0.5


@pytest.mark.parametrize("jitter", ["corners", "one_ulp_inside", "random"])
def test_ods_culled_pixels_miss_for_every_jitter(ods_pano, jitter):
    """Each culled pixel's rays, from their own origin', miss the root box and the sphere under the oracle's float32 arithmetic."""
    from test_miss_cull_cpu import box_hits
    s = ods_pano
    cam, W, H, od = s["cam"], s["W"], s["H"], s["od"]
    ys, xs = np.nonzero(s["mask"])
    one_m = np.nextafter(f32(1), f32(0)); tiny = np.nextafter(f32(0), f32(1))
    if jitter == "corners":
        js = [(a, b) for a in (f32(0), f32(1)) for b in (f32(0), f32(1))]
    elif jitter == "one_ulp_inside":
        js = [(a, b) for a in (tiny, one_m) for b in (tiny, one_m)]
    else:
        rng = np.random.RandomState(7)
        js = [(rng.rand(len(xs)).astype(f32), rng.rand(len(xs)).astype(f32)) for _ in range(2)]
    step = 1 << 20
    for jx, jy in js:
        for i in range(0, len(xs), step):
            sl = slice(i, i + step)
            jxs = jx[sl] if np.ndim(jx) else np.full(len(xs[sl]), jx, f32)
            jys = jy[sl] if np.ndim(jy) else np.full(len(xs[sl]), jy, f32)
            org, llc, _, _ = O.ods_camera(cam, od, W, H, xs[sl], ys[sl], jxs, jys)
            b = (llc - org).astype(f32)
            assert (b != 0).all() and (org != 0).all(), "a culled sample would take the literal order"
            n = np.sqrt(((b[:, 0] * b[:, 0]).astype(f32) + (b[:, 1] * b[:, 1]).astype(f32) + (b[:, 2] * b[:, 2]).astype(f32)).astype(f32)).astype(f32)
            d = [(b[:, k] / n).astype(f32) for k in range(3)]
            o = [org[:, k] for k in range(3)]
            assert not box_hits(s["pmin"], s["pmax"], o, d).any(), "a culled pixel's ray hits the root box"
            assert not _sphere_hits(s["sph_center"], s["sph_radius"], o, d).any(), "a culled pixel's ray hits the sphere"


def test_ods_cull_bound_holds_every_origin(headline):
    cam = headline["cam"]
    od = O.params(ipd=2.0)
    R, _ = O.cull_bounds(cam, od)
    x, y, jx, jy = random_pixels(4096, 2048, 20000, 4)
    org, _, _, _ = O.ods_camera(cam, od, 4096, 2048, x, y, jx, jy)
    d = np.abs(org.astype(np.float64) - np.asarray(cam["origin"], np.float64)).max()
    assert d <= R and R < 1.01 * float(od["half_ipd"]) + 1e-5
    assert O.cull_bounds(dict(cam, u=(cam["u"] * f32(1.01)).astype(f32)), od) is None
    assert O.cull_bounds(dict(cam, origin=np.array([cam["origin"][0], 0.5, cam["origin"][2]], f32)), O.params(ipd=2.0)) is None
