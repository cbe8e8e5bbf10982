"""k_miss_cull restated in NumPy (tests/miss_cull_ref.py) on the headline frame: how much it culls, and that every pixel it culls is a miss
for every jitter under the CPU oracle's camera, box and sphere arithmetic (oracle/vpt_oracle.c: get_ray, box_intersect, sphere_intersect)."""
import numpy as np
import pytest

import miss_cull_ref as M

f32 = np.float32
SPP = 64


@pytest.fixture(scope="module")
def headline():
    s = M.headline_setup()
    s["mask"] = M.cull_mask(s["cam"], s["W"], s["H"], s["pmin"], s["pmax"], s["sph_center"], s["sph_radius"])
    return s


def oracle_ray(cam, W, H, x, y, jx, jy):
    """vpt_oracle.c's pinhole ray in float32: u = (x + jx) / W, dir = normalize(llc + u h + v vv - origin), each operation rounded."""
    u = ((x.astype(f32) + jx).astype(f32) / f32(W)).astype(f32)
    v = ((y.astype(f32) + jy).astype(f32) / f32(H)).astype(f32)
    d = [(((f32(cam["lower_left_corner"][k]) + (f32(cam["horizontal"][k]) * u).astype(f32)).astype(f32)
           + (f32(cam["vertical"][k]) * v).astype(f32)).astype(f32) - f32(cam["origin"][k])).astype(f32) for k in range(3)]
    n = np.sqrt(((d[0] * d[0]).astype(f32) + (d[1] * d[1]).astype(f32) + (d[2] * d[2]).astype(f32)).astype(f32)).astype(f32)
    return [(c / n).astype(f32) for c in d]


def box_hits(pmin, pmax, o, d):
    """box_intersect of vpt_oracle.c (AABB.h:182-205) in float32, vectorised."""
    with np.errstate(divide="ignore", invalid="ignore"):
        t = []
        for k in range(3):
            inv = (f32(1) / d[k]).astype(f32)
            t.append(((f32(pmin[k]) - f32(o[k])) * inv).astype(f32)); t.append(((f32(pmax[k]) - f32(o[k])) * inv).astype(f32))
    tmin = np.fmax(np.fmax(np.fmin(t[0], t[1]), np.fmin(t[2], t[3])), np.fmin(t[4], t[5]))
    tmax = np.fmin(np.fmin(np.fmax(t[0], t[1]), np.fmax(t[2], t[3])), np.fmax(t[4], t[5]))
    hit = (tmax > 0) & ~(tmin > tmax)
    tmin = np.where(tmin < 0, tmax, tmin)
    return hit & ~(tmin < 0)


def sphere_hits(c, r, o, d):
    """sphere_intersect of vpt_oracle.c (geometry.h:114-137) in float32, vectorised."""
    oc = [f32(o[k]) - f32(c[k]) for k in range(3)]
    A = ((d[0] * d[0]).astype(f32) + (d[1] * d[1]).astype(f32) + (d[2] * d[2]).astype(f32)).astype(f32)
    B = (f32(2) * ((d[0] * oc[0]).astype(f32) + (d[1] * oc[1]).astype(f32) + (d[2] * oc[2]).astype(f32)).astype(f32)).astype(f32)
    C = f32(sum(float(f32(v) * f32(v)) for v in oc) - float(f32(r) * f32(r)))
    discr = ((B * B).astype(f32) - (f32(4) * A * C).astype(f32)).astype(f32)
    ok = discr >= 0
    sq = np.sqrt(np.maximum(discr, 0)).astype(f32)
    q = np.where(B < 0, f32(-0.5) * (B - sq), f32(-0.5) * (B + sq)).astype(f32)
    with np.errstate(divide="ignore", invalid="ignore"):
        x1 = (q / A).astype(f32); x2 = (C / q).astype(f32)
    lo, hi = np.minimum(x1, x2), np.maximum(x1, x2)
    return ok & ((lo >= 0) | (hi >= 0))


def test_headline_culled_fraction_and_saving(headline):
    m = headline["mask"]
    frac = float(m.mean())
    culled = int(m.sum())
    tiles = m.reshape(headline["H"] // 4, 4, headline["W"] // 32, 32).all(axis=(1, 3)).mean()
    records = culled * SPP
    print(f"\nheadline: {culled} of {m.size} pixels culled ({100 * frac:.1f} %), {100 * tiles:.1f} % of the 32x4 tiles wholly; "
          f"{records / 1e6:.1f} M miss records per {SPP}-pass step not written ({records * 16 / 1e9:.2f} GB) and not read back "
          f"({records * 16 / 1e9:.2f} GB); k_resolve reads {records * 8 / 1e9:.2f} GB of L2-resident jitter table instead")
    assert 0.5 < frac < 0.7                  # the dragon's root box covers part of the frame; ~70 % of the samples are misses


@pytest.mark.parametrize("jitter", ["corners", "one_minus_ulp", "random"])
def test_culled_pixels_miss_for_every_jitter(headline, jitter):
    s = headline
    cam, W, H = s["cam"], s["W"], s["H"]
    ys, xs = np.nonzero(s["mask"])
    assert len(xs) > 0
    one_m = np.nextafter(f32(1), f32(0))
    if jitter == "corners":
        js = [(a, b) for a in (f32(0), f32(1)) for b in (f32(0), f32(1))]
    elif jitter == "one_minus_ulp":
        js = [(one_m, one_m), (f32(0), one_m), (one_m, f32(0)), (f32(0.5), one_m)]
    else:
        rng = np.random.RandomState(11)
        js = [(rng.rand(len(xs)).astype(f32), rng.rand(len(xs)).astype(f32)) for _ in range(4)]
    o = cam["origin"]
    for jx, jy in js:
        d = oracle_ray(cam, W, H, xs, ys, jx, jy)
        assert all(np.all(c != 0) for c in d)
        assert not box_hits(s["pmin"], s["pmax"], o, d).any(), "a culled pixel's ray hits the root box"
        assert not sphere_hits(s["sph_center"], s["sph_radius"], o, d).any(), "a culled pixel's ray hits the sphere"
        # and the kernel's own b0 (the fma chain) keeps the strict signs the cull relied on
        b0 = M.pinhole_b0(cam, W, H, xs, ys, jx, jy)
        assert np.all(np.sign(b0) == np.sign(M.pinhole_b0(cam, W, H, xs, ys, f32(0), f32(0))))


def test_pixels_next_to_the_silhouette_are_kept(headline):
    """Sanity of the margin: every pixel with a box-hitting jitter is kept, and the kept band around the hits is narrow."""
    s = headline
    cam, W, H = s["cam"], s["W"], s["H"]
    ys, xs = np.mgrid[0:H, 0:W]
    d = oracle_ray(cam, W, H, xs.ravel(), ys.ravel(), f32(0.5), f32(0.5))
    hit = box_hits(s["pmin"], s["pmax"], cam["origin"], d).reshape(H, W)
    assert not (hit & (s["mask"] == 1)).any()
    kept_miss = (~hit) & (s["mask"] == 0)
    assert kept_miss.mean() < 0.05


def test_thin_lens_and_degenerate_scenes_cull_nothing(headline):
    s = headline
    lens = dict(s["cam"], lens_radius=0.1)
    assert not M.cull_mask(lens, 64, 36, s["pmin"], s["pmax"], s["sph_center"], s["sph_radius"]).any()
    zero_o = dict(s["cam"], origin=np.array([0.0, 14.2, 15.0], np.float32))
    assert not M.cull_mask(zero_o, 64, 36, s["pmin"], s["pmax"], s["sph_center"], s["sph_radius"]).any()
    empty = (np.full(3, 3.4e38, np.float32), np.full(3, -3.4e38, np.float32))
    assert not M.cull_mask(s["cam"], 64, 36, *empty, s["sph_center"], s["sph_radius"]).any()
    inside = dict(s["cam"], origin=((s["pmin"] + s["pmax"]) / 2).astype(np.float32))
    assert not M.cull_mask(inside, 64, 36, s["pmin"], s["pmax"], s["sph_center"], s["sph_radius"]).any()
    # a sphere straight ahead of pixel (6, 32) of a 64x36 frame (u = 0.1, v = 0.9: far from the box) keeps that pixel
    toward = (s["cam"]["lower_left_corner"] + s["cam"]["horizontal"] * 0.1 + s["cam"]["vertical"] * 0.9 - s["cam"]["origin"])
    c = s["cam"]["origin"] + 3.0 * toward / np.linalg.norm(toward)
    assert M.cull_mask(s["cam"], 64, 36, s["pmin"], s["pmax"], s["sph_center"], s["sph_radius"])[32, 6] == 1
    assert M.cull_mask(s["cam"], 64, 36, s["pmin"], s["pmax"], c, 0.3)[32, 6] == 0
