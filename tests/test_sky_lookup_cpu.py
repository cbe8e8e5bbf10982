"""The sky look-up case table (tests/sky_cases.py) restated in float64: each frame reaches every branch it claims, on pixels that stay on
their side for any jitter, and no ray of any frame can reach the volume's root box or the reference sphere.  This keeps
tests/test_sky_lookup_gpu.py from quietly ceasing to exercise a branch when a case is edited."""
import math

import numpy as np
import pytest

import sky_cases as S

MIN_PIXELS = 2                      # robust pixels required on each side of a split


@pytest.mark.parametrize("case", S.CASES, ids=S.case_id)
def test_case_reaches_its_branches(case):
    g = S.GEOMETRY[case[0]]
    claims = S.claims_of(g, case[1])
    c = S.classify(g, case[1])
    report = {k: (int((c[k] == 1).sum()), int((c[k] == -1).sum())) for k in S.SPLITS}
    print(S.case_id(case), report)
    assert claims, "a case that claims nothing tests nothing"
    for k in claims:
        if k in S.SPLITS:
            yes, no = report[k]
            assert yes >= MIN_PIXELS and no >= MIN_PIXELS, f"{k}: {yes} pixels on its true side, {no} on its false side"
        elif k == "all_past":
            assert report["past"][0] == g.size[0] * g.size[1], "not every pixel passes the atmosphere"
        elif k == "below_ground":
            assert c["r"] < S.RG
        else:
            assert S.band_present(c["mu_s"], k), f"no look-up in band {k}"


def test_every_branch_is_claimed_somewhere():
    """The table as a whole reaches both sides of every split, every mu_s band, a camera below the ground and a frame wholly past the
    atmosphere; and covers the sun elevations 90, 45, 3, -0.5, -15 and -40, each at two azimuths."""
    claimed = {k for g in S.GEOMETRIES for i in range(len(g.suns)) for k in S.claims_of(g, i)}
    assert set(S.SPLITS) | {"all_past", "below_ground", "mu_s+", "mu_s0", "mu_s-"} <= claimed
    for el in (90.0, 45.0, 3.0, -0.5, -15.0, -40.0):
        az = {s.azimuth for g in S.GEOMETRIES for s in g.suns if s.elevation == el}
        assert len(az) >= 2 or el == 90.0, (el, az)     # at the zenith the azimuth does not move the sun
    altitudes = {g.pos[1] for g in S.GEOMETRIES}
    assert {1.5, 10.0, 500.0, 2000.0, 5000.0, 12000.0, 20000.0, 40000.0, 45000.0, 59900.0, 150000.0, 1500000.0, -2.0} <= altitudes
    assert any(a < S.RT - S.RG and a > S.RT - S.RG - 2 for a in altitudes) and any(a > S.RT - S.RG and a < S.RT - S.RG + 2 for a in altitudes)


@pytest.mark.parametrize("name", list(S.GEOMETRY))
def test_frame_cannot_reach_the_volume_or_the_sphere(name):
    """Every pinhole ray has d . w = -focus / |b0| < 0 (w: the camera's backward axis), so a point p with (p - origin) . w > 0 is never
    reached at t > 0.  All eight corners of the root box and the whole sphere lie on that side, by far more than any rounding."""
    g = S.GEOMETRY[name]
    cam = S.camera(g)
    a = S.cam_arrays(cam)
    o, w = a["origin"], a["w"]
    assert abs(np.linalg.norm(w) - 1) < 1e-6
    for j in S.JITTERS:
        d = S.rays(cam, g.size, j)
        assert (d @ w).max() < -0.1                       # every frame is well inside a half space
    pos, centre = S.placement(g)
    lo, hi = S.root_box(pos)
    corners = np.array([[(hi if (i >> k) & 1 else lo)[k] for k in range(3)] for i in range(8)], np.float64)
    assert ((corners - o) @ w).min() > S.BEHIND / 2
    assert (np.asarray(centre) - o) @ w - S.SPHERE_RADIUS > S.BEHIND / 2


def test_constants_match_the_model():
    """sky_cases' copy of the model's scalars: cos(120 degrees) with pi as a float (the parameter block's mu_s_min)."""
    assert S.MU_S_MIN == float(np.float32(-0.50000006))
    assert S.SUN_ANGULAR_RADIUS == float(np.float32(0.004675))
    assert math.isclose(S.dip(45000.0), 6.8, abs_tol=0.1)
