"""float64 restatement of the motion vectors (vpt_set_motion_vectors, include/vpt_b200.h; DESIGN.md section 8o) for the tests: the film
projection of a camera, the per-sample vector and the running mean.

A camera is anything with the four fields the projection reads -- a ctypes vpt_camera or a dict of 3-vectors -- and points are (..., 3)
arrays.  Nothing here reads the reference sources or binaries built from them."""
import numpy as np

FIELDS = ("origin", "lower_left_corner", "horizontal", "vertical")


def fields(cam):
    """The four projection fields of `cam` as float64 3-vectors."""
    if isinstance(cam, dict):
        return {f: np.asarray(cam[f], dtype=np.float64) for f in FIELDS}
    return {f: np.array([getattr(getattr(cam, f), a) for a in "xyz"], dtype=np.float64) for f in FIELDS}


def project(cam, P, W, H):
    """(st, ok): pi_K(P) = (s W, t H) of camera K for points P (..., 3), and whether P is in front of K with a finite result.
    d = P - origin, e = llc - origin, n = horizontal x vertical, k = (e . n) / (d . n), q = k d - e = s horizontal + t vertical."""
    f = fields(cam)
    o, h, v = f["origin"], f["horizontal"], f["vertical"]
    e = f["lower_left_corner"] - o
    n = np.cross(h, v)
    d = np.asarray(P, dtype=np.float64) - o
    with np.errstate(divide="ignore", invalid="ignore"):
        k = (e @ n) / (d @ n)
        q = k[..., None] * d - e
        hh, hv, vv = h @ h, h @ v, v @ v
        qh, qv = q @ h, q @ v
        if hv == 0.0:
            s, t = qh / hh, qv / vv
        else:
            det = hh * vv - hv * hv
            s, t = (vv * qh - hv * qv) / det, (hh * qv - hv * qh) / det
        st = np.stack([s * W, t * H], axis=-1)
    ok = (k > 0) & np.isfinite(st).all(axis=-1)
    return st, ok


def film_point(cam, x, y, jx, jy, W, H, dist=1.0):
    """The point at `dist` times b0 along the pinhole ray through film position (x + jx, y + jy): origin + dist * b0,
    b0 = llc + s horizontal + t vertical - origin with s = (x + jx) / W, t = (y + jy) / H."""
    f = fields(cam)
    s, t = (np.asarray(x, np.float64) + jx) / W, (np.asarray(y, np.float64) + jy) / H
    b0 = f["lower_left_corner"] - f["origin"] + s[..., None] * f["horizontal"] + t[..., None] * f["vertical"]
    return f["origin"] + np.asarray(dist, np.float64)[..., None] * b0


def sample_vectors(a, b, P, covered, W, H):
    """The per-sample vector pi_B(P) - pi_A(P) where `covered` (c = depth > 0) holds and both projections are valid, else 0: (..., 2)."""
    pa, oka = project(a, P, W, H)
    pb, okb = project(b, P, W, H)
    keep = np.asarray(covered, bool) & oka & okb
    return np.where(keep[..., None], pb - pa, 0.0)


def lens_point(stream, accept, t2, t3):
    """The accepted lens point (2 vdc2[i] - 1, 2 vdc3[j] - 1) of the lens rejection loop on `stream` (a tests/motion_ref.py Stream; accept,
    t2, t3: its accept_table and vdc_table(2), vdc_table(3)), as float64 of the float32 table values; the stream is left at the shutter
    draw.  The thin-lens ray starts at origin + lens_radius (p.x u + p.y v)."""
    while True:
        i = int(np.float32(stream.next() * np.float32(100)))
        j = int(np.float32(stream.next() * np.float32(100)))
        if accept[i, j]:
            return 2.0 * float(t2[i]) - 1.0, 2.0 * float(t3[j]) - 1.0


def running_mean(x, s, iteration, max_interactions):
    """One pass of accum's rule: iteration 0 assigns, iteration < max_interactions updates x + (s - x) / (iteration + 1), later passes
    keep x."""
    x, s = np.asarray(x, np.float64), np.asarray(s, np.float64)
    if iteration == 0:
        return s.copy()
    if iteration < max_interactions:
        return x + (s - x) / (iteration + 1)
    return x.copy()
