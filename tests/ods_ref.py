"""NumPy restatement of the omni-directional stereo camera (ods_camera in vpt_frame.cuh).  Used by tests/test_ods_cpu.py and
tests/test_ods_gpu.py.

Pixel (x, y) at jitter (jx, jy): the layout gives the eye e (-1 left, +1 right), the row y_e within the eye and the eye's height H_e;
(phi, theta) and b0 are the equirectangular projection's (projection_ref) at (W, H_e), row y_e; the pole merge k is 1 for |theta| <= from,
0 for |theta| >= to, (to - |theta|) * inv_span in between; s = (e ipd/2) k, r = cos phi u + sin phi w, origin' = fma(s, r, origin) and
lower_left_corner' = origin' + b0, in float32 with the kernel's operation order.  np.sin / np.cos stand in for __sinf / __cosf (within
1e-6 of them), so origin' and llc' agree with the kernel to a few ulp; e and k do not depend on them and agree bit for bit.
"""
import numpy as np

import projection_ref as P

f32 = np.float32
LEFT, RIGHT, OVER_UNDER = 0, 1, 2                     # VPT_ODS_* of vpt_b200.h


def params(hfov_deg=360.0, vfov_deg=180.0, ipd=0.064, layout=OVER_UNDER, merge=(60.0, 75.0)):
    """The projection as vpt_set_projection_ods rounds it to float."""
    rad = np.pi / 180.0
    lo, hi = float(merge[0]), float(merge[1])
    return dict(hfov=f32(hfov_deg * rad), vfov=f32(vfov_deg * rad), half_ipd=f32(float(f32(ipd)) / 2.0), layout=layout,
                merge_from=f32(lo * rad), merge_to=f32(hi * rad), inv_span=f32(1.0 / ((hi - lo) * rad)) if hi > lo else f32(0.0))


def eye_rows(layout, H, y):
    """(e, y_e, H_e) of global row y."""
    y = np.asarray(y)
    if layout == OVER_UNDER:
        top = y >= H // 2
        return np.where(top, f32(-1), f32(1)), np.where(top, y - H // 2, y), H // 2
    return np.full(y.shape, f32(-1) if layout == LEFT else f32(1)), y, H


def pole_merge(od, theta):
    at = np.abs(np.asarray(theta, np.float32))
    mid = ((od["merge_to"] - at).astype(f32) * od["inv_span"]).astype(f32)
    return np.where(at <= od["merge_from"], f32(1), np.where(at >= od["merge_to"], f32(0), mid)).astype(f32)


def _fma(a, b, c):
    """float32 fma: the float64 product of two floats is exact, one rounding of the sum (a second one to float32 is rare and ignored)."""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(f32)


def ods_camera(cam, od, W, H, x, y, jx, jy):
    """-> origin' [..., 3], lower_left_corner' [..., 3], e, k (float32)."""
    e, ye, He = eye_rows(od["layout"], H, y)
    phi, theta = P.pano_angles(od["hfov"], od["vfov"], W, He, x, ye, jx, jy)
    b0 = P.pano_b0(cam, od["hfov"], od["vfov"], W, He, x, ye, jx, jy)
    k = pole_merge(od, theta)
    s = (np.where(e < 0, -od["half_ipd"], od["half_ipd"]).astype(f32) * k).astype(f32)
    sp, cp = np.sin(phi), np.cos(phi)
    org, llc = [], []
    for c in range(3):
        r = _fma(cp, f32(cam["u"][c]), (sp * f32(cam["w"][c])).astype(f32))
        o = _fma(s, r, f32(cam["origin"][c]))
        org.append(o)
        llc.append((o + b0[..., c]).astype(f32))
    return np.stack(org, -1), np.stack(llc, -1), e, k


def cull_bounds(cam, od):
    """(R, delta) of ods_cull_bounds in vpt_kernels.cu, or None when the camera cannot be culled."""
    U, V, Wd = (np.asarray(cam[k], np.float64) for k in ("u", "v", "w"))
    M = np.stack([U, V, Wd], axis=1)
    e = float(np.abs(M.T @ M - np.eye(3)).max())
    if not e < 1e-4:
        return None
    u24, s3 = 2.0 ** -24, np.sqrt(3.0)
    rb = np.sqrt((1 + 2 * e) * (1 + 1e-5)) + s3 * 2 * u24
    h = abs(float(od["half_ipd"]))
    o = np.abs(np.asarray(cam["origin"], np.float64))
    R = (h * rb + s3 * u24 * (o.max() + h * rb)) * (1 + 1e-12)
    err = s3 * 2 * u24 * (o.max() + R + 2)
    if not (np.isfinite(R) and o.min() > R and err < 0.45):
        return None
    return R, float(np.arcsin(min(1.0, err / (0.9 - err))))


def cull_mask(cam, od, W, H, pmin, pmax, sph_center, sph_radius):
    """uint8 [H, W] of k_miss_cull_ods, in double: the equirectangular cull (projection_ref.cull_mask) of each eye's rows from the camera
    origin, with the root box grown by R on every axis, the sphere grown by R (line_misses_sphere's growth taken at distance L + R), alpha
    widened by delta, and every direction component further than alpha + SLACK from 0."""
    from miss_cull_ref import SLACK, STRIP, box_planes
    out = np.zeros((H, W), np.uint8)
    b = cull_bounds(cam, od)
    pmin = np.asarray(pmin, np.float64); pmax = np.asarray(pmax, np.float64)
    if b is None or cam["lens_radius"] != 0.0 or not np.all(pmin <= pmax) or not np.all(np.isfinite(np.r_[pmin, pmax])):
        return out
    R, delta = b
    U, V, Wd = (np.asarray(cam[k], np.float64) for k in ("u", "v", "w"))
    M = np.stack([U, V, Wd], axis=1)
    e = float(np.abs(M.T @ M - np.eye(3)).max())
    k = np.sqrt((1 + 3 * e) / (1 - 3 * e))
    o = np.asarray(cam["origin"], np.float64)
    a = np.asarray(sph_center, np.float64) - o
    L2 = float(a @ a)
    L = np.sqrt(L2) + R
    r2 = (np.sqrt(1.02 * float(sph_radius) ** 2 + 2e-3 * L * L + 1e-6) + R) ** 2
    if not (np.isfinite(r2) and L2 > r2):
        return out
    y = np.arange(H)
    _, ye, He = eye_rows(od["layout"], H, y)
    x0 = np.arange(0, W, STRIP); x1 = np.minimum(x0 + STRIP, W)
    ys = np.repeat(ye[:, None], len(x0), axis=1)
    p0, t0 = P.pano_angles(od["hfov"], od["vfov"], W, He, np.broadcast_to(x0, ys.shape), ys, 0.0, 0.0)
    p1, t1 = P.pano_angles(od["hfov"], od["vfov"], W, He, np.broadcast_to(x1, ys.shape), ys, 0.0, 1.0)
    p0, p1, t0, t1 = (q.astype(np.float64) for q in (p0, p1, t0, t1))
    pc, tc = (p0 + p1) / 2, (t0 + t1) / 2
    cmax = np.where((t0 <= 0) & (t1 >= 0), 1.0, np.maximum(np.cos(t0), np.cos(t1)))
    alpha = (t1 - t0) / 2 + cmax * (p1 - p0) / 2 + 2 * np.arcsin((k - 1) / (k + 1)) + delta
    ok = alpha + SLACK < np.pi / 2
    f = (np.cos(tc)[..., None] * (np.sin(pc)[..., None] * U - np.cos(pc)[..., None] * Wd) + np.sin(tc)[..., None] * V)
    f /= np.linalg.norm(f, axis=-1, keepdims=True)
    ok &= (np.abs(f) > (alpha + SLACK)[..., None]).all(-1)
    lim = -np.sin(alpha + SLACK)
    box_miss = np.zeros(ys.shape, bool)
    for n in box_planes(o, pmin - R, pmax + R):
        box_miss |= f @ n < lim
    gamma = alpha + np.arcsin(np.sqrt(r2 / L2)) + SLACK
    sph_miss = f @ (a / np.sqrt(L2)) < np.cos(gamma)
    out[:] = np.repeat((ok & box_miss & sph_miss).astype(np.uint8), STRIP, axis=1)[:, :W]
    return out
