"""NumPy restatement of the equirectangular projection (pano_angles / pano_b0 in vpt_frame.cuh) and of its miss cull
(k_miss_cull_equirect, pano_strip_culled in vpt_kernels.cu).  Used by tests/test_projection_cpu.py.

Pixel (x, y) at jitter (jx, jy): s = (x + jx) / W, t = (y + jy) / H, phi = (s - 1/2) hfov, theta = (t - 1/2) vfov, and the ray is
(origin, normalize(b0)) with b0 = cos theta (sin phi u - cos phi w) + sin theta v.

A strip of STRIP pixels of a row is culled when
  * the camera has no lens and its basis M = [u v w] is orthonormal up to e < 1e-4 in every entry of M^T M - I;
  * its float angles, [phi(x0), phi(x1)] x [theta(y), theta(y + 1)], fit in a cone around the direction f of the range's centre of
    half-angle alpha = dtheta / 2 + max cos(theta) dphi / 2 + 2 asin((k - 1) / (k + 1)) (k^2 = (1 + 3e) / (1 - 3e)), with
    alpha + SLACK < pi / 2;
  * a candidate plane n of the root box (miss_cull_ref.box_planes) has f . n < -sin(alpha + SLACK);
  * the grown sphere (as in the pinhole cull) is further than alpha + SLACK from f.
"""
import ctypes as C

import numpy as np

from miss_cull_ref import SLACK, STRIP, box_planes

f32 = np.float32


def pano_angles(hfov, vfov, W, H, x, y, jx, jy):
    """phi, theta of pano_angles in float32."""
    s = ((np.asarray(x, np.float32) + np.asarray(jx, np.float32)).astype(f32) / f32(W)).astype(f32)
    t = ((np.asarray(y, np.float32) + np.asarray(jy, np.float32)).astype(f32) / f32(H)).astype(f32)
    return ((s - f32(0.5)).astype(f32) * f32(hfov)).astype(f32), ((t - f32(0.5)).astype(f32) * f32(vfov)).astype(f32)


def pano_b0(cam, hfov, vfov, W, H, x, y, jx, jy):
    """b0 of pano_b0 in float32 (np.sin / np.cos in place of __sinf / __cosf: within 1e-6 of them)."""
    phi, th = pano_angles(hfov, vfov, W, H, x, y, jx, jy)
    sp, cp, st, ct = np.sin(phi), np.cos(phi), np.sin(th), np.cos(th)
    out = []
    for k in range(3):
        h = (sp * f32(cam["u"][k]) - (cp * f32(cam["w"][k])).astype(f32)).astype(f32)
        out.append((st * f32(cam["v"][k]) + (ct * h).astype(f32)).astype(f32))
    return np.stack(out, axis=-1)


def oracle_dir(cam, hfov, vfov, W, H, x, y, jx, jy):
    """The traced direction, normalize(b0), in float32 as the reference kernel's normalize does it (per-operation rounding)."""
    b = pano_b0(cam, hfov, vfov, W, H, x, y, jx, jy)
    d = [b[..., k] for k in range(3)]
    n = np.sqrt(((d[0] * d[0]).astype(f32) + (d[1] * d[1]).astype(f32) + (d[2] * d[2]).astype(f32)).astype(f32)).astype(f32)
    return [(c / n).astype(f32) for c in d]


def cull_mask(cam, hfov, vfov, W, H, pmin, pmax, sph_center, sph_radius, rows=None):
    """uint8 [len(rows), W]: 1 = every jitter of the pixel misses both the root box and the sphere (see the module text)."""
    rows = np.arange(H) if rows is None else np.asarray(rows)
    out = np.zeros((len(rows), W), dtype=np.uint8)
    pmin = np.asarray(pmin, np.float64); pmax = np.asarray(pmax, np.float64)
    if cam["lens_radius"] != 0.0 or not np.all(pmin <= pmax) or not np.all(np.isfinite(np.r_[pmin, pmax])):
        return out
    U, V, Wd = (np.asarray(cam[k], np.float64) for k in ("u", "v", "w"))
    M = np.stack([U, V, Wd], axis=1)
    e = float(np.abs(M.T @ M - np.eye(3)).max())
    if not e < 1e-4:
        return out
    k = np.sqrt((1 + 3 * e) / (1 - 3 * e))
    o = np.asarray(cam["origin"], np.float64)
    a = np.asarray(sph_center, np.float64) - o
    L2 = float(a @ a)
    r2 = 1.02 * float(sph_radius) ** 2 + 2e-3 * L2 + 1e-6
    if not (np.isfinite(r2) and L2 > r2):
        return out
    x0 = np.arange(0, W, STRIP); x1 = np.minimum(x0 + STRIP, W)
    ys = np.repeat(rows[:, None], len(x0), axis=1)
    p0, t0 = pano_angles(hfov, vfov, W, H, np.broadcast_to(x0, ys.shape), ys, 0.0, 0.0)
    p1, t1 = pano_angles(hfov, vfov, W, H, np.broadcast_to(x1, ys.shape), ys, 0.0, 1.0)
    p0, p1, t0, t1 = (q.astype(np.float64) for q in (p0, p1, t0, t1))
    pc, tc = (p0 + p1) / 2, (t0 + t1) / 2
    cmax = np.where((t0 <= 0) & (t1 >= 0), 1.0, np.maximum(np.cos(t0), np.cos(t1)))
    alpha = (t1 - t0) / 2 + cmax * (p1 - p0) / 2 + 2 * np.arcsin((k - 1) / (k + 1))
    ok = alpha + SLACK < np.pi / 2
    f = (np.cos(tc)[..., None] * (np.sin(pc)[..., None] * U - np.cos(pc)[..., None] * Wd) + np.sin(tc)[..., None] * V)
    f /= np.linalg.norm(f, axis=-1, keepdims=True)
    lim = -np.sin(alpha + SLACK)
    box_miss = np.zeros(ys.shape, bool)
    for n in box_planes(o, pmin, pmax):
        box_miss |= f @ n < lim
    gamma = alpha + np.arcsin(np.sqrt(r2 / L2)) + SLACK
    sph_miss = f @ (a / np.sqrt(L2)) < np.cos(gamma)
    out[:] = np.repeat((ok & box_miss & sph_miss).astype(np.uint8), STRIP, axis=1)[:, :W]
    return out


def camera_dict(cam):
    g = lambda v: np.array([v.x, v.y, v.z], dtype=np.float32)
    return dict(origin=g(cam.origin), u=g(cam.u), v=g(cam.v), w=g(cam.w), lens_radius=float(cam.lens_radius))


def headline_pano_setup(W=4096, H=2048, hfov_deg=360.0, vfov_deg=180.0):
    """A panorama from the headline camera position (miss_cull_ref.headline_setup: the root box and the sphere), looking at the root box's
    centre; hfov / vfov are rounded to float32 radians as vpt_set_projection rounds them."""
    import miss_cull_ref as M
    from vpt_b200 import _native as N
    s = M.headline_setup()
    centre = ((s["pmin"] + s["pmax"]) / f32(2)).astype(f32)
    cam = N.camera()
    N.lib.vpt_camera_look_at(C.byref(cam), N.fvec(s["cam"]["origin"]), N.fvec(centre), N.fvec((0, 1, 0)), 30.0, 1.0, 0.0)
    return dict(cam=camera_dict(cam), W=W, H=H, hfov=f32(np.deg2rad(hfov_deg)), vfov=f32(np.deg2rad(vfov_deg)),
                pmin=s["pmin"], pmax=s["pmax"], sph_center=s["sph_center"], sph_radius=s["sph_radius"])
