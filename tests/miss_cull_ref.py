"""NumPy restatement of k_miss_cull (vpt_kernels.cu): which pixels of a pinhole frame cannot reach the volume's root box or the
reference sphere with any jitter, and so need no sample record.  Used by tests/test_miss_cull_cpu.py.

A pixel is culled when
  * the camera is a pinhole (lens_radius == 0, no origin component exactly 0: the condition under which k_generate builds the
    pinhole ray, b0 = lower_left_corner + u * horizontal + v * vertical - origin, before any random draw);
  * pixels are tested in strips of STRIP pixels of a row.  Every component of b0 at the four corners of the strip's jitter range
    (x + jx from x0 to x1, y + jy from y to y + 1) has one strict sign, away from 0 by 1e-3 of |b0|.  Each float operation of that
    expression is monotone in x + jx and y + jy, so every b0 of the strip lies in the box D spanned by the four corner values:
    k_generate takes the pinhole branch for every sample of those pixels;
  * a plane through the camera origin separates the cone over D from the root box: all box corners on one side, every d of D at
    least kSlack * |d| inside the other.  Candidate planes: the three coordinate planes and the planes through two box corners
    (the facets of the cone over the box);
  * the sphere, grown as in line_misses_sphere (r'^2 = 1.02 r^2 + 2e-3 |c - o|^2 + 1e-6), lies outside a circular cone around D
    widened by kSlack.
"""
import ctypes as C

import numpy as np

SLACK = 1e-3           # angular margin (radians): ~8000 float ulps, against the normalize and the slab / quadratic arithmetic
SIGN_MARGIN = 1e-3     # |b0_c| > SIGN_MARGIN * max|b0| at all four corners
STRIP = 4              # pixels of one row tested together (k_miss_cull's kCullStrip)
PLANE_TOL = 1e-9       # a box corner this close to a candidate plane (relative, double rounding) still counts as on it

f32 = np.float32


def _fma32(a, b, c):
    # float32 a*b is exact in float64; the sum is then rounded twice (float64, float32): equal to a fused multiply-add except in
    # ties far below the margins used here
    return (np.float64(a) * np.float64(b) + np.float64(c)).astype(np.float32)


def pinhole_b0(cam, W, H, x, y, jx, jy):
    """b0 of k_generate's pinhole ray in float32: (x + jx) / W, (y + jy) / H, then the fma chain and the subtraction."""
    x = np.asarray(x, dtype=np.float32); y = np.asarray(y, dtype=np.float32)
    u = ((x + np.asarray(jx, dtype=np.float32)).astype(np.float32) / f32(W)).astype(np.float32)
    v = ((y + np.asarray(jy, dtype=np.float32)).astype(np.float32) / f32(H)).astype(np.float32)
    out = []
    for k in range(3):
        inner = _fma32(cam["horizontal"][k], u, cam["lower_left_corner"][k])
        out.append((_fma32(cam["vertical"][k], v, inner) - f32(cam["origin"][k])).astype(np.float32))
    return np.stack(out, axis=-1)


def is_pinhole(cam):
    o = cam["origin"]
    return cam["lens_radius"] == 0.0 and o[0] != 0.0 and o[1] != 0.0 and o[2] != 0.0


def box_planes(o, pmin, pmax):
    """Unit normals n (float64) with n . (corner - o) >= 0 for every root-box corner: the candidate separating planes."""
    o = np.asarray(o, np.float64)
    corners = np.array([[(pmax if (i >> a) & 1 else pmin)[a] for a in range(3)] for i in range(8)], dtype=np.float64) - o
    cands = [np.eye(3)[k] * s for k in range(3) for s in (1.0, -1.0)]
    for i in range(8):
        for j in range(i + 1, 8):
            n = np.cross(corners[i], corners[j])
            cands += [n, -n]
    out = []
    for n in cands:
        ln = np.linalg.norm(n)
        if not ln > 0.0:
            continue
        n = n / ln
        if np.all(corners @ n >= -PLANE_TOL * np.linalg.norm(corners, axis=1)):
            out.append(n)
    return np.array(out).reshape(-1, 3)


def cull_mask(cam, W, H, pmin, pmax, sph_center, sph_radius, rows=None):
    """uint8 [len(rows), W]: 1 = every jitter of the pixel misses both the root box and the sphere (see the module text)."""
    rows = np.arange(H) if rows is None else np.asarray(rows)
    out = np.zeros((len(rows), W), dtype=np.uint8)
    pmin = np.asarray(pmin, np.float64); pmax = np.asarray(pmax, np.float64)
    if not is_pinhole(cam) or not np.all(pmin <= pmax) or not np.all(np.isfinite(np.r_[pmin, pmax])):
        return out
    o = np.asarray(cam["origin"], np.float64)
    x0 = np.arange(0, W, STRIP); x1 = np.minimum(x0 + STRIP, W)
    ys = np.repeat(np.asarray(rows)[:, None], len(x0), axis=1)
    cs = np.stack([pinhole_b0(cam, W, H, np.broadcast_to(xe, ys.shape), ys, 0.0, jy).astype(np.float64)
                   for xe in (x0, x1) for jy in (0.0, 1.0)])                                                          # [4, R, strips, 3]
    lo, hi = cs.min(axis=0), cs.max(axis=0)
    big = np.abs(cs).max(axis=(0, 3))
    signs = np.all((lo > SIGN_MARGIN * big[..., None]) | (hi < -SIGN_MARGIN * big[..., None]), axis=-1)

    # the eight corners of D; |d| is convex, so its largest value over D is at a corner
    dc = np.stack([np.stack([np.where((i >> a) & 1, hi[..., a], lo[..., a]) for a in range(3)], axis=-1) for i in range(8)])   # [8, R, W, 3]
    dmax = np.linalg.norm(dc, axis=-1).max(axis=0)
    mid, half = (lo + hi) / 2, (hi - lo) / 2
    box_miss = np.zeros_like(signs)
    for n in box_planes(o, pmin, pmax):
        worst = mid @ n + np.abs(half) @ np.abs(n)             # max over D of n . d
        box_miss |= worst + SLACK * dmax < 0.0

    a = np.asarray(sph_center, np.float64) - o
    L2 = float(a @ a)
    r2 = 1.02 * float(sph_radius) ** 2 + 2e-3 * L2 + 1e-6
    if not (np.isfinite(r2) and L2 > r2):
        return out
    alpha = np.arcsin(np.sqrt(r2 / L2))
    f = dc.sum(axis=0); f /= np.linalg.norm(f, axis=-1, keepdims=True)
    du = dc / np.linalg.norm(dc, axis=-1, keepdims=True)
    theta = np.arccos(np.clip(np.einsum("kijc,ijc->kij", du, f), -1.0, 1.0)).max(axis=0)   # cone around f holding all of D
    beta = np.arccos(np.clip(f @ (a / np.sqrt(L2)), -1.0, 1.0))
    sph_miss = beta > theta + alpha + SLACK
    out[:] = np.repeat((signs & box_miss & sph_miss).astype(np.uint8), STRIP, axis=1)[:, :W]
    return out


def camera_dict(cam):
    g = lambda v: np.array([v.x, v.y, v.z], dtype=np.float32)
    return dict(origin=g(cam.origin), lower_left_corner=g(cam.lower_left_corner), horizontal=g(cam.horizontal), vertical=g(cam.vertical),
                lens_radius=float(cam.lens_radius))


def headline_setup(width=1920, height=1080, fov=30.0, aperture=0.0):
    """The headline frame's camera, root box and sphere, built on the host exactly as Scene / Renderer build them (no GPU)."""
    import vpt_b200 as V
    from vpt_b200 import _native as N
    from vpt_b200.scene import load_vdb_grid, instance_xform
    _, meta = load_vdb_grid(V.find_asset("dragon.vdb"), "density")
    g = N.GPU_VDB()
    g.vdb_info.bmin = N.f3(*[float(b) for b in meta["bbox_min"]]); g.vdb_info.bmax = N.f3(*[float(b) for b in meta["bbox_max"]])
    X = instance_xform(np.array(meta["xform"], dtype=np.float32), (0, 0, 0), (0, 0, 0, 1), 1.0)
    for a in range(4):
        for b in range(4):
            g.xform[a][b] = float(X[a][b])
    b6 = (C.c_float * 6)()
    N.lib.vpt_volume_bounds(C.byref(g), b6)
    b = np.array(list(b6), dtype=np.float32)
    pmin, pmax = b[:3] - f32(1), b[3:] + f32(1)                    # vpt_octree_build: the union of instance bounds, +-1
    # Scene.world_bounds / frame_camera: the instance corners through the xform, the origin included
    lo = np.zeros(3, np.float32); hi = np.zeros(3, np.float32)
    for corner, agg in ((meta["bbox_min"], "lo"), (meta["bbox_max"], "hi")):
        p = np.array([corner[0], corner[1], corner[2], 1.0], dtype=np.float32)
        w = np.array([np.dot(X[r], p) for r in range(3)], dtype=np.float32)
        lo, hi = (np.minimum(lo, w), hi) if agg == "lo" else (lo, np.maximum(hi, w))
    center = (hi + lo) / f32(2)
    lookfrom = center + f32(float(np.linalg.norm(hi - lo)))
    cam = N.camera()
    N.lib.vpt_camera_look_at(C.byref(cam), N.fvec(lookfrom), N.fvec(center), N.fvec((0, 1, 0)), float(fov), float(width) / float(height), float(aperture))
    return dict(cam=camera_dict(cam), W=width, H=height, pmin=pmin, pmax=pmax, sph_center=np.array([0, 1000, 0], np.float32), sph_radius=1.0)
