"""Restatement of the collision AOVs (vpt_set_collision_aovs; DESIGN.md section 8q) in NumPy: the per-volume world -> texture coordinate
(volume_coord), the texture filter (texfilter_ref.sample), the octree leaf that contains a point and its leaf list, the central differences
of the density, the colour LUT index, the sphere branch and the running mean.

Arithmetic.  Every float32 operation the kernel rounds is rounded here at the same place: additions, subtractions and products with
numpy float32, fused multiply-adds as one rounding of the exact float64 value a * b + c (exact when a * b + c fits float64, which holds
for the small-integer and power-of-two transforms the tests build).  The kernel's fast-math divisions and reciprocal square roots are
not correctly rounded; where they enter (the LUT index argument, the albedo, the normal's length) the callers' tolerances say so.
volume_rec restates make_volume_rec in float64 and is exact only for transforms whose cofactors and determinant are exact in float32
(small integers, power-of-two scales) and for power-of-two dimensions (1 / dim is then exact whatever the reciprocal's rounding)."""
import numpy as np

import texfilter_ref as T

F32 = np.float32


def fma32(a, b, c):
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(F32)


# ---- volumes ---------------------------------------------------------------------------------------------------------------------------
def volume_rec(xform, bmin, dims):
    """make_volume_rec of a GPU_VDB with 4x4 `xform` (row-major, as GPU_VDB::xform), index-space bmin and dims (dx, dy, dz): dict of
    m [3][3], adj3 [3], idet, bmin [3], rdim [3] as float32."""
    n = np.asarray(xform, np.float64)
    inv = np.linalg.inv(n)                                  # index = inv @ (p, 1): the reference's transpose().inverse().transform_point
    det = np.linalg.det(n)
    idet = 1.0 / det
    adj = inv * det                                         # the adjugate (unscaled) entries the kernel multiplies by idet
    m = np.array([[inv[r][c] for c in range(3)] for r in range(3)])
    return dict(m=m.astype(F32), adj3=adj[:3, 3].astype(F32), idet=F32(idet), bmin=np.asarray(bmin, F32),
                rdim=(1.0 / np.asarray(dims, np.float64)).astype(F32))


def volume_coord(rec, P):
    """(uvw [n, 3] float32, inside [n]) of world points P [n, 3] float32: volume_coord's chain mul(y), fma(x), fma(z), fma(adj, idet), then
    (i - bmin) * rdim; inside = every component in [0, 1]."""
    P = np.asarray(P, F32)
    m, adj, idet = rec["m"], rec["adj3"], rec["idet"]
    out = []
    for r in range(3):
        v = fma32(adj[r], idet, fma32(P[:, 2], m[r][2], fma32(P[:, 0], m[r][0], (P[:, 1] * m[r][1]).astype(F32))))
        out.append(((v - rec["bmin"][r]).astype(F32) * rec["rdim"][r]).astype(F32))
    uvw = np.stack(out, 1)
    inside = ~((uvw < 0) | (uvw > 1)).any(1)
    return uvw, inside


def volume_density(rec, grid, P):
    """The filtered density of one volume at P (0 outside its box), and the largest corner texel |t| of each look-up (0 outside)."""
    uvw, inside = volume_coord(rec, P)
    s = T.sample(grid, np.where(inside[:, None], uvw, 0).astype(F32))
    return np.where(inside, s["value"], F32(0)), np.where(inside, np.abs(s["texels"]).max(1), F32(0))


def volume_color(rec, rgb, P):
    """volume_color: the colour grid rgb [z][y][x][3] filtered per channel at P (0 outside), (1, 1, 1) for rgb None."""
    if rgb is None:
        return np.ones((len(P), 3), F32)
    uvw, inside = volume_coord(rec, P)
    uvw = np.where(inside[:, None], uvw, 0).astype(F32)
    c = np.stack([T.sample(rgb[..., k], uvw)["value"] for k in range(3)], 1)
    return np.where(inside[:, None], c, F32(0))


# ---- the octree: leaf location and leaf lists ------------------------------------------------------------------------------------------
class Octree:
    """The flat tables of a scene's octree: root box, the 73 internal nodes' split planes and child-empty masks, the 512 leaf lists.
    nodes: {node number: OCTNode} (mixed_scenes.read_tree); leaf_lists: Scene.leaf_lists()."""

    def __init__(self, nodes, leaf_lists):
        root = nodes[0]
        self.pmin = np.array([root.bbox.pmin.x, root.bbox.pmin.y, root.bbox.pmin.z], F32)
        self.pmax = np.array([root.bbox.pmax.x, root.bbox.pmax.y, root.bbox.pmax.z], F32)
        self.half = np.zeros((73, 3), F32)
        self.empty = np.full((73, 8), True)
        for j in range(73):
            if j not in nodes or nodes[j].num_volumes <= 0:
                continue
            kids = [(1 + c if j == 0 else (9 + (j - 1) * 8 + c if j < 9 else 73 + (j - 9) * 8 + c)) for c in range(8)]
            k0 = nodes[kids[0]]
            self.half[j] = (k0.bbox.pmax.x, k0.bbox.pmin.y, k0.bbox.pmax.z)
            self.empty[j] = [kids[c] not in nodes or nodes[kids[c]].num_volumes == 0 for c in range(8)]
        self.lists = leaf_lists

    def leaf(self, X):
        """collision_leaf: the leaf index c1 * 64 + c2 * 8 + c3 of each point, -1 outside the root box or in an empty node."""
        X = np.asarray(X, F32)
        out = np.full(len(X), -1, np.int64)
        inside = ((X >= self.pmin) & (X <= self.pmax)).all(1)
        for i in np.nonzero(inside)[0]:
            p, node, leaf = X[i], 0, 0
            for lvl in range(3):
                h = self.half[node]
                c = int(not p[0] <= h[0]) + 2 * int(not p[1] >= h[1]) + 4 * int(not p[2] <= h[2])
                if self.empty[node][c]:
                    leaf = -1
                    break
                leaf = leaf * 8 + c
                node = 1 + c if lvl == 0 else 9 + (node - 1) * 8 + c
            out[i] = leaf
        return out


class Scene:
    """What rho and Cd read: the volume records and grids (volume 0 first) and, for more than one volume, the octree."""

    def __init__(self, recs, grids, colors=None, octree=None):
        self.recs, self.grids = recs, grids
        self.colors = colors or [None] * len(recs)
        self.octree = octree

    def density(self, X):
        """(rho [n] float32, error bound [n]): rho(X) and a bound on |tex3D's rho - rho| (one ulp of the largest corner texel of every
        look-up, DESIGN.md section 3a, plus one ulp of the running sum per added term); the brick and cell samplers give rho exactly."""
        X = np.asarray(X, F32)
        if len(self.recs) == 1:
            v, tmax = volume_density(self.recs[0], self.grids[0], X)
            return (F32(0) + v).astype(F32), np.spacing(tmax.astype(F32)).astype(np.float64)
        leaf = self.octree.leaf(X)
        rho = np.zeros(len(X), F32); err = np.zeros(len(X))
        per = [volume_density(r, g, X) for r, g in zip(self.recs, self.grids)]
        for i in range(len(X)):
            if leaf[i] < 0:
                continue
            for v in self.octree.lists[leaf[i]]:
                rho[i] = F32(rho[i] + per[v][0][i])
                err[i] += float(np.spacing(F32(per[v][1][i]))) + float(np.spacing(F32(abs(rho[i]) + per[v][1][i])))
        return rho, err

    def color(self, X):
        """Cd(X): fmax3(0, volume_color) of volume 0 for one volume, else the component-wise max over the leaf list (0 in no leaf)."""
        X = np.asarray(X, F32)
        if len(self.recs) == 1:
            return np.maximum(volume_color(self.recs[0], self.colors[0], X), F32(0))
        leaf = self.octree.leaf(X)
        per = [volume_color(r, c, X) for r, c in zip(self.recs, self.colors)]
        out = np.zeros((len(X), 3), F32)
        for i in range(len(X)):
            if leaf[i] >= 0:
                for v in self.octree.lists[leaf[i]]:
                    out[i] = np.maximum(out[i], per[v][i])
        return out


# ---- normal and albedo -------------------------------------------------------------------------------------------------------------------
def offsets(P, h):
    """The six points P +- h e_i, rounded as the kernel rounds them: [6, n, 3] in the order +x, -x, +y, -y, +z, -z."""
    P = np.asarray(P, F32); h = F32(h)
    out = []
    for a in range(3):
        for s in (1, -1):
            Q = P.copy()
            Q[:, a] = (P[:, a] + h).astype(F32) if s > 0 else (P[:, a] - h).astype(F32)
            out.append(Q)
    return np.stack(out)


def gradient(scene, P, h):
    """(g [n, 3] float64, bound [n, 3]): the central differences (rho(P + h e_i) - rho(P - h e_i)) / (2h) of the exact float32 densities,
    and the bound their density errors put on each component."""
    Q = offsets(P, h)
    rho, err = zip(*[scene.density(q) for q in Q])
    g = np.stack([(rho[2 * a].astype(np.float64) - rho[2 * a + 1]) / (2.0 * float(F32(h))) for a in range(3)], 1)
    e = np.stack([(err[2 * a] + err[2 * a + 1]) / (2.0 * float(F32(h))) for a in range(3)], 1)
    return g, e


def normal_of_gradient(g):
    """n = -g / |g|, (0, 0, 0) where |g| is 0 or not finite."""
    g = np.asarray(g, np.float64)
    L = np.linalg.norm(g, axis=-1, keepdims=True)
    ok = (L > 0) & np.isfinite(L)
    return np.where(ok, -g / np.where(ok, L, 1.0), 0.0)


def lut_argument(rho, max_extinction, emission_pivot):
    """rho / max_extinction * 255 / emission_pivot in float64 (the kernel's fast divisions differ by a few ulps: callers excuse ties)."""
    return np.asarray(rho, np.float64) * (1.0 / float(F32(max_extinction))) * 255.0 / float(F32(emission_pivot))


def lut_index(arg):
    """floor(clamp(arg, 0, 255)); NaN -> 0 as fmaxf(NaN, 0) gives."""
    a = np.where(np.isnan(arg), 0.0, arg)
    return np.floor(np.clip(a, 0.0, 255.0)).astype(np.int64)


def volume_albedo(albedo, Cd, lut, index, extinction, energy_inject):
    """albedo * Cd * density_color[index] / extinction * energy_inject, in float64."""
    return (np.asarray(albedo, np.float64) * np.asarray(Cd, np.float64) * np.asarray(lut, np.float64)[index]
            / np.asarray(extinction, np.float64) * float(np.float32(energy_inject)))


def sphere_normal(P, centre):
    """(P - centre) / |P - centre|: on the sphere, (P - c) / r."""
    d = np.asarray(P, np.float64) - np.asarray(centre, np.float64)
    return d / np.linalg.norm(d, axis=-1, keepdims=True)


def ray_box(org, d, pmin, pmax):
    """Entry distance of the slab test (float64), +inf on a miss."""
    with np.errstate(divide="ignore", invalid="ignore"):
        t0 = (np.asarray(pmin, np.float64) - org) / d
        t1 = (np.asarray(pmax, np.float64) - org) / d
    tmin = np.nanmax(np.minimum(t0, t1), axis=-1); tmax = np.nanmin(np.maximum(t0, t1), axis=-1)
    return np.where(tmax >= np.maximum(tmin, 0), tmin, np.inf)


def ray_sphere(org, d, centre, radius):
    """Nearest non-negative hit distance of the sphere (float64), +inf on a miss."""
    oc = org - np.asarray(centre, np.float64)
    b = (d * oc).sum(-1); cc = (oc * oc).sum(-1) - radius * radius; a = (d * d).sum(-1)
    disc = b * b - a * cc
    s = np.sqrt(np.maximum(disc, 0))
    t0 = (-b - s) / a; t1 = (-b + s) / a
    t = np.where(t0 >= 0, t0, t1)
    return np.where((disc >= 0) & (t >= 0), t, np.inf)


# ---- the running mean ----------------------------------------------------------------------------------------------------------------------
def running_mean(x, s, iteration, max_interactions):
    """One pass of accum's rule in float64: iteration 0 assigns, iteration < max_interactions updates x + (s - x) / (iteration + 1), later
    passes keep x (the kernel's float32 update with a fast division is within a few ulps of it)."""
    x, s = np.asarray(x, np.float64), np.asarray(s, np.float64)
    if iteration == 0:
        return s.copy()
    if iteration < max_interactions:
        return x + (s - x) / (iteration + 1)
    return x.copy()
