"""NumPy restatement of the instance mattes (include/vpt_b200.h, vpt_set_instance_mattes).

Which instance.  The walk accepts a collision when pmul(inv_max, density) > u, density the float32 sum over the start leaf's instance list
in list order at the collision point.  The instance is the first list entry i whose prefix sum (entries 0..i, the same float32 additions)
passes the same test.

Means.  Matte k of a pixel keeps, pass by pass, accum's running mean of the coverage sample [id maps to k] and of the colour sample (the
sample where its id maps to k, +0 elsewhere); a sample the NaN / Inf guard replaced gives every matte its own mean as colour."""
import numpy as np

SPHERE = 0xFFFFFFFF                      # kMatteSphereId: the id of a camera ray that hit the sphere before the volume box


def prefix_sums(densities):
    """float32 prefix sums in list order, added one by one as leaf_density adds them"""
    out = np.empty(len(densities), np.float32)
    acc = np.float32(0.0)
    for i, d in enumerate(np.asarray(densities, np.float32)):
        acc = np.float32(acc + d)
        out[i] = acc
    return out


def accepted(inv_max, density, u):
    return bool(np.float32(np.float32(inv_max) * np.float32(density)) > np.float32(u))


def collision_entry(inv_max, densities, u):
    """the first list position whose prefix passes the acceptance test, -1 when none does"""
    p = prefix_sums(densities)
    ok = np.float32(inv_max) * p > np.float32(u)        # float32 products, round to nearest (pmul)
    hit = np.flatnonzero(ok)
    return int(hit[0]) if hit.size else -1


def matte_bins(depth, ids, matte_of, sphere=-1):
    """-> int array shaped like `depth`: the matte of each sample, -1 for none (depth not > 0, or an id mapped to none)"""
    d = np.asarray(depth, np.float32)
    ids = np.asarray(ids, np.uint64)
    table = np.asarray(matte_of, np.int64)
    out = np.full(d.shape, -1, np.int64)
    with np.errstate(invalid="ignore"):
        c = d > 0
    inst = c & (ids != SPHERE)
    out[inst] = table[ids[inst].astype(np.int64)]
    out[c & (ids == SPHERE)] = sphere
    return out


def matte_means(values, bins, k, it0=0, max_interactions=1 << 30, guarded=None, prev=None):
    """float32 running means (r, g, b, w) of matte k for one pixel over its passes: values (P, 3), bins (P,); guarded (P,) marks the samples
    the guard replaced; prev: the buffer's previous content (read at iteration 0 by a guarded sample only)"""
    x = np.zeros(4, np.float32) if prev is None else np.asarray(prev, np.float32).copy()
    for p, (v, b) in enumerate(zip(np.asarray(values, np.float32), bins)):
        it = it0 + p
        cov = np.float32(1.0 if b == k else 0.0)
        if guarded is not None and guarded[p]:
            col = x[:3].copy()
        else:
            col = v if b == k else np.zeros(3, np.float32)
        if it == 0:
            x = np.concatenate([col, [cov]]).astype(np.float32)
        elif it < max_interactions:
            n = np.float32(it + 1)
            x[:3] = x[:3] + (col - x[:3]) / n
            x[3] = x[3] + (cov - x[3]) / n
    return x
