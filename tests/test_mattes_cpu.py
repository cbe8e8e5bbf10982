"""Instance mattes without a GPU: the prefix rule that names the instance of an accepted collision (tests/matte_ref.py, restating
include/vpt_b200.h), the binning of samples to mattes, and the binned running means."""
import numpy as np

from matte_ref import SPHERE, accepted, collision_entry, matte_bins, matte_means, prefix_sums


def leaf_lists(seed, n_lists=400):
    """random instance lists up to 600 long: positive, zero and negative densities, some lists all zero or all negative"""
    rng = np.random.default_rng(seed)
    for j in range(n_lists):
        n = int(rng.integers(1, 601)) if j % 4 else int(rng.integers(1, 9))
        d = rng.lognormal(-1.0, 2.0, n).astype(np.float32)
        d[rng.random(n) < 0.3] = 0.0
        neg = rng.random(n) < (0.5 if j % 7 == 0 else 0.1)
        d[neg] = -d[neg]
        if j % 23 == 0:
            d[:] = 0.0
        yield d


def test_last_prefix_is_the_list_order_sum():
    for d in leaf_lists(1):
        acc = np.float32(0.0)
        for v in d:
            acc = np.float32(acc + v)
        assert prefix_sums(d)[-1].tobytes() == acc.tobytes()


def test_every_accepted_collision_finds_an_instance():
    rng = np.random.default_rng(2)
    n_accepted = 0
    for d in leaf_lists(3):
        density = prefix_sums(d)[-1]
        inv_max = np.float32(1.0 / max(float(np.abs(d).sum()), 1e-3) * rng.uniform(0.5, 1.0))
        t = np.float32(inv_max * density)
        # u one ulp either side of the threshold, and random draws in [0, 1)
        for u in (np.nextafter(t, np.float32(-np.inf)), t, np.nextafter(t, np.float32(np.inf)), *rng.random(4).astype(np.float32)):
            if not accepted(inv_max, density, u):
                continue
            n_accepted += 1
            i = collision_entry(inv_max, d, u)
            assert 0 <= i < len(d)
            # i is the first entry that passes: no earlier prefix does
            p = prefix_sums(d)
            assert not (np.float32(inv_max) * p[:i] > u).any()
    assert n_accepted > 300


def test_the_threshold_is_strict():
    d = np.array([0.25, 0.25], np.float32)
    inv_max = np.float32(1.0)
    assert collision_entry(inv_max, d, np.float32(0.25)) == 1              # 0.25 > 0.25 fails, 0.5 > 0.25 passes
    assert collision_entry(inv_max, d, np.nextafter(np.float32(0.25), np.float32(0))) == 0
    assert collision_entry(inv_max, d, np.float32(0.5)) == -1              # not accepted: no instance is asked for
    # a negative density first: the prefix is not monotone, "first i" still names the instance
    d = np.array([-0.5, 0.75, 0.25], np.float32)
    assert collision_entry(inv_max, d, np.float32(0.2)) == 1
    assert collision_entry(inv_max, d, np.float32(0.3)) == 2


def test_matte_bins():
    depth = np.array([1.0, 2.0, 0.0, np.nan, 3.0, 4.0, -1.0, 5.0], np.float32)
    ids = np.array([0, 2, 1, 1, SPHERE, 1, 0, 3], np.uint64)
    assert matte_bins(depth, ids, [0, -1, 1, 1], sphere=1).tolist() == [0, 1, -1, -1, 1, -1, -1, 1]
    assert matte_bins(depth, ids, [0, -1, 1, 1]).tolist() == [0, 1, -1, -1, -1, -1, -1, 1]


def test_means_identities():
    """K = 1 with everything mapped is the AOV restatement; the mattes of a full map sum to the AOVs up to rounding"""
    rng = np.random.default_rng(5)
    P = 40
    values = rng.uniform(0, 2, (P, 3)).astype(np.float32)
    depth = np.where(rng.random(P) < 0.6, rng.uniform(0.5, 9, P), 0.0).astype(np.float32)
    ids = rng.integers(0, 5, P).astype(np.uint64)
    ids[rng.random(P) < 0.1] = SPHERE
    one = matte_means(values, matte_bins(depth, ids, [0] * 5, sphere=0), 0)
    # the AOVs: alpha = mean of [depth > 0], volume = mean of the sample where depth > 0
    a, v = np.float32(0), np.zeros(3, np.float32)
    for p in range(P):
        c = depth[p] > 0
        s_a, s_v = np.float32(1.0 if c else 0.0), (values[p] if c else np.zeros(3, np.float32))
        if p == 0:
            a, v = s_a, s_v.copy()
        else:
            n = np.float32(p + 1)
            a = a + (s_a - a) / n
            v = v + (s_v - v) / n
    assert one[3].tobytes() == np.float32(a).tobytes() and one[:3].tobytes() == v.astype(np.float32).tobytes()
    table = [0, 1, 2, 3, 1]
    bins = matte_bins(depth, ids, table, sphere=2)
    total = sum(matte_means(values, bins, k).astype(np.float64) for k in range(4))
    assert np.allclose(total, one, rtol=1e-5, atol=1e-6)
