"""Deep slices without a GPU: the binning rule's edge cases (tests/deep_ref.py, restating include/vpt_b200.h) and the host functions
deep.flatten / deep.exr_samples on synthetic slices against a float64 NumPy restatement."""
import numpy as np
import pytest
import torch

from vpt_b200 import deep
from deep_ref import slice_of

INF = float("inf")


def test_binning_edge_cases():
    b = [1.0, 2.0, 4.0, INF]
    d = np.array([1.0, 2.0, 3.999, 4.0, 1e30, INF, 0.0, -0.0, np.nan, 0.5, -3.0], np.float32)
    want = [0, 1, 1, 2, 2, 2, -1, -1, -1, -1, -1]
    assert slice_of(d, b).tolist() == want
    # a finite last bound: a depth at or beyond z_K and +inf fall in no slice
    b2 = [0.0, 1.0, 2.0]
    d2 = np.array([1e-30, 0.999, 1.0, 1.999, 2.0, 7.0, INF, 0.0], np.float32)
    assert slice_of(d2, b2).tolist() == [0, 0, 1, 1, -1, -1, -1, -1]
    # K = 1 with {0, inf} is the coverage decision of the AOVs: depth > 0
    d3 = np.array([0.0, 1e-38, 5.0, INF, np.nan], np.float32)
    assert (slice_of(d3, [0.0, INF]) == 0).tolist() == [False, True, True, True, False]


def synthetic(seed=7, K=5, H=6, W=7):
    """slices whose coverages of a pixel sum to at most 1: a Dirichlet split of a random total per pixel, with some slices empty, some
    pixels empty and some fully covered before their last slice"""
    rng = np.random.default_rng(seed)
    p = rng.dirichlet(np.ones(K + 1), size=(H, W)).astype(np.float32)[..., :K]     # (H, W, K), the rest is transmitted
    p[rng.random((H, W, K)) < 0.3] = 0.0
    p[0, 0] = 0.0                                                                  # an empty pixel
    p[1, 1] = [0.25, 0.75, 0, 0, 0]                                                # fully covered after slice 1: T_2 = 0
    p[1, 2] = [0.0, 1.0, 0, 0, 0]
    c = (p[..., None] * rng.uniform(0.1, 3.0, (H, W, K, 3))).astype(np.float32)
    s = np.concatenate([c, p[..., None]], -1).transpose(2, 0, 1, 3)                 # (K, H, W, 4)
    return np.ascontiguousarray(s)


def test_flatten_against_the_restatement():
    s = synthetic()
    K, H, W, _ = s.shape
    b = [0.0, 1.0, 1.5, 3.0, 8.0, INF]
    rng = np.random.default_rng(3)
    zmap = rng.choice([0.5, 1.0, 1.2, 3.0, 8.0, 100.0, INF], size=(H, W)).astype(np.float32)
    for z in (None, 0.0, 1.0, 1.5, 7.9, 8.0, INF, zmap):
        col, cov = deep.flatten(torch.from_numpy(s), b, z=None if z is None else (torch.from_numpy(z) if isinstance(z, np.ndarray) else z))
        zz = np.full((H, W), INF) if z is None else np.broadcast_to(np.float64(z), (H, W))
        keep = np.array(b[1:], np.float64)[:, None, None] <= zz[None]
        want = np.where(keep[..., None], s.astype(np.float64), 0.0).sum(0)
        assert col.shape == (H, W, 3) and cov.shape == (H, W)
        assert np.allclose(col.numpy(), want[..., :3], rtol=1e-6, atol=1e-7)
        assert np.allclose(cov.numpy(), want[..., 3], rtol=1e-6, atol=1e-7)
    # every slice: the sums; nothing in front of the first back bound: zero
    col, cov = deep.flatten(torch.from_numpy(s), b, z=0.5)
    assert float(col.abs().max()) == 0.0 and float(cov.abs().max()) == 0.0


def over(samples):
    """the deep 'over' of OpenEXR, front to back per pixel, in float64: -> (colour (H, W, 3), alpha (H, W))"""
    count = samples.count.numpy()
    a, rgb = samples.a.numpy().astype(np.float64), samples.rgb.numpy().astype(np.float64)
    H, W = count.shape
    col, t = np.zeros((H, W, 3)), np.ones((H, W))
    i = 0
    for y in range(H):
        for x in range(W):
            for _ in range(count[y, x]):
                col[y, x] += t[y, x] * rgb[i]
                t[y, x] *= 1.0 - a[i]
                i += 1
    assert i == len(a)
    return col, 1.0 - t


def test_exr_samples_against_the_restatement():
    s = synthetic()
    K, H, W, _ = s.shape
    b = [0.0, 1.0, 1.5, 3.0, 8.0, INF]
    e = deep.exr_samples(torch.from_numpy(s), b)
    # float64 restatement: non-empty slices, T_k, A_k = p_k / T_k, RGB_k = c_k / T_k, pixel-major then front to back
    s64 = s.astype(np.float64)
    zs, zbs, As, rgbs, counts = [], [], [], [], np.zeros((H, W), np.int64)
    for y in range(H):
        for x in range(W):
            t = 1.0
            for k in range(K):
                c, p = s64[k, y, x, :3], s64[k, y, x, 3]
                if p != 0 or (c != 0).any():
                    counts[y, x] += 1
                    zs.append(b[k]); zbs.append(b[k + 1])
                    As.append(p / t if t > 0 else 1.0); rgbs.append(c / t if t > 0 else np.zeros(3))
                t -= p
    assert e.count.tolist() == counts.tolist()
    assert counts[0, 0] == 0 and counts[1, 1] == 2 and counts[1, 2] == 1
    assert e.z.tolist() == [np.float32(v) for v in zs] and e.zback.tolist() == [np.float32(v) for v in zbs]
    assert np.allclose(e.a.numpy(), As, rtol=1e-5, atol=1e-7)
    assert np.allclose(e.rgb.numpy(), np.array(rgbs).reshape(-1, 3), rtol=1e-5, atol=1e-6)
    # the fully covered pixel: its last sample is opaque and takes the rest of the coverage
    i11 = int(counts.reshape(-1)[: 1 * W + 1].sum())
    assert e.a[i11 + 1].item() == pytest.approx(1.0, abs=1e-7)
    # compositing the samples with 'over' gives back the sums of the slices
    col, alpha = over(e)
    assert np.allclose(col, s64[..., :3].sum(0), rtol=1e-5, atol=1e-6)
    assert np.allclose(alpha, s64[..., 3].sum(0), rtol=1e-5, atol=1e-6)


def rays(seed=11, H=4, W=5, N=64):
    """per pixel N camera samples: first-collision depth (0 = miss) and premultiplied colour, float64"""
    rng = np.random.default_rng(seed)
    depth = np.where(rng.random((H, W, N)) < 0.35, 0.0, rng.uniform(0.1, 12.0, (H, W, N)))
    colour = rng.uniform(0.0, 2.0, (H, W, N, 3)) * (depth > 0)[..., None]
    return depth, colour


def slices_of(depth, colour, bounds):
    """the slices of these samples, the kernel's definition with exact means: (K, H, W, 4) float64"""
    sl = slice_of(depth, bounds)
    K = len(bounds) - 1
    s = np.zeros((K,) + depth.shape[:2] + (4,))
    for k in range(K):
        m = (sl == k).astype(np.float64)
        s[k, ..., :3] = (colour * m[..., None]).mean(2)
        s[k, ..., 3] = m.mean(2)
    return s


def test_insert_is_the_per_sample_composite():
    """deep.insert against the composite restated sample by sample: a sample whose slice lies in front of z is the volume's; otherwise the
    element covers a fraction a of it, and the rest collides behind z or reaches the plate.  An empty element gives back the flat composite
    of the AOVs, volume + (1 - alpha) * plate."""
    H, W = 4, 5
    depth, colour = rays(H=H, W=W)
    b = [0.0, 2.0, 4.0, 6.0, 9.0, INF]
    s = torch.from_numpy(slices_of(depth, colour, b))
    rng = np.random.default_rng(5)
    plate = rng.uniform(0.0, 3.0, (H, W, 3))
    a = rng.uniform(0.0, 1.0, (H, W))
    element = np.concatenate([rng.uniform(0.0, 1.0, (H, W, 3)) * a[..., None], a[..., None]], -1)
    hit = depth > 0
    volume, alpha = (colour * hit[..., None]).mean(2), hit.mean(2)
    zmap = rng.choice([2.0, 4.0, 9.0], size=(H, W))
    for z in (0.0, 2.0, 6.0, 9.0, INF, zmap):
        zz = np.broadcast_to(np.asarray(z, np.float64), (H, W))
        back = np.array(b[1:])[slice_of(depth, b).clip(0)]                   # back bound of each sample's slice
        front = hit & (back <= zz[..., None])
        for e in (element, np.zeros((H, W, 4))):
            per = np.where(front[..., None], colour,
                           e[:, :, None, :3] + (1 - e[:, :, None, 3:]) * np.where(hit[..., None], colour, plate[:, :, None, :]))
            cov = np.where(front, 1.0, e[:, :, None, 3] + (1 - e[:, :, None, 3]) * hit)
            zt = torch.from_numpy(z) if isinstance(z, np.ndarray) else z
            got_c, got_a = deep.insert(s, b, zt, torch.from_numpy(e), torch.from_numpy(plate))
            assert np.allclose(got_c.numpy(), per.mean(2), rtol=1e-12, atol=1e-12), z
            assert np.allclose(got_a.numpy(), cov.mean(2), rtol=1e-12, atol=1e-12), z
        # the empty element: the flat composite of the AOVs, at every depth
        got_c, got_a = deep.insert(s, b, zt, torch.zeros(H, W, 4, dtype=torch.float64), torch.from_numpy(plate))
        assert np.allclose(got_c.numpy(), volume + (1 - alpha)[..., None] * plate, rtol=1e-12, atol=1e-12)
        assert np.allclose(got_a.numpy(), alpha, rtol=1e-12, atol=1e-12)
    # an opaque element: the volume in front of it over the element
    opaque = np.concatenate([rng.uniform(0.0, 1.0, (H, W, 3)), np.ones((H, W, 1))], -1)
    fc, fa = deep.flatten(s, b, 4.0)
    got_c, got_a = deep.insert(s, b, 4.0, torch.from_numpy(opaque), torch.from_numpy(plate))
    assert np.allclose(got_c.numpy(), fc.numpy() + (1 - fa.numpy())[..., None] * opaque[..., :3], rtol=1e-12, atol=1e-12)
    assert np.allclose(got_a.numpy(), 1.0)


def test_shapes_are_checked():
    s = torch.zeros(3, 2, 2, 4)
    with pytest.raises(ValueError):
        deep.flatten(s, [0.0, 1.0, 2.0])
    with pytest.raises(ValueError):
        deep.exr_samples(torch.zeros(3, 2, 2, 3), [0.0, 1.0, 2.0, 3.0])
