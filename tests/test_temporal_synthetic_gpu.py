"""The temporal filter and its layers on the GPU against the NumPy restatement (tests/temporal_ref.py, tests/temporal_layers_ref.py), on
synthetic frames passed in through the C ABI (vpt_temporal, vpt_temporal_layers) on a bare context: every max_history and clip_sigma
value with and without history and display words, from 1x1 to the 65535-pixel caps; q on the frame edge and one float32 step either
side of it, integer px, non-finite and huge motions; B == A, a skewed B and a B turned away from the environment under every kind of
M.z; non-finite, +-3e38, denormal, negative and cancelling colours, histories and lengths; and up to 16 layers of 1 to 4 channels.

The restatement decides the footprint in the kernel's float32 order (footprint_dt, motion_dt) and makes the kernel's float32 decisions
(diff32, clip32, ftz), so the taps, `used` and L are the device's.  Every pixel is checked (temporal_ref.compare): L bit for bit; a pixel
without history, and every layer value there, equals its input bit for bit; non-finite values match in kind; every finite value is
within 1e-5 + RTOL M, M the largest finite |value| the pixel read.  Display words, for every pixel, are within 1 LSB of the packing of
the device's own colour with the device's NaN rules."""
import ctypes as C

import numpy as np
import pytest
import torch

import vpt_b200 as V
from vpt_b200 import _native as N
import temporal_layers_ref as TL
import temporal_ref as T

pytestmark = pytest.mark.gpu
F32 = np.float32
INF = float("inf")
FLT_MAX = float(np.finfo(np.float32).max)
DENORMAL = float(F32(1e-40))
MAX_HISTORY = (1, 2, 3, 16, 1 << 24)
CLIP = (DENORMAL, 0.25, 1.5, 64.0, FLT_MAX, INF)
SIZES = [(1, 1), (1, 2), (2, 1), (31, 9), (33, 9), (97, 41), (65535, 2), (2, 65535)]
LENGTHS = np.array([np.nan, np.inf, -np.inf, 0, -1, -0.5, 2.5, 2 ** 24, 2 ** 25], np.float32)
WORST = {}                                                     # label -> the largest |d| / (1e-5 + M), printed per test


@pytest.fixture(scope="module")
def ctx():
    c = C.c_void_p(0)
    assert V.lib.vpt_create(C.byref(c)) == 0
    yield c
    torch.cuda.synchronize()
    V.lib.vpt_destroy(c)


def look_at(frm, at, w, h, fov=35.0):
    cam = N.camera()
    V.lib.vpt_camera_look_at(C.byref(cam), N.fvec(frm), N.fvec(at), N.fvec((0, 1, 0)), fov, w / h, 0.0)
    return cam


def cameras(w, h):
    return look_at((3.0, 2.0, 9.0), (0.2, 0.1, 0.0), w, h), look_at((3.1, 2.0, 8.9), (0.25, 0.1, 0.0), w, h)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def run(ctx, w, h, color, vectors, a, b, hist, ln, mh, clip, display, layers=None):
    """vpt_temporal (layers None) or vpt_temporal_layers of NumPy inputs; layers = [(src, history, channels, count)] with src / history
    (count, N, channels).  -> (out (N, 3), L (N,), words (N,) or None, [dst (count, N, channels)])"""
    n = w * h
    c, m = dev(color), dev(vectors)
    hh, hl = (dev(hist), dev(ln)) if hist is not None else (None, None)
    out = torch.empty(n, 3, dtype=torch.float32, device="cuda")
    out_len = torch.empty(n, dtype=torch.float32, device="cuda")
    words = torch.empty(n, dtype=torch.int32, device="cuda") if display else None
    opt = N.temporal_options(mh, clip)
    args = (ctx, w, h, ptr(c), ptr(m), C.byref(a), C.byref(b), ptr(hh), ptr(hl), C.byref(opt), 1.0, ptr(out), ptr(out_len), ptr(words))
    keep, dsts = [], []
    if layers is None:
        rc = V.lib.vpt_temporal(*args, None)
    else:
        descs = []
        for src, lh, ch, k in layers:
            s, d = dev(src), torch.empty(k * n * ch, dtype=torch.float32, device="cuda")
            hs = dev(lh) if lh is not None else None
            keep += [s, hs]; dsts.append((d, ch, k))
            descs.append(N.temporal_layer(s.data_ptr(), hs.data_ptr() if hs is not None else None, d.data_ptr(), ch, k))
        arr = (N.temporal_layer * max(1, len(descs)))(*descs)
        rc = V.lib.vpt_temporal_layers(*args, arr, len(descs), None)
    assert rc == 0, V.lib.vpt_last_error(ctx).decode()
    torch.cuda.synchronize()
    got_words = words.cpu().numpy().view(np.uint32) if display else None
    return (out.cpu().numpy(), out_len.cpu().numpy(), got_words, [d.cpu().numpy().reshape(k, n, ch) for d, ch, k in dsts])


def check(label, w, h, color, vectors, a, b, hist, ln, mh, clip, got, layers=()):
    """Every pixel of the device's beauty, lengths, display words and layers against the restatement -> the restatement's dict"""
    out, L, words, dsts = got
    ref = T.temporal(w, h, color, vectors, a, b, hist, ln, max_history=mh, clip_sigma=clip, motion_dt=F32, footprint_dt=F32)
    want_L = ref["L"].astype(F32)
    bad = L.view(np.uint32) != want_L.view(np.uint32)
    assert not bad.any(), f"{label}: {int(bad.sum())} history lengths differ, first {np.flatnonzero(bad)[0]}: " \
                          f"{L[bad][0]} vs {want_L[bad][0]}"
    copied = ~ref["used"]
    fails, st = T.compare(out, ref["out"], color, copied, ref["M"])
    assert not fails, f"{label}: " + "; ".join(fails)
    worst = st["ratio"]
    if words is not None:
        want = T.display_words(out)
        lsb = max(int(np.abs(((words >> s) & 0xff).astype(int) - ((want >> s) & 0xff).astype(int)).max()) for s in (0, 8, 16))
        assert lsb <= 1 and (words >> 24 == 0xff).all(), f"{label}: display words {lsb} LSB away"
    for i, ((src, lh, ch, k), dst) in enumerate(zip(layers, dsts)):
        want = TL.blend_layer(ref, src, lh, ch, k)
        M = TL.layer_reach(ref, src, lh, ch, k)
        for p in range(k):
            fails, s = T.compare(dst[p], want[p], src[p], copied, M[p])
            assert not fails, f"{label}, layer {i} ({ch} ch) plane {p}: " + "; ".join(fails)
            worst = max(worst, s["ratio"])
    key = label.split(":")[0]
    WORST[key] = max(WORST.get(key, 0.0), worst)
    return ref


@pytest.fixture(autouse=True)
def report(request):
    WORST.clear()
    yield
    for k, v in WORST.items():
        print(f"[{request.node.name}] {k}: worst |d| / (1e-5 + M) {v:.3g}")


def frame(w, h, seed, hostile=False):
    """Colours, premultiplied vectors, histories and lengths: fractional and integer motions under M.z in {0, 0.3, 1}, 5 % off the frame.
    hostile: NaN / +-inf in single channels of C and H, every kind of length, +-3e38 blocks of alternating sign in C and H, denormals,
    negative colours, cancelling histories (+-1e30 side by side) and M.z in {NaN, -0.5, 0, 1 - 2^-24, 1, 2}."""
    rng = np.random.default_rng(seed)
    n = w * h
    lo = -1.0 if hostile else 0.0
    c = rng.uniform(lo, 2.0, (n, 3)).astype(F32)
    hist = rng.uniform(lo, 2.0, (n, 3)).astype(F32)
    ln = rng.integers(1, 12, n).astype(F32)
    m = np.zeros((n, 3), F32)
    zs = [np.nan, -0.5, 0.0, 1 - 2.0 ** -24, 1.0, 2.0] if hostile else [0.0, 0.3, 1.0]
    m[:, 2] = rng.choice(np.array(zs, F32), n)
    frac = rng.random(n) < 0.5
    m[:, :2] = np.where(frac[:, None], rng.uniform(-3.0, 3.0, (n, 2)), rng.integers(-3, 4, (n, 2)))
    m[:, :2] *= np.where(np.isfinite(m[:, 2:3]) & (m[:, 2:3] > 0), m[:, 2:3], 1)
    far = rng.random(n) < 0.05
    m[far, :2] = 1e4
    if not hostile:
        return c, m, hist, ln
    pick = lambda frac: rng.random(n) < frac
    for val, frac in ((np.nan, 0.02), (np.inf, 0.01), (-np.inf, 0.01)):
        c[pick(frac), rng.integers(0, 3)] = val
        hist[pick(frac), rng.integers(0, 3)] = val
    sel = pick(0.3)
    ln[sel] = rng.choice(LENGTHS, int(sel.sum()))
    c[pick(0.02)] = F32(3e-39)                                                  # denormal colours
    hist[pick(0.02), rng.integers(0, 3)] = F32(-7e-40)
    cancel = np.flatnonzero(pick(0.03))
    hist[cancel] = F32(1e30); hist[(cancel + 1) % n] = F32(-1e30)                # side by side: a bilinear mean cancels
    for arr, off in ((c, 0), (hist, n // 3)):                                   # 3x3 blocks of +-3e38, alternating sign
        y, x = divmod((n // 2 + off) % n, w)
        for dy in range(3):
            for dx in range(3):
                if y + dy < h and x + dx < w:
                    arr[(y + dy) * w + x + dx] = F32(3e38 if (dx + dy) % 2 == 0 else -3e38)
    return c, m, hist, ln


# ---- 1. the options, every size ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("wh", SIZES)
def test_every_option_at_every_size(ctx, wh):
    """Every (max_history, clip_sigma) pair with history, display words on every other call; then no history, with and without display"""
    w, h = wh
    a, b = cameras(w, h)
    c, m, hist, ln = frame(w, h, w * 7 + h)
    k = 0
    for mh in MAX_HISTORY:
        for clip in CLIP:
            got = run(ctx, w, h, c, m, a, b, hist, ln, mh, clip, display=k % 2 == 0)
            check(f"{w}x{h} max_history {mh} clip {clip:g}: ", w, h, c, m, a, b, hist, ln, mh, clip, got)
            k += 1
    for display in (False, True):
        got = run(ctx, w, h, c, m, a, b, None, None, 16, 1.5, display)
        ref = check(f"{w}x{h} no history", w, h, c, m, a, b, None, None, 16, 1.5, got)
        assert not ref["used"].any() and (got[1] == 1).all()
    if w * h > 100:
        ref = T.temporal(w, h, c, m, a, b, hist, ln, motion_dt=F32, footprint_dt=F32)
        assert ref["used"].any() and (~ref["used"]).any()


# ---- 2. the frame edge ---------------------------------------------------------------------------------------------------------------

def edge_motions(w, h, seed):
    """Per-pixel motions (M.z = 1, 2 or NaN: v = M.xy) putting q on 0, W or H, one float32 step inside or outside them, px on an integer,
    or v at +-inf, NaN or +-1e30; the other axis fractional or on an integer."""
    rng = np.random.default_rng(seed)
    n = w * h
    y, x = np.divmod(np.arange(n), w)
    m = np.zeros((n, 3), F32)
    m[:, 2] = rng.choice(np.array([1.0, 2.0, np.nan], F32), n)
    m[:, :2] = np.where(rng.random((n, 1)) < 0.5, rng.uniform(-2, 2, (n, 2)), rng.integers(-2, 3, (n, 2)))
    for axis, pos, size in ((0, x, w), (1, y, h)):
        kind = rng.integers(0, 4, n)
        step = rng.integers(-1, 2, n)
        for i in range(n):
            if kind[i] == 3:
                continue                                                    # the other axis decides
            if kind[i] == 2:                                                    # px = q - 1/2 an integer
                m[i, axis] = F32(np.floor(rng.uniform(0, size)) - pos[i])
                continue
            edge = F32(0.0 if kind[i] == 0 else size)
            target, toward = edge, F32(np.inf if step[i] > 0 else -np.inf)
            for _ in range(abs(step[i])):
                target = np.nextafter(target, toward)
            v = F32(np.float64(target) - (pos[i] + 0.5))
            if F32(pos[i] + 0.5) + v != target:                                 # q one step of v past the edge instead
                v = F32(np.float64(edge) - (pos[i] + 0.5))
                for _ in range(abs(step[i])):
                    v = np.nextafter(v, toward)
            m[i, axis] = v
    special = rng.random(n) < 0.04
    m[special, rng.integers(0, 2)] = rng.choice(np.array([np.inf, -np.inf, np.nan, 1e30, -1e30], F32), int(special.sum()))
    return m


@pytest.mark.parametrize("wh", [(1, 1), (2, 1), (1, 2), (31, 9), (33, 9), (97, 41), (65535, 2), (2, 65535)])
def test_q_on_the_frame_edge(ctx, wh):
    w, h = wh
    a, b = cameras(w, h)
    c, _, hist, ln = frame(w, h, w + 3 * h)
    m = edge_motions(w, h, w * h)
    if w * h > 1000:                                                        # q exactly on each edge somewhere
        y, x = np.divmod(np.arange(w * h), w)
        q = np.stack([(x + 0.5).astype(F32) + m[:, 0], (y + 0.5).astype(F32) + m[:, 1]], 1)
        for axis, size in ((0, w), (1, h)):
            assert (q[:, axis] == 0).any() and (q[:, axis] == size).any() and (q[:, axis] < 0).any() and (q[:, axis] > size).any()
    for mh, clip in ((16, INF), (3, 1.5)):
        got = run(ctx, w, h, c, m, a, b, hist, ln, mh, clip, display=True, layers=[(c[None], hist[None], 3, 1)])
        check(f"{w}x{h} edge max_history {mh} clip {clip:g}", w, h, c, m, a, b, hist, ln, mh, clip, got, [(c[None], hist[None], 3, 1)])
        assert np.array_equal(got[3][0][0].view(np.uint32), got[0].view(np.uint32)) or clip != INF, "the colour as a layer != the beauty"


# ---- 3. cameras ----------------------------------------------------------------------------------------------------------------------

def test_b_equal_to_a_reads_one_texel_bit_for_bit(ctx):
    """B == A with M.z in [0, 1) and M.xy = 0: v = +0, so every pixel reads its own texel with weight 1.  With C == H every output, and a
    layer whose src is its history, equal their inputs bit for bit."""
    w, h = 97, 41
    a, _ = cameras(w, h)
    rng = np.random.default_rng(1)
    n = w * h
    m = np.zeros((n, 3), F32)
    m[:, 2] = rng.uniform(0, 1, n).astype(F32)
    c = rng.uniform(-1, 3, (n, 3)).astype(F32)
    ln = rng.integers(1, 30, n).astype(F32)
    lay = rng.uniform(-5, 5, (2, n, 4)).astype(F32)
    for mh, clip in ((16, INF), (1 << 24, 64.0)):
        got = run(ctx, w, h, c, m, a, a, c, ln, mh, clip, True, [(lay, lay, 4, 2)])
        ref = check(f"B == A max_history {mh}", w, h, c, m, a, a, c, ln, mh, clip, got, [(lay, lay, 4, 2)])
        assert ref["used"].all() and (ref["v"] == 0).all() and not np.signbit(ref["v"]).any()
        assert np.array_equal(got[0].view(np.uint32), c.view(np.uint32)) and np.array_equal(got[3][0].view(np.uint32), lay.view(np.uint32))
        assert np.array_equal(got[1], np.minimum(ln + 1, mh))
    hist = rng.uniform(-1, 3, (n, 3)).astype(F32)
    got = run(ctx, w, h, c, m, a, a, hist, ln, 16, INF, True)
    check("B == A, C != H", w, h, c, m, a, a, hist, ln, 16, INF, got)


def test_a_skewed_b(ctx):
    """A B whose vertical is not perpendicular to its horizontal: film_project_dir solves the 2x2 system (the det branch)"""
    for w, h in ((97, 41), (33, 9)):
        a, b = cameras(w, h)
        for skew in (0.15, -0.4):
            s = N.camera.from_buffer_copy(bytes(b))
            s.vertical = N.f3(*(float(F32(getattr(b.vertical, k)) + F32(skew) * F32(getattr(b.horizontal, k))) for k in "xyz"))
            assert T.film_cam(s, F32)["hv"] != 0
            c, m, hist, ln = frame(w, h, 11, hostile=True)
            for mh, clip in ((16, INF), (2, 1.5)):
                got = run(ctx, w, h, c, m, a, s, hist, ln, mh, clip, True)
                ref = check(f"{w}x{h} skew {skew} max_history {mh}", w, h, c, m, a, s, hist, ln, mh, clip, got)
                env = m[:, 2] < 1
                assert ref["used"][env].any()


def test_a_b_turned_away_from_the_environment(ctx):
    """Every environment direction of A lies behind B: no history where M.z < 1, the vectors' motion where M.z >= 1 or NaN"""
    w, h = 97, 41
    a = look_at((3.0, 2.0, 9.0), (0.2, 0.1, 0.0), w, h)
    b = look_at((3.0, 2.0, 9.0), (5.8, 3.9, 18.0), w, h)
    c, m, hist, ln = frame(w, h, 5, hostile=True)
    got = run(ctx, w, h, c, m, a, b, hist, ln, 16, 1.5, True)
    ref = check("B turned away", w, h, c, m, a, b, hist, ln, 16, 1.5, got)
    env = m[:, 2] < 1
    assert not ref["used"][env].any() and ref["used"][~env].any()


# ---- 4. hostile values ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("wh", [(97, 41), (33, 9), (65535, 2)])
def test_hostile_values(ctx, wh):
    w, h = wh
    a, b = cameras(w, h)
    c, m, hist, ln = frame(w, h, w - h, hostile=True)
    rng = np.random.default_rng(w)
    n = w * h
    src = rng.uniform(-2, 2, (3, n, 2)).astype(F32)
    lh = rng.uniform(-2, 2, (3, n, 2)).astype(F32)
    for arr in (src, lh):
        for val in (np.nan, np.inf, -np.inf, F32(3e38), F32(-3e38), F32(2e-39)):
            arr[rng.random((3, n, 2)) < 0.01] = val
    layers = [(src, lh, 2, 3), (c[None], hist[None], 3, 1)]
    for mh in (1, 16, 1 << 24):
        for clip in (INF, 1.5, DENORMAL, FLT_MAX):
            got = run(ctx, w, h, c, m, a, b, hist, ln, mh, clip, True, layers)
            check(f"{w}x{h} hostile max_history {mh} clip {clip:g}", w, h, c, m, a, b, hist, ln, mh, clip, got, layers)


# ---- 5. layers -----------------------------------------------------------------------------------------------------------------------

def layer_set(specs, n, seed, hostile):
    rng = np.random.default_rng(seed)
    out = []
    for ch, k in specs:
        src, lh = (rng.uniform(-2, 2, (k, n, ch)).astype(F32) for _ in range(2))
        if hostile:
            for arr in (src, lh):
                for val in (np.nan, np.inf, -np.inf, F32(3e38), F32(-3e38), F32(2e-39)):
                    arr[rng.random((k, n, ch)) < 0.004] = val
        out.append((src, lh, ch, k))
    return out


@pytest.mark.parametrize("count", [1, 3, 8])
def test_layers_of_every_channel_count(ctx, count):
    w, h = 97, 41
    a, b = cameras(w, h)
    c, m, hist, ln = frame(w, h, count, hostile=True)
    layers = layer_set([(ch, count) for ch in (1, 2, 3, 4)], w * h, count, hostile=True)
    for mh, clip in ((16, INF), (3, 0.25)):
        got = run(ctx, w, h, c, m, a, b, hist, ln, mh, clip, count % 2 == 1, layers)
        check(f"count {count} max_history {mh}", w, h, c, m, a, b, hist, ln, mh, clip, got, layers)
    got = run(ctx, w, h, c, m, a, b, None, None, 16, INF, True, [(s, None, ch, k) for s, _, ch, k in layers])
    check(f"count {count} no history", w, h, c, m, a, b, None, None, 16, INF, got, [(s, None, ch, k) for s, _, ch, k in layers])


@pytest.mark.parametrize("wh", [(97, 41), (65535, 2), (2, 65535)])
def test_sixteen_layers_in_one_call(ctx, wh):
    """All 16 layers, 1 to 4 channels and counts up to 8, with hostile values; at the width and height caps too"""
    w, h = wh
    a, b = cameras(w, h)
    c, m, hist, ln = frame(w, h, 16 + w, hostile=True)
    specs = [(1 + i % 4, (1, 3, 8, 2)[i // 4]) for i in range(16)]
    layers = layer_set(specs, w * h, w, hostile=True)
    got = run(ctx, w, h, c, m, a, b, hist, ln, 16, 1.5, True, layers)
    check(f"{w}x{h} 16 layers", w, h, c, m, a, b, hist, ln, 16, 1.5, got, layers)
