"""Restatement of camera motion (vpt_set_camera_motion, include/vpt_b200.h) for the tests: which Philox draw of a pixel's stream is its
shutter draw xi, and the camera xi gives.

A camera sample of the reference (camera::get_ray) runs the lens rejection loop -- two draws per trial, each mapped through
vanDerCorput(int(draw * 100)) in bases 2 and 3 -- and then takes one more draw, the shutter time; xi is that draw.  The draws come from
the plain-C oracle's Philox block function (orc_philox_block, pinned to Random123's vectors and curand's stream addressing by
tests/test_oracle_cpu.py).  The acceptance of a trial is decided exactly (fractions) over the 101 x 101 table pairs, so the restatement
does not depend on how a float library rounds the fma of the test."""
import ctypes as C
from fractions import Fraction

import numpy as np

FIELDS = ("origin", "lower_left_corner", "horizontal", "vertical", "u", "v")


def vdc_table(base):
    """vanDerCorput(n), n = 0..100, in float32 (camera.h:49-62; the division is IEEE here, see accept_table for why that is enough)."""
    out = []
    for n0 in range(101):
        n, r, denom, inv = n0, np.float32(0), np.float32(1), np.float32(1) / np.float32(base)
        while n:
            denom = np.float32(denom * np.float32(base))
            r = np.float32(r + np.float32(np.float32(n % base) / denom))
            n = int(np.float32(np.float32(n) * inv))
        out.append(r)
    return np.array(out, dtype=np.float32)


def _rn32(q):
    """Fraction -> the nearest float32 (ties to even), as a Fraction.  float(q) rounds to double first, so the float32 it rounds to may
    be one step off (double rounding): the nearest of it and its two neighbours is the answer."""
    f = np.float32(float(q))
    cands = [f, np.nextafter(f, np.float32(-np.inf)), np.nextafter(f, np.float32(np.inf))]
    best = min(cands, key=lambda c: (abs(Fraction(float(c)) - q), int(np.array(c).view(np.int32)) & 1))
    return Fraction(float(best))


def accept_table(t2=None, t3=None):
    """accept[i, j]: the trial with table entries vdc2[i], vdc3[j] ends the loop, i.e. fma(px, px, py * py) < 1 in float32 with
    px = fma(a, 2, -1), py = fma(b, 2, -1) (each rounded once, as the kernels compute them)."""
    t2 = vdc_table(2) if t2 is None else t2
    t3 = vdc_table(3) if t3 is None else t3
    px = [_rn32(2 * Fraction(float(a)) - 1) for a in t2]
    py = [_rn32(2 * Fraction(float(b)) - 1) for b in t3]
    pyy = [_rn32(p * p) for p in py]
    return np.array([[_rn32(p * p + q) < 1 for q in pyy] for p in px], dtype=bool)


def unit(u32):
    """curand_uniform: x * 2^-32 + 2^-33 in float32 with one rounding (exact in float64 before it)."""
    return np.float32(float(np.float32(u32)) * 2.0 ** -32 + 2.0 ** -33)


class Stream:
    """The Philox stream of global pixel `idx` at pass `iteration` (curand_init(idx, 0, iteration * 4096))."""

    def __init__(self, lib, idx, iteration):
        self.lib, self.key, self.base, self.k, self.blk = lib, idx, ((iteration * 4096) & 0xffffffff) >> 2, 0, {}

    def next(self):
        b = self.k >> 2
        if b not in self.blk:
            c = self.base + b
            out = (C.c_uint32 * 4)()
            self.lib.orc_philox_block(c & 0xffffffff, c >> 32, self.key, out)
            self.blk = {b: tuple(out)}
        v = self.blk[b][self.k & 3]
        self.k += 1
        return unit(v)


def shutter_draw(stream, accept):
    """(xi, index of the draw): the lens loop on `stream`, then the shutter draw."""
    while True:
        i = int(np.float32(stream.next() * np.float32(100)))
        j = int(np.float32(stream.next() * np.float32(100)))
        if accept[i, j]:
            break
    k = stream.k
    return stream.next(), k


def oracle_lib():
    import oracle_cpu
    lib = C.CDLL(oracle_cpu.LIB)
    lib.orc_philox_block.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(C.c_uint32)]; lib.orc_philox_block.restype = None
    return lib


def shutter_draws(width, height, iteration, rows=None, lib=None):
    """float32 (len(rows), width) xi of every pixel of the given global rows (default: all) at pass `iteration`."""
    lib = lib or oracle_lib()
    acc = accept_table()
    rows = range(height) if rows is None else rows
    return np.array([[shutter_draw(Stream(lib, y * width + x, iteration), acc)[0] for x in range(width)] for y in rows], dtype=np.float32)


def camera_fields(cam):
    """The six interpolated fields of a ctypes camera as a (6, 3) float32 array."""
    return np.array([[getattr(getattr(cam, f), c) for c in "xyz"] for f in FIELDS], dtype=np.float32)


def lerp64(o, c, xi):
    """float64 o + xi (c - o) of (6, 3) poses at draws xi (any shape): (..., 6, 3)."""
    o, c = o.astype(np.float64), c.astype(np.float64)
    return o + np.asarray(xi, dtype=np.float64)[..., None, None] * (c - o)
