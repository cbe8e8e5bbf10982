"""The Bruneton sky precompute (SURVEY 8(f) row N2), one kernel at a time: each of this library's six table kernels
(vpt_debug_bruneton_stage) against the reference's own compiled kernel for that stage (oracle/_ref/atmo, launched by
vptref_atmosphere_stage with atmosphere::precompute's launch shape and argument bytes), both given the same inputs.

Identical inputs: the parameter block is V.Atmosphere(...)'s (equal to the reference's field for field,
test_atmosphere_gpu.py::test_parameter_block_equals_reference) with its buffer pointers swapped for test-owned tables, and the
tables a stage reads are the REFERENCE's outputs of the stages before it: the test drives the reference chain transmittance ->
direct irradiance -> single scattering -> {scattering density, indirect irradiance, multiple scattering} for orders 2, 3, 4 one
stage at a time and hands each intermediate state to both sides.  Every table a stage writes is compared in all four channels.

Attribution by experiment: every reference table sits inside 2 MB guards on both sides, and each reference stage runs twice,
once with the guards holding 0 and once holding 3.0.  A texel whose reference output changes between the two runs read memory
outside the reference's buffers; that set is O.  This library clamps its indices to the tables, so only texels in O may differ
by construction; every texel outside O must meet the stage's bound, and the size of O is pinned per stage at its measured
value.  Measured on an H100 (sm_90a, both sides fp32 --use_fast_math from the same operand types):

    stage                 |O| per table (both option sets)                        worst rel err outside O   bound
    transmittance         0                                                       bit for bit               bit for bit
    direct irradiance     0                                                       bit for bit               bit for bit
    single scattering     Rayleigh, scattering 3982 / 3983; Mie, single Mie      bit for bit               bit for bit
                          3133 / 3137
    scattering density    0 (orders 2-4)                                          1.66e-6                   3.3e-6
    indirect irradiance   0 (orders 2-4)                                          bit for bit               bit for bit
    multiple scattering   2048 per order, delta and running table                 2.62e-4                   5.2e-4
    blend = 1, first triple's matrix: the same, except single scattering's running scattering table (|O| 3931) and single Mie
    (|O| 0); the blended running tables are bit for bit outside O except multiple scattering's (2.07e-5).

What O contains.  Single scattering reads only the transmittance table, and the reference clamps that look-up's LINEAR index to
[0, W*H] -- one texel past the end (atmosphere_kernels.cu:161-171); its O are those reads, all with the sun below the horizon
(mu_s -0.11 .. -0.24), at every r.  Multiple scattering's O are the 2048 texels of the first five mu rows (rays just below the
horizon, mu -0.004 .. -0.013) at the 2nd-5th r layers (63 m .. 1 km): their look-ups along the ray down to r = Rg leave the delta
scattering-density buffer.  Upward the coordinates of an in-range look-up stay inside the table (u_r <= 1 - 1/64, u_mu <= 1 -
1/256; the x overflow at nu = 1 enters with weight 0), so these reads land BEFORE the buffer: the ground branch's
(d - d_min) / (d_max - d_min) cancels near r = Rg and the mu coordinate goes negative in the lowest r slice.  No stage reads past
the end of a scattering buffer with non-zero weight, and scattering density and indirect irradiance read no memory outside the
reference's buffers.  The same negative coordinate in a higher r slice addresses the previous slice's last row INSIDE the buffer;
the library follows the reference's linear index there and clamps only an index outside the table, so those texels agree and O's
own differ by at most 9e-7.  Two findings of this test were fixed in vpt_bruneton.cu: the nu clamp's bounds are formed in double
and rounded once as the reference's are (single scattering was off by 6.6e-5, scattering density by 2.3e-5), and the scattering
look-up no longer clamps each texel coordinate (that per-axis clamp was the whole of the end-to-end test's 0.18 % of scattering
texels off by > 2e-3).  Multiple scattering still differs outside O by up to 2.6e-4; the operation behind it is not found yet.

Sensitivity: a build whose multiple_scattering drops the 0.5 trapezoid end weight fails test_stages_against_reference_kernels
and test_tables_against_reference_precompute[default]; one whose single scattering ignores blend_mie
fails test_blend_and_matrix_paths_against_reference_kernels and test_tables_against_reference_precompute[luminance2].

The blend and matrix paths (luminance mode PRECOMPUTED accumulates five wavelength triples through non-identity
luminance-from-radiance matrices) are driven once more from random positive running tables with blend = 1 and the first
triple's matrix, including the reference's doubling of the running irradiance in direct irradiance (it adds the value it read
after writing nothing).
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import vpt_b200 as V
from vpt_b200 import _native as N
import oracle_ref

has_atmo = os.path.exists(os.path.join(oracle_ref.REF_DIR, "atmo", "atmosphere_kernels.ptx"))
needs_atmo_build = pytest.mark.skipif(not (oracle_ref.available() and has_atmo), reason="oracle/_ref/atmo (the reference's precompute) not built")

TRANSMITTANCE, DIRECT_IRRADIANCE, SINGLE_SCATTERING = N.BRUNETON_TRANSMITTANCE, N.BRUNETON_DIRECT_IRRADIANCE, N.BRUNETON_SINGLE_SCATTERING
SCATTERING_DENSITY, INDIRECT_IRRADIANCE, MULTIPLE_SCATTERING = N.BRUNETON_SCATTERING_DENSITY, N.BRUNETON_INDIRECT_IRRADIANCE, N.BRUNETON_MULTIPLE_SCATTERING
STAGE_NAMES = ("transmittance", "direct irradiance", "single scattering", "scattering density", "indirect irradiance", "multiple scattering")

# the nine tables in the order of the parameter block's buffer pointers (definitions.h:82-90)
TABLES = ("delta_irradiance", "delta_rayleigh", "delta_mie", "delta_density", "delta_multiple", "transmittance", "irradiance", "scattering", "single_mie")
SMALL, BIG = 256 * 64, 256 * 128 * 32
COUNTS = (SMALL, BIG, BIG, BIG, BIG, SMALL, SMALL, BIG, BIG)
IRRADIANCE_TABLES = {"delta_irradiance", "irradiance", "transmittance"}
WRITES = {TRANSMITTANCE: ("transmittance",), DIRECT_IRRADIANCE: ("delta_irradiance", "irradiance"),
          SINGLE_SCATTERING: ("delta_rayleigh", "delta_mie", "scattering", "single_mie"), SCATTERING_DENSITY: ("delta_density",),
          INDIRECT_IRRADIANCE: ("delta_irradiance", "irradiance"), MULTIPLE_SCATTERING: ("delta_multiple", "scattering")}
CHAIN = [(TRANSMITTANCE, 0), (DIRECT_IRRADIANCE, 0), (SINGLE_SCATTERING, 0)] + [(s, k) for k in (2, 3, 4) for s in (SCATTERING_DENSITY, INDIRECT_IRRADIANCE, MULTIPLE_SCATTERING)]
GUARD = (2 << 20) // 16                  # float4 texels of guard before and after every table
CANARY = 3.0
IDENTITY = (1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0)
# luminance_from_radiance of the first of luminance mode PRECOMPUTED's five triples, row-major (vpt_atmosphere_host.cpp:218-223:
# wavelengths 375.67, 407, 438.33 nm, CIE 1931 -> linear sRGB times the 31.33 nm step), rounded to float as the library passes it
FIRST_TRIPLE_LFR = (0.0219768286, 0.809137344, 7.03783941, -0.0185755603, -0.705908537, -6.92410851, 0.129827589, 4.98654032, 56.9538689)
VPT_ERR_INVALID = -1                     # include/vpt_b200.h

OPTION_SETS = {"default": dict(), "solar_no_ozone": dict(use_constant_solar_spectrum=False, use_ozone=False)}

# relative error bound outside O per stage (floor 1e-6 x the channel's largest |value| in the table); None = bit for bit.  Twice the
# worst case measured (module docstring)
STAGE_BOUND = {TRANSMITTANCE: None, DIRECT_IRRADIANCE: None, SINGLE_SCATTERING: None, SCATTERING_DENSITY: 3.3e-6,
               INDIRECT_IRRADIANCE: None, MULTIPLE_SCATTERING: 5.2e-4}
BLEND_BOUND = STAGE_BOUND                # a blended table's error is taken relative to its two parts (compare), so the same bounds hold
# measured size of O: (option set, stage, order, table) -> texels; anything not listed is 0
PINNED_O = {}
for _opts, _ray, _mie in (("default", 3982, 3133), ("solar_no_ozone", 3983, 3137)):
    PINNED_O.update({(_opts, SINGLE_SCATTERING, 0, "delta_rayleigh"): _ray, (_opts, SINGLE_SCATTERING, 0, "scattering"): _ray,
                     (_opts, SINGLE_SCATTERING, 0, "delta_mie"): _mie, (_opts, SINGLE_SCATTERING, 0, "single_mie"): _mie})
    for _order in (2, 3, 4):
        PINNED_O.update({(_opts, MULTIPLE_SCATTERING, _order, "delta_multiple"): 2048, (_opts, MULTIPLE_SCATTERING, _order, "scattering"): 2048})
PINNED_O_BLEND = {("blend", SINGLE_SCATTERING, 0, "delta_rayleigh"): 3982, ("blend", SINGLE_SCATTERING, 0, "delta_mie"): 3133,
                  ("blend", SINGLE_SCATTERING, 0, "scattering"): 3931, ("blend", MULTIPLE_SCATTERING, 2, "delta_multiple"): 2048,
                  ("blend", MULTIPLE_SCATTERING, 2, "scattering"): 2048}


class Slab:
    """The nine tables in one device allocation, each inside GUARD float4 texels of guard on both sides."""

    def __init__(self):
        self.mem = torch.zeros((GUARD + sum(c + GUARD for c in COUNTS), 4), dtype=torch.float32, device="cuda")
        self.tables, self.guards = [], [self.mem[:GUARD]]
        off = GUARD
        for c in COUNTS:
            self.tables.append(self.mem[off:off + c]); off += c
            self.guards.append(self.mem[off:off + GUARD]); off += GUARD
        self.ptrs = (C.c_uint64 * 9)(*[t.data_ptr() for t in self.tables])

    def load(self, state, guard=0.0):
        for t, s in zip(self.tables, state): t.copy_(s)
        for g in self.guards: g.fill_(guard)
        torch.cuda.synchronize()

    def read(self):
        torch.cuda.synchronize()
        return [t.clone() for t in self.tables]


def run_own(slab, params, state, stage, blend, lfr, order):
    slab.load(state)
    N.check(N.lib.vpt_debug_bruneton_stage(stage, C.byref(params), slab.ptrs, (C.c_float * 9)(*lfr), blend, order), None, "vpt_debug_bruneton_stage")
    return slab.read()


def run_ref(orc, slab, params, state, stage, blend, lfr, order, guard):
    slab.load(state, guard)
    p = N.AtmosphereParameters.from_buffer_copy(bytes(params))
    p.scratch_buffers[:] = list(slab.ptrs)
    orc.atmosphere_stage(stage, p, blend=blend, lfr=lfr, order=order)
    return slab.read()


def texel_coordinates(name, i, p):
    """(x, y[, z]) of texel i and the (r, mu, mu_s, nu) or (r, mu_s) its centre stands for (the tables' parametrisation,
    atmosphere_kernels.cu:249-357, 572-586), for the report only."""
    Rg, Rt, mu_s_min = float(p.bottom_radius), float(p.top_radius), float(p.mu_s_min)
    H = np.sqrt(Rt * Rt - Rg * Rg)
    unit = lambda u, n: (u - 0.5 / n) / (1.0 - 1.0 / n)
    if name in IRRADIANCE_TABLES:
        x, y = i % 256, i // 256
        return f"({x}, {y}) -> r - Rg = {unit((y + 0.5) / 64, 64) * (Rt - Rg):.1f} m, mu_s = {2 * unit((x + 0.5) / 256, 256) - 1:.4f}"
    x, y, z = i % 256, (i // 256) % 128, i // (256 * 128)
    rho = H * unit((z + 0.5) / 32, 32); r = np.sqrt(rho * rho + Rg * Rg)
    u_mu = (y + 0.5) / 128
    if u_mu < 0.5:
        d = (r - Rg) + (rho - (r - Rg)) * unit(1 - 2 * u_mu, 64)
        mu = -1.0 if d == 0 else np.clip(-(rho * rho + d * d) / (2 * r * d), -1, 1)
    else:
        d = (Rt - r) + (rho + H - (Rt - r)) * unit(2 * u_mu - 1, 64)
        mu = 1.0 if d == 0 else np.clip((H * H - rho * rho - d * d) / (2 * r * d), -1, 1)
    A = -2 * mu_s_min * Rg / (H - (Rt - Rg)); xs = unit(((x + 0.5) % 32) / 32, 32)
    a = (A - xs * A) / (1 + xs * A); ds = (Rt - Rg) + min(a, A) * (H - (Rt - Rg))
    mu_s = 1.0 if ds == 0 else np.clip((H * H - ds * ds) / (2 * Rg * ds), -1, 1)
    nu = np.clip(np.floor((x + 0.5) / 32) / 7 * 2 - 1, -1, 1)
    return f"({x}, {y}, {z}) -> r - Rg = {r - Rg:.1f} m, mu = {mu:.5f}, mu_s = {mu_s:.4f}, nu = {nu:.3f}"


BLENDED = {DIRECT_IRRADIANCE: ("irradiance",), SINGLE_SCATTERING: ("scattering", "single_mie"), INDIRECT_IRRADIANCE: ("irradiance",),
           MULTIPLE_SCATTERING: ("scattering",)}                # the running tables a stage adds to when blend = 1


def compare(label, stage, own, ref0, ref3, state, params, blend=0):
    """Per table the stage writes: (|O|, worst relative error outside O, bit-identical outside O); prints where O lies.
    A blended table's error is relative to |prefilled| + |new term| (the new term as the reference computed it): the two parts
    cancel where the matrix has a negative row, and a result near 0 says nothing about how exactly either part was formed."""
    out = {}
    for name in WRITES[stage]:
        k = TABLES.index(name)
        a, b, b3 = (t[k].double().cpu().numpy() for t in (own, ref0, ref3))
        in_o = (b != b3).any(axis=1)
        scale = np.abs(b)
        if blend and name in BLENDED.get(stage, ()):
            prev = state[k].double().cpu().numpy()
            scale = np.abs(prev) + np.abs(b - prev)
        floor = np.maximum(1e-6 * scale.max(axis=0), 1e-30)
        rel = (np.abs(a - b) / np.maximum(scale, floor)).max(axis=1)
        outside = rel[~in_o]
        worst = float(outside.max()) if outside.size else 0.0
        exact = bool((a[~in_o] == b[~in_o]).all())
        n_o = int(in_o.sum())
        print(f"{label:38s} {name:16s} |O| = {n_o:6d}   worst rel err outside O {worst:.3g}{'  (bit for bit)' if exact else ''}"
              f"   |err| in O up to {float(rel[in_o].max()) if n_o else 0.0:.3g}")
        if n_o:
            idx = np.nonzero(in_o)[0]
            if name not in IRRADIANCE_TABLES:
                xs, ys, zs = idx % 256, (idx // 256) % 128, idx // (256 * 128)
                print(f"    O lies at y (mu) in {sorted(set(ys.tolist()))[:12]}, z (r) in {sorted(set(zs.tolist()))[:12]}, "
                      f"x (nu, mu_s) in [{xs.min()}, {xs.max()}]")
            for i in idx[:: max(1, len(idx) // 6)][:6]:
                print("      ", texel_coordinates(name, int(i), params))
        out[name] = (n_o, worst, exact)
    # a stage writes nothing but its own tables
    for k, name in enumerate(TABLES):
        if name not in WRITES[stage]:
            assert torch.equal(own[k], state[k]), f"{label}: {name} was written"
    return out


@pytest.fixture(scope="module")
def slabs():
    s = (Slab(), Slab())
    yield s
    del s
    torch.cuda.empty_cache()


def check_report(report, pins, bounds, failures):
    for key, (n_o, worst, exact) in report.items():
        bound = bounds[key[1]]
        if bound is None:
            if not exact: failures.append(f"{key}: not bit for bit outside O (worst rel err {worst:.3g})")
        elif worst > bound:
            failures.append(f"{key}: worst rel err outside O {worst:.3g} > {bound:.3g}")
        if n_o != pins.get(key, 0):
            failures.append(f"{key}: |O| = {n_o}, measured {pins.get(key, 0)}")


@pytest.mark.gpu
@needs_atmo_build
@pytest.mark.parametrize("opts", list(OPTION_SETS))
def test_stages_against_reference_kernels(slabs, opts):
    """The reference chain, one stage at a time; at every stage both kernels start from the reference's tables."""
    atm = V.Atmosphere(**OPTION_SETS[opts])
    params = atm.params
    orc = oracle_ref.RefOracle()
    own_slab, ref_slab = slabs
    state = [torch.zeros((c, 4), dtype=torch.float32, device="cuda") for c in COUNTS]
    report = {}
    for stage, order in CHAIN:
        label = f"[{opts}] {STAGE_NAMES[stage]}" + (f" order {order}" if order else "")
        ref0 = run_ref(orc, ref_slab, params, state, stage, 0, IDENTITY, order, 0.0)
        ref3 = run_ref(orc, ref_slab, params, state, stage, 0, IDENTITY, order, CANARY)
        own = run_own(own_slab, params, state, stage, 0, IDENTITY, order)
        for name, r in compare(label, stage, own, ref0, ref3, state, params).items():
            report[(opts, stage, order, name)] = r
        state = ref0
    atm.destroy()
    failures = []
    check_report(report, PINNED_O, STAGE_BOUND, failures)
    assert not failures, "\n".join(failures)


@pytest.mark.gpu
@needs_atmo_build
def test_blend_and_matrix_paths_against_reference_kernels(slabs):
    """blend = 1 and the first triple's luminance-from-radiance matrix in the four kernels that take them, the running tables
    (irradiance, scattering, single Mie) prefilled with random positive values, the other inputs from the reference chain."""
    atm = V.Atmosphere()
    params = atm.params
    orc = oracle_ref.RefOracle()
    own_slab, ref_slab = slabs
    state = [torch.zeros((c, 4), dtype=torch.float32, device="cuda") for c in COUNTS]
    inputs = {}                                         # stage -> the reference chain's tables it starts from
    for stage, order in CHAIN[:5]:
        inputs[stage] = state
        state = run_ref(orc, ref_slab, params, state, stage, 0, IDENTITY, order, 0.0)
    inputs[MULTIPLE_SCATTERING] = state
    g = torch.Generator(device="cuda"); g.manual_seed(20260418)
    report = {}
    for stage in (DIRECT_IRRADIANCE, SINGLE_SCATTERING, INDIRECT_IRRADIANCE, MULTIPLE_SCATTERING):
        order = 2 if stage >= SCATTERING_DENSITY else 0
        st = list(inputs[stage])
        for name in ("irradiance", "scattering", "single_mie"):
            k = TABLES.index(name)
            st[k] = 0.1 + torch.rand(st[k].shape, generator=g, device="cuda", dtype=torch.float32)
        label = f"[blend, lfr] {STAGE_NAMES[stage]}" + (f" order {order}" if order else "")
        ref0 = run_ref(orc, ref_slab, params, st, stage, 1, FIRST_TRIPLE_LFR, order, 0.0)
        ref3 = run_ref(orc, ref_slab, params, st, stage, 1, FIRST_TRIPLE_LFR, order, CANARY)
        own = run_own(own_slab, params, st, stage, 1, FIRST_TRIPLE_LFR, order)
        for name, r in compare(label, stage, own, ref0, ref3, st, params, blend=1).items():
            report[("blend", stage, order, name)] = r
        if stage == DIRECT_IRRADIANCE:                  # irradiance += what it held: twice the prefilled table on both sides
            k = TABLES.index("irradiance")
            assert torch.equal(ref0[k], st[k] * 2) and torch.equal(own[k], st[k] * 2)
    atm.destroy()
    failures = []
    check_report(report, PINNED_O_BLEND, BLEND_BOUND, failures)
    assert not failures, "\n".join(failures)


_REFUSALS = """
import ctypes as C, sys
sys.path.insert(0, sys.argv[1])
from vpt_b200 import _native as N
p = N.AtmosphereParameters()
ptrs = (C.c_uint64 * 9)(*([16] * 9))
lfr = (C.c_float * 9)(1, 0, 0, 0, 1, 0, 0, 0, 1)
calls = [(s, C.byref(p), ptrs, lfr, b, o) for s, b, o in ((-1, 0, 0), (6, 0, 0), (0, 2, 0), (1, -1, 0), (3, 0, 1), (4, 0, 17), (5, 0, 0))]
calls += [(0, None, ptrs, lfr, 0, 0), (0, C.byref(p), None, lfr, 0, 0), (0, C.byref(p), ptrs, None, 0, 0)]
for k, v in ((0, 0), (8, 0), (3, 8)):                       # a null or misaligned table
    q = (C.c_uint64 * 9)(*([16] * 9)); q[k] = v
    calls.append((0, C.byref(p), q, lfr, 0, 0))
print(" ".join(str(N.lib.vpt_debug_bruneton_stage(*c)) for c in calls))
"""


def test_stage_entry_refuses_bad_arguments():
    """Every bad argument is refused with VPT_ERR_INVALID.  The calls run in a child process that sees no GPU
    (CUDA_VISIBLE_DEVICES empty): a check that stopped refusing would fail to launch there, never launch on a device."""
    import subprocess, sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", PYTHONNOUSERSITE="1")
    r = subprocess.run([sys.executable, "-c", _REFUSALS, root], env=env, capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    codes = [int(c) for c in r.stdout.split()]
    assert len(codes) == 13 and all(c == VPT_ERR_INVALID for c in codes), codes
