"""The shape of each k_trace instantiation (trace_threads, trace_min_ctas, trace_ray_words, trace_smem_bytes and the carveout in
csrc/device/vpt_kernels.h; DESIGN.md section 4) against what an H100 SM offers: 233 472 B of shared memory for its CTAs, 1 KB more
reserved per CTA, and 65 536 registers.  The lean kernels at 2 rays per lane park 29 words per ray and have three shapes
(VPT_LEAN2_SHAPE): 4 CTAs of 224 threads (28 warps, the default), 3 CTAs of 256 threads, or the same under the 196 KB carveout, so that
the L1 keeps 60 KB.  The cell-table kernel keeps 3 CTAs of 256 threads in every shape.

The 29-word record packs no field into fewer bits than the 34-word one: rd and vd keep their 16 bits, the pass its 6 (start_path
masks it to 0..63), and the flag it adds takes bit 24 of the packed word, above the pass.  So no frame the API accepts needs the 34-word
record, and the host picks the lean kernels at 2 rays per lane for every lean frame, as before (tests/test_kernel_choice_cpu.py)."""
import subprocess

import pytest

from test_kernel_choice_cpu import DEVICE, cuda_include

SM_SMEM = 233472            # shared memory per SM available to CTAs (228 KB)
RESERVE = 1024              # reserved by the hardware per CTA
SM_REGS = 65536
TABLES = 4352               # static shared memory of k_trace (FrameShared + the empty-ahead table), asserted in vpt_kernels.cu
CARVEOUTS_KB = (0, 8, 16, 32, 64, 100, 132, 164, 196, 228)   # shared-memory capacities of an sm_90 SM; the L1 gets the rest of 256 KB

PROBE = r'''
#include "vpt_kernels.h"
#include <cstdio>
int main() {
    std::printf("%d %d %d %d\n", vpt::kTraceTablesBytes, vpt::kSmemPerSm, vpt::kSmemReservePerCta, vpt::kTraceThreads);
    for (int lean = 0; lean < 2; ++lean) for (int slots = 2; slots <= 3; ++slots)
    for (int cells = 0; cells < 2; ++cells)
        std::printf("%d %d %d %d %d %d %zu %zu %d\n", lean, slots, cells, vpt::trace_threads(lean, slots, cells), vpt::trace_min_ctas(lean, slots, cells),
                    vpt::trace_ray_words(lean, slots), vpt::trace_smem_bytes(lean, slots, cells), vpt::trace_sm_smem_bytes(lean, slots, cells),
                    vpt::trace_carveout_percent(lean, slots, cells));
}
'''


def shapes(tmp_path, shape):
    src = tmp_path / "probe.cpp"
    src.write_text(PROBE)
    exe = tmp_path / f"probe{shape}"
    subprocess.run(["g++", "-std=c++17", f"-DVPT_LEAN2_SHAPE={shape}", "-I", cuda_include(), "-I", DEVICE, str(src), "-o", str(exe)],
                   check=True)
    lines = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    consts = tuple(int(v) for v in lines[0].split())
    rows = {}
    for line in filter(None, lines[1:]):
        lean, slots, cells, threads, ctas, words, smem, sm_smem, carveout = (int(v) for v in line.split())
        if cells and not (lean and slots == 2):
            continue                                                  # only the lean kernel at 2 rays per lane has a cell-table form
        rows[(lean, slots) + ((1,) if cells else ())] = dict(threads=threads, ctas=ctas, words=words, smem=smem, sm_smem=sm_smem, carveout=carveout)
    return consts, rows


def register_cap(threads, ctas):
    """The registers per thread __launch_bounds__(threads, ctas) leaves: whole warps, allocated in units of 8 registers."""
    warps = -(-threads // 32)
    return SM_REGS // (ctas * warps * 32) // 8 * 8


@pytest.mark.parametrize("shape", [0, 1, 2])
def test_every_trace_shape_fits_an_sm(tmp_path, shape):
    consts, rows = shapes(tmp_path, shape)
    assert consts == (TABLES, SM_SMEM, RESERVE, 128)
    for (lean, slots, *cells), r in rows.items():
        assert r["smem"] == r["threads"] // 32 * 32 * slots * r["words"] * 4, (lean, slots)
        assert r["sm_smem"] == r["ctas"] * (r["smem"] + TABLES + RESERVE) <= SM_SMEM, (lean, slots)
        assert r["ctas"] * r["threads"] * register_cap(r["threads"], r["ctas"]) <= SM_REGS, (lean, slots)
        assert r["threads"] % 32 == 0
        assert r["words"] == (29 if (lean, slots) == (1, 2) else 34)
    # every other instantiation keeps its parent shape: 128 threads, 34 words, 4 CTAs at 3 rays per lane, 5 at 2
    assert [(rows[k]["threads"], rows[k]["ctas"]) for k in ((0, 2), (0, 3), (1, 3))] == [(128, 5), (128, 4), (128, 4)]
    # the cell-table kernel runs 3 CTAs of 256 threads at 80 registers in every shape
    assert (rows[(1, 2, 1)]["threads"], rows[(1, 2, 1)]["ctas"]) == (256, 3)


@pytest.mark.parametrize("shape", [0, 1])
def test_lean_shapes_0_and_1_keep_24_warps_and_fit_the_196_kb_carveout(tmp_path, shape):
    _, rows = shapes(tmp_path, shape)
    r = rows[(1, 2)]
    assert (r["threads"], r["ctas"], register_cap(r["threads"], r["ctas"])) == (256, 3, 80)
    assert r["smem"] == 59392                                         # 8 warps x 64 rays x 29 words
    assert r["sm_smem"] == 194304
    # the driver takes the smallest capacity at or above the carveout asked for; the three CTAs must fit it
    asked = r["carveout"] * SM_SMEM / 100
    capacity = min(c for c in CARVEOUTS_KB if c * 1024 >= asked)
    assert capacity == 196 and r["sm_smem"] <= capacity * 1024
    assert 256 - capacity == 60                                       # KB of L1, against 28 KB under the 228 KB carveout
    assert (r["carveout"] - 1) * SM_SMEM / 100 < r["sm_smem"]          # the least percentage that holds them


def test_lean_shape_2_runs_28_warps(tmp_path):
    _, rows = shapes(tmp_path, 2)
    r = rows[(1, 2)]
    assert (r["threads"], r["ctas"], register_cap(r["threads"], r["ctas"])) == (224, 4, 72)
    assert r["smem"] == 51968 and r["sm_smem"] == 229376
    assert min(c for c in CARVEOUTS_KB if c * 1024 >= r["carveout"] * SM_SMEM / 100) == 228
