"""Which trace kernel a frame runs (vpt::pick_trace_kernel in csrc/device/vpt_kernels.h), for every input frame_setup can pass.

Several trace kernels give bit-identical images (2 vs 3 rays per lane, lean vs generic), so no GPU test sees a wrong pick: only a
lost CTA per SM or a slower kernel would.  This test compiles a small probe against the header with the host compiler and pins the
choice, and the default of option "sched_min_lanes" that follows from it, to the table below."""
import itertools
import os
import shutil
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEVICE = os.path.join(ROOT, "volumetric-path-tracer_b200", "csrc", "device")

KERNELS = ["TK_GENERIC_3", "TK_LEAN_3", "TK_VOL_3", "TK_BRICK", "TK_GENERIC_2", "TK_LEAN_2", "TK_LEAN_2_CELLS",
           "TK_GENERIC_3_GROUPS", "TK_VOL_3_GROUPS"]

PROBE = r'''
#include "vpt_kernels.h"
#include <cstdio>
#define NAME(x) if (k == vpt::x) return #x;
static const char* name(vpt::TraceKernel k) { %s return "?"; }
int main() {
    std::printf("%%d\n", (int)vpt::kTraceKernels);
    for (int brick = 0; brick < 2; ++brick) for (int cells = 0; cells < 2; ++cells) for (int vol = 0; vol < 2; ++vol)
    for (int lean = 0; lean < 2; ++lean) for (int groups = 0; groups < 2; ++groups) for (int slots = 2; slots <= 3; ++slots) {
        const vpt::TraceKernel k = vpt::pick_trace_kernel(brick, cells, vol, lean, groups, slots);
        std::printf("%%d %%d %%d %%d %%d %%d %%s %%d\n", brick, cells, vol, lean, groups, slots, name(k), vpt::trace_sched_min_lanes(k));
    }
}
''' % " ".join(f"NAME({k})" for k in KERNELS)


def cuda_include():
    nvcc = shutil.which("nvcc")
    home = os.path.dirname(os.path.dirname(os.path.realpath(nvcc))) if nvcc else os.environ.get("CUDA_HOME", "/usr/local/cuda")
    return os.path.join(home, "include")


def reachable(brick, cells, vol, lean, groups, slots):
    """The inputs frame_setup can produce: a lean scene has one volume, the direct integrator and no light-group planes; brick and cell
    mode run lean scenes only, never together, cell mode at 2 rays per lane; brick mode and the volumetric integrator at 3.  Group planes
    come with whatever rays per lane the scene asks for (the group kernels run 3)."""
    if lean and (vol or groups):
        return False
    if (brick or cells) and not lean:
        return False
    if brick and cells:
        return False
    if cells and slots != 2:
        return False
    return not ((brick or vol) and slots != 3)


def expected(brick, cells, vol, lean, groups, slots):
    if groups:
        return "TK_VOL_3_GROUPS" if vol else "TK_GENERIC_3_GROUPS"
    if brick:
        return "TK_BRICK"
    if cells:
        return "TK_LEAN_2_CELLS"
    if vol:
        return "TK_VOL_3"
    if slots == 2:
        return "TK_LEAN_2" if lean else "TK_GENERIC_2"
    return "TK_LEAN_3" if lean else "TK_GENERIC_3"


def test_trace_kernel_choice_and_sched_min_lanes(tmp_path):
    src = tmp_path / "probe.cpp"
    src.write_text(PROBE)
    exe = tmp_path / "probe"
    subprocess.run(["g++", "-std=c++17", "-I", cuda_include(), "-I", DEVICE, str(src), "-o", str(exe)], check=True)
    lines = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    assert int(lines[0]) == len(KERNELS)
    got = {}
    for line in filter(None, lines[1:]):
        *bits, kernel, lanes = line.split()
        got[tuple(int(b) for b in bits)] = (kernel, int(lanes))
    assert len(got) == 64

    cases = [c for c in itertools.product((0, 1), (0, 1), (0, 1), (0, 1), (0, 1), (2, 3)) if reachable(*c)]
    for c in cases:
        want = expected(*c)
        assert got[c] == (want, 26 if want == "TK_LEAN_3" else 20), f"brick, cells, vol, lean, groups, slots = {c}"
    assert sorted({expected(*c) for c in cases}) == sorted(KERNELS)      # every trace kernel is the pick of some frame
