#!/usr/bin/env python3
"""Static shared-memory instruction counts per kernel: python tools/smem_ops.py LIB [NAME_REGEX]

LIB is a cubin or shared library built with csrc/build.sh's flags.  For every kernel whose demangled name matches NAME_REGEX (default
k_trace) prints its instruction count and its LDS / STS instructions by access width (32, 64, 128 bit), with REG / STACK / SHARED from
`cuobjdump -res-usage`.  Static counts: how often each runs is a matter of the counters (option "count_stats")."""
import collections, re, sys

from sass_compare import demangle, kernels


def width(op):
    m = re.search(r"\.(64|128)\b", op)
    return int(m.group(1)) if m else 32


def main(path, pattern="k_trace"):
    ks = kernels(path)
    names = demangle(sorted(ks))
    print(f"{'kernel':70s} {'insns':>6s} {'LDS32':>6s} {'LDS64':>6s} {'LDS128':>6s} {'STS32':>6s} {'STS64':>6s} {'STS128':>6s}  resources")
    for n in sorted(ks, key=lambda k: names[k]):
        if not re.search(pattern, names[n]): continue
        insns, res = ks[n]
        cnt = collections.Counter()
        for t in insns or []:
            op = t.split()[1] if t.startswith("@") else t.split()[0]
            base = op.split(".")[0]
            if base in ("LDS", "STS"): cnt[base, width(op)] += 1
        print(f"{names[n][:70]:70s} {len(insns or []):6d} " + " ".join(f"{cnt[b, w]:6d}" for b in ("LDS", "STS") for w in (32, 64, 128)) + f"  {res}")


if __name__ == "__main__":
    if len(sys.argv) < 2: sys.exit(__doc__)
    main(*sys.argv[1:3])
