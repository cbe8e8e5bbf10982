#!/usr/bin/env python3
"""Compare the machine code of two builds kernel by kernel: python tools/sass_compare.py OLD NEW

OLD and NEW are cubins or shared libraries built with csrc/build.sh's flags.  For every kernel in either file prints
  identical  the SASS instruction text is equal once the address column and the encodings are stripped
  same-ops   the sorted opcode histograms are equal (register renaming, reordered independent instructions)
  different  / missing
followed by REG / STACK / SHARED of both builds from `cuobjdump -res-usage`.  Exit status 1 when any kernel is not
identical or changed its resources.  Needs cuobjdump (and cu++filt for readable names) on PATH or under $CUDA_HOME/bin.
"""
import collections, os, re, shutil, subprocess, sys

CUDA_BIN = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin")
INSN = re.compile(r"^\s*/\*[0-9a-f]+\*/\s*(.*?)\s*;")


def tool(name):
    return shutil.which(name) or os.path.join(CUDA_BIN, name)


def run(*cmd):
    return subprocess.run(cmd, check=True, capture_output=True, text=True).stdout


def kernels(path):
    """{name: (instruction texts, {REG, STACK, SHARED})}"""
    sass, res, name = {}, {}, None
    for line in run(tool("cuobjdump"), "-sass", path).splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
            sass[name] = []
        elif name and (m := INSN.match(line)):
            sass[name].append(" ".join(m.group(1).split()))
    for line in run(tool("cuobjdump"), "-res-usage", path).splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            name = m.group(1)
        elif name and "REG:" in line:
            res[name] = {k: int(v) for k, v in re.findall(r"(REG|STACK|SHARED):(\d+)", line)}
            name = None
    return {n: (sass.get(n), res.get(n, {})) for n in set(sass) | set(res)}


def opcodes(insns):
    # the mnemonic with its modifiers, without the predicate guard (guards are renamed registers too)
    return sorted(t.split()[1] if t.startswith("@") else t.split()[0] for t in insns)


def demangle(names):
    try:
        out = run(tool("cu++filt"), *names).splitlines()
        return dict(zip(names, out)) if len(out) == len(names) else {n: n for n in names}
    except (OSError, subprocess.CalledProcessError):
        return {n: n for n in names}


def main(old_path, new_path):
    old, new = kernels(old_path), kernels(new_path)
    names = sorted(set(old) | set(new))
    pretty = demangle(names)
    clean = True
    for n in sorted(names, key=lambda n: pretty[n]):
        (a, ra), (b, rb) = old.get(n, (None, {})), new.get(n, (None, {}))
        if a is None or b is None:
            verdict = "missing in " + ("OLD" if a is None else "NEW")
        elif a == b:
            verdict = "identical"
        elif opcodes(a) == opcodes(b):
            verdict = "same-ops"
        else:
            verdict = "different (%d -> %d instructions)" % (len(a), len(b))
        usage = "  ".join("%s %s -> %s" % (k, ra.get(k, "-"), rb.get(k, "-")) if ra.get(k) != rb.get(k) else "%s %s" % (k, ra.get(k))
                          for k in ("REG", "STACK", "SHARED"))
        clean &= verdict == "identical" and ra == rb
        print("%-10s %s   [%s]" % (verdict, pretty[n], usage))
    return 0 if clean else 1


if __name__ == "__main__":
    if len(sys.argv) != 3:
        sys.exit(__doc__)
    sys.exit(main(sys.argv[1], sys.argv[2]))
