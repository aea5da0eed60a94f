#!/usr/bin/env python
"""Compares the SASS of two builds kernel by kernel, instruction by instruction.

  cuobjdump -sass old/als.cubin > old.sass; cuobjdump -sass new/als.cubin > new.sass
  python benchmarks/sass_compare.py old.sass new.sass

A change that adds a defaulted template parameter (such as the ALS kernels' `DET = false`) renames every existing
instantiation; its code must not change.  Kernels are therefore matched by demangled name after dropping trailing
`false` template arguments (and an all-default `<false>`), and a kernel of the old build must match exactly one kernel
of the new build.  An instruction is the text between the address and the encoding comment of a `cuobjdump -sass` line:
opcode, modifiers, registers, immediates and constant-bank offsets all count.  Prints the kernels that differ or are
missing and exits 1 if there are any.  Needs `cu++filt` (CUDA toolkit) on the PATH.
"""
import re
import subprocess
import sys


def kernels(path):
    """{mangled name: [instruction, ...]} of a `cuobjdump -sass` dump."""
    out, cur = {}, None
    for line in open(path):
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = out.setdefault(m.group(1), [])
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?;)", line)
        if m and cur is not None:
            cur.append(m.group(1))
    return out


def canonical(name):
    """Demangled kernel name without trailing `false` template arguments."""
    m = re.match(r"(.*?)<(.*)>(\(.*)$", name)
    if not m:
        return name
    head, args, tail = m.groups()
    parts = [a.strip() for a in args.split(",")]
    while parts and parts[-1] in ("(bool)0", "false"):
        parts.pop()
    return head + ("<" + ", ".join(parts) + ">" if parts else "") + tail


def demangle(names):
    txt = subprocess.run(["cu++filt"] + names, stdout=subprocess.PIPE, text=True, check=True).stdout
    return dict(zip(names, [re.sub(r"^void ", "", l) for l in txt.strip().split("\n")]))


def main():
    old, new = kernels(sys.argv[1]), kernels(sys.argv[2])
    d_old, d_new = demangle(list(old)), demangle(list(new))
    by_name = {}
    for k, v in d_new.items():
        by_name.setdefault(canonical(v), []).append(k)
    same, bad = 0, 0
    for k, name in sorted(d_old.items(), key=lambda kv: kv[1]):
        hits = by_name.get(canonical(name), [])
        if len(hits) != 1:
            print("%s: %s" % ("MISSING" if not hits else "AMBIGUOUS", name))
            bad += 1
        elif old[k] != new[hits[0]]:
            a, b = old[k], new[hits[0]]
            first = next((i for i, (x, y) in enumerate(zip(a, b)) if x != y), min(len(a), len(b)))
            print("DIFFERENT: %s (%d vs %d instructions, first difference at %d)" % (name, len(a), len(b), first))
            bad += 1
        else:
            same += 1
    print("%d kernels in the old build: %d identical, %d different or missing; %d kernels in the new build"
          % (len(old), same, bad, len(new)))
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
