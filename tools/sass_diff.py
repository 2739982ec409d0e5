#!/usr/bin/env python3
"""Compare the SASS of two builds of one object, kernel by kernel, ignoring addresses and encodings.

    python tools/sass_diff.py old/flow.o new/flow.o

For each kernel: "same" when the instruction streams are equal; "REORDERED" when they hold the same multiset of
instructions once register names and branch targets are ignored; "DIFFERENT" otherwise, with the first differing
instruction.  REORDERED is not a proof of equal arithmetic: with the register names gone, FFMA R2, R6, 0.5, R9 and
FFMA R2, R9, 0.5, R6 look alike, so such a kernel's dataflow has to be checked by hand (the differing positions are
printed).  The anonymous-namespace hash in the mangled names (which depends on the file name) is dropped, so a copy
of a source compiled under another name compares too.  Exit status: 0 when every kernel is the same, 2 when some are
only REORDERED, 1 when any is DIFFERENT or exists in one object only.
"""
import collections
import re
import subprocess
import sys


def kernels(path):
    txt = subprocess.run(["cuobjdump", "-sass", path], stdout=subprocess.PIPE, text=True, check=True).stdout
    cur, out = None, {}
    for line in txt.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = re.sub(r"_ZN\d+scn\d+_GLOBAL__N__.*?_cu_[0-9a-f]{8}", "", m.group(1))
            out[cur] = []
            continue
        m = re.search(r"/\*[0-9a-f]{4,6}\*/\s+(.*?;)", line)
        if m and cur:
            out[cur].append(m.group(1).strip())
    return out


def skeleton(ins):
    return collections.Counter(re.sub(r"0x[0-9a-f]+|\bU?R\d+\b|\bU?P\d\b", "_", i.replace(".reuse", "")) for i in ins)


def main():
    a, b = kernels(sys.argv[1]), kernels(sys.argv[2])
    bad = reordered = False
    for k in sorted(set(a) | set(b)):
        if k not in a or k not in b:
            print(f"only in {'new' if k in b else 'old'}: {k}")
            bad = True
        elif a[k] == b[k]:
            print(f"same       {len(a[k]):5d}  {k}")
        elif skeleton(a[k]) == skeleton(b[k]):
            diff = [i for i, (x, y) in enumerate(zip(a[k], b[k])) if x != y]
            print(f"REORDERED  {len(a[k]):5d}  {k}  ({len(diff)} positions differ; check their dataflow by hand)")
            for i in diff:
                print(f"    {i:5d}  {a[k][i]:<48s} | {b[k][i]}")
            reordered = True
        else:
            i = next((i for i, (x, y) in enumerate(zip(a[k], b[k])) if x != y), min(len(a[k]), len(b[k])))
            print(f"DIFFERENT  {len(a[k])}/{len(b[k])}  {k}  first at {i}: {a[k][i:i + 1]} vs {b[k][i:i + 1]}")
            bad = True
    sys.exit(1 if bad else 2 if reordered else 0)


if __name__ == "__main__":
    main()
