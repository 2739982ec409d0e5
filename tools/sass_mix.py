#!/usr/bin/env python3
"""Instruction mix of the loop that holds most of a kernel's conversions (I2F) / PRMTs, from `cuobjdump -sass`.

    python tools/sass_mix.py scanner_b200/lib/libscn_kernels.so nv12_stream_kernel [anchor-mnemonic]

nv12_stream_kernel's hot loop runs a block of 4 steps: divide its count by 4 for one 32-pixel step.
"""
import collections
import re
import subprocess
import sys


def main():
    so, pat = sys.argv[1], sys.argv[2]
    anchor = sys.argv[3] if len(sys.argv) > 3 else "I2F"
    txt = subprocess.run(["cuobjdump", "-sass", so], stdout=subprocess.PIPE, text=True).stdout
    cur, funcs = None, {}
    for line in txt.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs[cur] = []
            continue
        m = re.search(r"/\*([0-9a-f]{4,6})\*/\s+(.*?);", line)
        if m and cur:
            funcs[cur].append((int(m.group(1), 16), m.group(2).strip()))
    for name, ins in funcs.items():
        if pat not in name:
            continue
        anchors = sorted(a for a, t in ins if anchor in t)
        mid = anchors[len(anchors) // 2]
        best = None
        for a, t in ins:
            m = re.search(r"BRA\S*\s+(?:\S+,\s*)?0x([0-9a-f]+)", t)
            if m:
                tgt = int(m.group(1), 16)
                if tgt <= mid <= a and (best is None or a - tgt < best[0]):
                    best = (a - tgt, tgt, a)
        _, lo, hi = best
        loop = [t for a, t in ins if lo <= a <= hi]
        c = collections.Counter()
        for t in loop:
            t = re.sub(r"^@!?U?P\d\s+", "", t)
            c[t.split()[0]] += 1
        cls = collections.Counter()
        for k, v in c.items():
            base = k.split(".")[0]
            if base in ("IMAD", "FFMA2", "FADD2", "FMUL2", "HFMA2", "HADD2", "HMUL2"):
                cls["fma2"] += v
            elif base in ("FFMA", "FADD", "FMUL"):
                cls["fma1"] += v
            elif base in ("I2F", "F2I", "POPC", "MUFU", "F2F"):
                cls["xu"] += v
            elif base in ("LOP3", "PRMT", "SHF", "IADD3", "LEA", "VIADD", "ISETP", "SEL", "VIMNMX", "VIMNMX3", "FMNMX", "FMNMX3",
                          "PLOP3", "MOV", "FSETP", "I2FP"):
                cls["alu"] += v
            else:
                cls["other"] += v
        n = len(loop)
        print(f"{name}: loop {lo:#x}..{hi:#x}, {n} instructions (static)")
        print("  classes:", dict(cls), f"-> issue {n}, ALU clk {2 * cls['alu']}, FMA clk {cls['fma1'] + 2 * cls['fma2']}, XU clk {8 * cls['xu']}")
        print("  ", ", ".join(f"{k} {v}" for k, v in c.most_common()))


if __name__ == "__main__":
    main()
