#!/usr/bin/env python3
"""Per-kernel measured-bytes roofline of the Farneback path from an ncu CSV log.

On a GPU:
  ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum,lts__t_bytes.sum,\
smsp__issue_active.avg.pct_of_peak_sustained_active,smsp__inst_executed.sum --clock-control none \
      -k regex:'gray|gauss|poly|resize_f32|update_matrices|box_' -c 200 --csv --log-file flow_ncu.csv \
      python tools/flow_roofline.py drive
Then:  python tools/flow_roofline.py table flow_ncu.csv [peak GB/s]
`drive` runs 3 consecutive 1080p pairs of one clip (the op's access pattern; the first pair expands two frames).
"""
import csv
import collections
import sys


def drive():
    import torch
    sys.path.insert(0, ".")
    from scanner_b200 import kernels
    g = torch.Generator(device="cuda").manual_seed(3)
    a = torch.randint(0, 256, (4, 1080, 1920, 3), dtype=torch.uint8, device="cuda", generator=g)
    kernels.optical_flow_sequence(a)
    torch.cuda.synchronize()


def table(path, peak):
    rows = [r for r in csv.reader(l for l in open(path) if not l.startswith("=="))]
    hdr = rows[0]
    ki, gi, mi, vi = hdr.index("Kernel Name"), hdr.index("Grid Size"), hdr.index("Metric Name"), hdr.index("Metric Value")
    ii = hdr.index("ID")
    launches = collections.OrderedDict()
    for r in rows[1:]:
        if len(r) <= vi:
            continue
        launches.setdefault(r[ii], {"kernel": r[ki].split("(")[0].split("::")[-1], "grid": r[gi]})[r[mi]] = float(r[vi].replace(",", ""))
    agg = collections.OrderedDict()
    for l in launches.values():
        k = (l["kernel"], l["grid"])
        a = agg.setdefault(k, {"n": 0, "ns": 0.0, "rd": 0.0, "wr": 0.0, "l2": 0.0, "issue": 0.0, "inst": 0.0})
        a["n"] += 1
        a["ns"] += l.get("gpu__time_duration.sum", 0)
        a["rd"] += l.get("dram__bytes_read.sum", 0)
        a["wr"] += l.get("dram__bytes_write.sum", 0)
        a["l2"] += l.get("lts__t_bytes.sum", 0)
        a["issue"] += l.get("smsp__issue_active.avg.pct_of_peak_sustained_active", 0)
        a["inst"] += l.get("smsp__inst_executed.sum", 0)
    total_ns = sum(a["ns"] for a in agg.values())
    print("| kernel | grid | launches | us / launch | DRAM read MB | DRAM write MB | DRAM GB/s | frac of %.0f GB/s | L2 GB/s | issue active %% | share of time |" % peak)
    print("|---|---|---|---|---|---|---|---|---|---|---|")
    for (k, g), a in agg.items():
        n = a["n"]
        us = a["ns"] / n / 1e3
        bw = (a["rd"] + a["wr"]) / a["ns"]
        print(f"| `{k}` | {g} | {n} | {us:.1f} | {a['rd'] / n / 1e6:.1f} | {a['wr'] / n / 1e6:.1f} | {bw:.0f} | {bw / peak:.2f} | "
              f"{a['l2'] / a['ns']:.0f} | {a['issue'] / n:.0f} | {100 * a['ns'] / total_ns:.1f} % |")
    print(f"\ntotal {total_ns / 1e3:.0f} us over {sum(a['n'] for a in agg.values())} launches (ncu: serialised, cold caches between replays)")


if __name__ == "__main__":
    if sys.argv[1] == "drive":
        drive()
    else:
        table(sys.argv[2], float(sys.argv[3]) if len(sys.argv) > 3 else 6567.4)
