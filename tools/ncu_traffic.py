"""Reduce `ncu -i step.ncu-rep --page raw --csv` (an `ncu --set full --profile-from-start off ... python tools/profile_step.py`
capture of ONE eager training step) to
  * <out.json> : per conv family {launches, dram_bytes, time_us_under_ncu}
  * a per-launch table on stdout       : time, DRAM read/write, SM / tensor-pipe / L2 throughput %, grid
Usage: python tools/ncu_traffic.py raw.csv out.json > table.txt
Family = the role of the kernel in the step (what bench.py's CUDA-event families time as tc_fwd / tc_dgrad / tc_wgrad / dw_*).
"""
import csv
import json
import re
import sys


def family(name):
    n = name
    if "wgrad" in n and ("pconv_tc" in n or "smallco" in n):
        return "tc_wgrad"
    if "dw4_s1_wgrad" in n or "dw3_wgrad" in n or "dw_wgrad" in n:
        return "dw_wgrad"
    m = re.search(r"pconv_tc_(tma|persistent)_kernel<\s*(?:\(int\))?\s*(\d+),\s*(?:\(int\))?\s*(\d+)", n)
    if m:
        return "tc_dgrad" if m.group(3) == "1" else "tc_fwd"
    if "pconv_tc_sp_kernel" in n:
        return "tc_dgrad"
    if "smallco_fwd" in n or "k2r_combine" in n:
        return "tc_fwd"
    if "smallco_dgrad" in n:
        return "tc_dgrad"
    if "k2r_dbuild" in n:
        return "tc_dgrad" if re.search(r"k2r_dbuild_kernel<\s*(?:\(bool\))?\s*(0|false)", n) else "tc_wgrad"
    m = re.search(r"dw4_s1_kernel<[^,]+,\s*(?:\(bool\))?\s*(\w+)", n)
    if m:
        return "dw_dgrad" if m.group(1) in ("1", "true") else "dw_fwd"
    if "dw3_fwd" in n or "dw_fwd" in n:
        return "dw_fwd"
    if "dw3_dgrad" in n or "dw_dgrad" in n:
        return "dw_dgrad"
    return None


def main():
    rows = list(csv.reader(open(sys.argv[1], errors="replace")))
    hi = next(i for i, r in enumerate(rows) if "Kernel Name" in r)
    hdr, units = rows[hi], rows[hi + 1]
    col = {c: i for i, c in enumerate(hdr)}

    def get(r, key, default=0.0):
        i = col.get(key)
        if i is None or i >= len(r):
            return default
        try:
            v = float(r[i].replace(",", ""))
        except ValueError:
            return default
        u = units[i].lower()
        scale = {"byte": 1.0, "kbyte": 1e3, "mbyte": 1e6, "gbyte": 1e9, "ns": 1e-3, "us": 1.0, "ms": 1e3, "s": 1e6}.get(u, 1.0)
        return v * scale

    fams = {}
    print("# one eager training step under ncu (--clock-control none; serialised, cold caches): per launch time, DRAM bytes, SM and L2 throughput % of peak")
    print(f"{'family':9s} {'us':>8s} {'rd MB':>8s} {'wr MB':>8s} {'SM%':>6s} {'L2%':>6s} {'grid':>16s}  kernel")
    for r in rows[hi + 2:]:
        if len(r) <= col["Kernel Name"]:
            continue
        name = r[col["Kernel Name"]]
        f = family(name)
        t = get(r, "gpu__time_duration.sum")
        rd, wr = get(r, "dram__bytes_read.sum"), get(r, "dram__bytes_write.sum")
        sm = get(r, "sm__throughput.avg.pct_of_peak_sustained_elapsed")
        l2 = get(r, "lts__throughput.avg.pct_of_peak_sustained_elapsed")
        grid = r[col["Grid Size"]] if "Grid Size" in col else ""
        short = re.sub(r"void <unnamed>::|\(.*$", "", name)[:70]
        print(f"{f or '-':9s} {t:8.1f} {rd / 1e6:8.2f} {wr / 1e6:8.2f} {sm:6.1f} {l2:6.1f} {grid:>16s}  {short}")
        if f:
            d = fams.setdefault(f, {"launches": 0, "dram_bytes": 0.0, "time_us_under_ncu": 0.0})
            d["launches"] += 1
            d["dram_bytes"] += rd + wr
            d["time_us_under_ncu"] += t
    if len(sys.argv) > 2:
        json.dump(fams, open(sys.argv[2], "w"), indent=1)
    for k, d in sorted(fams.items()):
        print(f"== {k:9s} launches {d['launches']:4d}  DRAM {d['dram_bytes'] / 1e6:9.1f} MB  {d['time_us_under_ncu']:9.1f} us under ncu")


if __name__ == "__main__":
    main()
