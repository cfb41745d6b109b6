#!/usr/bin/env python
"""Summarise .ncu-rep files (read here, no GPU needed) into a markdown table.

    python tools/ncu_summary.py r1_volume.ncu-rep [more.ncu-rep ...] > ncu_summary.md
"""
import csv
import io
import subprocess
import sys

METRICS = [
    ("gpu__time_duration.sum", "time"),
    ("dram__bytes_read.sum", "dram read"),
    ("dram__bytes_write.sum", "dram write"),
    ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram % of peak"),
    ("lts__t_bytes.sum", "L2 bytes"),
    ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "SM throughput %"),
    ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue active %"),
    ("sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "FMA pipe %"),
    ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "tensor pipe %"),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "warps active %"),
    ("launch__registers_per_thread", "regs/thread"),
    ("launch__grid_size", "grid"),
    ("launch__block_size", "block"),
    ("launch__shared_mem_per_block_dynamic", "dyn smem/block"),
    ("smsp__inst_executed.sum", "warp instructions"),
]


def rows_of(path):
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL,
                         text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    hdr, units = rows[0], rows[1]
    for r in rows[2:]:
        if len(r) == len(hdr):
            yield hdr, units, r


def aggregate(path):
    """One row per distinct kernel name: launches, total / mean duration, launch-averaged metrics."""
    groups, order = {}, []
    hdr = units = None
    for hdr, units, r in rows_of(path):
        name = r[hdr.index("Kernel Name")]
        if name not in groups:
            groups[name] = []
            order.append(name)
        groups[name].append(r)
    print("## %s (aggregated per kernel)\n" % path.split("/")[-1])
    cols = [(k, l) for k, l in METRICS if hdr and k in hdr]
    print("| kernel | launches | total time | " + " | ".join(l for _, l in cols[1:]) + " |")
    print("|---|---|---|" + "---|" * (len(cols) - 1))

    def num(x):
        try:
            return float(x.replace(",", ""))
        except ValueError:
            return None

    ti = hdr.index("gpu__time_duration.sum")
    for name in order:
        rs = groups[name]
        total = sum(num(r[ti]) or 0.0 for r in rs)
        cells = []
        for k, _ in cols[1:]:
            vals = [num(r[hdr.index(k)]) for r in rs]
            vals = [v for v in vals if v is not None]
            cells.append("%.4g %s" % (sum(vals) / len(vals), units[hdr.index(k)]) if vals else "")
        print("| `%s` | %d | %.4g %s | %s |" % (name[:110], len(rs), total, units[ti], " | ".join(cells)))
    print()


def main():
    if len(sys.argv) > 2 and sys.argv[1] == "--aggregate":
        for path in sys.argv[2:]:
            aggregate(path)
        return
    for path in sys.argv[1:]:
        print("## %s\n" % path.split("/")[-1])
        for hdr, units, r in rows_of(path):
            name = r[hdr.index("Kernel Name")]
            print("**%s**\n" % name)
            print("| metric | value |\n|---|---|")
            for key, label in METRICS:
                if key in hdr:
                    i = hdr.index(key)
                    print("| %s (`%s`) | %s %s |" % (label, key, r[i], units[i]))
            print()


if __name__ == "__main__":
    main()
