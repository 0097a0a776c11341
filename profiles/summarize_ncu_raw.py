#!/usr/bin/env python
"""Per-kernel summary of an `ncu --set full` capture:  ncu -i X.ncu-rep --page raw --csv | python profiles/summarize_ncu_raw.py [title]

One line per profiled launch: grid, duration, DRAM bytes (read + write), tensor-pipe / issue / DRAM / L2 / shared-memory utilisation,
registers, occupancy, shared-memory bank conflicts.  Times under ncu are cold-cache and serialised: use the shares."""
import csv
import sys

WANT = [
    ("dur_us", "gpu__time_duration.sum", 1e-3),
    ("dram_rd_MB", "dram__bytes_read.sum", 1e-6),
    ("dram_wr_MB", "dram__bytes_write.sum", 1e-6),
    ("tensor%", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", 1),
    ("tensor_subpipe%", "sm__pipe_tensor_subpipe_umma_cycles_active.avg.pct_of_peak_sustained_active", 1),
    ("issue%", "sm__inst_issued.avg.pct_of_peak_sustained_active", 1),
    ("dram%", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", 1),
    ("l2%", "lts__throughput.avg.pct_of_peak_sustained_elapsed", 1),
    ("smem%", "l1tex__data_pipe_lsu_wavefronts_mem_shared.avg.pct_of_peak_sustained_elapsed", 1),
    ("l1tex%", "l1tex__throughput.avg.pct_of_peak_sustained_active", 1),
    ("occ%", "sm__warps_active.avg.pct_of_peak_sustained_active", 1),
    ("regs", "launch__registers_per_thread", 1),
    ("bankconf", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", 1),
]


def main():
    rows = list(csv.reader(sys.stdin))
    hdr = next(i for i, r in enumerate(rows) if "Kernel Name" in r)
    names, units = rows[hdr], rows[hdr + 1]
    col = {n: i for i, n in enumerate(names)}
    title = sys.argv[1] if len(sys.argv) > 1 else "ncu --set full --clock-control none"
    print(f"# {title}")
    print("# columns: " + " ".join(k for k, _, _ in WANT))
    for r in rows[hdr + 2:]:
        if len(r) < len(names):
            continue
        kn = r[col["Kernel Name"]]
        grid = r[col["Grid Size"]] if "Grid Size" in col else "?"
        out = []
        for label, metric, scale in WANT:
            if metric not in col:
                continue
            raw = r[col[metric]].replace(",", "")
            try:
                v = float(raw)
            except ValueError:
                continue
            unit = units[col[metric]]
            if label == "dur_us":
                v *= {"ns": 1e-3, "us": 1.0, "ms": 1e3, "s": 1e6, "nsecond": 1e-3, "usecond": 1.0, "msecond": 1e3}.get(unit, 1e-3)
            elif label.endswith("_MB"):
                v *= {"byte": 1e-6, "Kbyte": 1e-3, "Mbyte": 1.0, "Gbyte": 1e3}.get(unit, 1e-6)
            out.append(f"{label}={v:.1f}" if abs(v) < 1e6 else f"{label}={v:.3g}")
        print(f"{kn[:78]:78s} grid={grid:>14s} " + " ".join(out))


if __name__ == "__main__":
    main()
