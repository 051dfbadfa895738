#!/usr/bin/env python
"""The columns of an `ncu --set full ... --page raw --csv` export that the roofline discussion uses, one line per launch.

    python tools/ncu_summary.py full_frame_raw.csv > ncu_full_summary.tsv
"""
import csv
import re
import sys

COLS = [("regs", "launch__registers_per_thread", 1), ("time_us", "gpu__time_duration.sum", None),
        ("dram_rd_MB", "dram__bytes_read.sum", None), ("dram_wr_MB", "dram__bytes_write.sum", None),
        ("issue_pct", "smsp__issue_active.avg.pct_of_peak_sustained_active", 1),
        ("warps_pct", "sm__warps_active.avg.pct_of_peak_sustained_active", 1),
        ("cyc_act_avg", "sm__cycles_active.avg", 1), ("cyc_act_max", "sm__cycles_active.max", 1), ("cyc_elapsed", "sm__cycles_elapsed.max", 1),
        ("smem_conflicts", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", 1), ("l2_hit_pct", "lts__t_sector_hit_rate.pct", 1),
        ("tensor_pct", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", 1),
        ("tma_pct", "sm__pipe_tma_cycles_active.avg.pct_of_peak_sustained_active", 1)]
TIME = {"ns": 1e-3, "us": 1.0, "ms": 1e3, "s": 1e6, "nsecond": 1e-3, "usecond": 1.0, "msecond": 1e3, "second": 1e6}
BYTES = {"byte": 1e-6, "Kbyte": 1e-3, "Mbyte": 1.0, "Gbyte": 1e3}


def main(path):
    rows = list(csv.reader(open(path, newline="")))
    rows = [r for r in rows if len(r) > 20]
    head, units = rows[0], rows[1]
    idx = {name: i for i, name in enumerate(head)}
    print("kernel\tgrid\tblock\t" + "\t".join(c[0] for c in COLS))
    for r in rows[2:]:
        name = re.sub(r"\(.*", "", r[idx["Kernel Name"]])
        name = re.sub(r"^void\s+", "", name).replace("unnamed>::", "")
        out = [name, r[idx["Grid Size"]].strip("() ").split(",")[0], r[idx["Block Size"]].strip("() ").split(",")[0]]
        for label, col, scale in COLS:
            if col not in idx or r[idx[col]] in ("", "n/a"):
                out.append("")
                continue
            v = float(r[idx[col]].replace(",", ""))
            u = units[idx[col]]
            if label == "time_us":
                v *= TIME.get(u, 1.0)
            elif label.startswith("dram_"):
                v *= BYTES.get(u, 1.0)
            out.append("%.4g" % v)
        print("\t".join(out))


if __name__ == "__main__":
    main(sys.argv[1])
