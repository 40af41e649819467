"""Condenses an `ncu --set full --csv --page raw` capture of one bench step (e.g. of scripts/profile_step.py) into a
per-launch summary, and (optionally) an `ncu --page source --csv` capture into its top stall lines.

  python scripts/ncu_summary.py raw.csv conv_ncu_summary.csv [layer names...]
  python scripts/ncu_summary.py --stalls src.csv top_stalls.txt
"""
import csv
import sys

COLS = [
    ("gpu__time_duration.sum", "ms", 1e-6),
    ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed", "tensor_pipe_active_pct", 1),
    ("sm__cycles_elapsed.avg.per_second", "sm_ghz", 1e-9),
    ("dram__bytes_read.sum", "dram_read_GB", 1e-9),
    ("dram__bytes_write.sum", "dram_write_GB", 1e-9),
    ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram_pct", 1),
    ("l1tex__m_xbar2l1tex_read_bytes_mem_global_op_tma_ld.sum", "tma_load_GB", 1e-9),
    ("l1tex__m_xbar2l1tex_read_bytes.sum.per_second", "xbar2l1tex_TBps", 1e-12),
    ("l1tex__m_xbar2l1tex_read_bytes.sum.pct_of_peak_sustained_elapsed", "xbar2l1tex_pct", 1),
    ("lts__throughput.avg.pct_of_peak_sustained_elapsed", "l2_throughput_pct", 1),
    ("lts__t_sector_hit_rate.pct", "l2_hit_pct", 1),
    ("sm__inst_issued.avg.pct_of_peak_sustained_active", "issue_active_pct", 1),
    ("launch__registers_per_thread", "regs", 1),
    ("launch__grid_size", "grid", 1),
]


def summary(src, dst, names):
    rows = list(csv.reader(open(src)))
    hi = [i for i, r in enumerate(rows) if r and r[0] == "ID"][0]
    hdr, data = rows[hi], rows[hi + 2:]
    kn = hdr.index("Kernel Name")
    with open(dst, "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(["layer", "kernel"] + [c[1] for c in COLS])
        for i, r in enumerate(data):
            out = [names[i] if i < len(names) else str(i), r[kn].split("(")[0].replace("void ", "")]
            for metric, _, scale in COLS:
                try:
                    v = float(r[hdr.index(metric)].replace(",", "")) * scale
                    out.append("%.4g" % v)
                except (ValueError, IndexError):
                    out.append("")
            w.writerow(out)
    print(open(dst).read())


def stalls(src, dst, top=30):
    rows = list(csv.reader(open(src)))
    hdr, data = rows[1], rows[2:]
    si, ie = hdr.index("# Samples"), hdr.index("Instructions Executed")
    sc = [i for i, c in enumerate(hdr) if c.startswith("stall_") and "Not Issued" not in c]
    tot = sum(int(r[si]) for r in data if len(r) > si and r[si].isdigit())
    best = sorted(((int(r[si]), i) for i, r in enumerate(data) if len(r) > si and r[si].isdigit()), reverse=True)[:top]
    with open(dst, "w") as f:
        f.write("%s\n%s\ntotal warp-stall samples %d; top %d SASS lines\n" % (rows[0][1], src, tot, top))
        for s, i in best:
            r = data[i]
            st = sorted(((int(r[j]), hdr[j]) for j in sc if r[j].isdigit() and int(r[j]) > 0), reverse=True)[:2]
            f.write("%6d %5.1f%%  executed %9s  %-64s %s\n" % (s, 100.0 * s / tot, r[ie], r[1].strip()[:64],
                                                             ", ".join("%s %d" % (n, c) for c, n in st)))
    print(open(dst).read())


if __name__ == "__main__":
    if sys.argv[1] == "--stalls":
        stalls(sys.argv[2], sys.argv[3])
    else:
        summary(sys.argv[1], sys.argv[2], sys.argv[3:])
