"""Per-launch summary (markdown) of an ``ncu --set full`` capture exported with ``--page raw --csv``.

  python tools/ncu_full_summary.py step_full_raw.csv step_full_summary.md
"""
import csv
import re
import sys

COLS = [
    ("us", "gpu__time_duration.sum"),
    ("dram rd MB", "dram__bytes_read.sum"),
    ("dram wr MB", "dram__bytes_write.sum"),
    ("dram %", "dram__throughput.avg.pct_of_peak_sustained_elapsed"),
    ("L2 %", "lts__throughput.avg.pct_of_peak_sustained_elapsed"),
    ("L1 %", "l1tex__throughput.avg.pct_of_peak_sustained_elapsed"),
    ("SM %", "sm__throughput.avg.pct_of_peak_sustained_elapsed"),
    ("tensor %", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed"),
    ("issue %", "sm__inst_issued.avg.pct_of_peak_sustained_elapsed"),
    ("fma %", "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active"),
    ("occ %", "sm__warps_active.avg.pct_of_peak_sustained_active"),
    ("regs", "launch__registers_per_thread"),
    ("smem KB", "launch__shared_mem_per_block_dynamic"),
]


def short(name):
    name = re.sub(r"\(anonymous namespace\)::|<unnamed>::", "", name)
    m = re.match(r"(?:void )?([A-Za-z0-9_:]+(?:<[^>(]*>)?)", name)
    return (m.group(1) if m else name)[:48]


def num(x):
    try:
        return float(x.replace(",", ""))
    except ValueError:
        return None


def main(src, out):
    rows = list(csv.reader(open(src)))
    hdr, units, data = rows[0], rows[1], rows[2:]
    ix = {h: i for i, h in enumerate(hdr)}

    def find(metric):
        if metric in ix:
            return ix[metric]
        c = [i for h, i in ix.items() if h.endswith(metric)]
        return c[0] if c else None

    sel = [(t, find(m)) for t, m in COLS]
    scale = {"byte": 1e-6, "Kbyte": 1e-3, "Mbyte": 1.0, "Gbyte": 1e3, "ns": 1e-3, "us": 1.0, "ms": 1e3}
    lines = ["| # | kernel | grid | block | " + " | ".join(t for t, _ in sel) + " |", "|" + "---|" * (4 + len(sel))]
    tot_us = tot_rd = tot_wr = 0.0
    for k, r in enumerate(data):
        cells = []
        for t, i in sel:
            if i is None:
                cells.append("-")
                continue
            v = num(r[i])
            if v is None:
                cells.append(r[i])
                continue
            u = units[i]
            if t in ("us", "dram rd MB", "dram wr MB"):
                v *= scale.get(u, 1.0)
            if t == "smem KB":
                v *= {"byte": 1 / 1024, "Kbyte": 1.0}.get(u, 1.0 / 1024)
            if t == "us":
                tot_us += v
            if t == "dram rd MB":
                tot_rd += v
            if t == "dram wr MB":
                tot_wr += v
            cells.append(f"{v:.1f}" if t not in ("regs",) else f"{v:.0f}")
        lines.append(f"| {k} | {short(r[ix['Kernel Name']])} | {r[ix['Grid Size']]} | {r[ix['Block Size']]} | " + " | ".join(cells) + " |")
    lines.append("")
    lines.append(f"Total: {tot_us:.1f} us (serialised, cold-cache under ncu), DRAM read {tot_rd:.1f} MB, write {tot_wr:.1f} MB")
    open(out, "w").write("\n".join(lines) + "\n")
    print("\n".join(lines))


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2])
