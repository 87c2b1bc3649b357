"""Summarise an ``ncu --csv --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum``
launch list of ``bench.py`` into a per-kernel table (markdown) + the DRAM traffic of the tensor-core conv
launches of one step (JSON, read back by bench.py for ``roofline.traffic``).

  python tools/ncu_summarize.py launches.csv launches_summary.md tc_traffic.json [steps]

`steps` = number of bottom-up steps inside the capture (``bench.py --ncu-step --steps K`` under
``ncu --profile-from-start off``).  Without it the count is taken from the kernels that run exactly once per step
(the grouping kernel for the post-processing chain, the first-layer kernel for the network).  Round 1 divided the
post-processing kernels by the step count but the conv launches by 1 whenever the first layer ran as the Toeplitz
view (no ``k_conv_first`` launch): ``traffic_bytes_per_step`` was the sum over all captured steps.
"""
import csv
import json
import re
import sys
from collections import OrderedDict


def short(name):
    name = re.sub(r"<unnamed>::", "", name)
    name = re.sub(r"\b[a-z_0-9]+::", "", name)
    m = re.match(r"(?:void )?([A-Za-z0-9_]+(?:<[^>(]*>)?)", name)
    return m.group(1) if m else name[:60]


def main(src, out_md, out_json, steps=None):
    rows = []
    with open(src, newline="") as f:
        lines = [l for l in f if l.startswith('"')]
    for r in csv.DictReader(lines):
        rows.append(r)
    launches = OrderedDict()
    for r in rows:
        d = launches.setdefault(int(r["ID"]), {"name": short(r["Kernel Name"]), "grid": r["Grid Size"], "block": r["Block Size"]})
        v = float(r["Metric Value"].replace(",", ""))
        unit = r["Metric Unit"]
        if r["Metric Name"].startswith("gpu__time_duration"):
            d["ns"] = v * {"ns": 1, "us": 1e3, "ms": 1e6, "s": 1e9}.get(unit, 1)
        else:
            mult = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(unit, 1)
            key = "rd" if "read" in r["Metric Name"] else "wr"
            d[key] = v * mult
    ls = list(launches.values())
    n_full = sum(1 for l in ls if l["name"].startswith("k_group")) or 1
    n_fwd = max(sum(1 for l in ls if l["name"].startswith("k_first_view")), sum(1 for l in ls if l["name"].startswith("k_conv_first")),
                sum(1 for l in ls if l["name"].startswith("k_conv01"))) or n_full
    if steps:
        n_full = n_fwd = int(steps)
    per = OrderedDict()
    for l in ls:
        p = per.setdefault(l["name"], {"n": 0, "ns": 0.0, "rd": 0.0, "wr": 0.0})
        p["n"] += 1; p["ns"] += l.get("ns", 0); p["rd"] += l.get("rd", 0); p["wr"] += l.get("wr", 0)
    post = {"k_local_scan", "k_local_emit", "k_score_match", "k_group", "k_integral", "k_lines", "k_lsap_batch"}
    tot_step_ns = 0.0
    table = []
    for name, p in per.items():
        steps = n_full if name.split("<")[0] in post else n_fwd
        per_step_ns = p["ns"] / steps
        tot_step_ns += per_step_ns
        table.append((name, p["n"], p["n"] / steps, p["ns"] / p["n"] / 1e3, per_step_ns / 1e3, (p["rd"] + p["wr"]) / steps / 1e6))
    with open(out_md, "w") as f:
        f.write(f"# ncu launch list summary ({src})\n\n")
        f.write(f"{len(ls)} launches captured; {n_fwd} forward passes, {n_full} full bottom-up steps. Times are ncu's serialised, "
                "cold-cache per-launch durations (shares matter, absolutes do not).\n\n")
        f.write("| kernel | launches | per step | avg us | us / step | share | DRAM MB / step |\n|---|---|---|---|---|---|---|\n")
        for name, n, nps, avg, ps, mb in sorted(table, key=lambda t: -t[4]):
            f.write(f"| {name} | {n} | {nps:.1f} | {avg:.1f} | {ps:.1f} | {ps * 1e3 / tot_step_ns:.1%} | {mb:.1f} |\n")
        f.write(f"\nsum of kernel time per step: {tot_step_ns / 1e6:.3f} ms\n")
    tc = [(n, p) for n, p in per.items() if n.startswith("k_conv_tc") or n.startswith("k_conv01") or n.startswith("k_head")]
    tr = sum(p["rd"] + p["wr"] for _, p in tc) / n_fwd
    tns = sum(p["ns"] for _, p in tc) / n_fwd
    json.dump({"source": src, "steps_captured": n_fwd, "tc_kernels": [n for n, _ in tc], "traffic_bytes_per_step": tr, "tc_launches_per_step": sum(p["n"] for _, p in tc) / n_fwd,
               "tc_ns_per_step_under_ncu": tns, "tc_share_of_step_under_ncu": tns / tot_step_ns if tot_step_ns else None},
              open(out_json, "w"), indent=1)
    print(open(out_md).read())


if __name__ == "__main__":
    main(*sys.argv[1:5])
