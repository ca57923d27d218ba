"""Turns Nsight Compute reports (*.ncu-rep) and launch-list CSVs into small text summaries.

  python tools/ncu_summary.py launches launches.csv > launches.md
  python tools/ncu_summary.py kernel   conv_tc.ncu-rep > conv_tc.md
"""
import collections
import csv
import re
import subprocess
import sys


def launches(path):
    rows = list(csv.reader(open(path)))
    hi = [i for i, r in enumerate(rows) if "Kernel Name" in r][0]
    h = rows[hi]
    ki, vi = h.index("Kernel Name"), h.index("Metric Value")
    agg = collections.OrderedDict()
    n = 0
    for r in rows[hi + 1:]:
        if len(r) <= vi:
            continue
        name = re.sub(r"\(.*", "", r[ki])
        name = re.sub(r".*::", "", name)
        a = agg.setdefault(name, [0, 0.0])
        a[0] += 1
        a[1] += float(r[vi].replace(",", "")) / 1e3
        n += 1
    tot = sum(v[1] for v in agg.values())
    print(f"# launch list ({path}): {n} launches, {tot / 1e3:.2f} ms of kernel time (ncu: cold cache, serialised -- compare shares)\n")
    print("| kernel | launches | total us | share |\n|---|---:|---:|---:|")
    for k, v in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print(f"| `{k}` | {v[0]} | {v[1]:.1f} | {100 * v[1] / tot:.1f} % |")


WANT = ["gpu__time_duration.sum", "dram__bytes_read.sum ", "dram__bytes_write.sum ", "dram__bytes_read.sum.per_second", "dram__bytes_write.sum.per_second",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__pipe_tensor_cycles_active_realtime.avg.pct_of_peak_sustained_elapsed", "sm__pipe_tensor_subpipe_hmma_cycles_active_realtime.avg ",
        "sm__inst_executed_pipe_tensor_subpipe_hmma.avg.pct_of_peak_sustained_active", "sm__mem_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed",
        "l1tex__m_xbar2l1tex_read_bytes.sum ", "l1tex__m_xbar2l1tex_read_bytes.sum.per_second", "launch__grid_size", "launch__block_size",
        "launch__registers_per_thread ", "launch__occupancy_limit_shared_mem", "sm__cycles_elapsed.avg ", "sm__cycles_elapsed.avg.per_second",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__cycles_active.avg ", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "launch__shared_mem_per_block_dynamic", "sm__cycles_active.avg "]


def kernel(path):
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    hdr, units = rows[0], rows[1]
    for vals in rows[2:]:
        d = dict(zip(hdr, vals))
        print(f"# {d.get('Kernel Name', '?')[:120]}\n")
        print("| metric | unit | value |\n|---|---|---:|")
        for h, u, v in zip(hdr, units, vals):
            if any(h == w.strip() or (w.endswith(" ") and h == w.strip()) for w in WANT) or h in [w.strip() for w in WANT]:
                print(f"| {h} | {u} | {v} |")
        print()




TABLE = [("gpu__time_duration.sum", "us", 1e-3), ("sm__pipe_tensor_cycles_active_realtime.avg.pct_of_peak_sustained_elapsed", "tensor pipe % of elapsed", 1),
         ("sm__cycles_elapsed.avg.per_second", "SM GHz", 1), ("dram__bytes_read.sum", "DRAM rd MB", 1), ("dram__bytes_write.sum", "DRAM wr MB", 1),
         ("lts__throughput.avg.pct_of_peak_sustained_elapsed", "L2 %", 1), ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "SM %", 1),
         ("launch__grid_size", "grid", 1), ("launch__registers_per_thread", "regs", 1)]


def table(path, out_json=None):
    """One row per kernel of an `ncu --page raw --csv` dump: time, tensor-pipe %, SM clock, DRAM bytes, L2 %."""
    import json
    rows = list(csv.reader(open(path)))
    hi = [i for i, r in enumerate(rows) if "Kernel Name" in r][0]
    hdr, units = rows[hi], rows[hi + 1]
    print(f"# {path}: ncu --set full --clock-control none (cold-cache, serialised replays: compare shares and per-launch metrics)\n")
    print("| # | kernel | grid | us | tensor pipe % of elapsed | smem->tensor operand path % | SM GHz | DRAM rd MB | DRAM wr MB | L2 % | SM % | regs |\n|---|---|---:|---:|---:|---:|---:|---:|---:|---:|---:|---:|")
    recs = []
    for n, vals in enumerate(rows[hi + 2:]):
        if len(vals) < len(hdr):
            continue
        d = dict(zip(hdr, vals))
        u = dict(zip(hdr, units))

        def num(key, to=None):
            v = d.get(key, "")
            try:
                x = float(v.replace(",", ""))
            except ValueError:
                return float("nan")
            unit = u.get(key, "")
            if to == "MB":
                x *= {"byte": 1e-6, "Kbyte": 1e-3, "Mbyte": 1, "Gbyte": 1e3}.get(unit, 1e-6)
            if to == "us":
                x *= {"ns": 1e-3, "us": 1, "ms": 1e3, "s": 1e6}.get(unit, 1e-3)
            if to == "GHz":
                x *= {"Hz": 1e-9, "Khz": 1e-6, "Mhz": 1e-3, "Ghz": 1, "hz": 1e-9, "cycle/nsecond": 1, "cycle/usecond": 1e-3, "cycle/second": 1e-9}.get(unit, 1)
            return x
        name = re.sub(r"\(CUtensorMap.*", "", d["Kernel Name"])
        name = re.sub(r".*::", "", name)
        rec = {"kernel": name, "grid": d.get("launch__grid_size", ""), "us": num("gpu__time_duration.sum", "us"),
               "tensor_pct": num("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed"),
               "mem_tensor_pct": num("sm__mem_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed"),
               "sm_ghz": num("sm__cycles_elapsed.avg.per_second", "GHz"), "dram_rd_mb": num("dram__bytes_read.sum", "MB"),
               "dram_wr_mb": num("dram__bytes_write.sum", "MB"), "l2_pct": num("lts__throughput.avg.pct_of_peak_sustained_elapsed"),
               "sm_pct": num("sm__throughput.avg.pct_of_peak_sustained_elapsed"), "regs": d.get("launch__registers_per_thread", "")}
        recs.append(rec)
        print(f"| {n} | `{name}` | {rec['grid']} | {rec['us']:.1f} | {rec['tensor_pct']:.1f} | {rec['mem_tensor_pct']:.1f} | {rec['sm_ghz']:.2f} | {rec['dram_rd_mb']:.1f} | "
              f"{rec['dram_wr_mb']:.1f} | {rec['l2_pct']:.1f} | {rec['sm_pct']:.1f} | {rec['regs']} |")
    if out_json:
        json.dump(recs, open(out_json, "w"), indent=1)


if __name__ == "__main__" and len(sys.argv) > 1 and sys.argv[1] == "table":
    table(sys.argv[2], sys.argv[3] if len(sys.argv) > 3 else None)
elif __name__ == "__main__":
    {"launches": launches, "kernel": kernel}[sys.argv[1]](sys.argv[2])
