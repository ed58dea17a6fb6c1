"""Summarise an `ncu --set full` report (.ncu-rep) into a table: one row per launch with time,
DRAM bytes, achieved DRAM GB/s, tensor-pipe / LSU / L2 / DRAM utilisation, IPC, registers, grid.
Usage: python tools/ncu_table.py prof.ncu-rep [title]"""
import csv
import io
import subprocess
import sys

rep = sys.argv[1]
title = sys.argv[2] if len(sys.argv) > 2 else ""
if rep.endswith(".csv"):          # already exported with `ncu -i x.ncu-rep --page raw --csv` (the reports themselves are large)
    raw = open(rep).read()
else:
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], stdout=subprocess.PIPE, text=True, check=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
hdr, units, data = rows[0], rows[1], rows[2:]
col = {k: i for i, k in enumerate(hdr)}


def get(r, k, default=""):
    return r[col[k]] if k in col else default


def num(x):
    try:
        return float(x.replace(",", ""))
    except ValueError:
        return float("nan")


def scaled(r, k, to):
    """value of metric k converted to unit `to` (us, MB)"""
    v, u = num(get(r, k, "nan")), units[col[k]] if k in col else ""
    f = {"ns": 1e-3, "nsecond": 1e-3, "us": 1.0, "usecond": 1.0, "ms": 1e3, "msecond": 1e3, "s": 1e6, "second": 1e6}
    g = {"byte": 1e-6, "Kbyte": 1e-3, "Mbyte": 1.0, "Gbyte": 1e3}
    return v * (f.get(u, 1.0) if to == "us" else g.get(u, 1.0))


print("# %s" % title)
print("# ncu --set full --clock-control none (times under the profiler: cold cache, serialised; compare shares / utilisations)")
print("%-46s %8s %9s %9s %9s %8s %7s %7s %7s %6s %5s %5s" % ("kernel", "us", "dram_rdMB", "dram_wrMB", "dram_GB/s", "tensor%", "lsu%", "l2%", "dram%",
                                                              "ipc", "regs", "grid"))
for r in data:
    name = get(r, "Kernel Name").replace("void ", "").replace("riqn::", "").replace("(int)", "")
    name = name.split("(")[0][:46]
    us = scaled(r, "gpu__time_duration.sum", "us")
    rd, wr = scaled(r, "dram__bytes_read.sum", "MB"), scaled(r, "dram__bytes_write.sum", "MB")
    print("%-46s %8.1f %9.1f %9.1f %9.0f %8.1f %7.1f %7.1f %7.1f %6.2f %5s %5s" % (
        name, us, rd, wr, (rd + wr) / us * 1e3 if us else 0.0,
        num(get(r, "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "nan")),
        num(get(r, "l1tex__data_pipe_lsu_wavefronts.avg.pct_of_peak_sustained_elapsed", "nan")),
        num(get(r, "lts__t_sectors.avg.pct_of_peak_sustained_elapsed", "nan")),
        num(get(r, "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "nan")),
        num(get(r, "sm__inst_executed.avg.per_cycle_elapsed", get(r, "smsp__inst_executed.avg.per_cycle_active", "nan"))),
        get(r, "launch__registers_per_thread"), get(r, "launch__grid_size")))
