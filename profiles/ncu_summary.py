"""Summarise an `ncu --set full` report (read on the CPU box): per kernel duration, DRAM bytes, achieved GB/s, % of the
measured HBM copy bandwidth (MEASURED_PEAKS.json), tensor-pipe %, registers.

    python profiles/ncu_summary.py profiles_out/x.ncu-rep > profiles_out/ncu_x.txt
"""
import csv
import io
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
rep = sys.argv[1]
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
hdr, units = rows[0], rows[1]
idx = {h: i for i, h in enumerate(hdr)}
try:
    hbm = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]
except Exception:
    hbm = 6650.0


def val(r, k, scale):
    v, u = float(r[idx[k]]), units[idx[k]]
    return v * scale[u]


T = {"s": 1e6, "ms": 1e3, "us": 1.0, "ns": 1e-3, "usecond": 1.0, "msecond": 1e3, "nsecond": 1e-3, "second": 1e6}
B = {"Gbyte": 1.0, "Mbyte": 1e-3, "Kbyte": 1e-6, "byte": 1e-9}
print(f"# {os.path.basename(rep)}  (ncu --set full --clock-control none; HBM roofline denominator = {hbm:.1f} GB/s measured copy)")
print(f"{'kernel':58s} {'us':>8s} {'rd GB':>7s} {'wr GB':>7s} {'GB/s':>7s} {'%HBM':>6s} {'tensor%':>8s} {'sm%':>6s} {'L2hit%':>7s} {'regs':>5s}")
for r in rows[2:]:
    t = val(r, "gpu__time_duration.sum", T)
    rd, wr = val(r, "dram__bytes_read.sum", B), val(r, "dram__bytes_write.sum", B)
    gbs = (rd + wr) / t * 1e6
    name = r[idx["Kernel Name"]].split("(")[0].replace("void ", "")[:58]
    tp = r[idx["sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active"]] if "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active" in idx else "0"
    print(f"{name:58s} {t:8.1f} {rd:7.3f} {wr:7.3f} {gbs:7.0f} {100 * gbs / hbm:6.1f} {float(tp):8.1f} "
          f"{float(r[idx['sm__throughput.avg.pct_of_peak_sustained_elapsed']]):6.1f} {float(r[idx['lts__t_sector_hit_rate.pct']]):7.1f} "
          f"{r[idx['launch__registers_per_thread']]:>5s}")
