"""Key metrics of an ncu report as a small CSV (no GPU needed):  python scripts/ncu_key.py rep.ncu-rep > x_ncu_key.csv
Also summarises an `ncu --csv --log-file` launch list:          python scripts/ncu_key.py --launches launches.csv > y_summary.csv"""
import collections
import csv
import io
import subprocess
import sys

KEYS = ["Kernel Name", "Grid Size", "Block Size", "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "dram__throughput.avg.pct_of_peak_sustained_elapsed", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__inst_issued.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum", "launch__registers_per_thread",
        "launch__shared_mem_per_block_dynamic", "lts__t_sector_hit_rate.pct", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "lts__t_bytes.sum", "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum",
        "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio"]


def key_report(path):
    raw = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units, data = rows[0], rows[1], rows[2:]
    idx = [hdr.index(k) for k in KEYS if k in hdr]
    w = csv.writer(sys.stdout)
    w.writerow([hdr[i] for i in idx])
    w.writerow([units[i] for i in idx])
    for r in data:
        w.writerow([r[i] for i in idx])


def launch_summary(path):
    txt = open(path).read()
    start = txt.find('"ID"')
    rows = list(csv.DictReader(io.StringIO(txt[start:])))
    agg = collections.OrderedDict()
    for r in rows:
        if r.get("Metric Name") is None:
            continue
        k = r["Kernel Name"]
        a = agg.setdefault(k, collections.defaultdict(float))
        try:
            v = float(r["Metric Value"].replace(",", ""))
        except ValueError:
            continue
        m, u = r["Metric Name"], r["Metric Unit"]
        if m == "gpu__time_duration.sum":
            a["us"] += v / 1e3 if u in ("ns", "nsecond") else (v if u in ("us", "usecond") else v * 1e3)
            a["n"] += 1
        elif m.startswith("dram__bytes"):
            scale = {"byte": 1e-6, "Kbyte": 1e-3, "Mbyte": 1.0, "Gbyte": 1e3}.get(u, 1e-6)
            a["dram_mb"] += v * scale
        elif m.startswith("sm__pipe_tensor"):
            a["tensor"] += v
        elif m.startswith("sm__inst_issued"):
            a["issue"] += v
    tot = sum(a["us"] for a in agg.values())
    print("kernel,launches,total_us,share_pct,avg_us,avg_dram_MB,avg_tensor_pipe_pct,avg_issue_pct")
    for k, a in sorted(agg.items(), key=lambda kv: -kv[1]["us"]):
        n = max(a["n"], 1)
        name = k.replace("vox::<unnamed>::", "").replace("void ", "")
        print(f"{name.split('(')[0]},{int(a['n'])},{a['us']:.1f},{100 * a['us'] / tot:.2f},{a['us'] / n:.2f},{a['dram_mb'] / n:.3f},"
              f"{a['tensor'] / n:.1f},{a['issue'] / n:.1f}")


if __name__ == "__main__":
    if sys.argv[1] == "--launches":
        launch_summary(sys.argv[2])
    else:
        key_report(sys.argv[1])
