"""One markdown row per distinct kernel of an `ncu --page raw --csv` export (longest launch of each):
duration, DRAM bytes and GB/s against the measured HBM peak, tensor-pipe / LSU-wavefront / issue
utilisation, registers.    python tools/ncu_kernel_table.py raw.csv > <name>.md"""
import csv, json, os, re, sys

rows = list(csv.reader(open(sys.argv[1])))
hdr, units, data = rows[0], rows[1], rows[2:]
col = {k: i for i, k in enumerate(hdr)}
try:
    peak = float(json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "MEASURED_PEAKS.json")))["hbm_gbs"])
except Exception:
    peak = 3350.0


def num(row, key, default=0.0):
    try:
        return float(row[col[key]].replace(",", ""))
    except Exception:
        return default


def scaled(row, key):
    """value in base units (bytes, ns) whatever unit prefix ncu picked"""
    v = num(row, key)
    u = units[col[key]] if key in col else ""
    mult = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "ns": 1, "us": 1e3, "ms": 1e6, "s": 1e9,
            "nsecond": 1, "usecond": 1e3, "msecond": 1e6, "second": 1e9}
    return v * mult.get(u, 1)


best = {}
for r in data:
    name = re.sub(r"^void ", "", r[col["Kernel Name"]])
    name = re.sub(r"hdrnet_b200::", "", name)
    name = re.sub(r"\(.*$", "", name)
    t = scaled(r, "gpu__time_duration.sum")
    n = best.setdefault(name, {"n": 0, "t": -1, "row": None})
    n["n"] += 1
    if t > n["t"]:
        n["t"], n["row"] = t, r
print(f"| kernel (longest of n launches) | n | time us | DRAM MB | GB/s | % of {peak:.0f} GB/s | tensor pipe % | LSU smem wavefronts % | issue active % | regs | grid x block |")
print("|---|---|---|---|---|---|---|---|---|---|---|")
for name, e in sorted(best.items(), key=lambda kv: -kv[1]["t"]):
    r = e["row"]
    t_ns = e["t"]
    dram = scaled(r, "dram__bytes_read.sum") + scaled(r, "dram__bytes_write.sum")
    gbs = dram / t_ns if t_ns > 0 else 0.0
    print(f"| `{name[:110]}` | {e['n']} | {t_ns / 1e3:.1f} | {dram / 1e6:.1f} | {gbs:.0f} | {100 * gbs / peak:.1f} | "
          f"{num(r, 'sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed'):.1f} | "
          f"{num(r, 'l1tex__data_pipe_lsu_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed'):.1f} | "
          f"{num(r, 'smsp__issue_active.avg.pct_of_peak_sustained_active'):.1f} | "
          f"{int(num(r, 'launch__registers_per_thread'))} | {int(num(r, 'launch__grid_size'))} x {int(num(r, 'launch__block_size'))} |")
