"""Condense `ncu --page raw --csv` exports into the few numbers the roofline argument needs, one row per kernel launch.

    python tools/ncu_summary.py gpurun_out/ncu/gemm.raw.csv gpurun_out/ncu/attn.raw.csv ... > profiles/ncu_summary_r1.md
"""

import csv
import json
import re
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
WANT = {
    "gpu__time_duration.sum": "dur_us",
    "dram__bytes_read.sum": "dram_rd_MB",
    "dram__bytes_write.sum": "dram_wr_MB",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed": "dram_pct",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active": "tensor_pct",
    "sm__inst_executed_pipe_tensor.sum": "tensor_inst",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed": "sm_pct",
    "sm__warps_active.avg.pct_of_peak_sustained_active": "warps_active_pct",
    "launch__registers_per_thread": "regs",
    "launch__grid_size": "grid",
    "launch__block_size": "block",
    "launch__shared_mem_per_block_dynamic": "dyn_smem",
    "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum": "smem_bank_conflicts",
    "lts__t_sector_hit_rate.pct": "l2_hit_pct",
    "sm__cycles_active.avg": "sm_cycles_active",
    "smsp__cycles_active.avg": "smsp_cycles",
}


def to_float(v: str) -> float | None:
    try:
        return float(v.replace(",", ""))
    except ValueError:
        return None


def scale(value: float, unit: str, target: str) -> float:
    u = unit.lower()
    if target == "us":
        return value * {"ns": 1e-3, "nsecond": 1e-3, "us": 1, "usecond": 1, "ms": 1e3, "msecond": 1e3, "s": 1e6, "second": 1e6}.get(u, 1)
    if target == "MB":
        return value * {"byte": 1e-6, "kbyte": 1e-3, "mbyte": 1, "gbyte": 1e3}.get(u, 1e-6)
    return value


def rows_of(path: Path):
    with open(path, newline="") as f:
        lines = [ln for ln in f if not ln.startswith("==")]
    rd = list(csv.reader(lines))
    if len(rd) < 3:
        return []
    header, units = rd[0], rd[1]
    out = []
    for r in rd[2:]:
        if len(r) != len(header):
            continue
        rec = dict(zip(header, r))
        # kernels in anonymous namespaces are reported as "<unnamed>::name<args>(…)": strip the qualifier BEFORE cutting at the
        # first template bracket (round 1 printed blank names for the GEMM / attention rows because of it)
        full = rec.get("Kernel Name", "?").replace("void ", "")
        full = re.sub(r"(<unnamed>|\(anonymous namespace\))::", "", full)
        row = {"kernel": re.sub(r"\(.*", "", re.sub(r"<.*", "", full)).strip(), "id": rec.get("ID")}
        tmpl = re.search(r"<([^>]*)>", full)
        if tmpl:
            row["tmpl"] = tmpl.group(1)
        for metric, short in WANT.items():
            if metric in rec:
                v = to_float(rec[metric])
                if v is None:
                    continue
                unit = units[header.index(metric)]
                if short == "dur_us":
                    v = scale(v, unit, "us")
                elif short.endswith("_MB"):
                    v = scale(v, unit, "MB")
                row[short] = round(v, 2)
        out.append(row)
    return out


def main(paths):
    peaks = {}
    try:
        peaks = json.loads((ROOT / "MEASURED_PEAKS.json").read_text())
    except Exception:
        pass
    hbm = peaks.get("hbm_gbs", 3350.0)  # default: H100 SXM data-sheet HBM3 bandwidth (not a measured rate)
    print("# ncu summary (one row per captured launch; `--set full --clock-control none`, durations are under the profiler's cache control — "
          "compare shares and utilisations, not absolute times; event-timed numbers live in the *_bench JSON files)\n")  # fmt: skip
    cols = ["kernel", "tmpl", "dur_us", "dram_rd_MB", "dram_wr_MB", "dram_GBps", "dram_pct", "tensor_pct", "sm_pct", "warps_active_pct", "regs", "grid", "block",
            "dyn_smem", "l2_hit_pct"]  # fmt: skip
    for p in paths:
        rows = rows_of(Path(p))
        print(f"## {Path(p).name}  ({len(rows)} launches)\n")
        print("| " + " | ".join(cols) + " |")
        print("|" + "---|" * len(cols))
        for r in rows:
            if "dur_us" in r and r["dur_us"] > 0:
                r["dram_GBps"] = round((r.get("dram_rd_MB", 0) + r.get("dram_wr_MB", 0)) / r["dur_us"] * 1e3, 0)
            print("| " + " | ".join(str(r.get(c, "")) for c in cols) + " |")
        print()
    print(f"\nMeasured copy bandwidth (MEASURED_PEAKS.json): {hbm} GB/s; measured sustained cuBLAS bf16: {peaks.get('bf16_tflops_sustained')} TFLOP/s.")


if __name__ == "__main__":
    main(sys.argv[1:])
