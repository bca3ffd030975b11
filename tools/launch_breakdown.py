"""Step composition from an ``ncu --metrics gpu__time_duration.sum --csv`` launch list: time share per kernel family.

    python tools/launch_breakdown.py gpurun_out/launches_1gpu_step_r2_final.csv > profiles/step_composition_r2_final.md

Durations are taken under the profiler (serialised launches, no overlap), so the shares — not the absolute sum — are the result.
GEMM rows are split by template arguments <A_MN, B_MN, PAIR, EPI, IO> (EPI 0 plain · 1 RoPE · 2 SwiGLU · 3 SwiGLU backward; IO 0
local · 1 all-gather A · 2 reduce-scatter C · 3 parameter gather).
"""

import csv
import re
import sys
from collections import defaultdict

FAMILIES = [
    (r"gemm_bf16_kernel", "GEMM (wgmma)"),
    (r"gemm_mxfp8|quantize_mxfp8", "MXFP8 GEMM / quantisers"),
    (r"flash_fwd|bwd_dkdv|bwd_dq|bwd_delta", "attention"),
    (r"rmsnorm|colsum", "RMSNorm (fwd, bwd, weight-grad column sums)"),
    (r"adamw_push|grad_reduce|norm_publish|cast_push|barrier", "inner optimizer (reduce ⊕ norm ⊕ AdamW ⊕ push)"),
    (r"outer_nesterov|pseudograd", "outer step"),
    (r"cross_entropy|ce_count|ce_finalize", "loss"),
    (r"embedding", "embedding"),
    (r"rope|swiglu", "stand-alone RoPE / SwiGLU"),
    (r"at::native|at_cuda|cub::|elementwise_kernel|vectorized|Memset|memcpy", "torch / runtime kernels"),
]


def family(name: str) -> str:
    for pat, fam in FAMILIES:
        if re.search(pat, name):
            return fam
    return "other"


def short(name: str) -> str:
    m = re.search(r"(\w+)(<[^>]*>)?\(", name)
    return (m.group(1) + (m.group(2) or "")) if m else name[:60]


def main(path: str) -> None:
    rows = []
    with open(path, newline="") as f:
        lines = [ln for ln in f if ln.startswith('"')]
    for r in csv.DictReader(lines):
        if r.get("Metric Name") == "gpu__time_duration.sum":
            ns = float(r["Metric Value"].replace(",", ""))
            if r.get("Metric Unit") in ("us", "usecond"):
                ns *= 1e3
            rows.append((r["Kernel Name"], ns))
    total = sum(ns for _, ns in rows)
    fam = defaultdict(lambda: [0, 0.0])
    ker = defaultdict(lambda: [0, 0.0])
    for name, ns in rows:
        fam[family(name)][0] += 1
        fam[family(name)][1] += ns
        ker[short(name)][0] += 1
        ker[short(name)][1] += ns
    print(f"# Step composition — `{path}`\n\n{len(rows)} launches, {total / 1e6:.2f} ms summed kernel time (under the profiler: serialised)\n")
    print("| family | launches | ms | share |\n|---|---|---|---|")
    for k, (n, ns) in sorted(fam.items(), key=lambda kv: -kv[1][1]):
        print(f"| {k} | {n} | {ns / 1e6:.3f} | {100 * ns / total:.2f} % |")
    print("\n| kernel | launches | ms | mean µs | share |\n|---|---|---|---|---|")
    for k, (n, ns) in sorted(ker.items(), key=lambda kv: -kv[1][1])[:40]:
        print(f"| `{k}` | {n} | {ns / 1e6:.3f} | {ns / n / 1e3:.1f} | {100 * ns / total:.2f} % |")


if __name__ == "__main__":
    main(sys.argv[1])
