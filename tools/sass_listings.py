#!/usr/bin/env python
"""Per-kernel SASS listings of the built library → ``profiles/sass/`` (local output, not committed).

    python tools/sass_listings.py            # every kernel family, one representative instantiation each, + INDEX.md
    python tools/sass_listings.py --all      # every instantiation (≈30 MB of text: not committed)

A listing is the ``cuobjdump -sass -fun <mangled>`` output with the encoding words stripped: address + instruction per line.
INDEX.md tabulates, per listed kernel, the instruction count and the mnemonics that prove the hardware path
(HGMMA = wgmma, HMMA = mma.sync, LDSM = ldmatrix, UTMA* = TMA, SYNCS = mbarrier, *.SYS = peer traffic, LDGMC/multimem = NVLS).
"""

from __future__ import annotations

import argparse
import re
import subprocess
from collections import Counter
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
LIB = ROOT / "prime_b200" / "_C" / "libprime_b200.so"
OUT = ROOT / "profiles" / "sass"
PROOF = ["HGMMA", "UTMALDG", "UTMASTG", "SYNCS", "LDSM", "HMMA", "MUFU.EX2", "LDGMC"]
# representative instantiation per family (demangled-name regex → short file name); first match wins.
# gemm_bf16_kernel<A_MN, B_MN, EPI, IO>: EPI 0 plain | 1 RoPE | 2 SwiGLU | 3 SwiGLU backward; IO 0 local | 1 all-gather | 2 reduce-scatter | 3 weight gather
PICK = [
    (r"gemm_bf16_kernel<0, 0, 0, 0>", "gemm_bf16_kmajor"),
    (r"gemm_bf16_kernel<1, 1, 0, 0>", "gemm_bf16_wgrad_mnmajor"),
    (r"gemm_bf16_kernel<0, 0, 1, 0>", "gemm_bf16_rope_epilogue"),
    (r"gemm_bf16_kernel<0, 0, 2, 0>", "gemm_bf16_swiglu_epilogue"),
    (r"gemm_bf16_kernel<0, 1, 3, 0>", "gemm_bf16_swiglu_bwd_epilogue"),
    (r"gemm_bf16_kernel<0, 0, 0, 1>", "gemm_allgather_activation_IO1"),
    (r"gemm_bf16_kernel<0, 0, 0, 2>", "gemm_reduce_scatter_IO2"),
    (r"gemm_bf16_kernel<0, 0, 0, 3>", "gemm_param_gather_fwd_IO3"),
    (r"gemm_bf16_kernel<0, 1, 0, 3>", "gemm_param_gather_dgrad_IO3"),
    (r"gemm_bf16_kernel<0, 0, 2, 3>", "gemm_param_gather_swiglu_IO3"),
    (r"gemm_mxfp8_kernel", "gemm_mxfp8"),
    (r"quantize_mxfp8_kernel", "quantize_mxfp8"),
    # attention kernels <D, kDoc>: kDoc = document masking
    (r"flash_fwd_kernel<128, false>", "flash_fwd_d128"),
    (r"bwd_dkdv_kernel<128, false>", "flash_bwd_dkdv_d128"),
    (r"bwd_dq_kernel<128, false>", "flash_bwd_dq_d128"),
    (r"flash_fwd_kernel<128, true>", "flash_fwd_doc_d128"),
    (r"bwd_dkdv_kernel<128, true>", "flash_bwd_dkdv_doc_d128"),
    (r"bwd_dq_kernel<128, true>", "flash_bwd_dq_doc_d128"),
    (r"doc_bounds_kernel", "doc_bounds"),
    (r"bwd_delta_kernel", "flash_bwd_delta"),
    (r"rmsnorm_fwd_kernel<4, true>", "rmsnorm_fwd_residual"),
    (r"rmsnorm_bwd_kernel<4, true>", "rmsnorm_bwd_residual"),
    (r"swiglu_bwd_kernel", "swiglu_bwd"),
    (r"cross_entropy_kernel", "cross_entropy_fwd_bwd"),
    (r"embedding_fwd_kernel", "embedding_fwd_peer_gather"),
    (r"embedding_sort_kernel", "embedding_bwd_sort"),
    (r"embedding_bwd_kernel", "embedding_bwd_segmented"),
    (r"^grad_reduce_kernel", "grad_reduce"),
    (r"adamw_push_kernel", "adamw_push"),
    (r"norm_publish_kernel", "norm_publish"),
    (r"pseudograd_quant_kernel", "outer_pseudograd_quant"),
    (r"^outer_nesterov_kernel", "outer_nesterov_int8"),
    (r"outer_nesterov_f32_kernel", "outer_nesterov_f32"),
    (r"barrier_kernel", "flag_barrier"),
    (r"mc_all_reduce", "nvls_all_reduce"),
]


def functions() -> list[tuple[str, str]]:
    txt = subprocess.run(["cuobjdump", "-sass", str(LIB)], capture_output=True, text=True, check=True).stdout
    mangled = re.findall(r"Function : (\S+)", txt)
    dem = subprocess.run(["c++filt"], input="\n".join(mangled), capture_output=True, text=True, check=True).stdout.splitlines()
    return [(m, d.replace("void ", "").replace("(anonymous namespace)::", "")) for m, d in zip(mangled, dem)]


def listing(mangled: str) -> list[str]:
    txt = subprocess.run(["cuobjdump", "-sass", "-fun", mangled, str(LIB)], capture_output=True, text=True, check=True).stdout
    out = []
    for ln in txt.splitlines():
        m = re.match(r"\s+/\*([0-9a-f]{4,})\*/\s+(.*?);\s*/\*", ln)
        if m:
            out.append(f"/*{m.group(1)}*/  {m.group(2).strip()} ;")
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--all", action="store_true")
    args = ap.parse_args()
    OUT.mkdir(parents=True, exist_ok=True)
    fns = functions()
    todo: list[tuple[str, str, str]] = []
    if args.all:
        todo = [(m, d, re.sub(r"[^A-Za-z0-9_]+", "_", d.split("(")[0])[:100]) for m, d in fns]
    else:
        for pat, short in PICK:
            for m, d in fns:
                if re.search(pat, d):
                    todo.append((m, d, short))
                    break
    rows = []
    for m, d, short in todo:
        lines = listing(m)
        (OUT / f"{short}.sass").write_text(f"// {d.split('(')[0]}\n// {m}\n" + "\n".join(lines) + "\n")
        c = Counter()
        for ln in lines:
            ins = ln.split("*/", 1)[1]
            for k in PROOF:
                if re.search(rf"\b{re.escape(k)}", ins):
                    c[k] += 1
            if re.search(r"\.SYS\b", ins):
                c["*.SYS"] += 1
        rows.append((short, d.split("(")[0], len(lines), c))
    cols = PROOF + ["*.SYS"]
    idx = ["# SASS listings (`cuobjdump -sass -fun`, encodings stripped)", "",
           f"{len(fns)} kernels in `libprime_b200.so`; one representative instantiation per family listed here "
           "(`python tools/sass_listings.py --all` writes every one).", "",
           "| file | kernel | instr | " + " | ".join(cols) + " |", "|---|---|---:|" + "---:|" * len(cols)]  # fmt: skip
    for short, d, n, c in rows:
        idx.append(f"| {short}.sass | `{d}` | {n} | " + " | ".join(str(c.get(k, "")) for k in cols) + " |")
    (OUT / "INDEX.md").write_text("\n".join(idx) + "\n")
    print(f"wrote {len(rows)} listings to {OUT}")


if __name__ == "__main__":
    main()
