"""Where do the warps of a kernel wait? Condense `ncu --page source --csv` (per-SASS-instruction stall samples) into regions.

    ncu -i gpurun_out/ncu/attn.ncu-rep --page source --csv --kernel-name regex:dkdv > /tmp/dkdv.csv
    python tools/ncu_source_hotspots.py /tmp/dkdv.csv

Instructions are grouped into runs with the same execution count (= same loop nest / branch); for every run the share of all
stall samples and the opcodes that collected them are printed, then the top single instructions. Useful to find which loads or
branches of a kernel collect the stalls.
"""

import collections
import csv
import re
import sys


def main(path: str, top: int = 25) -> None:
    rows = list(csv.reader(open(path)))
    hdr = next(i for i, r in enumerate(rows) if "# Samples" in r)
    h = rows[hdr]
    si, src, ex = h.index("# Samples"), h.index("Source"), h.index("Instructions Executed")
    launches = max(1, sum(1 for r in rows if r and r[0] == "Kernel Name"))
    data = [(int(r[si]), r[src].strip(), int(r[ex])) for r in rows[hdr + 1 :] if len(r) > si and r[si].isdigit()]
    data = data[: len(data) // launches]  # identical launches are concatenated: keep the first
    total = sum(d[0] for d in data) or 1
    print(f"{len(data)} instructions, {total} stall samples (first of {launches} captured launches)\n")
    print("runs of instructions with one execution count (>= 1 % of the samples):")
    runs, cur = [], None
    for i, (s, t, e) in enumerate(data):
        if cur is None or cur["exec"] != e:
            cur = {"exec": e, "first": i, "last": i, "samples": 0, "ops": collections.Counter()}
            runs.append(cur)
        cur["last"], cur["samples"] = i, cur["samples"] + s
        m = re.match(r"(@!?U?P\d+\s+)?([A-Z0-9_.]+)", t)
        cur["ops"][m.group(2).split(".")[0] if m else "?"] += s
    for r in runs:
        if r["samples"] * 100 >= total:
            ops = ", ".join(f"{k} {v}" for k, v in r["ops"].most_common(4))
            print(f"  exec {r['exec']:>9}  instr {r['first']:>5}-{r['last']:<5} samples {r['samples']:>6} ({100 * r['samples'] / total:4.1f} %)  {ops}")
    print(f"\ntop {top} instructions:")
    for s, t, e in sorted(data, reverse=True)[:top]:
        print(f"  {s:>6} ({100 * s / total:4.1f} %)  exec {e:>9}  {t[:100]}")


if __name__ == "__main__":
    main(sys.argv[1], int(sys.argv[2]) if len(sys.argv) > 2 else 25)
