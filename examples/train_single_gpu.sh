#!/bin/bash
# Llama-1B, seq 1024, 64 sequences/step, DiLoCo H=100 — one H100. Ctrl-C (or SIGTERM) writes a final checkpoint.
set -euo pipefail
cd "$(dirname "$0")/.."
python -c "import __graft_entry__ as g; g.build()"          # compile the sm_90a kernels in-tree (seconds)
python -m diloco.train @configs/1B/h100.toml \
    --ckpt.path "${CKPT:-/tmp/prime_b200/1b}" --ckpt.interval 500 --ckpt.resume latest \
    --monitor.jsonl_path "${CKPT:-/tmp/prime_b200/1b}/metrics.jsonl" "$@"
