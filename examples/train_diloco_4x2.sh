#!/bin/bash
# BASELINE config 2: 4 DiLoCo workers × 2-GPU FSDP on one 8×H100 NVSwitch box, fused P2P reduce/AdamW/all-gather kernels.
set -euo pipefail
cd "$(dirname "$0")/.."
python -c "import __graft_entry__ as g; g.build()"
python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 --master-port "${PORT:-29500}" \
    -m diloco.train @configs/1B/diloco_4x2.toml --ckpt.path "${CKPT:-/tmp/prime_b200/1b_4x2}" "$@"
