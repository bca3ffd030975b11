#!/bin/bash
# Run ON the GPU box: everything the profiles/ directory should contain for the current build, in one call (≈6-8 min).
set -u
mkdir -p gpurun_out/ncu
python -m pytest tests -m gpu -x -q 2>&1 | tail -3 | tee gpurun_out/pytest_gpu.txt
python __graft_entry__.py smoke 2>&1 | tail -1 | tee gpurun_out/smoke.txt
python bench.py --steps 10 --warmup 3 2>gpurun_out/bench_final.err | tee gpurun_out/bench_final.json | cut -c1-160
python bench.py --steps 6 --warmup 3 --no-fused-comm --attn sdpa 2>/dev/null | tee gpurun_out/bench_b0_sdpa_nccl.json | cut -c1-160
python tools/attn_bench.py > gpurun_out/attn_bench_final.json 2>/dev/null
python tools/op_bench.py > gpurun_out/op_bench_final.json 2>/dev/null
bash tools/profile.sh 2>&1 | tail -6
bash tools/sanitize.sh 2>&1 | tail -8
du -sh gpurun_out
