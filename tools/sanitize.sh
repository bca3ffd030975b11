#!/bin/bash
# Run ON the GPU box: compute-sanitizer over the kernel tests. memcheck = out-of-bounds / misaligned global+shared accesses,
# racecheck = shared-memory hazards, synccheck = invalid barrier usage. TMA / tensor-core kernels run ~50-100x slower under the tool,
# so each tool gets a focused subset; summaries land in gpurun_out/sanitizer_*.txt (copy to profiles/).
set -u
SAN=compute-sanitizer
run() { # tool, pytest -k expression, tag[, test file]
  timeout 600 $SAN --tool "$1" --print-limit 5 --error-exitcode 9 python -m pytest "${4:-tests/test_kernels_gpu.py}" -q -k "$2" -p no:cacheprovider \
    > gpurun_out/sanitizer_$3.log 2>&1
  echo "$1 [$2]: exit $? — $(grep -E 'ERROR SUMMARY|passed|failed' gpurun_out/sanitizer_$3.log | tr '\n' ' ')" | tee -a gpurun_out/sanitizer_summary.txt
}
: > gpurun_out/sanitizer_summary.txt
run memcheck  "rmsnorm or swiglu or rope_qkv or cross_entropy" memcheck_elementwise
run memcheck  "gemm_layouts or gemm_fp32 or split_k" memcheck_gemm
run memcheck  "flash_attention or rope_attention" memcheck_attention
run racecheck "rmsnorm or cross_entropy" racecheck_elementwise
run synccheck "gemm_transposed or flash_attention or rope_attention or qkv_gemm_rope" synccheck_tc
run memcheck  "mxfp8" memcheck_mxfp8
# tail rows, last vectors and partial tiles of the elementwise kernels and GEMM epilogues (the largest shapes are left to the plain run)
run memcheck  "gpu and not 16384 and not 128256 and not 14336" memcheck_edges tests/test_kernel_edges_gpu.py
run synccheck "mxfp8 or swiglu_epilogue" synccheck_mxfp8
# decode kernels: KV append, step bookkeeping and split-KV attention at the small shapes (the 32 K-key fp64 sweep is left to the plain run)
run memcheck  "gpu and (kv_append or decode_advance or graph_replay or generate_on_cuda)" memcheck_decode tests/test_kv_cache.py
# the e4m3 cache: append and prefill quantisers, verify attention at cap 2048, graphs and speculative rounds (the 32 K-key sweep, the
# 8 K bound check and the 1B models are left to the plain run)
run memcheck  "gpu and not decode_attn_fp8_matches and not analytic_bound and not 1b_shape" memcheck_kv_fp8 tests/test_kv_fp8_gpu.py
# e4m3 weights: dequantisation, the skinny GEMM at every M, strided outputs, graphs and speculation (the projection-shape sweep, the
# split-count sweep and the 1B models are left to the plain run)
run memcheck  "gpu and not projection_shapes and not split_count and not 1b" memcheck_weights_fp8 tests/test_weights_fp8_gpu.py
# flash attention against fp64: every instantiation, tile-edge documents and windows, probes (S >= 4096 is left to the plain run)
run memcheck  "gpu and not S4096 and not S8192 and not 32768" memcheck_attention_fp64 tests/test_attention_fp64_gpu.py
run racecheck "gpu and not S4096 and not S8192 and not 32768 and not doc_bounds" racecheck_attention_fp64 tests/test_attention_fp64_gpu.py
# bf16 GEMM in both tile widths (128 x 128 and the 128 x 256 setmaxnreg tile): every layout and epilogue at the small edge shapes
run memcheck  "gpu and not 5632" memcheck_gemm_wide tests/test_gemm_wide_gpu.py
run racecheck "gpu and not 5632" racecheck_gemm_wide tests/test_gemm_wide_gpu.py
# staged GEMM epilogue (shared-memory slots, TMA stores, TMA loads of the saved gate_up) in both tile widths
run memcheck  "gpu" memcheck_gemm_epilogue tests/test_gemm_epilogue_gpu.py
run racecheck "gpu" racecheck_gemm_epilogue tests/test_gemm_epilogue_gpu.py
run synccheck "gpu" synccheck_gemm_epilogue tests/test_gemm_epilogue_gpu.py
# the collective GEMMs (all-gather, reduce-scatter, weight-gather) with local buffers as the peers, against the local GEMM bit for
# bit: groups of 1 and 2 at the small shapes (a gated tile traps after 4 s, which the tool's slowdown would put at risk; P >= 3, the
# 7B MLP and the raster all-gather schedule are left to the plain run)
run memcheck  "gpu and (P1 or P2) and not llama7b and not raster" memcheck_gemm_collective tests/test_gemm_collective_epilogue_gpu.py
run racecheck "gpu and (P1 or P2) and not llama7b and not raster" racecheck_gemm_collective tests/test_gemm_collective_epilogue_gpu.py
run synccheck "gpu and (P1 or P2) and not llama7b and not raster" synccheck_gemm_collective tests/test_gemm_collective_epilogue_gpu.py
# optimizer, outer-step and peer-gather kernels with local buffers as peers, at the small shapes (block_sum / s_max shared memory;
# pseudograd_quant's __syncthreads inside the grid-stride loop needs the 4229-block case)
run memcheck  "gpu and not pass1 and not 4225 and not 1081352 and not 1600048 and not engine" memcheck_optimizer tests/test_optimizer_kernels_gpu.py
run racecheck "gpu and (grad_reduce or norm_publish or pseudograd) and not pass1" racecheck_optimizer tests/test_optimizer_kernels_gpu.py
run synccheck "gpu and pseudograd" synccheck_optimizer tests/test_optimizer_kernels_gpu.py
cat gpurun_out/sanitizer_summary.txt
