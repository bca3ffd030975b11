"""prime_b200 — an H100 (Hopper, sm_90a)-native DiLoCo / local-SGD training engine plus the
platform CLI & SDK surface of PrimeIntellect-ai/prime, rebuilt from scratch.

Layout
------
``prime_b200.ops``       hand-written sm_90a kernels (wgmma/TMA GEMM, flash attention, fused norm/rope/
                         swiglu/loss, fused collective+optimizer kernels) and their torch oracles
``prime_b200.models``    Llama family built on those ops
``prime_b200.parallel``  two-level mesh (DiLoCo workers × FSDP shards), symmetric NVLink heap,
                         fused reduce-scatter/AdamW/all-gather, int8 outer all-reduce, elasticity
``prime_b200.train``     the ``diloco.train`` entrypoint
``prime_b200.platform``  CLI + SDKs (pods, sandboxes, evals, tunnel, MCP …)
"""

__version__ = "0.1.1"
