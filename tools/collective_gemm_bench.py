"""Fused all-gather⊕GEMM and GEMM⊕reduce-scatter vs the NCCL formulation, on the tensor-parallel MLP shapes of Llama-1B.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 tools/collective_gemm_bench.py

Device-timed with CUDA events, max over ranks, median of 10, L2 flushed. Roofline: the slower of the GEMM at the measured
cuBLAS peak and the remote bytes at 900 GB/s per direction.
"""

import json
import sys
from pathlib import Path

import torch
import torch.distributed as dist

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from prime_b200 import ops  # noqa: E402
from prime_b200.parallel.collective_gemm import CollectiveGemm  # noqa: E402
from prime_b200.parallel.mesh import init_distributed  # noqa: E402
from prime_b200.parallel.symm import SymmetricHeap, dist_exchange  # noqa: E402


def timeit(fn, flush, iters=10, warm=3):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(iters):
        flush.zero_()
        dist.barrier()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        t = torch.tensor([e0.elapsed_time(e1)], device="cuda")
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ts.append(float(t))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    w = init_distributed("nccl")
    dev = torch.device("cuda", w.local_rank)
    n, r = w.world_size, w.rank
    heap = SymmetricHeap(2 << 30, r, n, dist_exchange(), dev)
    cg = CollectiveGemm(heap, list(range(n)))
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    from prime_b200.utils.clocks import ClockSampler

    sampler = ClockSampler(torch.cuda.current_device(), period_s=0.05)
    if r == 0:
        sampler.start()
    peaks = json.loads((ROOT / "MEASURED_PEAKS.json").read_text()) if (ROOT / "MEASURED_PEAKS.json").exists() else {}
    peak = float(peaks.get("bf16_tflops_sustained", 989.0)) * 1e12  # default: H100 SXM data-sheet dense bf16 (not a measured rate)
    T, D, FF = 16384, 2048, 5632
    rows = []
    # ---- all-gather ⊕ GEMM: sequence-sharded x [T/n, D] → gate/up columns of this rank [T, 2FF/n]
    M_local, N, K = T // n, (2 * FF // n) // 256 * 256, D
    a_sym = heap.alloc(M_local * K, torch.bfloat16).view(M_local, K)
    a_sym.normal_(0, 0.1)
    B = (torch.randn(N, K, device=dev) * 0.1).to(torch.bfloat16)
    out = torch.empty(T, N, device=dev, dtype=torch.bfloat16)
    gathered = torch.empty(T, K, device=dev, dtype=torch.bfloat16)
    t_fused = timeit(lambda: cg.all_gather_gemm(a_sym, B, out), flush)

    def nccl_ag():
        dist.all_gather_into_tensor(gathered, a_sym)
        ops.gemm(gathered, B, out=out)

    t_nccl = timeit(nccl_ag, flush)
    t_gemm = timeit(lambda: ops.gemm(gathered, B, out=out), flush)
    fl = 2.0 * T * N * K
    remote = (n - 1) * M_local * K * 2
    rows.append({"op": "all_gather⊕GEMM (x[T/n,D] → [T, 2FF/n])", "M": T, "N": N, "K": K, "fused_ms": round(t_fused, 4), "nccl_ag_plus_gemm_ms": round(t_nccl, 4),
                 "gemm_only_ms": round(t_gemm, 4), "speedup_vs_nccl": round(t_nccl / t_fused, 3), "fused_tflops": round(fl / t_fused / 1e9, 1),
                 "remote_GB_per_s": round(remote / t_fused / 1e6, 1), "roofline_ms": round(max(fl / peak, remote / 900e9) * 1e3, 4)})  # fmt: skip
    # ---- GEMM ⊕ reduce-scatter: h[T, FF/n] · W2[:, shard]ᵀ → y rows [T/n, D] (fp32)
    Kl = (FF // n) // 64 * 64
    a_k = (torch.randn(T, Kl, device=dev) * 0.1).to(torch.bfloat16)
    b_k = (torch.randn(D, Kl, device=dev) * 0.1).to(torch.bfloat16)
    out_sym = heap.alloc((T // n) * D, torch.float32).view(T // n, D)
    full = torch.empty(T, D, device=dev, dtype=torch.float32)
    shard = torch.empty(T // n, D, device=dev, dtype=torch.float32)
    t_fused = timeit(lambda: cg.gemm_reduce_scatter(a_k, b_k, out_sym), flush)

    def nccl_rs():
        ops.gemm(a_k, b_k, out=full)
        dist.reduce_scatter_tensor(shard, full)

    t_nccl = timeit(nccl_rs, flush)
    t_gemm = timeit(lambda: ops.gemm(a_k, b_k, out=full), flush)
    fl = 2.0 * T * D * Kl
    remote = (n - 1) * (T // n) * D * 4
    rows.append({"op": "GEMM⊕reduce_scatter (h[T,FF/n]·W2ᵀ → y[T/n, D] fp32)", "M": T, "N": D, "K": Kl, "fused_ms": round(t_fused, 4),
                 "gemm_plus_nccl_rs_ms": round(t_nccl, 4), "gemm_only_ms": round(t_gemm, 4), "speedup_vs_nccl": round(t_nccl / t_fused, 3),
                 "fused_tflops": round(fl / t_fused / 1e9, 1), "remote_GB_per_s": round(remote / t_fused / 1e6, 1),
                 "roofline_ms": round(max(fl / peak, remote / 900e9) * 1e3, 4)})  # fmt: skip
    heap.check_errors()
    if r == 0:
        print(json.dumps({"n_gpus": n, "rows": rows, "clocks": sampler.finish()}, indent=1))
    dist.barrier()
    heap.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
