"""Weight-gradient GEMMs (fp32 C += AᵀB into main_grad) with and without automatic split-K, vs cuBLAS (addmm_ on fp32 is not
comparable, so cuBLAS is timed as the bf16-output GEMM of the same shape — a lower bound on its cost)."""

import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from prime_b200 import ops  # noqa: E402


def timeit(fn, flush, iters=10, warm=3):
    """Median device time (ms) of fn over iters launches, L2 flushed before each."""
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    dev = torch.device("cuda", 0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    T = 16384
    rows = []
    for name, M, N in [("wqkv wgrad", 6144, 2048), ("wo wgrad", 2048, 2048), ("w13 wgrad", 11264, 2048), ("w2 wgrad", 2048, 5632), ("logits wgrad", 32000, 2048)]:
        A = torch.randn(T, M, device=dev, dtype=torch.bfloat16)  # dy  [K, M]
        B = torch.randn(T, N, device=dev, dtype=torch.bfloat16)  # x   [K, N]
        C = torch.zeros(M, N, device=dev, dtype=torch.float32)
        out16 = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
        res = {}
        for label, mode in (("no_split", 0), ("auto_split", -1)):
            ops.set_gemm_split_k(mode)
            res[label] = timeit(lambda: ops.gemm(A, B, a_mn_major=True, b_mn_major=True, out=C, accumulate=True), flush)
        ops.set_gemm_split_k(-1)
        res["cublas_bf16_out"] = timeit(lambda: torch.matmul(A.t(), B, out=out16), flush)
        fl = 2.0 * M * N * T
        rows.append({"shape": name, "M": M, "N": N, "K": T, **{f"{k}_ms": round(v, 4) for k, v in res.items()}, **{f"{k}_tflops": round(fl / v / 1e9, 1) for k, v in res.items()}})
        print(json.dumps(rows[-1]), flush=True)
    print(json.dumps({"rows": rows}))


if __name__ == "__main__":
    main()
