"""Time the wgmma GEMM against cuBLAS (torch.matmul) on the Llama shapes; report TFLOP/s and fraction
of the measured peak (MEASURED_PEAKS.json).  CUDA events, warm-up, L2 flushed between iterations."""

import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from prime_b200 import ops  # noqa: E402


def timeit(fn, iters=10, warm=3, flush=None):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        if flush is not None:
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
    peaks = {}
    try:
        peaks = json.loads((ROOT / "MEASURED_PEAKS.json").read_text())
    except Exception:
        pass
    peak = peaks.get("bf16_tflops", 1590.0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    from prime_b200.utils.clocks import ClockSampler

    sampler = ClockSampler(0, period_s=0.05)
    sampler.start()
    T = 16384
    shapes = [
        ("qkv fwd", T, 6144, 2048, False, False),
        ("wo fwd", T, 2048, 2048, False, False),
        ("w13 fwd", T, 11264, 2048, False, False),
        ("w2 fwd", T, 2048, 5632, False, False),
        ("logits fwd", T, 32000, 2048, False, False),
        ("w13 dgrad", T, 2048, 11264, False, True),
        ("w13 wgrad", 11264, 2048, T, True, True),
        ("w2 wgrad", 2048, 5632, T, True, True),
        ("square 8192", 8192, 8192, 8192, False, False),
    ]
    rows = []
    for name, M, N, K, amn, bmn in shapes:
        A = torch.randn((K, M) if amn else (M, K), device=dev, dtype=torch.bfloat16)
        B = torch.randn((K, N) if bmn else (N, K), device=dev, dtype=torch.bfloat16)
        out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
        ours = timeit(lambda: ops.gemm(A, B, a_mn_major=amn, b_mn_major=bmn, out=out), flush=flush)
        At = A.t() if amn else A
        Bt = B if bmn else B.t()
        ref = timeit(lambda: torch.matmul(At, Bt, out=out), flush=flush)
        fl = 2.0 * M * N * K
        rows.append({"shape": name, "M": M, "N": N, "K": K, "ours_ms": round(ours, 4), "cublas_ms": round(ref, 4),
                     "ours_tflops": round(fl / ours / 1e9, 1), "cublas_tflops": round(fl / ref / 1e9, 1),
                     "ours_frac_of_measured_peak": round(fl / ours / 1e9 / peak, 3)})  # fmt: skip
        print(rows[-1], flush=True)
    out_dir = ROOT / "gpurun_out"
    out_dir.mkdir(exist_ok=True)
    (out_dir / "gemm_bench.json").write_text(json.dumps({"rows": rows, "clocks": sampler.finish(), "peak_used_tflops": peak,
                                                         "timing": "CUDA events, median of 10, 256 MB L2 flush between iterations"}, indent=1))


if __name__ == "__main__":
    main()
