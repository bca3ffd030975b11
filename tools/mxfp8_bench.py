"""MXFP8 GEMM (e4m3 MMAs, per-32 block scales applied in registers) vs the bf16 wgmma GEMM on the Llama-1B projection shapes.

Device-timed with CUDA events, median of 20, L2 flushed between iterations. `python tools/mxfp8_bench.py > out.json`"""

import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from prime_b200 import ops  # noqa: E402


def timeit(fn, flush, iters=20, warm=3):
    for _ in range(warm):
        fn()
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
    shapes = [("qkv", T, 6144, 2048), ("wo", T, 2048, 2048), ("w13", T, 11264, 2048), ("w2", T, 2048, 5632), ("dgrad_w13", T, 2048, 11264)]
    rows = []
    for name, M, N, K in shapes:
        a = (torch.randn(M, K, device=dev) * 0.5).to(torch.bfloat16)
        b = (torch.randn(N, K, device=dev) * 0.05).to(torch.bfloat16)
        out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
        aq, asf = ops.quantize_mxfp8(a)
        bq, bsf = ops.quantize_mxfp8(b)
        t_fp8 = timeit(lambda: ops.gemm_mxfp8(aq, asf, bq, bsf, out=out), flush)
        t_bf16 = timeit(lambda: ops.gemm(a, b, out=out), flush)
        t_qa = timeit(lambda: ops.quantize_mxfp8(a), flush)
        t_qb = timeit(lambda: ops.quantize_mxfp8(b), flush)
        t_qbt = timeit(lambda: ops.quantize_mxfp8(b, transpose=True), flush) if N % 128 == 0 else None
        fl = 2.0 * M * N * K
        rows.append({"shape": name, "M": M, "N": N, "K": K, "mxfp8_ms": round(t_fp8, 4), "mxfp8_tflops": round(fl / t_fp8 / 1e9, 1),
                     "bf16_ms": round(t_bf16, 4), "bf16_tflops": round(fl / t_bf16 / 1e9, 1), "speedup": round(t_bf16 / t_fp8, 3),
                     "quantize_act_ms": round(t_qa, 4), "quantize_act_GBps": round(M * K * 3 / t_qa / 1e6, 1),
                     "quantize_w_ms": round(t_qb, 4), "quantize_w_transposed_ms": None if t_qbt is None else round(t_qbt, 4)})  # fmt: skip
    # sustained: 1.5 s of back-to-back GEMMs with the clocks sampled — under the ~1 kW power cap the SM clock, not the kernel,
    # sets the ceiling; efficiency is reported against the clock actually held
    from prime_b200.utils.clocks import ClockSampler

    M, N, K = 16384, 11264, 2048
    a = (torch.randn(M, K, device=dev) * 0.5).to(torch.bfloat16)
    b = (torch.randn(N, K, device=dev) * 0.05).to(torch.bfloat16)
    out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    aq, asf = ops.quantize_mxfp8(a)
    bq, bsf = ops.quantize_mxfp8(b)
    sustained = {}
    # library reference point: cuBLASLt fp8 through torch._scaled_mm (tensor-wise scales), same shape
    a8 = a.to(torch.float8_e4m3fn)
    b8t = b.to(torch.float8_e4m3fn).t()  # column-major [K, N]
    one = torch.ones((), device=dev, dtype=torch.float32)

    def cublaslt_fp8():
        return torch._scaled_mm(a8, b8t, scale_a=one, scale_b=one, out_dtype=torch.bfloat16)

    # dense tensor-core FLOP per clock per SM on H100: bf16 4096, fp8 8192 (data sheet: 989 / 1979 TFLOP/s at 1830 MHz on 132 SMs)
    cands = [("bf16", lambda: ops.gemm(a, b, out=out), 4096), ("mxfp8", lambda: ops.gemm_mxfp8(aq, asf, bq, bsf, out=out), 8192)]
    try:
        cublaslt_fp8()
        cands.append(("cublaslt_fp8_tensorwise", cublaslt_fp8, 8192))
    except Exception as e:  # noqa: BLE001
        sustained_err = f"torch._scaled_mm unavailable: {type(e).__name__}: {str(e)[:120]}"
    else:
        sustained_err = None
    n_sm = torch.cuda.get_device_properties(dev).multi_processor_count
    for name, fn, per_clk in cands:
        for _ in range(20):
            fn()
        torch.cuda.synchronize()
        cs = ClockSampler(0, period_s=0.05)
        cs.start()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        iters = 4000 if name == "bf16" else 5000
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        clocks = cs.finish()
        ms = e0.elapsed_time(e1) / iters
        tf = 2.0 * M * N * K / ms / 1e9
        mhz = clocks.get("sm_mhz") or 0
        sustained[name] = {"ms": round(ms, 4), "tflops": round(tf, 1), "clocks": clocks,
                           "fraction_of_tensor_peak_at_held_clock": round(tf * 1e12 / (n_sm * per_clk * mhz * 1e6), 3) if mhz else None}
    if sustained_err:
        sustained["cublaslt_fp8_tensorwise"] = {"error": sustained_err}
    print(json.dumps({"rows": rows, "sustained_w13_shape": sustained, "note": "fp8 dense peak 4.5 PFLOP/s nominal; bf16 2.25"}, indent=1))


if __name__ == "__main__":
    main()
