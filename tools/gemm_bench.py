"""Time every GEMM of the Llama-1B training step (16 × 1024 tokens per micro-batch) on the wgmma kernel, with the layouts and
fused epilogues the step uses, under every tile mode of the kernel and under cuBLAS (torch.matmul), the arms alternating in one
process.

    python tools/gemm_bench.py [--rounds 3] [--out profiles/gemm_bench.json]

Forward: QKV + RoPE, O, W13 + SwiGLU, W2, logits. Input gradients (dgrad): every weight, W2 with the SwiGLU-backward epilogue.
Weight gradients (wgrad): fp32 += into a main_grad-shaped buffer. cuBLAS runs the same product with the same operand layouts and
a bf16 output, without the fused epilogue: for the fused and fp32 shapes it is a lower bound on what cuBLAS would cost.
Modes: "auto" is the kernel's own choice (``ops.set_gemm_tile(-1)``), then every forced tile mode the library offers. CUDA
events, median of 10 launches with a 256 MB L2 flush before each, per round; the table reports the median over the rounds.
TFLOP/s are counted from the shapes; "of peak" is against the H100 SXM data-sheet dense BF16 rate, 989 TFLOP/s.
"""

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from prime_b200 import ops  # noqa: E402
from prime_b200.ops import _lib  # noqa: E402

DATASHEET_BF16_TFLOPS = 989.0  # H100 SXM, dense, at up to 700 W (NVIDIA data sheet); not a measured rate

T, DIM, FF, VOCAB, HEADS, HEAD_DIM, SEQ = 16384, 2048, 5632, 32000, 16, 128, 1024


def timeit(fn, flush, iters=10, warm=3):
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


def tile_modes() -> list:
    """(label, mode) of every tile mode: the automatic policy first, then each forced mode the library exposes."""
    lib = _lib.load()
    if not hasattr(lib, "pb_gemm_set_tile"):
        return [("kernel", None)]
    return [("auto", -1)] + [(f"tile{m}", m) for m in ops.GEMM_TILE_MODES]


def cases(dev):
    """(name, kernel call, cuBLAS call, FLOPs, (M, N, K, epilogue kind, fp32 +=)) for every GEMM of one micro-batch's forward,
    dgrad and wgrad."""
    g = torch.Generator(device=dev).manual_seed(0)

    def rnd(*shape, dtype=torch.bfloat16):
        return (torch.randn(*shape, device=dev, generator=g) * 0.1).to(dtype)

    weights = {"qkv": (3 * HEADS * HEAD_DIM, DIM), "o": (DIM, HEADS * HEAD_DIM), "w13": (2 * FF, DIM), "w2": (DIM, FF), "logits": (VOCAB, DIM)}
    W = {k: rnd(*s) for k, s in weights.items()}
    cos, sin = rnd(SEQ, HEAD_DIM // 2, dtype=torch.float32), rnd(SEQ, HEAD_DIM // 2, dtype=torch.float32)
    out = []
    # forward: y = x·Wᵀ
    for name, (n, k) in weights.items():
        x = rnd(T, k)
        y = torch.empty(T, n, device=dev, dtype=torch.bfloat16)
        kw = {}
        if name == "qkv":
            kw["rope"] = (cos, sin, SEQ, 2 * HEADS * HEAD_DIM, HEAD_DIM)
        if name == "w13":
            kw["swiglu_h"] = torch.empty(T, FF, device=dev, dtype=torch.bfloat16)
        label = {"qkv": "qkv+rope", "w13": "w13+swiglu"}.get(name, name)
        epi = {"qkv": 1, "w13": 2}.get(name, 0)
        out.append((f"fwd {label}", lambda x=x, w=W[name], y=y, kw=kw: ops.gemm(x, w, out=y, **kw),
                    lambda x=x, w=W[name], y=y: torch.matmul(x, w.t(), out=y), 2.0 * T * n * k, (T, n, k, epi, False)))  # fmt: skip
    # dgrad: dx = dy·W  (W read MN-major)
    for name, (n, k) in weights.items():
        dy = rnd(T, n)
        if name == "w2":  # dh never exists: d_gate_up from the saved gate_up
            gu = rnd(T, 2 * FF)
            dgu = torch.empty(T, 2 * FF, device=dev, dtype=torch.bfloat16)
            dh = torch.empty(T, FF, device=dev, dtype=torch.bfloat16)
            out.append(("dgrad w2+swiglu_bwd", lambda dy=dy, w=W[name], dgu=dgu, gu=gu: ops.gemm(dy, w, b_mn_major=True, out=dgu, swiglu_bwd_gu=gu),
                        lambda dy=dy, w=W[name], dh=dh: torch.matmul(dy, w, out=dh), 2.0 * T * n * k, (T, k, n, 3, False)))  # fmt: skip
            continue
        dx = torch.empty(T, k, device=dev, dtype=torch.bfloat16)
        out.append((f"dgrad {name}", lambda dy=dy, w=W[name], dx=dx: ops.gemm(dy, w, b_mn_major=True, out=dx),
                    lambda dy=dy, w=W[name], dx=dx: torch.matmul(dy, w, out=dx), 2.0 * T * n * k, (T, k, n, 0, False)))  # fmt: skip
    # wgrad: main_grad[n, k] += dyᵀ·x (both operands MN-major)
    for name, (n, k) in weights.items():
        dy, x = rnd(T, n), rnd(T, k)
        mg = torch.zeros(n, k, device=dev, dtype=torch.float32)
        o16 = torch.empty(n, k, device=dev, dtype=torch.bfloat16)
        out.append((f"wgrad {name}", lambda dy=dy, x=x, mg=mg: ops.gemm(dy, x, a_mn_major=True, b_mn_major=True, out=mg, accumulate=True),
                    lambda dy=dy, x=x, o16=o16: torch.matmul(dy.t(), x, out=o16), 2.0 * T * n * k, (n, k, T, 0, True)))  # fmt: skip
    return out


def card() -> dict:
    info = {"name": torch.cuda.get_device_name()}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()  # fmt: skip
        info["power_limit, max_sm_clock"] = q
    except Exception as e:  # noqa: BLE001 — the table stands without it, but says so
        info["power_limit, max_sm_clock"] = f"unavailable: {type(e).__name__}"
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=str(ROOT / "profiles" / "gemm_bench.json"))
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    from prime_b200.utils.clocks import ClockSampler

    sampler = ClockSampler(0, period_s=0.05)
    sampler.start()
    modes = tile_modes()
    rows = []
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    for name, ours, cublas, fl, shape in cases(dev):
        ts = {label: [] for label, _ in modes}
        ts["cublas"] = []
        for _ in range(args.rounds):
            for label, mode in modes:
                if mode is not None:
                    ops.set_gemm_tile(mode)
                ts[label].append(timeit(ours, flush))
            ts["cublas"].append(timeit(cublas, flush))
        if modes[0][1] is not None:
            ops.set_gemm_tile(-1)
        row = {"shape": name, "MNK": list(shape[:3])}
        if modes[0][1] is not None:
            M, N, K, epi, fp32 = shape
            row["auto_tile"] = ops.gemm_tile_policy(M, N, K, epilogue=epi, c_fp32=fp32, accumulate=fp32, num_sms=sms)
        for label, v in ts.items():
            ms = statistics.median(v)
            row[f"{label}_ms"] = round(ms, 4)
            row[f"{label}_tflops"] = round(fl / ms / 1e9, 1)
        row["best_ours_of_datasheet_peak"] = round(max(row[f"{lb}_tflops"] for lb, _ in modes) / DATASHEET_BF16_TFLOPS, 3)
        rows.append(row)
        print(json.dumps(row), flush=True)
    Path(args.out).parent.mkdir(parents=True, exist_ok=True)
    Path(args.out).write_text(json.dumps({"card": card(), "rows": rows, "clocks": sampler.finish(),
                                          "peak_tflops": DATASHEET_BF16_TFLOPS, "peak_source": "H100 SXM data sheet, dense BF16",
                                          "timing": "CUDA events, median of 10 with a 256 MB L2 flush before each, median over rounds"}, indent=1))  # fmt: skip


if __name__ == "__main__":
    main()
