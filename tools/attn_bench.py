"""Time the native flash-attention (fwd, bwd) against SDPA/cuDNN on the Llama shapes. CUDA events, median."""

import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from prime_b200.ops import attention_native as A  # noqa: E402


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
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    from prime_b200.utils.clocks import ClockSampler

    sampler = ClockSampler(0, period_s=0.05)
    sampler.start()
    rows = []
    for name, B, S, H, Hkv, D in [("1B mb16", 16, 1024, 16, 16, 128), ("7B-like", 8, 2048, 32, 32, 128), ("150M", 16, 1024, 16, 16, 64)]:
        W = (H + 2 * Hkv) * D
        qkv = (torch.randn(B, S, W, device=dev) * 0.5).to(torch.bfloat16).requires_grad_(True)
        out = A.flash_attention_qkv(qkv, H, Hkv, True)
        dout = torch.randn_like(out)
        fwd = timeit(lambda: A.flash_attention_qkv(qkv, H, Hkv, True), flush=flush)

        def fb():
            qkv.grad = None
            o = A.flash_attention_qkv(qkv, H, Hkv, True)
            o.backward(dout)

        both = timeit(fb, flush=flush)
        x = qkv.detach().view(B, S, H + 2 * Hkv, D)
        q = x[:, :, :H].transpose(1, 2).contiguous().requires_grad_(True)
        k = x[:, :, H : H + Hkv].transpose(1, 2).contiguous().requires_grad_(True)
        v = x[:, :, H + Hkv :].transpose(1, 2).contiguous().requires_grad_(True)
        sd = lambda: torch.nn.functional.scaled_dot_product_attention(q, k, v, is_causal=True, enable_gqa=H != Hkv)  # noqa: E731
        rfwd = timeit(sd, flush=flush)
        do2 = torch.randn(B, H, S, D, device=dev, dtype=torch.bfloat16)

        def rfb():
            q.grad = k.grad = v.grad = None
            sd().backward(do2)

        rboth = timeit(rfb, flush=flush)
        fl_f = 4.0 * B * H * S * S * D / 2
        rows.append({"shape": name, "B": B, "S": S, "H": H, "D": D, "native_fwd_ms": round(fwd, 4), "sdpa_fwd_ms": round(rfwd, 4),
                     "native_fwd_tflops": round(fl_f / fwd / 1e9, 1), "sdpa_fwd_tflops": round(fl_f / rfwd / 1e9, 1),
                     "native_bwd_ms": round(both - fwd, 4), "sdpa_bwd_ms": round(rboth - rfwd, 4),
                     "native_bwd_tflops_algorithmic": round(2.5 * fl_f / (both - fwd) / 1e9, 1),
                     "sdpa_bwd_tflops": round(2.5 * fl_f / (rboth - rfwd) / 1e9, 1)})  # fmt: skip
        print(rows[-1], flush=True)
    (ROOT / "gpurun_out").mkdir(exist_ok=True)
    (ROOT / "gpurun_out" / "attn_bench.json").write_text(json.dumps({"rows": rows, "clocks": sampler.finish(),
                                                                      "timing": "CUDA events, median, 256 MB L2 flush between iterations; same process for both arms"}, indent=1))


if __name__ == "__main__":
    main()
