"""Block-scaled fp8 (MXFP8) linear layer: quantise → block-scaled fp8 GEMM, against the bf16 GEMM. Runs on one H100; on CPU it
falls back to the torch reference of the same format (prime_b200/ops/reference.py), which is also its specification.

    python examples/mxfp8_linear.py
"""

import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from prime_b200 import ops  # noqa: E402
from prime_b200.ops import reference  # noqa: E402


def main() -> None:
    dev = torch.device("cuda", 0) if torch.cuda.is_available() else torch.device("cpu")
    torch.manual_seed(0)
    tokens, d_in, d_out = (16384, 2048, 6144) if dev.type == "cuda" else (256, 256, 384)
    x = torch.randn(tokens, d_in, device=dev, dtype=torch.bfloat16, requires_grad=True)
    w = (torch.randn(d_out, d_in, device=dev) * 0.02).to(torch.bfloat16).requires_grad_(True)

    xq, xsf = ops.quantize_mxfp8(x.detach())  # e4m3 bytes + one UE8M0 scale per 32 elements, already in the tensor-core layout
    print(f"x: {tuple(x.shape)} bf16 → {tuple(xq.shape)} e4m3 + {xsf.numel()} scale bytes; "
          f"round trip rel. error {float((reference.dequantize_mxfp8(xq, xsf) - x.detach().float()).norm() / x.detach().float().norm()):.4f}")

    y8 = ops.linear_mxfp8(x, w)   # forward + input-gradient GEMMs in MXFP8, weight gradient bf16 → fp32
    y16 = ops.linear(x.detach(), w.detach())
    print(f"y rel. difference MXFP8 vs bf16: {float((y8.detach().float() - y16.float()).norm() / y16.float().norm()):.4f}")
    y8.backward(torch.randn_like(y8))
    print(f"grads: dx {tuple(x.grad.shape)}, dw {tuple(w.grad.shape)}")


if __name__ == "__main__":
    main()
