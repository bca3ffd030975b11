"""Where the device time of one training step goes: the 1-GPU headline configuration of ``bench.py`` (Llama-1B, 16 × 1024 tokens
per micro-batch, 4 micro-batches per step) through ``Trainer``, profiled with ``torch.profiler`` (CUDA activities only) over a
few inner steps after warm-up.

    python tools/step_profile.py --steps 2 --out profiles/step_profile.json

Writes one JSON file: device time per kernel class (every GEMM instantiation on its own, the attention forward / dK-dV / dQ /
delta kernels, the elementwise kernels, cross-entropy, the optimizer and gradient kernels, anything else by name), each class's
share of the total kernel time, and for every GEMM class the FLOPs it ran — counted from the model's weight shapes, not measured —
over its device time. Run it on its own: tracing slows the host, so the step times it reports are not the benchmark's.
"""

from __future__ import annotations

import argparse
import json
import re
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

MODEL, SEQ, MICRO_BS, ACCUM, H = "1B", 1024, 16, 4, 100  # bench.py's 1-GPU headline configuration

# (substring of the kernel name, class); first match wins
CLASSES = [
    ("flash_fwd_kernel", "attention fwd"),
    ("bwd_dkdv_kernel", "attention dK/dV"),
    ("bwd_dq_kernel", "attention dQ"),
    ("bwd_delta_kernel", "attention delta"),
    ("doc_bounds_kernel", "attention doc bounds"),
    ("cross_entropy", "cross-entropy"),
    ("ce_count_kernel", "cross-entropy"),
    ("ce_finalize_kernel", "cross-entropy"),
    ("rmsnorm", "elementwise: rmsnorm"),
    ("colsum_partials", "elementwise: rmsnorm"),
    ("rope_inplace", "elementwise: rope"),
    ("swiglu", "elementwise: swiglu"),
    ("embedding", "embedding"),
    ("adamw", "optimizer"),
    ("grad_reduce", "gradient reduce / clip"),
    ("norm_publish", "gradient reduce / clip"),
    ("cast_push", "optimizer"),
    ("outer_nesterov", "outer step"),
    ("pseudograd", "outer step"),
]

# gemm_bf16_kernel<A_MN, B_MN, EPI, IO, ...>: the product each (layouts, epilogue) triple runs in this model
GEMM_ROLES = {
    (0, 0, 1): "forward QKV + RoPE",
    (0, 0, 2): "forward W13 + SwiGLU",
    (0, 0, 0): "forward O, W2, logits",
    (0, 1, 3): "dgrad W2 + SwiGLU backward",
    (0, 1, 0): "dgrad QKV, O, W13, logits",
    (1, 1, 0): "wgrad (fp32 += main_grad)",
}


def gemm_flops_per_microbatch(model, tokens: int) -> dict:
    """FLOPs of every GEMM of one micro-batch (forward, dgrad, wgrad), keyed by (A_MN, B_MN, EPI), from the weight shapes."""
    f = {k: 0.0 for k in GEMM_ROLES}
    for name, p in model.named_parameters():
        if p.dim() != 2 or "tok_embeddings" in name or "embed" in name:
            continue
        rows, cols = p.shape  # y = x·Wᵀ: N = rows, K = cols
        fl = 2.0 * tokens * rows * cols
        leaf = name.rsplit(".", 1)[-1]
        if leaf == "wqkv":
            f[(0, 0, 1)] += fl
            f[(0, 1, 0)] += fl
        elif leaf == "w13":
            f[(0, 0, 2)] += fl
            f[(0, 1, 0)] += fl
        elif leaf == "w2":
            f[(0, 0, 0)] += fl
            f[(0, 1, 3)] += fl
        else:  # wo, output
            f[(0, 0, 0)] += fl
            f[(0, 1, 0)] += fl
        f[(1, 1, 0)] += fl
    return f


def classify(name: str) -> str:
    m = re.search(r"gemm_bf16_kernel<([^>]*)>", name)
    if m:
        return "gemm<" + m.group(1).replace(" ", "") + ">"
    for key, cls in CLASSES:
        if key in name:
            return cls
    if "gemm_mxfp8" in name or "quantize_mxfp8" in name:
        return "mxfp8"
    return "other: " + name[:80]


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2, help="inner steps profiled (each is ACCUM micro-batches + optimizer)")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=str(ROOT / "profiles" / "step_profile.json"))
    args = ap.parse_args()

    from torch.profiler import ProfilerActivity, profile

    from prime_b200.config import Config
    from prime_b200.trainer import Trainer

    tree = {
        "name_model": MODEL,
        "type_model": "llama2",
        "data": {"seq_length": SEQ, "fake": True},
        "optim": {"batch_size": MICRO_BS * ACCUM, "warmup_steps": 10, "total_steps": 100000, "optim": {"lr": 4e-4}},
        "train": {"micro_bs": MICRO_BS, "fused_comm": True, "attn_impl": "auto", "cuda_graphs": False, "fp8": False,
                  "reshard_after_forward": None},
        "mesh": {"num_workers": 1, "fsdp_size": 1},
        "diloco": {"inner_steps": H, "compression": "int8", "outer_lr": 0.7},
    }  # fmt: skip
    trainer = Trainer(Config.model_validate(tree))
    for _ in range(args.warmup):
        trainer.inner_step()
    torch.cuda.synchronize()

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            trainer.inner_step()
        torch.cuda.synchronize()

    by_class: dict[str, dict] = {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        us = ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
        if "memcpy" in ev.name.lower() or "memset" in ev.name.lower():
            cls = "memcpy / memset"
        else:
            cls = classify(ev.name)
        row = by_class.setdefault(cls, {"us": 0.0, "launches": 0})
        row["us"] += us
        row["launches"] += 1
    total = sum(r["us"] for r in by_class.values())
    micro = args.steps * trainer.accum
    tokens = MICRO_BS * SEQ
    flops = gemm_flops_per_microbatch(trainer.model, tokens)
    gemm_us = 0.0
    gemm_groups: dict[tuple, float] = {}
    for cls, r in by_class.items():
        r["share"] = round(r["us"] / total, 4)
        r["ms_per_step"] = round(r["us"] / 1e3 / args.steps, 3)
        if cls.startswith("gemm<"):
            gemm_us += r["us"]
            key = tuple(int(x) for x in cls[5:-1].split(",")[:3])
            gemm_groups[key] = gemm_groups.get(key, 0.0) + r["us"]
    gemm = []
    for key, us in sorted(gemm_groups.items(), key=lambda kv: -kv[1]):
        fl = flops.get(key, 0.0) * micro
        gemm.append({"A_MN,B_MN,EPI": list(key), "role": GEMM_ROLES.get(key, "?"), "ms_per_step": round(us / 1e3 / args.steps, 3),
                     "tflop_per_step": round(fl / args.steps / 1e12, 2), "tflops": round(fl / (us * 1e-6) / 1e12, 1) if us else None})  # fmt: skip
    out = {
        "device": torch.cuda.get_device_name(),
        "config": f"Llama-{MODEL}, {MICRO_BS} x {SEQ} tokens per micro-batch, {ACCUM} micro-batches per step",
        "steps_profiled": args.steps,
        "kernel_ms_per_step": round(total / 1e3 / args.steps, 3),
        "gemm_share": round(gemm_us / total, 4),
        "gemm_tflops": round(sum(flops.values()) * micro / (gemm_us * 1e-6) / 1e12, 1) if gemm_us else None,
        "gemm_by_epilogue": gemm,
        "classes": dict(sorted(by_class.items(), key=lambda kv: -kv[1]["us"])),
        "timing": "torch.profiler CUDA activities, summed kernel device time over the profiled steps; FLOPs from the weight shapes",
    }
    Path(args.out).parent.mkdir(parents=True, exist_ok=True)
    Path(args.out).write_text(json.dumps(out, indent=1))
    print(json.dumps({k: out[k] for k in ("device", "kernel_ms_per_step", "gemm_share", "gemm_tflops")}))
    for g in gemm:
        print(g)
    for cls, r in list(out["classes"].items())[:20]:
        print(f"{r['ms_per_step']:9.3f} ms/step  {100 * r['share']:5.1f} %  {cls}")
    trainer.close()


if __name__ == "__main__":
    main()
