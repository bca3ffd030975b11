"""Roofline table for the memory-bound kernels at Llama-1B shapes (one 16×1024-token micro-batch; optimizer ops over all
1.1 G parameters): CUDA-event median, algorithmic bytes, achieved GB/s and fraction of the MEASURED copy bandwidth
(MEASURED_PEAKS.json). ``--once`` runs every op exactly once (what ``ncu --set full`` wraps).

    python tools/op_bench.py > gpurun_out/op_bench.json
"""

import argparse
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from prime_b200 import ops  # noqa: E402
from prime_b200.config import Config  # noqa: E402
from prime_b200.ops import functional as F  # noqa: E402
from prime_b200.trainer import Trainer  # noqa: E402


def timeit(fn, iters, warm, flush):
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
    ap = argparse.ArgumentParser()
    ap.add_argument("--once", action="store_true")
    ap.add_argument("--model", default="1B")
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    peaks = json.loads((ROOT / "MEASURED_PEAKS.json").read_text()) if (ROOT / "MEASURED_PEAKS.json").exists() else {}
    hbm = float(peaks.get("hbm_gbs", 3350.0))  # default: H100 SXM data-sheet HBM3 bandwidth (not a measured rate)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    from prime_b200.utils.clocks import ClockSampler

    sampler = ClockSampler(0)
    sampler.start()
    iters, warm = (1, 0) if a.once else (10, 3)
    B, S, D, FF, V, H, HD = 16, 1024, 2048, 5632, 32000, 16, 128
    T = B * S
    bf = torch.bfloat16
    rows = []

    def add(name, fn, nbytes):
        ms = timeit(fn, iters, warm, flush)
        rows.append({"op": name, "ms": round(ms, 4), "bytes": int(nbytes), "GBps": round(nbytes / ms / 1e6, 1), "frac_of_measured_hbm": round(nbytes / ms / 1e6 / hbm, 3)})

    x = torch.randn(T, D, device=dev, dtype=bf)
    res = torch.randn(T, D, device=dev, dtype=bf)
    w = torch.ones(D, device=dev, dtype=bf, requires_grad=True)
    add("rmsnorm_fwd", lambda: F.rmsnorm(x, w), 2 * T * D * 2)
    add("add_rmsnorm_fwd", lambda: F.add_rmsnorm(x, res, w), 4 * T * D * 2)
    xg = x.clone().requires_grad_(True)
    y = F.rmsnorm(xg, w)
    dy = torch.randn_like(y)
    add("rmsnorm_bwd(+colsum)", lambda: torch.autograd.grad(y, (xg, w), dy, retain_graph=True), 3 * T * D * 2)
    qkv = torch.randn(B, S, 3 * D, device=dev, dtype=bf)
    cos, sin = ops.reference.rope_tables(S, HD, 10000.0, device=dev)
    add("rope_inplace(q,k)", lambda: F.rope_qkv(qkv, cos, sin, H, H), 2 * T * 2 * D * 2)
    gu = torch.randn(T, 2 * FF, device=dev, dtype=bf, requires_grad=True)
    add("swiglu_fwd", lambda: F.swiglu(gu), 3 * T * FF * 2)
    o = F.swiglu(gu)
    do = torch.randn_like(o)
    add("swiglu_bwd", lambda: torch.autograd.grad(o, gu, do, retain_graph=True), 5 * T * FF * 2)
    logits = torch.randn(T, V, device=dev, dtype=bf)
    tg = torch.randint(0, V, (T,), device=dev)
    add("cross_entropy_fwd+bwd(in place)", lambda: F.cross_entropy(logits, tg, grad_scale=1.0, unit_upstream=True), 2 * T * V * 2)
    emb = torch.nn.Parameter(torch.randn(V, D, device=dev, dtype=bf))
    emb.main_grad = torch.zeros(V, D, device=dev, dtype=torch.float32)
    tok = torch.randint(0, V, (B, S), device=dev)
    add("embedding_fwd (native row gather)", lambda: F.embedding(tok, emb), 2 * T * D * 2)
    eo = F.embedding(tok, emb)
    deo = torch.randn_like(eo)
    add("embedding_bwd (sort + segmented sum into fp32 main_grad)", lambda: torch.autograd.grad(eo, emb, deo, retain_graph=True, allow_unused=True), T * D * 2 + 2 * T * D * 4)
    del x, res, xg, y, dy, qkv, gu, o, do, logits, emb, eo, deo
    torch.cuda.empty_cache()

    cfg = Config.model_validate({"name_model": a.model, "data": {"seq_length": S}, "optim": {"batch_size": 16}, "train": {"micro_bs": 16},
                                 "diloco": {"inner_steps": 100}})  # fmt: skip
    tr = Trainer(cfg)
    n = tr.engine.shard_total

    def inner():
        tr.engine.zero_grad()
        tr.engine.set_micro_step(True)
        tr.engine.finish_backward()
        tr.engine.step(1e-4)

    add("inner step: zero_grad + grad_reduce+norm + clip⊕AdamW⊕bf16 cast⊕param push (F=1)", inner, n * (4 + 8 + 30))
    add("outer step: pseudograd⊕int8 quant → dequant⊕Nesterov⊕master reset⊕bf16 push (W=1)", tr.outer.step, n * (9 + 23))
    out = {"shapes": {"tokens": T, "dim": D, "ffn": FF, "vocab": V, "params": n}, "hbm_gbs_measured": hbm, "mode": "once" if a.once else "median of 10, L2 flushed", "rows": rows,
           "launches": ops.launch_count(), "clocks": sampler.finish()}  # fmt: skip
    print(json.dumps(out, indent=1))
    tr.close()


if __name__ == "__main__":
    main()
