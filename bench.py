#!/usr/bin/env python
"""Headline benchmark (BASELINE.json): tokens/sec, Llama-1B DiLoCo H=100 on 1/2/4/8 H100; outer all-reduce GB/s.

    python bench.py --gpus 1 --steps 10 --warmup 3
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 \
        --master-port 29501 bench.py --gpus 8 --steps 10 --warmup 3

Mesh: N=1 → 1 worker × 1 GPU;  N>=2 → (N/2) DiLoCo workers × 2-GPU FSDP (config 2 of BASELINE.json).
Weak scaling: every GPU processes the same number of tokens per step for every N.
Other BASELINE configs through the same harness:  ``--model 7B --fsdp 8 --H 0`` (config 4, FSDP only, no outer step; 7B runs
micro-batch 1 × seq 4096 so that it fits 80 GB), ``--reshard 0|1`` picks replicated parameters vs ZeRO-3. Config 3 (7B DiLoCo,
2 workers × 4-GPU FSDP) does not fit an 80 GB H100: with 4-way sharding the replicated fp32 main_grad, the 1/4 optimizer shards and
the DiLoCo θ₀ + momentum alone take 76 GB per GPU before any activation (``python -m prime_b200.utils.memory_plan``).

A "step" is one full inner optimizer step (ACCUM micro-batches fwd+bwd, gradient reduce-scatter, clip, AdamW, parameter
all-gather).  The outer DiLoCo step (int8 pseudo-gradient all-reduce ⊕ Nesterov) runs every H inner steps *and* is forced at
the last step of each timed region so its cost is always inside the measurement (pessimistic when K < H).

Timed regions of K steps each, all through the public API ``Trainer.inner_step()`` and all including the per-micro-batch pinned
host→device input copies:
  * device-timed (CUDA events, max over ranks)                          → ``value``
  * end-to-end: same, plus a device→host read of the loss every step    → ``e2e``
Then, in the same invocation on the same box, the stock-PyTorch arm B0 (``baseline/torch_b0.py``: FSDP2 + NCCL + cuBLAS +
SDPA + fused AdamW, same config, same protocol) → ``b0`` and the ratio ``vs_b0``.  ``--impl torch_b0`` runs only that arm;
``--impl reference`` reports why the mounted reference cannot run the metric.

``--dump-outputs DIR`` writes, after the timed regions, what the last timed step computed for its caller: the step's loss and
gradient norm, and a fixed seeded sample of every parameter after the update, as ``DIR/<name>.npy`` (float32 / float64, < 64 MB).
The synthetic inputs and the initial weights are seeded, so two builds run with the same arguments can be compared output by output.
It needs replicated parameters (refused under ZeRO-3, where the model's parameters are views of one shared gather scratch).
"""

from __future__ import annotations

import argparse
import json
import os
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))

MODEL = "1B"
SEQ = 1024
MICRO_BS = 16
ACCUM = 4
H = 100


def reference_arm() -> None:
    """The mounted reference is the Prime CLI/SDK: there is no trainer in it to time (see DESIGN.md)."""
    ref = ROOT / "baseline" / "_ref"
    why = (
        "reference (PrimeIntellect-ai/prime @ d892ed8) is a pure-Python HTTP CLI/SDK with no model, trainer, "
        "GPU code or tokens/s benchmark (0 files import torch); nothing in it can run this metric"
    )
    if not ref.exists():
        why = "baseline/_ref not installed; and " + why
    print(json.dumps({"impl": "reference", "unavailable": why}))


from prime_b200.utils.clocks import ClockSampler, NvlinkCounters  # noqa: E402

DUMP_SAMPLE = 32768  # elements per parameter tensor written by --dump-outputs (seeded positions; whole tensor if smaller)


def dump_outputs(out_dir: Path, result, model) -> None:
    import numpy as np
    import torch

    out_dir.mkdir(parents=True, exist_ok=True)
    np.save(out_dir / "loss.npy", np.array([float(result.loss.item())], dtype=np.float64))
    if result.grad_norm is not None:
        np.save(out_dir / "grad_norm.npy", np.array([float(torch.as_tensor(result.grad_norm).item())], dtype=np.float64))
    for i, (name, p) in enumerate(model.named_parameters()):
        flat = p.detach().reshape(-1)
        if flat.numel() > DUMP_SAMPLE:
            gen = torch.Generator().manual_seed(i)
            idx = torch.randint(0, flat.numel(), (DUMP_SAMPLE,), generator=gen).to(flat.device)
            flat = flat[idx]
        np.save(out_dir / f"param.{name}.npy", flat.float().cpu().numpy())


MODEL_DESC = {"1B": "Llama-1B (dim 2048, 18 layers, 16 heads, vocab 32000)", "7B": "Llama-7B (dim 4096, 32 layers, 32 heads, vocab 32000)",
              "150M": "Llama-150M (dim 1024, 12 layers, 16 heads, vocab 32000)"}  # fmt: skip


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference", "torch_b0"])
    ap.add_argument("--model", default=MODEL)
    ap.add_argument("--micro-bs", type=int, default=None)
    ap.add_argument("--accum", type=int, default=None)
    ap.add_argument("--seq", type=int, default=None)
    ap.add_argument("--workers", type=int, default=0, help="DiLoCo workers (default: N/2 for N >= 2)")
    ap.add_argument("--fsdp", type=int, default=0, help="FSDP group size (default: 2 for N >= 2)")
    ap.add_argument("--H", type=int, default=H, help="inner steps per outer step; 0 = FSDP only (no [diloco])")
    ap.add_argument("--compression", default="int8", choices=["int8", "no"])
    ap.add_argument("--reshard", default="auto", choices=["auto", "0", "1"], help="ZeRO-3 parameter sharding (auto: on for >= 5 B params)")
    ap.add_argument("--no-fused-comm", action="store_true", help="engine with NCCL collectives instead of the fused P2P kernels")
    ap.add_argument("--attn", default="auto")
    ap.add_argument("--fp8", action="store_true", help="NON-headline: MXFP8 forward/dgrad GEMMs (reported with dtype 'mxfp8+bf16')")
    ap.add_argument("--graphs", type=int, default=0, help="capture each micro-step (fwd+bwd) in a CUDA graph")
    ap.add_argument("--no-b0", action="store_true", help="skip the stock-PyTorch comparison arm")
    ap.add_argument("--b0-compile", action="store_true", help="B0 with torch.compile on every block")
    ap.add_argument("--trace", action="store_true", help="per-rank device timeline of the step phases (stderr + JSON key step_trace)")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR", help="write the last timed step's outputs as DIR/<name>.npy (rank 0)")
    args = ap.parse_args()

    if args.impl == "reference":
        reference_arm()
        return

    import torch
    import torch.distributed as dist

    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world != args.gpus and args.gpus > 1:
        raise SystemExit(f"--gpus {args.gpus} needs torchrun with {args.gpus} ranks (WORLD_SIZE={world})")
    warmup = max(3, args.warmup)
    K = max(1, args.steps)
    seq = args.seq or (4096 if args.model == "7B" else SEQ)
    micro_bs = args.micro_bs or (1 if args.model == "7B" else MICRO_BS)  # 7B: micro-batch 4 × 4096 needs ≈ 119 GB per GPU at F = 8
    accum = args.accum or ACCUM

    fsdp = args.fsdp or (1 if world == 1 else 2)
    workers = args.workers or world // fsdp
    if workers * fsdp != world:
        raise SystemExit(f"mesh {workers}x{fsdp} does not match {world} ranks")
    use_diloco = args.H > 0

    def b0_arm() -> dict:
        from baseline.torch_b0 import B0Config, run_bench

        cfg = B0Config(model=args.model, seq=seq, micro_bs=micro_bs, accum=accum, workers=workers, fsdp=fsdp, inner_steps=args.H or 10**9,
                       compression=args.compression, compile=args.b0_compile, diloco=use_diloco)  # fmt: skip
        return run_bench(cfg, K, warmup)

    if args.impl == "torch_b0":
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
        sampler = ClockSampler(torch.cuda.current_device())
        if int(os.environ.get("RANK", 0)) == 0:
            sampler.start()
        r = b0_arm()
        if int(os.environ.get("RANK", 0)) == 0:
            r.update(metric="tokens/sec Llama-1B DiLoCo H=100; outer all-reduce GB/s", n_gpus=world, steps=K, warmup=warmup,
                     higher_is_better=True, scaling="weak", vs_baseline=None, dtype="bf16", data="synthetic tokens, random-init weights",
                     clocks=sampler.finish())  # fmt: skip
            r.pop("mfu_flops_per_step", None)
            print(json.dumps(r), flush=True)
        if dist.is_initialized():
            dist.barrier()
            dist.destroy_process_group()
        return

    from prime_b200 import ops
    from prime_b200.config import Config
    from prime_b200.trainer import Trainer

    tree = {
        "name_model": args.model,
        "type_model": "llama2",
        "data": {"seq_length": seq, "fake": True},
        # a randomly initialised 7B model diverges within ten steps of a 10-step ramp to 4e-4 (seen: NaN at step 8 on 4 GPUs); the
        # throughput does not depend on the learning rate, so the large models ramp over 1000 steps like their configs/ files
        "optim": {"batch_size": micro_bs * accum * fsdp, "warmup_steps": 10 if args.model in ("150M", "1B") else 1000, "total_steps": 100000,
                  "optim": {"lr": 4e-4 if args.model in ("150M", "1B") else 3e-4}},
        "train": {"micro_bs": micro_bs, "fused_comm": not args.no_fused_comm, "attn_impl": args.attn, "cuda_graphs": bool(args.graphs),
                  "fp8": args.fp8, "reshard_after_forward": None if args.reshard == "auto" else bool(int(args.reshard))},
        "mesh": {"num_workers": workers, "fsdp_size": fsdp},
    }  # fmt: skip
    if use_diloco:
        tree["diloco"] = {"inner_steps": args.H, "compression": args.compression, "outer_lr": 0.7}
    cfg = Config.model_validate(tree)
    trainer = Trainer(cfg)
    if args.dump_outputs and trainer.engine.shard_params:
        # under ZeRO-3 every model parameter is a view into one shared gather scratch (the embedding a zero placeholder): the
        # parameters a dump would read are not the trained weights
        raise SystemExit("--dump-outputs needs replicated parameters: add --reshard 0 (ZeRO-3 keeps only shards of the weights)")
    dev = trainer.device
    rank = trainer.mesh.world.rank
    if args.trace and trainer.engine.backend == "fused":
        from prime_b200.utils.steptrace import StepTrace

        trainer.engine.trace = None  # armed after the warm-up

    def sync_all():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    losses: list[float] = []
    last_step: dict = {}

    def run_region(n_steps: int, read_loss: bool) -> tuple[float, float, int]:
        """Returns (device ms, host s, launches) for n_steps inner steps incl. >= 1 outer step."""
        sync_all()
        ops.reset_launch_count()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record()
        did_outer = False
        last = None
        for i in range(n_steps):
            r = trainer.inner_step()
            last_step["result"] = r
            did_outer |= r.did_outer
            if i == n_steps - 1 and not did_outer and trainer.outer is not None:
                trainer.outer.step()
            if read_loss:
                last = float(r.loss.item())  # device→host read of the step result, every step
                losses.append(round(last, 4))
        e1.record()
        sync_all()
        host = time.perf_counter() - t0
        ms = torch.tensor([e0.elapsed_time(e1)], device=dev, dtype=torch.float64)
        hs = torch.tensor([host], device=dev, dtype=torch.float64)
        if world > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
            dist.all_reduce(hs, op=dist.ReduceOp.MAX)
        if read_loss and last is not None and not (last == last):
            raise RuntimeError("loss is NaN")
        return float(ms.item()), float(hs.item()), ops.launch_count()

    for _ in range(warmup):
        trainer.inner_step()
    if trainer.outer is not None:
        trainer.outer.step()  # warm the outer path too
        trainer.outer.reset_timing()
    sync_all()
    trainer.check_health()
    if args.trace and trainer.engine.backend == "fused":
        trainer.engine.trace = StepTrace(dev, max_steps=K)

    sampler = ClockSampler(torch.cuda.current_device())
    nvl = nvl0 = nvl1 = None
    if rank == 0:
        sampler.start()
        try:  # raw NVLink byte counters around the device-timed region (evidence for the multi-GPU lines; never fatal)
            nvl = NvlinkCounters(torch.cuda.current_device())
            nvl0 = nvl.read()
        except Exception:  # noqa: BLE001
            nvl = None
    dev_ms, _, launches = run_region(K, read_loss=False)
    if nvl is not None:
        try:
            nvl1 = nvl.read()
        except Exception:  # noqa: BLE001
            nvl1 = None
    trace = trainer.engine.trace.summary() if trainer.engine.trace is not None else None
    trainer.engine.trace = None
    e2e_ms, e2e_host_s, _ = run_region(K, read_loss=True)
    if args.dump_outputs and rank == 0:
        dump_outputs(Path(args.dump_outputs), last_step["result"], trainer.model)
    clocks = sampler.finish() if rank == 0 else {}
    trainer.check_health()
    memory = None
    try:  # the start-up memory plan next to what torch's allocator actually peaked at (before the B0 arm allocates anything); never fatal
        plan = getattr(trainer, "memory_plan", None)
        if plan is not None:
            gb = 1e9
            memory = {"planned_total_gb": round(plan.total_bytes / gb, 2), "planned_state_gb": round(plan.state_bytes / gb, 2),
                      "planned_heap_gb": round(plan.heap_bytes / gb, 2),
                      "planned_torch_gb": round(sum(r.nbytes for r in plan.rows if r.where == "torch") / gb, 2),
                      "torch_peak_gb": round(torch.cuda.max_memory_allocated() / gb, 2),
                      "heap_gb": round(getattr(trainer.heap, "nbytes", 0) / gb, 2) if trainer.heap is not None else 0.0,
                      "capacity_gb": round(plan.capacity / gb, 1)}  # fmt: skip
    except Exception:  # noqa: BLE001
        memory = None

    tokens = trainer.tokens_per_step * K
    value = tokens / (dev_ms / 1e3)
    e2e_value = tokens / max(e2e_host_s, e2e_ms / 1e3)
    h2d = trainer.loader.h2d_bytes_per_batch * trainer.accum
    outer_info = None
    if trainer.outer is not None:
        osec = trainer.outer.mean_device_seconds()
        t = torch.tensor([osec], device=dev, dtype=torch.float64)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        osec = float(t.item())
        skew = torch.tensor([trainer.outer.mean_skew_seconds()], device=dev, dtype=torch.float64)
        if world > 1:
            dist.all_reduce(skew, op=dist.ReduceOp.MAX)
        wire = trainer.outer.last_bytes_on_wire
        shard_elems = trainer.engine.shard_total
        outer_info = {
            "ms": round(osec * 1e3, 4),
            # device time the slowest-waiting rank spent at the alignment barrier IN FRONT of the timed window (workers drift apart
            # over the inner steps; that wait is arrival skew, not exchange time — it is inside `value`, outside `ms`)
            "arrival_skew_ms": round(float(skew.item()) * 1e3, 4),
            "bytes_on_wire_per_rank": wire,
            # bytes a rank must RECEIVE from the other workers (int8 payload + one fp32 scale per 1024) over the device time of the
            # whole fused outer step (quantise + barrier + peer loads ⊕ dequant-sum ⊕ Nesterov ⊕ bf16 write-back + barrier)
            "GBps": round(wire / osec / 1e9, 2) if wire and osec > 0 else None,
            # all local HBM traffic of the step (θ₀/θ/momentum/master read+write, payloads) over the same time, for W = 1 runs
            "local_GBps": round(shard_elems * (8 + 1 + 16 + 12 + 2 * fsdp) / osec / 1e9, 1) if osec > 0 else None,
            "timing": "CUDA events on the launching stream, mean over the outer steps of both timed regions, max over ranks",
        }
    if args.trace and trace is not None:
        rows = [None] * world
        if world > 1:
            dist.all_gather_object(rows, trace)
        else:
            rows = [trace]
        trace = rows
        if rank == 0:
            for i, row in enumerate(rows):
                print(f"[trace] rank {i}: {row}", file=sys.stderr)
    shard_mode = "zero3 (bf16 params sharded 1/F, gathered inside the GEMMs)" if trainer.engine.shard_params else "replicated bf16 params (ZeRO-1)"
    flops = trainer.flops_per_step() * K / world
    trainer.close()
    del trainer
    torch.cuda.empty_cache()

    b0 = None
    if not args.no_b0 and not args.fp8:
        try:
            b0 = b0_arm()
        except Exception as e:  # noqa: BLE001 — the comparison arm must never take the headline number down with it
            b0 = {"impl": "torch_b0", "error": f"{type(e).__name__}: {str(e)[:300]}"}

    if rank == 0:
        line = {
            "metric": "tokens/sec Llama-1B DiLoCo H=100; outer all-reduce GB/s",
            "value": round(value, 1),
            "unit": "tokens/s",
            "n_gpus": world,
            "steps": K,
            "warmup": warmup,
            "ms_per_step": round(dev_ms / K, 3),
            "higher_is_better": True,
            "scaling": "weak",
            "vs_baseline": None,
            "dtype": "bf16" if not args.fp8 else "mxfp8+bf16 (non-headline)",
            "data": "synthetic tokens, random-init weights",
            "impl": "ours",
            "config": {
                "model": MODEL_DESC.get(args.model, args.model),
                "global_batch": micro_bs * accum * world,
                "seq_len": seq,
                "micro_bs": micro_bs,
                "grad_accum": accum,
                "parallelism": f"diloco{workers}xfsdp{fsdp}",
                "diloco_H": args.H if use_diloco else None,
                "outer": f"{args.compression} pseudo-gradient exchange + Nesterov, forced >=1 per timed region" if use_diloco else None,
                "comm": "fused P2P kernels" if not args.no_fused_comm else "NCCL collectives",
                "params": shard_mode,
                "cuda_graphs": bool(args.graphs),
                "l2": "working set (params+activations, >20 GB/step) far larger than the 50 MB L2; no flush needed",
            },
            "clocks": clocks,
            "e2e": {
                "value": round(e2e_value, 1),
                "unit": "tokens/s",
                "h2d_bytes_per_step": h2d,
                "d2h_bytes_per_step": 4,
                "ms_per_step": round(max(e2e_host_s * 1e3, e2e_ms) / K, 3),
            },
            "gpu_launches": launches,
            "nvlink": NvlinkCounters.delta(nvl0, nvl1, K),
            "memory": memory,
            "losses_e2e_region": losses,
            "outer_allreduce": outer_info,
            "outer_allreduce_GBps": outer_info["GBps"] if outer_info else None,
            "mfu_of_measured_sustained_peak": None,
        }
        try:
            peaks = json.loads((ROOT / "MEASURED_PEAKS.json").read_text())
            line["mfu_of_measured_sustained_peak"] = round(flops / (dev_ms / 1e3) / (peaks["bf16_tflops_sustained"] * 1e12), 4)
        except Exception:
            pass
        if trace is not None:
            line["step_trace"] = trace
        if b0 is not None:
            b0.pop("mfu_flops_per_step", None)
            line["b0"] = b0
            if "value" in b0:
                line["vs_b0"] = {"value": round(value / b0["value"], 4), "e2e": round(e2e_value / b0["e2e"]["value"], 4),
                                 "note": "this engine ÷ stock PyTorch (FSDP2+NCCL+cuBLAS+SDPA), same config, same box, same invocation"}  # fmt: skip
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
