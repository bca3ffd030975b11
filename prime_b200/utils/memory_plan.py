"""Per-GPU HBM budget of a training configuration, computed BEFORE anything is allocated.

    python -m prime_b200.utils.memory_plan @configs/7B/fsdp_8.toml --world 8
    python -m prime_b200.utils.memory_plan --model 70B --fsdp 8 --micro-bs 1 --seq 4096

Why it exists: an H100 has 80 GB and the engine takes its big buffers once, at start-up, from two places — the symmetric NVLink
heap (``parallel/symm.py``: one ``cudaMalloc`` + IPC mapping per rank, invisible to torch's allocator statistics) and torch's caching
allocator. A configuration that cannot fit used to die inside ``cudaMalloc`` on one rank while its peers waited in the handle
exchange; on a shared box that is a hung job. ``Trainer`` now calls :func:`plan_from_config` first and refuses with the table below.

Two kinds of rows:

* **state** (exact): what ``ShardedEngine._allocate`` / ``DilocoOuter`` allocate, from the same formulas (``parallel/fsdp.py``,
  ``parallel/diloco.py``, ``trainer.py`` heap sizing) — parameters, fp32 ``main_grad``, fp32 master + AdamW moments, reduced
  gradient shard, DiLoCo θ₀ / momentum / int8 payload, ZeRO-3 gather scratch. Bucket padding (< 0.1 %) is covered by a margin.
* **activations** (estimate, conservative): tensors the autograd functions in ``ops/functional.py`` keep for the backward, per
  token and layer ``2·(5·dim + qkv_width + 3·ffn_hidden)`` bytes (residual, normed input, rotated QKV, attention output, second
  residual / normed input, gate‖up, SwiGLU output) + row statistics, plus the logits / loss workspace. Checked against a
  measured run (``bench.py --gpus 1`` on an H100 80GB HBM3, Llama-1B, micro-batch 16 × 1024, DiLoCo: 42.0 GB peak in torch's allocator;
  the torch rows of this plan sum to 42.8 GB for the same configuration).

Only the exact rows can make a configuration an error; the estimate produces a warning. (The reference has no counterpart: its
``prime rl`` / ``prime pods`` commands pick a GPU count from a table in the control plane — reference:
packages/prime/src/prime_cli/commands/rl.py — and never see the model.)
"""

from __future__ import annotations

import argparse
import json
import os
import sys
from dataclasses import dataclass, field

from ..models.llama import ModelArgs, get_model_args
from ..parallel.layout import SHARD_ALIGN, use_zero3

GB = 1e9
H100_HBM_BYTES = int(80 * GB)
CUDA_CONTEXT_BYTES = int(1.5 * GB)  # context + loaded modules + cuBLAS / NCCL workspaces of the comparison paths (measured ≈ 1.1 GB)


def count_params(a: ModelArgs) -> dict[str, int]:
    """Element counts by kind — the same shapes ``models/llama.py`` creates (fused wqkv and w13, untied output head)."""
    qkv_w = (a.n_heads + 2 * a.kv_heads) * a.head_dim
    layer_2d = qkv_w * a.dim + a.dim * a.n_heads * a.head_dim + 2 * a.ffn_hidden * a.dim + a.dim * a.ffn_hidden
    layer_1d = 2 * a.dim
    embed, head = a.vocab_size * a.dim, a.vocab_size * a.dim
    return {
        "embed": embed,
        "head": head,
        "layer_2d": layer_2d,
        "layers_2d": layer_2d * a.n_layers,
        "small_1d": layer_1d * a.n_layers + a.dim,
        "total": embed + head + layer_2d * a.n_layers + layer_1d * a.n_layers + a.dim,
        "qkv_width": qkv_w,
    }


@dataclass
class Row:
    name: str
    nbytes: int
    where: str  # "heap" (symmetric NVLink heap) | "torch" (caching allocator) | "driver"
    exact: bool = True
    note: str = ""


@dataclass
class MemoryPlan:
    rows: list[Row] = field(default_factory=list)
    capacity: int = H100_HBM_BYTES
    describe: str = ""

    def add(self, name: str, nbytes: float, where: str, exact: bool = True, note: str = "") -> None:
        if nbytes > 0:
            self.rows.append(Row(name, int(nbytes), where, exact, note))

    @property
    def state_bytes(self) -> int:
        return sum(r.nbytes for r in self.rows if r.exact)

    @property
    def total_bytes(self) -> int:
        return sum(r.nbytes for r in self.rows)

    @property
    def heap_bytes(self) -> int:
        return sum(r.nbytes for r in self.rows if r.where == "heap")

    @property
    def verdict(self) -> str:
        if self.state_bytes > self.capacity:
            return "does_not_fit"
        return "tight" if self.total_bytes > 0.95 * self.capacity else "fits"

    def largest(self) -> Row:
        return max(self.rows, key=lambda r: r.nbytes)

    def table(self) -> str:
        w = max(len(r.name) for r in self.rows) + 2
        lines = [self.describe, f"{'buffer':{w}s}{'GB':>9s}  {'where':7s} kind"]
        for r in self.rows:
            lines.append(f"{r.name:{w}s}{r.nbytes / GB:9.2f}  {r.where:7s} {'exact' if r.exact else 'estimate'}{'  — ' + r.note if r.note else ''}")
        lines.append(f"{'state (exact rows)':{w}s}{self.state_bytes / GB:9.2f}")
        lines.append(f"{'total':{w}s}{self.total_bytes / GB:9.2f}  of {self.capacity / GB:.0f} GB per GPU → {self.verdict}")
        return "\n".join(x for x in lines if x)

    def to_json(self) -> dict:
        return {"describe": self.describe, "capacity_bytes": self.capacity, "state_bytes": self.state_bytes, "total_bytes": self.total_bytes,
                "heap_bytes": self.heap_bytes, "verdict": self.verdict,
                "rows": [{"name": r.name, "bytes": r.nbytes, "where": r.where, "exact": r.exact} for r in self.rows]}  # fmt: skip


class MemoryPlanError(ValueError):
    """The exact part of the plan alone exceeds the GPU: refusing before the first allocation."""


def plan_memory(a: ModelArgs, *, fsdp_size: int = 1, micro_bs: int = 1, seq_len: int = 1024, shard_params: bool | None = None,
                ac_ckpt: bool | int = False, diloco: bool = False, compression: str = "int8", fused: bool = True, fp8: bool = False,
                capacity: int = H100_HBM_BYTES, name: str = "") -> MemoryPlan:  # fmt: skip
    """The budget of ONE rank. ``shard_params=None`` applies the Trainer's rule (ZeRO-3 from 5 B parameters when F > 1 and the fused
    backend is on)."""
    c = count_params(a)
    N, F = c["total"], max(1, fsdp_size)
    shard_params = use_zero3(shard_params, fused=fused, fsdp_size=F, n_params=N)
    pad = 1.001  # bucket padding to F·1024 elements and 16-byte parameter alignment
    shard = N / F * pad
    where = "heap" if fused else "torch"
    p = MemoryPlan(capacity=capacity)
    p.describe = (f"{name or 'model'}: {N / 1e9:.2f} B parameters (dim {a.dim}, {a.n_layers} layers, ffn {a.ffn_hidden}, vocab {a.vocab_size}) | "
                  f"fsdp {F} | micro_bs {micro_bs} × seq {seq_len} | {'ZeRO-3 (parameters sharded)' if shard_params else 'parameters replicated'}"
                  f"{' | DiLoCo ' + compression if diloco else ''}{' | ac_ckpt ' + str(ac_ckpt) if ac_ckpt else ''}")  # fmt: skip
    # ---- exact: engine state (parallel/fsdp.py:_allocate)
    if shard_params:
        p.add("bf16 parameter shard (rows 1/F of every weight)", 2 * shard, where)
        p.add("bf16 replicated 1-D parameters", 2 * c["small_1d"] * pad, where)
        p.add("bf16 gather scratch (one layer + head, reused by every layer)", 2 * (c["layer_2d"] + c["head"]), "torch")
    else:
        p.add("bf16 parameters (replicated inside the worker)", 2 * N * pad, where)
    p.add("fp32 main_grad (replicated; wgrad GEMMs accumulate into it)", 4 * N * pad, where,
          note="not sharded yet: the 1/F reduce happens after the backward")  # fmt: skip
    p.add("fp32 master weights (1/F)", 4 * shard, "torch")
    p.add("fp32 AdamW exp_avg + exp_avg_sq (1/F)", 8 * shard, "torch")
    if F > 1:
        p.add("fp32 reduced gradient shard (1/F)", 4 * shard, "torch")
    if diloco:
        p.add("fp32 DiLoCo θ₀ + outer momentum (1/F)", 8 * shard, "torch")
        if not fused:
            p.add("outer-step exchange buffers (1/F)", (4 if compression == "no" else 1 + 4 / SHARD_ALIGN) * shard, "torch")
    if fused:
        # trainer.py sizes the heap once, with room for the outer step's payload whether or not [diloco] is configured
        p.add("outer-step exchange reservation (int8 payload + block scales, 1/F)", 2 * shard, "heap")
        if diloco and compression == "no":
            p.add("fp32 master weights in the heap for the fused fp32 outer step (1/F)", 4 * shard, "heap",
                  note="instead of the torch-side master row")  # fmt: skip
            p.rows = [r for r in p.rows if r.name != "fp32 master weights (1/F)"]
        p.add("heap slack (flags, error words, alignment)", (64 << 20) + 4 * (a.n_layers + 4) * F * 1024, "heap")
    p.add("CUDA context, kernel images, library workspaces", CUDA_CONTEXT_BYTES, "driver")
    # ---- estimate: what the backward needs from the forward (ops/functional.py save_for_backward)
    tokens = micro_bs * seq_len
    per_tok_layer = 2 * (5 * a.dim + c["qkv_width"] + 3 * a.ffn_hidden) + 4 * a.n_heads + 8
    if fp8:
        per_tok_layer += (2 * a.dim + a.ffn_hidden) * 1.04  # MXFP8 copies of the GEMM inputs with their E8M0 scales
    L = a.n_layers
    if ac_ckpt:
        every = 1 if ac_ckpt is True else max(1, int(ac_ckpt))
        ckpt_layers = L // every
        kept = (L - ckpt_layers) * per_tok_layer + ckpt_layers * 2 * a.dim + per_tok_layer  # + the one block being recomputed
    else:
        kept = L * per_tok_layer
    p.add("saved activations", tokens * kept, "torch", exact=False, note=f"{per_tok_layer / 1024:.1f} KiB per token and layer")
    p.add("logits / loss workspace (bf16 logits, in-place gradient) + embedding output", tokens * (2 * a.vocab_size + 2 * a.dim + 16), "torch", exact=False)
    p.add("transient workspaces (attention dQ accumulators, dgrad outputs, allocator fragmentation)", tokens * (4 * a.dim + 2 * 2 * a.ffn_hidden) + 0.02 * tokens * kept,
          "torch", exact=False)  # fmt: skip
    return p


def plan_from_config(cfg, world_size: int, *, capacity: int = H100_HBM_BYTES, fused: bool | None = None, fsdp_size: int | None = None,
                     model_overrides: dict | None = None) -> MemoryPlan:  # fmt: skip
    """The plan of a ``prime_b200.config.Config`` on ``world_size`` ranks (mesh derivation as in ``parallel/mesh.py``; ``fsdp_size``
    overrides it when the caller already built the mesh)."""
    a = get_model_args(cfg.name_model, cfg.type_model, **dict(model_overrides or {}))
    F, W = fsdp_size or cfg.mesh.fsdp_size, cfg.mesh.num_workers
    if cfg.mesh.elastic:
        F = F or world_size
    elif not F:
        F = world_size // (W or 1)
    use_fused = cfg.train.fused_comm if fused is None else fused
    return plan_memory(a, fsdp_size=max(1, F), micro_bs=cfg.train.micro_bs, seq_len=cfg.data.seq_length, shard_params=cfg.train.reshard_after_forward,
                       ac_ckpt=cfg.train.ac_ckpt, diloco=cfg.diloco is not None, compression=cfg.diloco.compression if cfg.diloco else "int8",
                       fused=use_fused, fp8=cfg.train.fp8, capacity=capacity, name=f"{cfg.type_model}/{cfg.name_model}")  # fmt: skip


def check(plan: MemoryPlan, log=None) -> None:
    """Raise :class:`MemoryPlanError` when the exact rows alone exceed the GPU (``PB_SKIP_MEMORY_CHECK=1`` turns that into a warning);
    warn through ``log`` when only the estimate pushes the total over."""
    if plan.state_bytes > plan.capacity:
        big = plan.largest()
        msg = (f"this configuration cannot fit a {plan.capacity / GB:.0f} GB GPU: model and optimizer state alone need {plan.state_bytes / GB:.1f} GB "
               f"per rank (largest: {big.name}, {big.nbytes / GB:.1f} GB).\n{plan.table()}\n"
               "Raise mesh.fsdp_size, pick a smaller model, or see DESIGN.md §1.6 item 7 (gradient sharding) for what a 70B-class model still needs.")  # fmt: skip
        if os.environ.get("PB_SKIP_MEMORY_CHECK") == "1":
            if log is not None:
                log.warning("%s", msg)
            return
        raise MemoryPlanError(msg)
    if plan.total_bytes > plan.capacity and log is not None:
        log.warning("memory plan: state %.1f GB + estimated activations exceed %.0f GB per GPU — lower train.micro_bs or set train.ac_ckpt\n%s",
                    plan.state_bytes / GB, plan.capacity / GB, plan.table())  # fmt: skip


def largest_micro_bs(a: ModelArgs, **kw) -> int:
    """Largest power-of-two ``micro_bs`` whose total (estimate included) stays under 92 % of the GPU; 0 when even 1 does not."""
    best, mb = 0, 1
    while mb <= 1024:
        pl = plan_memory(a, micro_bs=mb, **kw)
        if pl.state_bytes > pl.capacity or pl.total_bytes > 0.92 * pl.capacity:
            break
        best, mb = mb, mb * 2
    return best


def main(argv: list[str] | None = None) -> int:
    ap = argparse.ArgumentParser(description="Per-GPU HBM budget of a training configuration (nothing is allocated)")
    ap.add_argument("config", nargs="*", help="@file.toml and dotted overrides, as for prime_b200.train")
    ap.add_argument("--world", type=int, default=8, help="ranks of the job (default 8: one NVSwitch box)")
    ap.add_argument("--model", help="model size instead of a config file (e.g. 7B)")
    ap.add_argument("--type", default="llama2", choices=("llama2", "llama3"))
    ap.add_argument("--fsdp", type=int, default=8)
    ap.add_argument("--micro-bs", type=int, default=1)
    ap.add_argument("--seq", type=int, default=4096)
    ap.add_argument("--ac-ckpt", action="store_true")
    ap.add_argument("--diloco", action="store_true")
    ap.add_argument("--reshard", type=int, choices=(0, 1), default=None)
    ap.add_argument("--capacity-gb", type=float, default=H100_HBM_BYTES / GB)
    ap.add_argument("--json", action="store_true")
    ns = ap.parse_args(argv)
    cap = int(ns.capacity_gb * GB)
    if ns.model:
        a = get_model_args(ns.model, ns.type)
        kw = dict(fsdp_size=ns.fsdp, seq_len=ns.seq, shard_params=None if ns.reshard is None else bool(ns.reshard), ac_ckpt=ns.ac_ckpt,
                  diloco=ns.diloco, capacity=cap, name=f"{ns.type}/{ns.model}")  # fmt: skip
        plan = plan_memory(a, micro_bs=ns.micro_bs, **kw)
        extra = {"largest_micro_bs": largest_micro_bs(a, **kw)}
    else:
        from ..config import load_config

        plan = plan_from_config(load_config(ns.config), ns.world, capacity=cap)
        extra = {}
    if ns.json:
        print(json.dumps({**plan.to_json(), **extra}))
    else:
        print(plan.table())
        for k, v in extra.items():
            print(f"{k}: {v}")
    return 0 if plan.verdict != "does_not_fit" else 1


if __name__ == "__main__":
    sys.exit(main())
