"""Shard layout of the sharded engine: where every parameter element lives, and which part of it each FSDP rank owns.

The engine's buffers, the checkpoints and the symmetric-heap size all follow it. It needs parameter names and shapes only, so
it can be planned on a ``meta``-device model. Bucket kinds: ``"flat"``, where rank r owns the r-th contiguous 1/F slice of the
bucket, and ``"rows"`` (ZeRO-3), where rank r owns rows [r·N/F, (r+1)·N/F) of every 2-D weight, one piece per weight.
"""

from __future__ import annotations

from dataclasses import dataclass

import torch
import torch.nn as nn

SHARD_ALIGN = 1024  # elements; also the int8 quantisation block of the outer step


def use_zero3(requested: bool | None, *, fused: bool, fsdp_size: int, n_params: int = 0) -> bool:
    """Whether the bf16 parameters are row-sharded (ZeRO-3, ``train.reshard_after_forward``). ``None`` asks for the default:
    on from 5 B parameters. It runs only with the fused backend and F > 1: peers read each other's shards inside the GEMMs."""
    want = n_params >= 5e9 if requested is None else bool(requested)
    return want and fused and fsdp_size > 1


@dataclass(frozen=True, eq=False)
class Bucket:
    name: str
    kind: str  # "flat" | "rows" (see the module docstring)
    params: tuple[tuple[str, nn.Parameter, int], ...]  # (qualified name, param, offset inside bucket)
    start: int  # offset in the flat main_grad buffer
    size: int  # padded element count (multiple of F * SHARD_ALIGN)
    shard_start: int  # offset in every rank's shard buffers
    shard_size: int
    pstart: int = 0  # flat kind: offset of the bucket in the replicated bf16 parameter buffer
    pieces: tuple[tuple[int, int], ...] = ()  # rows kind: per parameter (offset inside the bucket's shard, elements)

    def owned(self, rank: int) -> list[tuple[int, int, int]]:
        """Rank ``rank``'s part of this bucket as runs of (offset in the bucket, offset in its shard, elements); rows: one per param."""
        if self.kind == "flat":
            return [(rank * self.shard_size, self.shard_start, self.shard_size)]
        return [(off + rank * piece, self.shard_start + soff, piece) for (_, _, off), (soff, piece) in zip(self.params, self.pieces)]


@dataclass(frozen=True, eq=False)
class ShardLayout:
    F: int
    shard_params: bool
    buckets: tuple[Bucket, ...]
    total: int  # elements of the flat main_grad buffer
    shard_total: int  # elements of every rank's shard (fp32 master, AdamW moments, outer state)
    pflat_total: int  # elements of the replicated bf16 parameter buffer

    @property
    def signature(self) -> list[list]:
        """What checkpoints record of the layout, and compare on resume."""
        return [[b.name, b.start, b.size, b.shard_start, b.shard_size] for b in self.buckets]

    def matches(self, signature) -> bool:
        return [list(x) for x in signature] == self.signature

    def check_saved(self, signature, fsdp_size: int, shard_params: bool) -> None:
        """Raise ValueError unless state saved under (``signature``, ``fsdp_size``, ``shard_params``) fits this layout."""
        if fsdp_size != self.F:
            raise ValueError(f"checkpoint was written with fsdp_size={fsdp_size}, engine has {self.F}")
        if bool(shard_params) != self.shard_params:
            # the two modes cut the optimizer shards differently (contiguous 1/F slices of a bucket vs one row block per weight)
            raise ValueError(f"checkpoint was written with train.reshard_after_forward={bool(shard_params)} (shard layout differs), "
                             f"engine runs with {self.shard_params}: resume with the same setting")
        if signature is not None and not self.matches(signature):
            raise ValueError("checkpoint bucket layout does not match this model / mesh (different model size or parameter set)")

    def gather(self, shards: dict[int, torch.Tensor]) -> dict[str, torch.Tensor]:
        """Every rank's flat shard of one kind of state → {qualified parameter name: whole tensor in the parameter's shape}."""
        out = {}
        for b in self.buckets:
            flat = shards[0].new_zeros(b.size)
            for r in range(self.F):
                for src, dst, n in b.owned(r):
                    flat[src : src + n] = shards[r][dst : dst + n]
            out.update({qn: flat[off : off + p.numel()].view(p.shape) for qn, p, off in b.params})
        return out

    def scatter(self, full: dict[str, torch.Tensor], rank: int, dtype: torch.dtype = torch.float32) -> torch.Tensor:
        """Inverse of :meth:`gather` for one rank (padding stays zero)."""
        shard = torch.zeros(self.shard_total, dtype=dtype)
        for b in self.buckets:
            flat = torch.zeros(b.size, dtype=dtype)
            for qn, p, off in b.params:
                flat[off : off + p.numel()] = full[qn].reshape(-1)
            for src, dst, n in b.owned(rank):
                shard[dst : dst + n] = flat[src : src + n]
        return shard

    def heap_bytes(self, fp32_master: bool = False) -> int:
        """Symmetric-heap bytes: fp32 main_grad, bf16 parameters (+ ZeRO-3 row shards), the outer step's int8 payload and scales
        (reserved even without DiLoCo), the fp32 masters of the fused fp32 outer step, and 64 MiB of slack."""
        n = 4 * self.total + 2 * self.pflat_total + 2 * self.shard_total + (64 << 20)
        if self.shard_params:
            n += 2 * self.shard_total
        if fp32_master:
            n += 4 * self.shard_total
        return n


def _stages(model: nn.Module) -> list[tuple[str, list[tuple[str, nn.Parameter]]]]:
    """(stage name, [(qualified name, parameter)]): embedding, one stage per layer, head, then whatever is left."""
    named = dict(model.named_parameters())
    prefixes: list[tuple[str, list[str]]] = []
    if hasattr(model, "layers") and hasattr(model, "tok_embeddings"):
        prefixes = [("embed", ["tok_embeddings"]), *((f"layer{i}", [f"layers.{i}"]) for i in range(len(model.layers))), ("head", ["norm", "output"])]
    stages, used = [], set()
    for name, pre in prefixes:
        items = [(k, v) for k, v in named.items() if any(k == p or k.startswith(p + ".") for p in pre)]
        used.update(k for k, _ in items)
        stages.append((name, items))
    stages.append(("rest", [(k, v) for k, v in named.items() if k not in used]))
    return [s for s in stages if s[1]]


def _row_shardable(p: nn.Parameter, F: int) -> bool:
    return p.dim() == 2 and p.shape[0] % F == 0 and p.shape[1] % 64 == 0 and (p.numel() // F) % 8 == 0


def plan_layout(model: nn.Module, fsdp_size: int, shard_params: bool) -> ShardLayout:
    F = int(fsdp_size)
    gran = F * SHARD_ALIGN
    stages = _stages(model)
    plan = [(name, items, "flat") for name, items in stages]
    if shard_params:
        # every row-shardable 2-D weight goes to a "rows" bucket of its stage; the rest (norm gains, odd shapes) is collected
        # into ONE replicated flat bucket at the end of the shard space
        rows = [(name, [(k, v) for k, v in items if _row_shardable(v, F)], "rows") for name, items in stages]
        small = [(k, v) for _, items in stages for k, v in items if not _row_shardable(v, F)]
        plan = [x for x in rows if x[1]] + ([("small", small, "flat")] if small else [])
    buckets: list[Bucket] = []
    flat_off = shard_off = pflat_off = 0
    for name, items, kind in plan:
        off, plist = 0, []
        for qn, p in items:
            off = (off + 7) // 8 * 8  # 16-byte alignment of every bf16 parameter (TMA base address)
            plist.append((qn, p, off))
            off += p.numel()
        size = (off + gran - 1) // gran * gran
        if kind == "rows":
            soff, pieces = 0, []
            for _, p, _ in plist:
                piece = p.numel() // F
                pieces.append((soff, piece))
                soff += (piece + 7) // 8 * 8
            ssize = (soff + SHARD_ALIGN - 1) // SHARD_ALIGN * SHARD_ALIGN
            b = Bucket(name, kind, tuple(plist), flat_off, size, shard_off, ssize, pieces=tuple(pieces))
        else:
            b = Bucket(name, kind, tuple(plist), flat_off, size, shard_off, size // F, pstart=pflat_off)
            pflat_off += size
        buckets.append(b)
        flat_off += size
        shard_off += b.shard_size
    return ShardLayout(F, bool(shard_params), tuple(buckets), flat_off, shard_off, pflat_off)
