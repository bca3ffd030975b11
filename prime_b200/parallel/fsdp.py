"""Sharded inner-loop engine (the FSDP level of the two-level mesh).

Memory plan for 80 GB HBM3 parts: the bf16 parameters stay *resident and replicated* inside a
worker (one flat buffer), while everything optimizer-side — fp32 master weights, AdamW moments, the
reduced gradient — is partitioned 1/F per rank.  Per optimizer step the traffic is exactly FSDP's
(one gradient reduce-scatter + one parameter all-gather per bucket); what differs is *how*:

``backend="fused"`` (CUDA, symmetric NVLink heap — the product path)
    bucket ready in backward → flag signalled to peers → ``grad_reduce`` kernel pulls the peers'
    slices through NVSwitch (fixed rank order), scales, writes the fp32 shard gradient and the
    sum-of-squares partial;  after backward one ``adamw_push`` kernel per bucket does
    clip ⊕ AdamW ⊕ bf16 cast ⊕ *stores the new parameters straight into every peer's buffer*
    (the all-gather), then a flag barrier.  No NCCL call, no host sync, all on a side stream
    overlapped with the backward pass.

``backend="collective"`` (NCCL or gloo — the baseline "B0" and the CPU plumbing path)
    ``reduce_scatter`` / ``all_gather`` collectives around the same sharded optimizer.

Both share bucket layout and optimizer state, so checkpoints move freely between them.

``shard_params=True`` (``train.reshard_after_forward``; ZeRO-3, the default for 7B and larger)
    the bf16 parameters are NOT replicated: every 2-D weight is sharded by rows (dim 0, like FSDP2) and rank r keeps only
    rows [r·N/F, (r+1)·N/F) in its symmetric heap.  There is no all-gather collective at all — the GEMM that consumes a
    weight gathers it from the peers' shards while it multiplies (``pb_gemm_wgather``, IO = 3 of ``csrc/gemm_sm90.cu``:
    copier warps TMA the peer rows over NVLink into ONE layer-sized scratch that every layer reuses, the MMA tiles are
    released quarter block by quarter block), in the forward (y = x·Wᵀ, with the RoPE / SwiGLU epilogues) and again in the
    backward (dx = dy·W).  The embedding row gather reads the owners' shards directly.  The optimizer then updates only
    the local shard (no parameter push).  1-D parameters (norm gains, < 0.01 % of the model) stay replicated in one small
    flat bucket handled as above.  Per-GPU memory for Llama-7B at F = 8: 1.7 GB parameters + 0.4 GB scratch instead of 13.5 GB.
"""

from __future__ import annotations

import ctypes
from dataclasses import dataclass, field

import torch
import torch.distributed as dist
import torch.nn as nn

from ..ops import _lib, reference
from ..ops.functional import _count
from .layout import Bucket, ShardLayout, plan_layout, use_zero3
from .mesh import Mesh
from .symm import SymmetricHeap


@dataclass
class RowShard:
    """Attached to a row-sharded parameter as ``p.z3``: everything ``ops.functional`` needs to run the gather-fused GEMMs."""

    rows: int
    cols: int
    n: int
    rank: int
    rpr: int  # rows per rank
    peer_ptrs: object  # (c_void_p * n): rank i's [rpr, cols] bf16 block as mapped in this process
    full_ptr: int  # local [rows, cols] scratch the kernel gathers into (== the parameter tensor's storage)
    flags: torch.Tensor  # n * 4 readiness counters (zeroed by the launcher)
    shard: torch.Tensor  # this rank's [rpr, cols] block (view into the engine's bf16 shard buffer)
    full: torch.Tensor | None = None  # the scratch as a [rows, cols] tensor (plain kernels run on it when the weight is resident)
    # gather-ahead chain: the weight the NEXT GEMM of the pass consumes (forward order / backward dgrad order); the kernel that
    # computes with this weight also pulls that one into its scratch (ops.functional.gemm_wgather)
    next_fwd: "RowShard | None" = None
    next_bwd: "RowShard | None" = None
    ver: list = field(default_factory=lambda: [0])  # shared with the engine: bumped whenever the shards change (optimizer / outer step)


def reduce_segments(layout: ShardLayout, rank: int) -> list[_lib.SegTable]:
    """Per bucket, what rank ``rank``'s gradient reduce-scatter reads and writes: (offset in ``grad_flat``, offset in the reduced
    gradient shard, elements). A flat bucket is one piece, a row-sharded one a row block per parameter. At F = 1 the shard starts
    where the bucket does, so the reduction is in place in ``grad_flat``, which the shard aliases there."""
    return [_lib.SegTable.of((b.start + src, dst, n) for src, dst, n in b.owned(rank)) for b in layout.buckets]


class _Boundary(torch.autograd.Function):
    """Identity whose backward tells the engine "stage ``bucket_id`` has finished its backward"."""

    @staticmethod
    def forward(ctx, engine, bucket_id, *tensors):
        ctx.engine, ctx.bucket_id = engine, bucket_id
        return tuple(t.view_as(t) for t in tensors)

    @staticmethod
    def backward(ctx, *grads):
        ctx.engine._on_bucket_ready(ctx.bucket_id)
        return (None, None, *grads)


@dataclass
class AdamHyper:
    lr: float = 4e-4
    beta1: float = 0.9
    beta2: float = 0.95
    eps: float = 1e-8
    weight_decay: float = 0.1
    max_norm: float = 1.0


class ShardedEngine:
    def __init__(
        self,
        model: nn.Module,
        mesh: Mesh,
        hyper: AdamHyper,
        *,
        backend: str = "auto",
        heap: SymmetricHeap | None = None,
        overlap: bool = True,
        reduce_ctas: int = 32,
        shard_params: bool = False,
        master_in_heap: bool = False,
        fresh_grads: bool = True,
    ):
        self.model, self.mesh, self.hyper = model, mesh, hyper
        self.F = mesh.fsdp_size
        self.device = next(model.parameters()).device
        self.param_dtype = next(model.parameters()).dtype
        if backend == "auto":
            backend = "fused" if (self.device.type == "cuda" and heap is not None) else "collective"
        if backend == "fused" and (heap is None or self.device.type != "cuda"):
            raise ValueError("fused backend needs CUDA and a SymmetricHeap")
        self.backend, self.heap, self.overlap, self.reduce_ctas = backend, heap, overlap, reduce_ctas
        self.shard_params = use_zero3(bool(shard_params), fused=backend == "fused", fsdp_size=self.F)
        self.master_in_heap = bool(master_in_heap) and backend == "fused"
        # first weight-gradient write of a step overwrites (GEMM epilogue with accumulate=false) instead of adding into a buffer that
        # a 4·N-byte memset had to clear first; off while a CUDA graph is captured/replayed (the accumulate flag is baked in there)
        self.fresh_grads = bool(fresh_grads) and self.device.type == "cuda"
        self.step_count = 0
        self.last_grad_norm: torch.Tensor | None = None
        self._last_micro = True
        self._epoch = 0
        self._pver = [0]  # parameter-shard version: bumped whenever the bf16 shards change (gathered scratch copies go stale)
        self.capture_mode = False  # True while a CUDA graph of the micro-step is captured/replayed: no comm in backward
        self.trace = None  # optional StepTrace (utils/steptrace.py): CUDA events around the phases of the step
        if self.device.type == "cuda":
            self.lib = _lib.load()
            self.comm_stream = torch.cuda.Stream(device=self.device) if overlap else None
        else:
            self.lib, self.comm_stream = None, None
        from ..ops.functional import reset_gather_cache

        reset_gather_cache()
        self.layout = plan_layout(model, self.F, self.shard_params)
        self.buckets, self.total, self.shard_total = self.layout.buckets, self.layout.total, self.layout.shard_total
        self.bucket_index = {b.name: i for i, b in enumerate(self.buckets)}
        self._ready = [False] * len(self.buckets)
        self._work: list = [None] * len(self.buckets)  # async collective handles (collective backend)
        self._segs = reduce_segments(self.layout, mesh.fsdp_rank)
        self._allocate()
        self._install_hooks()

    # ------------------------------------------------------------------ buffers
    def _allocate(self) -> None:
        dev, F, r = self.device, self.F, self.mesh.fsdp_rank
        fused = self.backend == "fused"
        if fused:
            self.param_flat = self.heap.alloc(max(self.layout.pflat_total, 8), self.param_dtype)
            self.grad_flat = self.heap.alloc(self.total, torch.float32)
            self.pshard = self.heap.alloc(self.shard_total, self.param_dtype) if self.shard_params else None
            self.slot_grad = self.heap.alloc_flags(len(self.buckets) * F)
            self.slot_norm = self.heap.alloc_flags(F)
            self.slot_bar = self.heap.alloc_flags(F)
            # NVLS reduce-scatter: only when the heap has a multicast mapping AND it spans exactly this FSDP group (the switch
            # sums every device bound to the object, so a heap shared by several DiLoCo workers cannot use it)
            self._nvls = F > 1 and hasattr(self.heap, "mc_ptr") and self.heap.world_size == F
            self.sumsq_partial = torch.zeros(self.lib_grid(), dtype=torch.float32, device=dev)
            self.gnorm_buf = torch.zeros(1, dtype=torch.float32, device=dev)
        else:
            self.param_flat = torch.zeros(max(self.layout.pflat_total, 8), dtype=self.param_dtype, device=dev)
            self.grad_flat = torch.zeros(self.total, dtype=torch.float32, device=dev)
            self.pshard = None
        self.param_flat.zero_()
        self.grad_flat.zero_()
        if self.master_in_heap:
            self.master = self.heap.alloc(self.shard_total, torch.float32)
        else:
            self.master = torch.empty(self.shard_total, dtype=torch.float32, device=dev)
        self.master.zero_()
        if self.shard_params:
            self.pshard.zero_()
            # ONE layer-sized scratch for the gathered weights: every layer's wqkv lands at the same address (stream order makes the
            # reuse safe — a weight is gathered and consumed inside the same kernel), which also keeps the tensor-map cache tiny
            by_stage = {}
            for b in self.buckets:
                if b.kind == "rows" and b.name != "embed":
                    key = "layer" if b.name.startswith("layer") else b.name
                    by_stage[key] = max(by_stage.get(key, 0), b.size)
            self._scratch = {k: torch.empty(v, dtype=self.param_dtype, device=dev) for k, v in by_stage.items()}
            self._gather_flags = torch.zeros(64, dtype=torch.int32, device=dev)
        with torch.no_grad():
            for b in self.buckets:
                if b.kind == "rows":
                    self._attach_rows_bucket(b)
                    continue
                for _, p, off in b.params:
                    view = self.param_flat[b.pstart + off : b.pstart + off + p.numel()].view(p.shape)
                    view.copy_(p.data)
                    p.data = view
                    p.main_grad = self.grad_flat[b.start + off : b.start + off + p.numel()].view(p.shape)
                for src, dst, n in b.owned(r):
                    self.master[dst : dst + n] = self.param_flat[b.pstart + src : b.pstart + src + n].float()
        self.exp_avg = torch.zeros_like(self.master) if not self.master_in_heap else torch.zeros(self.shard_total, dtype=torch.float32, device=dev)
        self.exp_avg_sq = torch.zeros_like(self.exp_avg)
        # reduced gradient shard; with F == 1 the shard *is* the bucket, so alias instead of copying
        self.gshard = self.grad_flat if F == 1 else torch.zeros(self.shard_total, dtype=torch.float32, device=dev)
        self._params = [p for b in self.buckets for _, p, _ in b.params]
        if self.shard_params:
            self._link_gather_chain()

    def _link_gather_chain(self) -> None:
        """Order in which the GEMMs consume the sharded weights: forward wqkv → wo → w13 → w2 per layer, then the head; backward
        (input gradients) the reverse. Each weight points at its successor so the kernel computing with it can gather that one ahead."""
        m = self.model
        if not (hasattr(m, "layers") and hasattr(m, "output")):
            return
        seq = []
        for layer in m.layers:
            seq += [layer.attention.wqkv, layer.attention.wo, layer.feed_forward.w13, layer.feed_forward.w2]
        seq.append(m.output)
        zs = [getattr(p, "z3", None) for p in seq]
        if any(z is None for z in zs):
            return
        for a, b in zip(zs[:-1], zs[1:]):
            a.next_fwd = b
            b.next_bwd = a

    def _attach_rows_bucket(self, b: Bucket) -> None:
        """ZeRO-3: copy this rank's row block of every weight into the shard buffer, then re-point the parameter at the shared
        gather scratch (embedding: at a stride-0 placeholder — its rows are only ever read through the peers' shards)."""
        F, r, heap = self.F, self.mesh.fsdp_rank, self.heap
        ranks = self.mesh.fsdp_ranks
        key = "layer" if b.name.startswith("layer") else b.name
        for (qn, p, off), (src, lo, piece) in zip(b.params, b.owned(r)):
            rows, cols = p.shape
            rpr = rows // F
            shard = self.pshard[lo : lo + piece].view(rpr, cols)
            shard.view(-1).copy_(p.data.view(-1)[src - off : src - off + piece])
            self.master[lo : lo + piece] = shard.reshape(-1).float()
            if b.name == "embed":
                full = torch.zeros(1, dtype=self.param_dtype, device=self.device).expand(rows, cols)
                full_ptr = 0
            else:
                full = self._scratch[key][off : off + p.numel()].view(rows, cols)
                full_ptr = full.data_ptr()
            peers = (ctypes.c_void_p * F)(*[heap.peer_ptr(q, shard) for q in ranks])
            p.data = full
            p.main_grad = self.grad_flat[b.start + off : b.start + off + p.numel()].view(p.shape)
            p.z3 = RowShard(rows, cols, F, r, rpr, peers, full_ptr, self._gather_flags, shard, full=full if b.name != "embed" else None,
                            ver=self._pver)

    def lib_grid(self) -> int:
        return _lib.load().pb_grad_reduce_grid()

    # ------------------------------------------------------------------ hooks
    def _install_hooks(self) -> None:
        m = self.model
        if not (hasattr(m, "layers") and len(m.layers) > 0):
            return
        eng = self

        def pre_hook_for(bucket_id: int):
            def hook(module, args, kwargs):
                if not torch.is_grad_enabled():
                    return None
                idx = [i for i, a in enumerate(args) if isinstance(a, torch.Tensor) and a.requires_grad]
                if not idx:
                    return None
                outs = _Boundary.apply(eng, bucket_id, *[args[i] for i in idx])
                args = list(args)
                for i, o in zip(idx, outs):
                    args[i] = o
                return tuple(args), kwargs

            return hook

        for i, layer in enumerate(m.layers):
            layer.register_forward_pre_hook(pre_hook_for(self.bucket_index[f"layer{i}"]), with_kwargs=True)

        head_id = self.bucket_index.get("head")
        if head_id is not None:

            def post_hook(module, args, output):
                if not torch.is_grad_enabled():
                    return None
                outs = output if isinstance(output, tuple) else (output,)
                idx = [i for i, a in enumerate(outs) if isinstance(a, torch.Tensor) and a.requires_grad]
                if not idx:
                    return None
                wrapped = _Boundary.apply(eng, head_id, *[outs[i] for i in idx])
                outs = list(outs)
                for i, o in zip(idx, wrapped):
                    outs[i] = o
                return tuple(outs) if isinstance(output, tuple) else outs[0]

            m.layers[-1].register_forward_hook(post_hook)

    # ------------------------------------------------------------------ step protocol
    def zero_grad(self) -> None:
        if self.fresh_grads and not self.capture_mode:
            # no 4·N-byte memset: the first gradient write of every parameter in this step overwrites (ops check ``_mg_fresh``).
            # Only the embedding table is cleared — its backward scatters into a few rows and must find zeros elsewhere.
            for b in self.buckets:
                for qn, p, _ in b.params:
                    if "tok_embeddings" in qn:
                        p.main_grad.zero_()
                        p._mg_fresh = False
                    else:
                        p._mg_fresh = True
        else:
            self.grad_flat.zero_()
        self._ready = [False] * len(self.buckets)
        self._work = [None] * len(self.buckets)

    def set_micro_step(self, last: bool) -> None:
        """Tell the engine whether the coming backward is the last of the accumulation window."""
        self._last_micro = last
        if last:
            self._epoch += 1

    def _fold_autograd_grads(self, b: Bucket) -> None:
        """Ops without main_grad fusion (CPU reference ops) leave ``.grad``: fold into main_grad."""
        for _, p, _ in b.params:
            if p.grad is not None:
                if getattr(p, "_mg_fresh", False):
                    p.main_grad.copy_(p.grad)
                    p._mg_fresh = False
                else:
                    p.main_grad.add_(p.grad.to(torch.float32))
                p.grad = None

    def _settle_fresh(self, b: Bucket) -> None:
        """A parameter nobody wrote a gradient for in this step (unused in the graph) still holds last step's: clear it."""
        if not self.fresh_grads:
            return
        for _, p, _ in b.params:
            if getattr(p, "_mg_fresh", False):
                p.main_grad.zero_()
                p._mg_fresh = False

    def _on_bucket_ready(self, bucket_id: int) -> None:
        b = self.buckets[bucket_id]
        if self.capture_mode or not self._last_micro or self._ready[bucket_id]:
            return
        self._ready[bucket_id] = True
        self._fold_autograd_grads(b)
        self._settle_fresh(b)
        self._reduce_bucket(bucket_id)

    def _reduce_bucket(self, bucket_id: int) -> None:
        b, F, r = self.buckets[bucket_id], self.F, self.mesh.fsdp_rank
        if self.backend == "fused":
            main = torch.cuda.current_stream()
            cs = self.comm_stream or main
            if cs is not main:
                cs.wait_stream(main)
            with torch.cuda.stream(cs):
                s = cs.cuda_stream
                ranks = self.mesh.fsdp_ranks
                wait_flags = None
                slot_base = self.slot_grad + bucket_id * F
                if F > 1:
                    pp = self.heap.peers(ranks, self.heap.flags)
                    _lib.check(self.lib.pb_signal(ctypes.byref(pp), slot_base + r, self._epoch, s), "pb_signal")
                    _count()
                    wait_flags = self.heap.flags.data_ptr()
                ctas = self.reduce_ctas if (F > 1 and self.overlap) else 0
                gp = self.heap.peers(ranks, self.grad_flat)
                # NVLS: the switch sums the F copies, one multimem.ld_reduce per 16 bytes instead of F peer loads
                mc = self.heap.mc_ptr(self.grad_flat) if self._nvls else None
                _lib.check(
                    self.lib.pb_grad_reduce(
                        ctypes.byref(gp), mc, ctypes.byref(self._segs[bucket_id]), 1.0 / F, self.gshard.data_ptr(),
                        self.sumsq_partial.data_ptr(), wait_flags, slot_base, self._epoch, self.heap.err.data_ptr(), ctas, s,
                    ),
                    "pb_grad_reduce",
                )  # fmt: skip
                _count()
            return
        # ---- collective backend
        if F == 1:
            return
        src = self.grad_flat[b.start : b.start + b.size]
        dst = self.gshard[b.shard_start : b.shard_start + b.shard_size]
        g = self.mesh.fsdp_group
        if dist.get_backend(g) == "nccl":
            self._work[bucket_id] = dist.reduce_scatter_tensor(dst, src, op=dist.ReduceOp.AVG, group=g, async_op=True)
        else:  # gloo has no reduce_scatter: all-reduce the bucket, keep my slice
            dist.all_reduce(src, group=g)
            dst.copy_(src[r * b.shard_size : (r + 1) * b.shard_size])
            dst.mul_(1.0 / F)

    def finish_backward(self) -> None:
        """Call after ``loss.backward()`` of the last micro-step: reduces whatever has no boundary (embeddings)."""
        if self.trace is not None:
            self.trace.mark("backward_end")
        for i, b in enumerate(self.buckets):
            if not self._ready[i]:
                self._ready[i] = True
                self._fold_autograd_grads(b)
                self._settle_fresh(b)
                self._reduce_bucket(i)

    def fold_micro_grads(self) -> None:
        """After a non-final micro-step backward: fold stray ``.grad`` tensors into main_grad."""
        for b in self.buckets:
            self._fold_autograd_grads(b)

    # ------------------------------------------------------------------ optimizer
    def step(self, lr: float | None = None) -> None:
        h = self.hyper
        lr = h.lr if lr is None else lr
        self.step_count += 1
        t = self.step_count
        bc1, bc2 = 1.0 - h.beta1**t, 1.0 - h.beta2**t
        if self.backend == "fused":
            self._step_fused(lr, bc1, bc2)
        else:
            self._step_collective(lr, bc1, bc2)
        self._ready = [False] * len(self.buckets)
        self._work = [None] * len(self.buckets)
        self._pver[0] += 1

    def _param_dst(self, b: Bucket) -> tuple[_lib.PeerPtrs, int]:
        """Where the bf16 image of bucket ``b``'s master shard goes: (destination buffers, element offset)."""
        if b.kind == "rows":  # ZeRO-3: only the local shard; nothing is pushed over NVLink
            return _lib.PeerPtrs.of([self.pshard.data_ptr()]), b.shard_start
        return self.heap.peers(self.mesh.fsdp_ranks, self.param_flat), b.pstart + self.mesh.fsdp_rank * b.shard_size

    def outer_ranges(self) -> list[tuple[int, int, _lib.PeerPtrs, list[int], list[int]]]:
        """Shard-space ranges with one bf16 destination each, for the one-launch outer step: (lo, hi, dst, shard_starts
        relative to lo (+ the end), dst_starts)."""
        out: list = []
        for b in self.buckets:
            dst, off = self._param_dst(b)
            key = tuple(dst.p[i] for i in range(dst.n))
            if out and out[-1][5] == key:
                out[-1][3].append(b.shard_start - out[-1][0])
                out[-1][4].append(off)
                out[-1][1] = b.shard_start + b.shard_size
            else:
                out.append([b.shard_start, b.shard_start + b.shard_size, dst, [0], [off], key])
        return [(lo, hi, dst, starts + [hi - lo], dsts) for lo, hi, dst, starts, dsts, _ in out]

    def _step_fused(self, lr: float, bc1: float, bc2: float) -> None:
        h, F, r = self.hyper, self.F, self.mesh.fsdp_rank
        main = torch.cuda.current_stream()
        cs = self.comm_stream or main
        if cs is not main:
            cs.wait_stream(main)
        ranks = self.mesh.fsdp_ranks
        heap = self.heap
        with torch.cuda.stream(cs):
            s = cs.cuda_stream
            if self.trace is not None:
                self.trace.mark("reduce_end", cs)
            flags_pp = heap.peers(ranks, heap.flags)
            norm_pp = heap.peers(ranks, heap.norm_slots)
            _lib.check(
                self.lib.pb_norm_publish(self.sumsq_partial.data_ptr(), self.sumsq_partial.numel(), ctypes.byref(norm_pp),
                                         ctypes.byref(flags_pp), r, self.slot_norm, self._epoch, s),
                "pb_norm_publish",
            )  # fmt: skip
            _count(1 + len(self.buckets) + (1 if F > 1 else 0))
            args = _lib.AdamArgs(lr, h.beta1, h.beta2, h.eps, h.weight_decay, bc1, bc2, h.max_norm)
            for b in self.buckets:
                dst, dst_off = self._param_dst(b)
                sl = slice(b.shard_start, b.shard_start + b.shard_size)
                g = self.gshard[b.shard_start :] if F > 1 else self.grad_flat[b.start :]
                _lib.check(
                    self.lib.pb_adamw_push(
                        self.master[sl].data_ptr(), g.data_ptr(), self.exp_avg[sl].data_ptr(), self.exp_avg_sq[sl].data_ptr(),
                        b.shard_size, ctypes.byref(args), heap.norm_slots.data_ptr(), F, heap.flags.data_ptr(),
                        self.slot_norm, self._epoch, ctypes.byref(dst), dst_off,
                        self.gnorm_buf.data_ptr(), heap.err.data_ptr(),
                        # NVLS heap spanning exactly this FSDP group: the all-gather is ONE multicast store per 16 bytes
                        heap.mc_ptr(self.param_flat) if (self._nvls and b.kind == "flat") else None, s,
                    ),
                    "pb_adamw_push",
                )  # fmt: skip
            if self.trace is not None:
                self.trace.mark("adamw_end", cs)
            if F > 1:
                heap.barrier(ranks, self.slot_bar, self._epoch, s)
            if self.trace is not None:
                self.trace.mark("barrier_end", cs)
        if cs is not main:
            main.wait_stream(cs)
        self.last_grad_norm = self.gnorm_buf

    def _step_collective(self, lr: float, bc1: float, bc2: float) -> None:
        h, F, r = self.hyper, self.F, self.mesh.fsdp_rank
        g = self.mesh.fsdp_group
        for w in self._work:
            if w is not None:
                w.wait()
        gsh = self.gshard  # aliases grad_flat when F == 1 (identical layout)
        sumsq = gsh.pow(2).sum()
        if F > 1:
            dist.all_reduce(sumsq, group=g)
        gnorm = sumsq.sqrt()
        self.last_grad_norm = gnorm
        clip = torch.clamp(h.max_norm / (gnorm + 1e-6), max=1.0) if h.max_norm > 0 else torch.ones((), device=gnorm.device)
        gsh = gsh * clip
        reference.adamw_step(
            self.master, gsh, self.exp_avg, self.exp_avg_sq, lr=lr, beta1=h.beta1, beta2=h.beta2, eps=h.eps,
            weight_decay=h.weight_decay, step=self.step_count,
        )  # fmt: skip
        self.publish_params()

    @torch.no_grad()
    def publish_params(self) -> None:
        """fp32 master shard → parameter buffers of the whole FSDP group (cast + all-gather; ZeRO-3: cast into the local shard)."""
        F, r = self.F, self.mesh.fsdp_rank
        self._pver[0] += 1
        if self.backend == "fused":
            main = torch.cuda.current_stream()
            ranks = self.mesh.fsdp_ranks
            for b in self.buckets:
                dst, dst_off = self._param_dst(b)
                sl = slice(b.shard_start, b.shard_start + b.shard_size)
                _lib.check(
                    self.lib.pb_cast_push(self.master[sl].data_ptr(), b.shard_size, ctypes.byref(dst), dst_off, main.cuda_stream),
                    "pb_cast_push",
                )
            if F > 1:
                self._epoch += 1
                self.heap.barrier(ranks, self.slot_bar, self._epoch, main.cuda_stream)
            return
        for b in self.buckets:
            mine = self.param_flat[b.pstart + r * b.shard_size : b.pstart + (r + 1) * b.shard_size]
            mine.copy_(self.master[b.shard_start : b.shard_start + b.shard_size])
            if F > 1:
                dist.all_gather_into_tensor(self.param_flat[b.pstart : b.pstart + b.size], mine.clone(), group=self.mesh.fsdp_group)

    @torch.no_grad()
    def full_param(self, p: nn.Parameter) -> torch.Tensor:
        """The complete bf16 value of a parameter (ZeRO-3: gathered from the peers' shards into a fresh tensor)."""
        z = getattr(p, "z3", None)
        if z is None:
            return p.data
        out = torch.empty((z.rows, z.cols), dtype=self.param_dtype, device=self.device)
        pp = _lib.PeerPtrs.of(z.peer_ptrs[i] for i in range(z.n))
        _lib.check(self.lib.pb_allgather_copy(ctypes.byref(pp), z.rpr * z.cols * 2, out.data_ptr(), torch.cuda.current_stream().cuda_stream),
                   "pb_allgather_copy")  # fmt: skip
        return out

    # ------------------------------------------------------------------ state
    def state_dict(self) -> dict:
        return {
            "step": self.step_count,
            "master": self.master,
            "exp_avg": self.exp_avg,
            "exp_avg_sq": self.exp_avg_sq,
            "layout": self.layout.signature,
            "shard_params": self.shard_params,
            "fsdp_size": self.F,
            "fsdp_rank": self.mesh.fsdp_rank,
        }

    def load_state_dict(self, sd: dict) -> None:
        self.layout.check_saved(sd.get("layout"), sd["fsdp_size"], sd.get("shard_params", False))
        self.step_count = int(sd["step"])
        self.master.copy_(sd["master"])
        self.exp_avg.copy_(sd["exp_avg"])
        self.exp_avg_sq.copy_(sd["exp_avg_sq"])
        self.publish_params()

    def param_hash(self) -> float:
        """Cheap replica-consistency probe (sum of the bf16 parameter buffer)."""
        v = self.param_flat.float().sum()
        if self.shard_params:
            v = v + self.pshard.float().sum()
        return float(v.item())
