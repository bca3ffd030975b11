"""DiLoCo outer optimizer: every H inner steps, all-reduce the (int8-quantised) pseudo-gradient
across workers and take a Nesterov-SGD step on the replicated outer parameters θ₀.

State lives on the GPU (θ₀ and the momentum buffer are sharded exactly like the inner optimizer:
1/F per rank, so no host offload is needed).

Exchange design (SURVEY §7.3 #1): int8 payloads cannot be summed in the switch, so the all-reduce is
an *all-gather of (int8, per-1024 scales)* followed by a local dequantise-and-sum in fixed worker
order — every worker ends up with bitwise-identical θ₀ with one quantisation per contribution.

``backend="fused"``  : kernel 1 = pseudo-gradient ⊕ quantise (into the symmetric heap);
                       flag barrier; kernel 2 = peer int8 loads ⊕ dequant-sum ⊕ Nesterov ⊕ inner
                       master reset ⊕ bf16 parameter stores to the FSDP group.
``backend="collective"``: same math with ``all_gather`` / ``all_reduce`` (NCCL or gloo) — baseline + CPU path.
"""

from __future__ import annotations

import ctypes
import time
from dataclasses import dataclass

import torch
import torch.distributed as dist

from ..ops import _lib, reference
from ..ops.functional import _count
from .fsdp import ShardedEngine
from .layout import SHARD_ALIGN


@dataclass
class OuterHyper:
    lr: float = 0.7
    momentum: float = 0.9
    nesterov: bool = True
    compression: str = "int8"  # "int8" | "no"


def _all_gather(group, outs: list[torch.Tensor], t: torch.Tensor) -> None:
    """Works for registered groups and for the standalone per-epoch groups the elastic coordinator builds."""
    if group is None:
        dist.all_gather(outs, t)
    else:
        group.allgather([outs], [t]).wait()


def _all_reduce(group, t: torch.Tensor) -> None:
    if group is None:
        dist.all_reduce(t)
    else:
        group.allreduce([t]).wait()


class DilocoOuter:
    def __init__(self, engine: ShardedEngine, hyper: OuterHyper, *, diloco_group=None, diloco_ranks=None, collective: bool = False):
        self.engine, self.hyper = engine, hyper
        self.mesh = engine.mesh
        self.group = diloco_group if diloco_group is not None else self.mesh.diloco_group
        self.ranks = list(diloco_ranks) if diloco_ranks is not None else list(self.mesh.diloco_ranks)
        n = engine.shard_total
        dev = engine.device
        self.theta0 = engine.master.clone()
        self.momentum = torch.zeros(n, dtype=torch.float32, device=dev)
        self.outer_step_count = 0
        self.last_bytes_on_wire = 0
        self.last_seconds = 0.0  # host wall clock of the last step() call (enqueue time on CUDA: use device_seconds())
        self._ev: tuple | None = None
        self.total_device_ms = 0.0
        self.total_skew_ms = 0.0
        self._pre = None
        self.timed_steps = 0
        # ``collective=True``: the exchange goes through a (re-creatable) process group instead of the symmetric heap
        self.fused = engine.backend == "fused" and not collective
        self.exchange = None  # ElasticExchange: fused outer step across separately launched workers (attach_exchange)
        if engine.backend == "fused":
            # shard index → position in the bf16 parameter buffer, one entry per bucket (see BucketTable in csrc/comm.cu); one
            # launch per destination set (replicated engine: one; ZeRO-3: local shard buffer + the small replicated bucket)
            self._ranges = []
            for lo, hi, dst, starts, dsts in engine.outer_ranges():
                self._ranges.append((lo, hi, dst, torch.tensor(starts, dtype=torch.int64, device=dev),
                                     torch.tensor(dsts, dtype=torch.int64, device=dev)))  # fmt: skip
            self._ev_pool = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(2)]
        if self.fused:
            heap = engine.heap
            world = heap.world_size
            self.slot_bar = heap.alloc_flags(world)
            self.slot_bar2 = heap.alloc_flags(world)
            self.slot_align = heap.alloc_flags(world)
            self._epoch = 0
            if hyper.compression == "int8":
                self.q = heap.alloc(n, torch.int8)
                self.scales = heap.alloc(n // SHARD_ALIGN, torch.float32)
            else:
                if not engine.master_in_heap:
                    raise ValueError("fused fp32 outer step needs the inner masters in the symmetric heap (ShardedEngine(master_in_heap=True))")
                self.theta_new = torch.empty(n, dtype=torch.float32, device=dev)

    def attach_exchange(self, exchange) -> None:
        """Elastic jobs: run the fused kernel pair over an ``ElasticExchange`` (cudaIpc regions published through the global store)
        instead of a process group. Needs the fused engine; int8 compression only."""
        if self.engine.backend != "fused" or self.hyper.compression != "int8":
            raise ValueError("the elastic NVLink exchange needs the fused engine and int8 compression")
        self.exchange = exchange

    @property
    def num_workers(self) -> int:
        return len(self.exchange.members) if self.exchange is not None else len(self.ranks)

    def set_membership(self, ranks, group) -> None:
        """Elastic join/drop: swap the set of peers contributing to the next outer step."""
        self.ranks, self.group = list(ranks), group

    # ------------------------------------------------------------------ the outer step
    @torch.no_grad()
    def step(self) -> None:
        t0 = time.perf_counter()
        cuda = self.engine.device.type == "cuda"
        if cuda:
            if self.engine.backend == "fused":
                ev = self._ev_pool[self.outer_step_count % 2]
            else:
                ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
            self._harvest()
            if self.fused and self.engine.heap.world_size > 1:
                # line the ranks up first: workers drift apart over H inner steps, and the time a fast rank spends waiting for the
                # slowest one is arrival skew, not part of the exchange — it is timed separately (``last_skew_seconds``)
                pre = torch.cuda.Event(enable_timing=True)
                pre.record()
                self._epoch += 1
                self.engine.heap.barrier(list(range(self.engine.heap.world_size)), self.slot_align, self._epoch,
                                         torch.cuda.current_stream().cuda_stream)
                self._pre = pre
            ev[0].record()
        if self.exchange is not None:
            self._step_exchange()
        elif self.fused:
            self._step_fused()
        else:
            self._step_collective()
        if cuda:
            ev[1].record()
            self._ev = ev
        self.outer_step_count += 1
        if hasattr(self.engine, "_pver"):
            self.engine._pver[0] += 1  # the bf16 parameters changed: gathered scratch copies of the ZeRO-3 path are stale
        self.last_seconds = time.perf_counter() - t0

    def _harvest(self) -> None:
        if self._ev is not None:
            self._ev[1].synchronize()
            self.total_device_ms += self._ev[0].elapsed_time(self._ev[1])
            if getattr(self, "_pre", None) is not None:
                self.total_skew_ms += self._pre.elapsed_time(self._ev[0])
                self._pre = None
            self.timed_steps += 1
            self._ev = None

    def device_seconds(self) -> float:
        """Device time (CUDA events on the launching stream) of the most recent outer step; synchronises on its end event."""
        if self._ev is None:
            return self.last_seconds
        self._ev[1].synchronize()
        return self._ev[0].elapsed_time(self._ev[1]) / 1e3

    def reset_timing(self) -> None:
        self._harvest()
        self.total_device_ms, self.total_skew_ms, self.timed_steps = 0.0, 0.0, 0

    def mean_skew_seconds(self) -> float:
        """Mean device time a rank waited at the alignment barrier in front of the outer step (arrival skew between workers)."""
        self._harvest()
        return self.total_skew_ms / 1e3 / max(1, self.timed_steps)

    def mean_device_seconds(self) -> float:
        self._harvest()
        return self.total_device_ms / 1e3 / max(1, self.timed_steps)

    def _step_fused(self) -> None:
        eng, heap, lib = self.engine, self.engine.heap, self.engine.lib
        s = torch.cuda.current_stream().cuda_stream
        n = eng.shard_total
        W = self.num_workers
        all_ranks = list(range(heap.world_size))
        args = _lib.OuterArgs(self.hyper.lr, self.hyper.momentum, 1.0 / W, int(self.hyper.nesterov))
        if self.hyper.compression == "int8":
            _lib.check(lib.pb_pseudograd_quant(self.theta0.data_ptr(), eng.master.data_ptr(), self.q.data_ptr(),
                                               self.scales.data_ptr(), n, s), "pb_pseudograd_quant")  # fmt: skip
            self._epoch += 1
            heap.barrier(all_ranks, self.slot_bar, self._epoch, s)  # everyone's payload is published
            for lo, hi, dst, tab_s, tab_d in self._ranges:
                qs = _lib.PeerPtrs.of(heap.peer_ptr(w, self.q) + lo for w in self.ranks)
                ss = _lib.PeerPtrs.of(heap.peer_ptr(w, self.scales) + (lo // SHARD_ALIGN) * 4 for w in self.ranks)
                _lib.check(
                    lib.pb_outer_nesterov(ctypes.byref(qs), ctypes.byref(ss), self.theta0[lo:].data_ptr(), self.momentum[lo:].data_ptr(),
                                          eng.master[lo:].data_ptr(), hi - lo, ctypes.byref(args), ctypes.byref(dst), tab_s.data_ptr(),
                                          tab_d.data_ptr(), tab_d.numel(), heap.err.data_ptr(), s),
                    "pb_outer_nesterov",
                )  # fmt: skip
            self._epoch += 1
            heap.barrier(all_ranks, self.slot_bar2, self._epoch, s)  # payloads consumed, params landed
            self.last_bytes_on_wire = (W - 1) * (n + 4 * (n // SHARD_ALIGN))
            _count(3 + len(self._ranges))
        else:
            # uncompressed: every worker reads the peers' fp32 inner masters straight out of the heap
            self._epoch += 1
            heap.barrier(all_ranks, self.slot_bar, self._epoch, s)  # every worker finished its inner steps
            for lo, hi, dst, tab_s, tab_d in self._ranges:
                ths = _lib.PeerPtrs.of(heap.peer_ptr(w, eng.master) + lo * 4 for w in self.ranks)
                _lib.check(
                    lib.pb_outer_nesterov_f32(ctypes.byref(ths), self.theta0[lo:].data_ptr(), self.momentum[lo:].data_ptr(),
                                              self.theta_new[lo:].data_ptr(), hi - lo, ctypes.byref(args), ctypes.byref(dst),
                                              tab_s.data_ptr(), tab_d.data_ptr(), tab_d.numel(), heap.err.data_ptr(), s),
                    "pb_outer_nesterov_f32",
                )  # fmt: skip
            self._epoch += 1
            heap.barrier(all_ranks, self.slot_bar2, self._epoch, s)  # nobody reads the old masters any more
            eng.master.copy_(self.theta_new)
            self.last_bytes_on_wire = (W - 1) * 4 * n
            _count(3 + len(self._ranges))

    def _step_exchange(self) -> None:
        """Same kernel pair as ``_step_fused`` over the elastic exchange regions (see parallel/elastic_exchange.py). Synchronises at
        the end and raises if a member never reached a barrier — θ₀, momentum and the master are untouched in that case."""
        from .elastic_exchange import SLOT_A, SLOT_B

        eng, lib, x = self.engine, self.engine.lib, self.exchange
        s = torch.cuda.current_stream().cuda_stream
        n = eng.shard_total
        W = len(x.members)
        args = _lib.OuterArgs(self.hyper.lr, self.hyper.momentum, 1.0 / W, int(self.hyper.nesterov))
        _lib.check(lib.pb_pseudograd_quant(self.theta0.data_ptr(), eng.master.data_ptr(), x.q.data_ptr(), x.scales.data_ptr(), n, s),
                   "pb_pseudograd_quant")  # fmt: skip
        x.barrier(SLOT_A, s)  # every member's payload is published
        qs_all, ss_all = x.payload_ptrs()
        for lo, hi, dst, tab_s, tab_d in self._ranges:
            qs = _lib.PeerPtrs.of(qs_all.p[i] + lo for i in range(W))
            ss = _lib.PeerPtrs.of(ss_all.p[i] + (lo // SHARD_ALIGN) * 4 for i in range(W))
            _lib.check(
                lib.pb_outer_nesterov(ctypes.byref(qs), ctypes.byref(ss), self.theta0[lo:].data_ptr(), self.momentum[lo:].data_ptr(),
                                      eng.master[lo:].data_ptr(), hi - lo, ctypes.byref(args), ctypes.byref(dst), tab_s.data_ptr(),
                                      tab_d.data_ptr(), tab_d.numel(), x.err.data_ptr(), s),
                "pb_outer_nesterov",
            )  # fmt: skip
        x.barrier(SLOT_B, s)  # payloads consumed
        if eng.F > 1:  # the bf16 write-back went to the FSDP peers of THIS worker: close it like the inner step does
            eng._epoch += 1
            eng.heap.barrier(self.mesh.fsdp_ranks, eng.slot_bar, eng._epoch, s)
        self.last_bytes_on_wire = (W - 1) * (n + 4 * (n // SHARD_ALIGN))
        _count(3 + len(self._ranges))
        x.finish()

    def _step_collective(self) -> None:
        eng, h = self.engine, self.hyper
        W = self.num_workers
        pseudo = self.theta0 - eng.master
        if W > 1:
            if h.compression == "int8":
                q, sc = reference.quantize_int8_blockwise(pseudo, SHARD_ALIGN)
                qs = [torch.empty_like(q) for _ in range(W)]
                scs = [torch.empty_like(sc) for _ in range(W)]
                _all_gather(self.group, qs, q)
                _all_gather(self.group, scs, sc)
                avg = torch.zeros_like(pseudo)
                for qw, sw in zip(qs, scs):  # fixed worker order → identical result on every worker
                    avg += reference.dequantize_int8_blockwise(qw, sw, SHARD_ALIGN)
                avg /= W
                self.last_bytes_on_wire = (W - 1) * (q.numel() + 4 * sc.numel())
            else:
                avg = pseudo
                _all_reduce(self.group, avg)
                avg /= W
                self.last_bytes_on_wire = 2 * (W - 1) * 4 * avg.numel() // W
        else:
            if h.compression == "int8":
                q, sc = reference.quantize_int8_blockwise(pseudo, SHARD_ALIGN)
                avg = reference.dequantize_int8_blockwise(q, sc, SHARD_ALIGN)
            else:
                avg = pseudo
            self.last_bytes_on_wire = 0
        reference.nesterov_outer_step(self.theta0, avg, self.momentum, lr=h.lr, momentum=h.momentum, nesterov=h.nesterov)
        eng.master.copy_(self.theta0)
        eng.publish_params()

    # ------------------------------------------------------------------ state
    def state_dict(self) -> dict:
        return {"theta0": self.theta0, "momentum": self.momentum, "outer_step": self.outer_step_count}

    def load_state_dict(self, sd: dict) -> None:
        self.theta0.copy_(sd["theta0"])
        self.momentum.copy_(sd["momentum"])
        self.outer_step_count = int(sd["outer_step"])
