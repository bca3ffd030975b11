"""Fused collective ⊕ GEMM kernels over the NVLink symmetric heap — the tensor-parallel building blocks.

``all_gather_gemm``      C = [A₀; A₁; …] · Bᵀ where block r of A lives on rank r. The first column tile of every remote row block
                         TMA-loads its A tiles straight out of the owner's memory into the MMA ring and, as the MMAs retire them,
                         an idle warp stores them into a local gathered copy; per-block flags then release the block's other
                         column tiles. Every remote row crosses NVLink exactly once, hidden behind the local row blocks
                         (column-parallel linear on sequence-sharded input). The gathered copy is a by-product (``self.gathered``).
``gemm_reduce_scatter``  every rank multiplies its K-shard; the GEMM epilogue TMA-reduce-adds each fp32 tile into the buffer of the
                         rank that owns those rows (row-parallel linear → sequence-sharded output).

Both are ONE kernel each (``csrc/gemm_sm90.cu``, IO = 1 / 2); the only extra launches are two flag barriers that fence the
symmetric buffers. The NCCL formulation of the same ops (``all_gather_into_tensor`` + GEMM, GEMM + ``reduce_scatter_tensor``) is
the baseline they are benchmarked against in ``tools/collective_gemm_bench.py``.
"""

from __future__ import annotations

import ctypes
from typing import Sequence

import torch

from ..ops import _lib
from ..ops.functional import _count, _stream
from .symm import SymmetricHeap


class CollectiveGemm:
    def __init__(self, heap: SymmetricHeap, ranks: Sequence[int]):
        self.heap, self.ranks = heap, list(ranks)
        self.n = len(self.ranks)
        self.idx = self.ranks.index(heap.rank)
        self.slot = heap.alloc_flags(self.n)
        self.epoch = 0
        self.lib = heap.lib
        self._gathered: dict[tuple[int, int], torch.Tensor] = {}
        self._flags = torch.zeros(4096, dtype=torch.int32, device=heap.device)  # one per 256-row block (kernel zeroes what it uses)
        self.gathered: torch.Tensor | None = None  # last all_gather_gemm's [n·M_local, K] copy (remote blocks only)

    def _barrier(self) -> None:
        self.epoch += 1
        self.heap.barrier(self.ranks, self.slot, self.epoch, _stream())
        _count()

    def _peer_array(self, t: torch.Tensor):
        arr = (ctypes.c_void_p * self.n)(*[self.heap.peer_ptr(r, t) for r in self.ranks])
        return arr

    def all_gather_gemm(self, a_sym: torch.Tensor, b: torch.Tensor, out: torch.Tensor | None = None, *, b_mn_major: bool = False,
                        gathered: torch.Tensor | None = None, copy_local: bool = False) -> torch.Tensor:  # fmt: skip
        """``a_sym``: this rank's [M_local, K] bf16 block, allocated with ``heap.alloc`` at the SAME offset on every rank
        (M_local % 256 == 0); ``b``: [N, K] bf16 (local), or stored [K, N] with ``b_mn_major``. Returns C [n·M_local, N] bf16.

        ``gathered``: caller-owned [n·M_local, K] buffer for the by-product (kept for a backward pass); with ``copy_local`` the
        local block is copied in as well, so it ends up holding the complete gathered A."""
        M_local, K = a_sym.shape
        N = b.shape[1] if b_mn_major else b.shape[0]
        assert a_sym.dtype == torch.bfloat16 and b.dtype == torch.bfloat16 and b.shape[0 if b_mn_major else 1] == K and M_local % 256 == 0
        assert a_sym.is_contiguous() and b.stride(1) == 1
        if out is None:
            out = torch.empty((self.n * M_local, N), dtype=torch.bfloat16, device=a_sym.device)
        assert self.n * M_local // 256 <= self._flags.numel()
        full = gathered
        if full is None:
            full = self._gathered.get((M_local, K))
            if full is None:
                full = self._gathered[(M_local, K)] = torch.empty((self.n * M_local, K), dtype=torch.bfloat16, device=a_sym.device)
        assert full.shape == (self.n * M_local, K) and full.is_contiguous() and full.dtype == torch.bfloat16
        self.gathered = full
        self._barrier()  # every rank's block is written
        rc = self.lib.pb_gemm_allgather(self._peer_array(a_sym), self.n, self.idx, b.data_ptr(), out.data_ptr(), full.data_ptr(),
                                        self._flags.data_ptr(), M_local, N, K, a_sym.stride(0), b.stride(0), out.stride(0),
                                        int(b_mn_major), _stream())  # fmt: skip
        _lib.check(rc, "pb_gemm_allgather")
        _count()
        if copy_local:
            full[self.idx * M_local : (self.idx + 1) * M_local].copy_(a_sym)
        self._barrier()  # nobody may overwrite its block while a peer is still reading it
        return out

    def gemm_reduce_scatter(self, a: torch.Tensor, b: torch.Tensor, out_sym: torch.Tensor, *, b_mn_major: bool = False) -> torch.Tensor:
        """``a``: [M, K_local], ``b``: [N, K_local] (or stored [K_local, N] with ``b_mn_major``) — this rank's K shard, local memory;
        ``out_sym``: this rank's [M/n, N] fp32 buffer from ``heap.alloc`` (same offset everywhere). On return it holds rows
        [idx·M/n, (idx+1)·M/n) of Σ_ranks a·bᵀ."""
        M, K = a.shape
        N = b.shape[1] if b_mn_major else b.shape[0]
        assert b.shape[0 if b_mn_major else 1] == K and a.stride(1) == 1 and b.stride(1) == 1
        assert out_sym.dtype == torch.float32 and out_sym.shape == (M // self.n, N) and (M // self.n) % 256 == 0
        out_sym.zero_()
        self._barrier()  # all output buffers are zeroed
        rc = self.lib.pb_gemm_reduce_scatter(a.data_ptr(), b.data_ptr(), self._peer_array(out_sym), self.n, self.idx, M, N, K,
                                             a.stride(0), b.stride(0), out_sym.stride(0), int(b_mn_major), _stream())  # fmt: skip
        _lib.check(rc, "pb_gemm_reduce_scatter")
        _count()
        self._barrier()  # every rank's contributions have landed (TMA reduce completes before the kernel retires)
        return out_sym
