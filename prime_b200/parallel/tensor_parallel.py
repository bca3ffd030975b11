"""Sequence-parallel tensor parallelism for the Llama MLP on the fused collective GEMMs (``collective_gemm.py``).

Activations are sharded over the sequence (rank r holds tokens [r·T/n, (r+1)·T/n)), weights over the hidden dimension:
``w13`` column-parallel (rank r holds the gate and up rows of its FF/n features), ``w2`` row-parallel. Per MLP, forward and
backward, the only cross-GPU traffic is inside four GEMM kernels:

    forward    gate_up = all_gather(x) · W13ᵀ        all-gather ⊕ GEMM   (keeps the gathered x for dW13)
               y_local = reduce_scatter(h · W2ᵀ)     GEMM ⊕ reduce-scatter
    backward   dh      = all_gather(dy) · W2         all-gather ⊕ GEMM   (keeps the gathered dy for dW2)
               dx_local= reduce_scatter(dgu · W13)   GEMM ⊕ reduce-scatter
               dW2 += dy_fullᵀ · h,  dW13 += dguᵀ · x_full                local wgmma GEMMs (fp32 accumulate into main_grad)

The reference has no parallel-training code at all (SURVEY.md §2.4: every strategy ABSENT); this module exists because the
engine wants compute ⊕ collective kernels wherever a GEMM neighbours a collective.
"""

from __future__ import annotations

import torch

from .. import ops
from .collective_gemm import CollectiveGemm
from .symm import SymmetricHeap


class _SPMlpFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x_local: torch.Tensor, w13: torch.Tensor, w2: torch.Tensor, mod: "SequenceParallelMLP") -> torch.Tensor:
        cg, n = mod.cg, mod.cg.n
        t_local, d = x_local.shape
        mod.x_sym.copy_(x_local)
        x_full = torch.empty((n * t_local, d), dtype=torch.bfloat16, device=x_local.device)
        gate_up = cg.all_gather_gemm(mod.x_sym, w13, gathered=x_full, copy_local=True)  # [T, 2·FF/n]
        h = ops.swiglu(gate_up)                                                           # [T, FF/n]
        cg.gemm_reduce_scatter(h, w2, mod.y_sym)                                          # fp32 [T/n, D]
        ctx.save_for_backward(x_full, gate_up, h, w13, w2)
        ctx.mod = mod
        return mod.y_sym.to(torch.bfloat16)

    @staticmethod
    def backward(ctx, dy_local: torch.Tensor):
        x_full, gate_up, h, w13, w2 = ctx.saved_tensors
        mod = ctx.mod
        cg, n = mod.cg, mod.cg.n
        t_local, d = dy_local.shape
        mod.x_sym.copy_(dy_local)  # the forward's input slot is free again: reuse it for dy
        dy_full = torch.empty((n * t_local, d), dtype=torch.bfloat16, device=dy_local.device)
        dh = cg.all_gather_gemm(mod.x_sym, w2, b_mn_major=True, gathered=dy_full, copy_local=True)  # [T, FF/n] = dy_full · W2
        # dW2[D, FF/n] += dy_fullᵀ · h
        dw2 = _wgrad(dy_full, h, w2)
        dgu = _swiglu_bwd(gate_up, dh)
        # dW13[2FF/n, D] += dguᵀ · x_full
        dw13 = _wgrad(dgu, x_full, w13)
        cg.gemm_reduce_scatter(dgu, w13, mod.y_sym, b_mn_major=True)  # dx_local = RS(dgu · W13)
        return mod.y_sym.to(torch.bfloat16), dw13, dw2, None


def _wgrad(dy: torch.Tensor, x: torch.Tensor, weight: torch.Tensor) -> torch.Tensor | None:
    main_grad = getattr(weight, "main_grad", None)
    if main_grad is not None:
        ops.gemm(dy, x, a_mn_major=True, b_mn_major=True, out=main_grad, accumulate=True)
        return None
    return ops.gemm(dy, x, a_mn_major=True, b_mn_major=True)


def _swiglu_bwd(gate_up: torch.Tensor, dh: torch.Tensor) -> torch.Tensor:
    # reuse the fused backward kernel through autograd on a detached leaf (one kernel launch, no graph kept)
    gu = gate_up.detach().requires_grad_(True)
    with torch.enable_grad():
        out = ops.swiglu(gu)
    (dgu,) = torch.autograd.grad(out, gu, dh)
    return dgu


class SequenceParallelMLP(torch.nn.Module):
    """SwiGLU MLP with sequence-sharded activations and hidden-sharded weights over ``ranks`` of one NVSwitch box.

    ``w13_shard``: [2·FF/n, D] = [gate rows of this rank's features | up rows], ``w2_shard``: [D, FF/n]. ``forward(x_local)`` takes
    and returns [T/n, D] bf16 (T/n a multiple of 256). Buffers in the symmetric heap are allocated once for ``max_tokens_local``.
    """

    def __init__(self, heap: SymmetricHeap, ranks, dim: int, ffn_hidden: int, max_tokens_local: int, *, device=None):
        super().__init__()
        self.cg = CollectiveGemm(heap, ranks)
        n = self.cg.n
        assert ffn_hidden % n == 0 and max_tokens_local % 256 == 0
        self.dim, self.ff_local = dim, ffn_hidden // n
        dev = device or heap.device
        self.w13 = torch.nn.Parameter(torch.empty(2 * self.ff_local, dim, dtype=torch.bfloat16, device=dev))
        self.w2 = torch.nn.Parameter(torch.empty(dim, self.ff_local, dtype=torch.bfloat16, device=dev))
        self.x_sym = heap.alloc(max_tokens_local * dim, torch.bfloat16).view(max_tokens_local, dim)
        self.y_sym = heap.alloc(max_tokens_local * dim, torch.float32).view(max_tokens_local, dim)

    @torch.no_grad()
    def load_full_weights(self, w13_full: torch.Tensor, w2_full: torch.Tensor) -> None:
        """Shard an unsharded MLP: ``w13_full`` [2·FF, D] = [gate | up], ``w2_full`` [D, FF]."""
        n, r, f = self.cg.n, self.cg.idx, self.ff_local
        ff = f * n
        self.w13[:f].copy_(w13_full[r * f : (r + 1) * f])
        self.w13[f:].copy_(w13_full[ff + r * f : ff + (r + 1) * f])
        self.w2.copy_(w2_full[:, r * f : (r + 1) * f])

    def forward(self, x_local: torch.Tensor) -> torch.Tensor:
        assert x_local.shape == self.x_sym.shape, "token count is fixed by max_tokens_local (symmetric buffers)"
        return _SPMlpFn.apply(x_local.contiguous(), self.w13, self.w2, self)
