"""Flash attention on sm_90a over the fused QKV activation (mma.sync QKᵀ / P·V tiles, registers as accumulators).

Forward : ``csrc/attention_sm90.cu``      qkv [B,S,(H+2Hkv)·D] → out [B,S,H·D], lse2 [B,H,S]
Backward: ``csrc/attention_sm90.cu``    → dqkv [B,S,(H+2Hkv)·D]  (dK/dV kernel + dQ kernel + delta preprocess)

No transposes, slices or concatenations ever touch HBM: the kernels load Q/K/V head tiles straight from the fused buffer
with cp.async and write gradients from registers straight back in the same layout.
"""

from __future__ import annotations

import math

import torch

from . import _lib
from .functional import _launch, _ptr, _rope_inplace, _stream


def supported_shape(S: int, D: int, H: int, Hkv: int) -> bool:
    return D in (64, 128) and S % 128 == 0 and H % Hkv == 0


def supported(qkv: torch.Tensor, n_heads: int, n_kv_heads: int) -> bool:
    try:
        _lib.load()
    except Exception:
        return False
    D = qkv.shape[-1] // (n_heads + 2 * n_kv_heads)
    return qkv.dtype == torch.bfloat16 and qkv.is_contiguous() and supported_shape(qkv.shape[1], D, n_heads, n_kv_heads)


def _check_doc(doc, qkv: torch.Tensor, causal: bool) -> None:
    if not causal:
        raise ValueError("document masking implies causal attention: causal=False with doc=(doc_start, doc_end) is not supported")
    B, S = qkv.shape[:2]
    for t in doc:
        if t.dtype != torch.int32 or tuple(t.shape) != (B, S) or not t.is_contiguous() or t.device != qkv.device:
            raise ValueError(f"doc bounds must be contiguous int32 [{B}, {S}] tensors on {qkv.device} (ops.document_bounds)")


class _FlashAttnFn(torch.autograd.Function):
    """Attention over the fused QKV activation as ONE autograd node, optionally with RoPE on the Q/K heads (``cos`` / ``sin`` not
    None). The forward rotates in place on the QKV GEMM output (nobody else reads the un-rotated activation) unless the producer
    already did (``pre_rotated``); the backward folds the inverse rotation into the dQ / dK epilogues of the attention-backward
    kernels, so there is neither a copy of the 200 MB gradient (a stand-alone RoPE node may not mutate a gradient it does not own)
    nor a separate rotation pass over it. ``doc_start`` / ``doc_end``: document masking (both or neither)."""

    @staticmethod
    def forward(ctx, qkv: torch.Tensor, n_heads: int, n_kv_heads: int, causal: bool, cos=None, sin=None, pre_rotated: bool = False,
                doc_start=None, doc_end=None):  # fmt: skip
        B, S, W = qkv.shape
        D = W // (n_heads + 2 * n_kv_heads)
        if cos is not None and not pre_rotated:
            _rope_inplace(qkv, cos, sin, n_heads, n_kv_heads, 1.0)
        out = torch.empty((B, S, n_heads * D), dtype=qkv.dtype, device=qkv.device)
        lse2 = torch.empty((B, n_heads, S), dtype=torch.float32, device=qkv.device)
        scale = 1.0 / math.sqrt(D)
        _launch("pb_flash_attn_fwd", _ptr(qkv), _ptr(out), _ptr(lse2), _ptr(doc_start), B, S, n_heads, n_kv_heads, D, scale, int(causal),
                _stream())  # fmt: skip
        ctx.save_for_backward(qkv, out, lse2, cos, sin, doc_start, doc_end)
        ctx.meta = (n_heads, n_kv_heads, D, scale, causal)
        return out

    @staticmethod
    def backward(ctx, dout: torch.Tensor):
        qkv, out, lse2, cos, sin, doc_start, doc_end = ctx.saved_tensors
        n_heads, n_kv_heads, D, scale, causal = ctx.meta
        B, S, _ = qkv.shape
        dout = dout if dout.is_contiguous() else dout.contiguous()
        dqkv = torch.empty_like(qkv)
        delta = torch.empty_like(lse2)
        if cos is not None:
            # rotation is orthogonal: its backward is the inverse rotation, applied to dQ / dK inside the attention-backward epilogues
            # (in registers, before the 4-byte stores), so dQKV is written exactly once
            assert cos.dtype == torch.float32 and cos.is_contiguous() and sin.is_contiguous() and cos.shape[1] == D // 2 and cos.shape[0] >= S
        _launch("pb_flash_attn_bwd", _ptr(qkv), _ptr(out), _ptr(dout), _ptr(lse2), _ptr(delta), _ptr(dqkv), _ptr(doc_start), _ptr(doc_end),
                B, S, n_heads, n_kv_heads, D, scale, int(causal), _ptr(cos), _ptr(sin), _stream(), n=3)  # fmt: skip
        return dqkv, None, None, None, None, None, None, None, None


def flash_attention_qkv(qkv: torch.Tensor, n_heads: int, n_kv_heads: int, causal: bool = True, doc: tuple | None = None) -> torch.Tensor:
    """``doc=(doc_start, doc_end)`` (int32 [B, S], :func:`prime_b200.ops.document_bounds`): document-masked causal attention."""
    return rope_flash_attention_qkv(qkv, None, None, n_heads, n_kv_heads, causal, doc=doc)


def rope_flash_attention_qkv(qkv: torch.Tensor, cos: torch.Tensor | None, sin: torch.Tensor | None, n_heads: int, n_kv_heads: int,
                             causal: bool = True, pre_rotated: bool = False, doc: tuple | None = None) -> torch.Tensor:  # fmt: skip
    """RoPE (``cos`` / ``sin`` fp32 [S, D/2] tables; None = no rotation) ⊕ attention, see :class:`_FlashAttnFn`."""
    if doc is not None:
        _check_doc(doc, qkv, causal)
    return _FlashAttnFn.apply(qkv, n_heads, n_kv_heads, causal, cos, sin, pre_rotated, *(doc or (None, None)))


def document_bounds(tokens: torch.Tensor, eos_id: int | None, window: int | None = None) -> tuple[torch.Tensor, torch.Tensor]:
    """Native ``pb_doc_bounds``: int64 [B, S] CUDA tokens → (doc_start, doc_end) int32 [B, S]. ``eos_id`` None = no documents
    (passed as -1, which no token id equals), ``window`` None = no window (passed as 0)."""
    B, S = tokens.shape
    t = tokens if tokens.is_contiguous() else tokens.contiguous()
    assert t.dtype == torch.int64
    doc_start = torch.empty((B, S), dtype=torch.int32, device=t.device)
    doc_end = torch.empty((B, S), dtype=torch.int32, device=t.device)
    eos = -1 if eos_id is None else int(eos_id)
    _launch("pb_doc_bounds", _ptr(t), B, S, eos, int(window or 0), _ptr(doc_start), _ptr(doc_end), _stream())
    return doc_start, doc_end
