"""Flash attention on sm_90a over the fused QKV activation (mma.sync QKᵀ / P·V tiles, registers as accumulators).

Forward : ``csrc/attention_sm90.cu``      qkv [B,S,(H+2Hkv)·D] → out [B,S,H·D], lse2 [B,H,S]
Backward: ``csrc/attention_sm90.cu``    → dqkv [B,S,(H+2Hkv)·D]  (dK/dV kernel + dQ kernel + delta preprocess)

No transposes, slices or concatenations ever touch HBM: the kernels address Q/K/V heads inside the fused buffer
through one TMA tensor map and write gradients straight back in the same layout.
"""

from __future__ import annotations

import math

import torch

from . import _lib
from .functional import _count, _ptr, _stream


def supported_shape(S: int, D: int, H: int, Hkv: int) -> bool:
    return D in (64, 128) and S % 128 == 0 and H % Hkv == 0


def supported(qkv: torch.Tensor, n_heads: int, n_kv_heads: int) -> bool:
    try:
        lib = _lib.load()
    except Exception:
        return False
    if getattr(lib, "pb_flash_attn_fwd", None) is None:
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


def _fwd(lib, qkv: torch.Tensor, n_heads: int, n_kv_heads: int, causal: bool, doc) -> tuple[torch.Tensor, torch.Tensor, int, float]:
    B, S, W = qkv.shape
    D = W // (n_heads + 2 * n_kv_heads)
    out = torch.empty((B, S, n_heads * D), dtype=qkv.dtype, device=qkv.device)
    lse2 = torch.empty((B, n_heads, S), dtype=torch.float32, device=qkv.device)
    scale = 1.0 / math.sqrt(D)
    if doc is None:
        rc = lib.pb_flash_attn_fwd(_ptr(qkv), _ptr(out), _ptr(lse2), B, S, n_heads, n_kv_heads, D, scale, int(causal), _stream())
        _lib.check(rc, "pb_flash_attn_fwd")
    else:
        rc = lib.pb_flash_attn_fwd_doc(_ptr(qkv), _ptr(out), _ptr(lse2), _ptr(doc[0]), B, S, n_heads, n_kv_heads, D, scale, _stream())
        _lib.check(rc, "pb_flash_attn_fwd_doc")
    _count()
    return out, lse2, D, scale


def _bwd_doc(lib, qkv, out, dout, lse2, delta, dqkv, doc_start, doc_end, n_heads, n_kv_heads, D, scale, cos=None, sin=None) -> None:
    B, S, _ = qkv.shape
    rc = lib.pb_flash_attn_bwd_doc(_ptr(qkv), _ptr(out), _ptr(dout), _ptr(lse2), _ptr(delta), _ptr(dqkv), _ptr(doc_start), _ptr(doc_end),
                                   B, S, n_heads, n_kv_heads, D, scale, _ptr(cos), _ptr(sin), _stream())  # fmt: skip
    _lib.check(rc, "pb_flash_attn_bwd_doc")


class _FlashAttnQKVFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, qkv: torch.Tensor, n_heads: int, n_kv_heads: int, causal: bool, doc_start=None, doc_end=None):
        lib = _lib.load()
        doc = None if doc_start is None else (doc_start, doc_end)
        out, lse2, D, scale = _fwd(lib, qkv, n_heads, n_kv_heads, causal, doc)
        ctx.save_for_backward(qkv, out, lse2, *(doc or ()))
        ctx.meta = (n_heads, n_kv_heads, D, scale, causal)
        return out

    @staticmethod
    def backward(ctx, dout: torch.Tensor):
        lib = _lib.load()
        qkv, out, lse2, *doc = ctx.saved_tensors
        n_heads, n_kv_heads, D, scale, causal = ctx.meta
        B, S, _ = qkv.shape
        dout = dout if dout.is_contiguous() else dout.contiguous()
        dqkv = torch.empty_like(qkv)
        delta = torch.empty_like(lse2)
        if doc:
            _bwd_doc(lib, qkv, out, dout, lse2, delta, dqkv, doc[0], doc[1], n_heads, n_kv_heads, D, scale)
        else:
            rc = lib.pb_flash_attn_bwd(_ptr(qkv), _ptr(out), _ptr(dout), _ptr(lse2), _ptr(delta), _ptr(dqkv), B, S, n_heads,
                                       n_kv_heads, D, scale, int(causal), _stream())  # fmt: skip
            _lib.check(rc, "pb_flash_attn_bwd")
        _count(3)
        return dqkv, None, None, None, None, None


def flash_attention_qkv(qkv: torch.Tensor, n_heads: int, n_kv_heads: int, causal: bool = True, doc: tuple | None = None) -> torch.Tensor:
    """``doc=(doc_start, doc_end)`` (int32 [B, S], :func:`prime_b200.ops.document_bounds`): document-masked causal attention."""
    if doc is None:
        return _FlashAttnQKVFn.apply(qkv, n_heads, n_kv_heads, causal)
    _check_doc(doc, qkv, causal)
    return _FlashAttnQKVFn.apply(qkv, n_heads, n_kv_heads, causal, doc[0], doc[1])


def _rope_inplace(lib, t: torch.Tensor, cos, sin, n_heads: int, n_kv_heads: int, D: int, sign: float) -> None:
    tokens = t.numel() // t.shape[-1]
    rc = lib.pb_rope_inplace(_ptr(t), _ptr(cos), _ptr(sin), tokens, t.shape[1], n_heads + n_kv_heads, n_heads + 2 * n_kv_heads, D,
                             sign, _stream())  # fmt: skip
    _lib.check(rc, "pb_rope_inplace")
    _count()


class _RopeFlashAttnFn(torch.autograd.Function):
    """RoPE ⊕ attention as ONE autograd node: forward rotates in place on the QKV GEMM output (nobody else reads the un-rotated
    activation); backward folds the inverse rotation into the dQ / dK epilogues of the attention-backward kernels, so there is
    neither a copy of the 200 MB gradient (a stand-alone RoPE node may not mutate a gradient it does not own) nor a separate
    rotation pass over it."""

    @staticmethod
    def forward(ctx, qkv: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, n_heads: int, n_kv_heads: int, causal: bool,
                pre_rotated: bool = False, doc_start=None, doc_end=None):  # fmt: skip
        lib = _lib.load()
        B, S, W = qkv.shape
        D = W // (n_heads + 2 * n_kv_heads)
        if not pre_rotated:  # otherwise the QKV GEMM epilogue already did it
            _rope_inplace(lib, qkv, cos, sin, n_heads, n_kv_heads, D, 1.0)
        doc = None if doc_start is None else (doc_start, doc_end)
        out, lse2, D, scale = _fwd(lib, qkv, n_heads, n_kv_heads, causal, doc)
        ctx.save_for_backward(qkv, out, lse2, cos, sin, *(doc or ()))
        ctx.meta = (n_heads, n_kv_heads, D, scale, causal)
        return out

    @staticmethod
    def backward(ctx, dout: torch.Tensor):
        lib = _lib.load()
        qkv, out, lse2, cos, sin, *doc = ctx.saved_tensors
        n_heads, n_kv_heads, D, scale, causal = ctx.meta
        B, S, _ = qkv.shape
        dout = dout if dout.is_contiguous() else dout.contiguous()
        dqkv = torch.empty_like(qkv)
        delta = torch.empty_like(lse2)
        # rotation is orthogonal: its backward is the inverse rotation, applied to dQ / dK inside the attention-backward epilogues
        # (registers → smem → TMA store), so dQKV is written exactly once
        assert cos.dtype == torch.float32 and cos.is_contiguous() and sin.is_contiguous() and cos.shape[1] == D // 2 and cos.shape[0] >= S
        if doc:
            _bwd_doc(lib, qkv, out, dout, lse2, delta, dqkv, doc[0], doc[1], n_heads, n_kv_heads, D, scale, cos, sin)
        else:
            rc = lib.pb_flash_attn_bwd_rope(_ptr(qkv), _ptr(out), _ptr(dout), _ptr(lse2), _ptr(delta), _ptr(dqkv), B, S, n_heads,
                                            n_kv_heads, D, scale, int(causal), _ptr(cos), _ptr(sin), _stream())  # fmt: skip
            _lib.check(rc, "pb_flash_attn_bwd_rope")
        _count(3)
        return dqkv, None, None, None, None, None, None, None, None


def rope_flash_attention_qkv(qkv: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, n_heads: int, n_kv_heads: int,
                             causal: bool = True, pre_rotated: bool = False, doc: tuple | None = None) -> torch.Tensor:  # fmt: skip
    if doc is None:
        return _RopeFlashAttnFn.apply(qkv, cos, sin, n_heads, n_kv_heads, causal, pre_rotated)
    _check_doc(doc, qkv, causal)
    return _RopeFlashAttnFn.apply(qkv, cos, sin, n_heads, n_kv_heads, causal, pre_rotated, doc[0], doc[1])


def document_bounds(tokens: torch.Tensor, eos_id: int) -> tuple[torch.Tensor, torch.Tensor]:
    """Native ``pb_doc_bounds``: int64 [B, S] CUDA tokens → (doc_start, doc_end) int32 [B, S]."""
    B, S = tokens.shape
    t = tokens if tokens.is_contiguous() else tokens.contiguous()
    assert t.dtype == torch.int64
    doc_start = torch.empty((B, S), dtype=torch.int32, device=t.device)
    doc_end = torch.empty((B, S), dtype=torch.int32, device=t.device)
    _lib.check(_lib.load().pb_doc_bounds(_ptr(t), B, S, int(eos_id), _ptr(doc_start), _ptr(doc_end), _stream()), "pb_doc_bounds")
    _count()
    return doc_start, doc_end
