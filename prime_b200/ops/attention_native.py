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


class _FlashAttnQKVFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, qkv: torch.Tensor, n_heads: int, n_kv_heads: int, causal: bool):
        lib = _lib.load()
        B, S, W = qkv.shape
        D = W // (n_heads + 2 * n_kv_heads)
        out = torch.empty((B, S, n_heads * D), dtype=qkv.dtype, device=qkv.device)
        lse2 = torch.empty((B, n_heads, S), dtype=torch.float32, device=qkv.device)
        scale = 1.0 / math.sqrt(D)
        rc = lib.pb_flash_attn_fwd(_ptr(qkv), _ptr(out), _ptr(lse2), B, S, n_heads, n_kv_heads, D, scale, int(causal), _stream())
        _lib.check(rc, "pb_flash_attn_fwd")
        _count()
        ctx.save_for_backward(qkv, out, lse2)
        ctx.meta = (n_heads, n_kv_heads, D, scale, causal)
        return out

    @staticmethod
    def backward(ctx, dout: torch.Tensor):
        lib = _lib.load()
        qkv, out, lse2 = ctx.saved_tensors
        n_heads, n_kv_heads, D, scale, causal = ctx.meta
        B, S, _ = qkv.shape
        dout = dout if dout.is_contiguous() else dout.contiguous()
        dqkv = torch.empty_like(qkv)
        delta = torch.empty_like(lse2)
        rc = lib.pb_flash_attn_bwd(_ptr(qkv), _ptr(out), _ptr(dout), _ptr(lse2), _ptr(delta), _ptr(dqkv), B, S, n_heads,
                                   n_kv_heads, D, scale, int(causal), _stream())  # fmt: skip
        _lib.check(rc, "pb_flash_attn_bwd")
        _count(3)
        return dqkv, None, None, None


def flash_attention_qkv(qkv: torch.Tensor, n_heads: int, n_kv_heads: int, causal: bool = True) -> torch.Tensor:
    return _FlashAttnQKVFn.apply(qkv, n_heads, n_kv_heads, causal)


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
                pre_rotated: bool = False):  # fmt: skip
        lib = _lib.load()
        B, S, W = qkv.shape
        D = W // (n_heads + 2 * n_kv_heads)
        if not pre_rotated:  # otherwise the QKV GEMM epilogue already did it
            _rope_inplace(lib, qkv, cos, sin, n_heads, n_kv_heads, D, 1.0)
        out = torch.empty((B, S, n_heads * D), dtype=qkv.dtype, device=qkv.device)
        lse2 = torch.empty((B, n_heads, S), dtype=torch.float32, device=qkv.device)
        scale = 1.0 / math.sqrt(D)
        rc = lib.pb_flash_attn_fwd(_ptr(qkv), _ptr(out), _ptr(lse2), B, S, n_heads, n_kv_heads, D, scale, int(causal), _stream())
        _lib.check(rc, "pb_flash_attn_fwd")
        _count()
        ctx.save_for_backward(qkv, out, lse2, cos, sin)
        ctx.meta = (n_heads, n_kv_heads, D, scale, causal)
        return out

    @staticmethod
    def backward(ctx, dout: torch.Tensor):
        lib = _lib.load()
        qkv, out, lse2, cos, sin = ctx.saved_tensors
        n_heads, n_kv_heads, D, scale, causal = ctx.meta
        B, S, _ = qkv.shape
        dout = dout if dout.is_contiguous() else dout.contiguous()
        dqkv = torch.empty_like(qkv)
        delta = torch.empty_like(lse2)
        # rotation is orthogonal: its backward is the inverse rotation, applied to dQ / dK inside the attention-backward epilogues
        # (registers → smem → TMA store), so dQKV is written exactly once
        assert cos.dtype == torch.float32 and cos.is_contiguous() and sin.is_contiguous() and cos.shape[1] == D // 2 and cos.shape[0] >= S
        rc = lib.pb_flash_attn_bwd_rope(_ptr(qkv), _ptr(out), _ptr(dout), _ptr(lse2), _ptr(delta), _ptr(dqkv), B, S, n_heads,
                                        n_kv_heads, D, scale, int(causal), _ptr(cos), _ptr(sin), _stream())  # fmt: skip
        _lib.check(rc, "pb_flash_attn_bwd_rope")
        _count(3)
        return dqkv, None, None, None, None, None, None


def rope_flash_attention_qkv(qkv: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, n_heads: int, n_kv_heads: int,
                             causal: bool = True, pre_rotated: bool = False) -> torch.Tensor:  # fmt: skip
    return _RopeFlashAttnFn.apply(qkv, cos, sin, n_heads, n_kv_heads, causal, pre_rotated)
