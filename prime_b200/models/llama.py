"""Llama-2/3 family on prime_b200 ops.

Hopper-first choices:
  * fused ``wqkv`` ([H+2Hkv]·D × dim) and ``w13`` (2·hidden × dim) parameters → one wgmma GEMM each;
  * RoPE applied in place on the fused QKV activation; attention reads strided Q/K/V views of it;
  * the residual add is fused into the following RMSNorm (``add_rmsnorm``): a block returns
    ``(residual_stream, pending_delta)`` so no stand-alone elementwise add ever touches HBM;
  * cross-entropy is fused forward+backward and overwrites the logits with their gradient.

Sizes follow the DiLoCo engine's model zoo named in BASELINE.json (150M / 1B / 7B …).
``to_reference_state_dict`` / ``from_reference_state_dict`` convert to the split
``attention.wq/wk/wv``, ``feed_forward.w1/w3`` naming for checkpoint interchange.
"""

from __future__ import annotations

import math
from dataclasses import dataclass, replace

import torch
import torch.nn as nn

from .. import ops


@dataclass(frozen=True)
class ModelArgs:
    dim: int = 4096
    n_layers: int = 32
    n_heads: int = 32
    n_kv_heads: int | None = None
    vocab_size: int = 32000
    multiple_of: int = 256
    ffn_dim_multiplier: float | None = None
    norm_eps: float = 1e-5
    rope_theta: float = 10000.0
    max_seq_len: int = 2048
    depth_init: bool = True
    intermediate_size: int | None = None  # explicit FFN width (imported checkpoints); None = derived from dim / multiple_of
    # sliding-window attention in every layer (Mistral): query q attends only keys q - W + 1 .. q. None = full causal attention
    sliding_window: int | None = None

    @property
    def head_dim(self) -> int:
        return self.dim // self.n_heads

    @property
    def kv_heads(self) -> int:
        return self.n_kv_heads or self.n_heads

    @property
    def ffn_hidden(self) -> int:
        if self.intermediate_size is not None:
            return self.intermediate_size
        hidden = int(2 * (4 * self.dim) / 3)
        if self.ffn_dim_multiplier is not None:
            hidden = int(self.ffn_dim_multiplier * hidden)
        return self.multiple_of * ((hidden + self.multiple_of - 1) // self.multiple_of)


LLAMA2_CONFIGS: dict[str, ModelArgs] = {
    "debugmodel": ModelArgs(dim=256, n_layers=2, n_heads=8, vocab_size=2048),
    "10M": ModelArgs(dim=64, n_layers=5, n_heads=4),
    "150M": ModelArgs(dim=1024, n_layers=12, n_heads=16),
    "271M": ModelArgs(dim=1024, n_layers=16, n_heads=8),
    "1B": ModelArgs(dim=2048, n_layers=18, n_heads=16),
    "7B": ModelArgs(dim=4096, n_layers=32, n_heads=32),
    "10B": ModelArgs(dim=5120, n_layers=32, n_heads=40),
    "13B": ModelArgs(dim=5120, n_layers=40, n_heads=40),
    "26B": ModelArgs(dim=5120, n_layers=80, n_heads=40),
    "70B": ModelArgs(dim=8192, n_layers=80, n_heads=64, n_kv_heads=8, ffn_dim_multiplier=1.3, multiple_of=4096),
}

LLAMA3_CONFIGS: dict[str, ModelArgs] = {
    "debugmodel": ModelArgs(dim=256, n_layers=2, n_heads=8, vocab_size=2048, rope_theta=500000),
    "10M": ModelArgs(dim=64, n_layers=5, n_heads=4, vocab_size=128256, rope_theta=500000),
    "150M": ModelArgs(dim=1024, n_layers=12, n_heads=16, vocab_size=128256, rope_theta=500000),
    "1B": ModelArgs(dim=2048, n_layers=18, n_heads=16, vocab_size=128256, rope_theta=500000),
    "7B": ModelArgs(dim=4096, n_layers=32, n_heads=32, n_kv_heads=8, ffn_dim_multiplier=1.3, multiple_of=1024,
                    vocab_size=128256, rope_theta=500000),  # fmt: skip
    "10B": ModelArgs(dim=4096, n_layers=42, n_heads=32, n_kv_heads=8, ffn_dim_multiplier=1.3, multiple_of=1024,
                     vocab_size=128256, rope_theta=500000),  # fmt: skip
    "70B": ModelArgs(dim=8192, n_layers=80, n_heads=64, n_kv_heads=8, ffn_dim_multiplier=1.3, multiple_of=4096,
                     vocab_size=128256, rope_theta=500000),  # fmt: skip
}


def get_model_args(name: str, type_model: str = "llama2", **overrides) -> ModelArgs:
    table = LLAMA2_CONFIGS if type_model == "llama2" else LLAMA3_CONFIGS
    if name not in table:
        raise KeyError(f"unknown {type_model} size {name!r}; have {sorted(table)}")
    return replace(table[name], **overrides)


class RMSNormWeight(nn.Module):
    def __init__(self, dim: int):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(dim))


class Attention(nn.Module):
    def __init__(self, args: ModelArgs):
        super().__init__()
        self.n_heads, self.n_kv_heads, self.head_dim = args.n_heads, args.kv_heads, args.head_dim
        qkv_out = (self.n_heads + 2 * self.n_kv_heads) * self.head_dim
        self.wqkv = nn.Parameter(torch.empty(qkv_out, args.dim))
        self.wo = nn.Parameter(torch.empty(args.dim, self.n_heads * self.head_dim))
        self.fp8 = False  # train.fp8: MXFP8 forward / input-gradient GEMMs (Transformer.set_fp8)

    def forward(self, x: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, attn_impl: str = "auto", doc: tuple | None = None,
                kv=None) -> torch.Tensor:  # fmt: skip
        """``doc``: (doc_start, doc_end) of ``ops.document_bounds`` for document-masked and / or sliding-window attention, None =
        plain causal. ``kv``: this layer's handle of an ``inference.KVCache``, None outside generation. When prefilling, the rotated
        K|V columns of every position are also copied into the cache; when decoding, ``x`` is [B, 1, dim], the new token is appended
        to the cache and attends over it; when verifying, ``x`` is [B, T, dim], the T tokens are appended and each attends over the
        cache up to itself, within its document (``cache.lo_q``) and window."""
        B, S, _ = x.shape
        H, Hkv, D = self.n_heads, self.n_kv_heads, self.head_dim
        if kv is not None and kv.verifying:
            qkv = ops.linear(x, self.wqkv)  # M = B·T
            ops.kv_append_tokens(qkv, kv.kv, kv.cache.len, cos, sin, H, Hkv, kv_scale=kv.kv_scale)
            out = ops.verify_attention(qkv, kv.kv, kv.cache.len, kv.cache.lo_q, kv.cache.window, H, Hkv, kv_scale=kv.kv_scale)
            return ops.linear(out, self.wo)
        if kv is not None and kv.decoding:
            qkv = ops.linear(x, self.wqkv).view(B, -1)  # M = B: the new token of every row
            ops.kv_append(qkv, kv.kv, kv.cache.len, cos, sin, H, Hkv, kv_scale=kv.kv_scale)
            out = ops.decode_attention(qkv, kv.kv, kv.cache.len, kv.cache.lo, kv.cache.window, H, Hkv, kv_scale=kv.kv_scale)
            return ops.linear(out.view(B, 1, H * D), self.wo)
        if self.fp8:
            qkv = ops.linear_mxfp8(x, self.wqkv)
            out = self._prefill_attention(qkv, cos, sin, attn_impl, doc, kv)
            return ops.linear_mxfp8(out, self.wo)
        if attn_impl in ("auto", "native") and ops.rope_fusable(x, H, Hkv, D):
            # RoPE rides in the QKV GEMM epilogue (forward) and in the dQ/dK epilogues of the attention backward: no rotation pass
            qkv = ops.linear_qkv_rope(x, self.wqkv, cos, sin, H, Hkv)  # [B, S, (H+2Hkv)·D], Q/K heads rotated
            if kv is not None:
                kv.store(qkv, H * D)
            out = ops.rope_attention_qkv(qkv, cos, sin, H, Hkv, causal=True, impl=attn_impl, pre_rotated=True, doc=doc)
        else:
            qkv = ops.linear(x, self.wqkv)  # [B, S, (H+2Hkv)·D]
            out = self._prefill_attention(qkv, cos, sin, attn_impl, doc, kv)  # [B, S, H·D], no layout shuffles
        return ops.linear(out, self.wo)

    def _prefill_attention(self, qkv: torch.Tensor, cos, sin, attn_impl: str, doc: tuple | None, kv) -> torch.Tensor:
        """RoPE ⊕ attention of the un-rotated fused QKV. With a cache handle the rotation runs as its own op (``rope_qkv``: in place
        on CUDA, a new tensor on the CPU), so that the rotated K|V can be copied into the cache before the attention reads them."""
        H, Hkv = self.n_heads, self.n_kv_heads
        if kv is None:
            return ops.rope_attention_qkv(qkv, cos, sin, H, Hkv, causal=True, impl=attn_impl, doc=doc)
        qkv = ops.rope_qkv(qkv, cos, sin, H, Hkv)
        kv.store(qkv, H * self.head_dim)
        return ops.attention_qkv(qkv, H, Hkv, causal=True, impl=attn_impl, doc=doc)


class FeedForward(nn.Module):
    def __init__(self, args: ModelArgs):
        super().__init__()
        hidden = args.ffn_hidden
        self.w13 = nn.Parameter(torch.empty(2 * hidden, args.dim))  # rows [0,hidden)=w1 (gate), [hidden,2h)=w3 (up)
        self.w2 = nn.Parameter(torch.empty(args.dim, hidden))
        self.fp8 = False

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if self.fp8:
            return ops.linear_mxfp8(ops.swiglu(ops.linear_mxfp8(x, self.w13)), self.w2)
        return ops.mlp_swiglu(x, self.w13, self.w2)  # SwiGLU forward AND backward ride in GEMM epilogues on CUDA


class TransformerBlock(nn.Module):
    def __init__(self, layer_id: int, args: ModelArgs):
        super().__init__()
        self.layer_id = layer_id
        self.attention = Attention(args)
        self.feed_forward = FeedForward(args)
        self.attention_norm = RMSNormWeight(args.dim)
        self.ffn_norm = RMSNormWeight(args.dim)
        self.eps = args.norm_eps
        self.init_std = 0.02 / math.sqrt(2 * (layer_id + 1)) if args.depth_init else 0.02 / math.sqrt(2 * args.n_layers)

    def forward(self, h: torch.Tensor, delta: torch.Tensor | None, cos, sin, attn_impl: str = "auto", doc: tuple | None = None, kv=None):
        """``h`` = residual stream, ``delta`` = output of the previous sub-block not yet added, ``doc`` = document bounds or None,
        ``kv`` = this layer's KV-cache handle or None (see :meth:`Attention.forward`)."""
        if delta is None:
            x = ops.rmsnorm(h, self.attention_norm.weight, self.eps)
        else:
            x, h = ops.add_rmsnorm(delta, h, self.attention_norm.weight, self.eps)
        a = self.attention(x, cos, sin, attn_impl, doc, kv)
        y, h = ops.add_rmsnorm(a, h, self.ffn_norm.weight, self.eps)
        return h, self.feed_forward(y)

    def init_weights(self, generator: torch.Generator | None = None) -> None:
        nn.init.ones_(self.attention_norm.weight)
        nn.init.ones_(self.ffn_norm.weight)
        nn.init.normal_(self.attention.wqkv, 0.0, 0.02, generator=generator)
        nn.init.normal_(self.feed_forward.w13, 0.0, 0.02, generator=generator)
        nn.init.normal_(self.attention.wo, 0.0, self.init_std, generator=generator)
        nn.init.normal_(self.feed_forward.w2, 0.0, self.init_std, generator=generator)


class Transformer(nn.Module):
    def __init__(self, args: ModelArgs):
        super().__init__()
        self.args = args
        self.tok_embeddings = nn.Embedding(args.vocab_size, args.dim)
        self.layers = nn.ModuleList(TransformerBlock(i, args) for i in range(args.n_layers))
        self.norm = RMSNormWeight(args.dim)
        self.output = nn.Parameter(torch.empty(args.vocab_size, args.dim))
        self.ac_ckpt: bool | int = False  # True = every block, n = every n-th block (train.ac_ckpt)
        self.attn_impl = "auto"
        # document masking of packed rows (data.document_mask): a token attends only to earlier tokens of its own document, where a
        # document ends with this EOS id. None = plain causal attention
        self.doc_eos_id: int | None = None
        self._rope: tuple[torch.Tensor, torch.Tensor] | None = None

    # ------------------------------------------------------------------ init
    def set_fp8(self, on: bool) -> None:
        """MXFP8 (block-scaled e4m3) for the forward and input-gradient GEMMs of every block's four
        projections; weight gradients, the LM head, norms and attention stay bf16 / fp32."""
        for blk in self.layers:
            blk.attention.fp8 = blk.feed_forward.fp8 = bool(on)

    def init_weights(self, seed: int | None = None) -> None:
        dev = self.output.device
        gen = None
        if seed is not None:
            gen = torch.Generator(device=dev)
            gen.manual_seed(seed)
        nn.init.normal_(self.tok_embeddings.weight, 0.0, 1.0, generator=gen)
        for layer in self.layers:
            layer.init_weights(gen)
        nn.init.ones_(self.norm.weight)
        cutoff = 3
        std = self.args.dim**-0.5
        nn.init.trunc_normal_(self.output, 0.0, std, -cutoff * std, cutoff * std, generator=gen)

    def rope_tables(self, seq_len: int, device) -> tuple[torch.Tensor, torch.Tensor]:
        if self._rope is None or self._rope[0].shape[0] < seq_len or self._rope[0].device != torch.device(device):
            n = max(seq_len, self.args.max_seq_len)
            self._rope = ops.reference.rope_tables(n, self.args.head_dim, self.args.rope_theta, device=device)
        return self._rope

    # ------------------------------------------------------------------ forward
    def forward_hidden(self, tokens: torch.Tensor, cache=None) -> torch.Tensor:
        """Final hidden states [B, S, dim]. ``cache``: an ``inference.KVCache`` that receives every layer's rotated K|V (prefill)."""
        B, S = tokens.shape
        cos, sin = self.rope_tables(S, tokens.device)
        h = ops.embedding(tokens, self.tok_embeddings.weight)
        # computed once per micro-batch, read by every layer: documents and / or the sliding window bound the keys a query sees
        win = self.args.sliding_window
        doc = ops.document_bounds(tokens, self.doc_eos_id, win) if self.doc_eos_id is not None or win is not None else None
        delta = None
        ac = self.ac_ckpt if torch.is_grad_enabled() else False
        for i, layer in enumerate(self.layers):
            if ac and (ac is True or i % int(ac) == 0):
                # activation checkpointing: keep only the block's inputs, re-run its forward inside backward. The in-place ops of
                # the block (RoPE on the QKV GEMM output) act on tensors the block itself creates, so replaying it is safe.
                from torch.utils.checkpoint import checkpoint

                h, delta = checkpoint(layer, h, delta, cos, sin, self.attn_impl, doc, use_reentrant=False)
            else:
                h, delta = layer(h, delta, cos, sin, self.attn_impl, doc, None if cache is None else cache.layer(i))
        x, _ = ops.add_rmsnorm(delta, h, self.norm.weight, self.args.norm_eps)
        return x

    def forward(self, tokens: torch.Tensor) -> torch.Tensor:
        return ops.linear(self.forward_hidden(tokens), self.output)

    def decode_step(self, tokens: torch.Tensor, cache) -> torch.Tensor:
        """One generation step over a filled ``inference.KVCache``: ``tokens`` int64 [B], the next token of every row → logits [B, V]
        of the token after it. The same blocks run on [B, 1, dim]; only attention appends to the cache and reads it. Every input that
        changes between steps is on the device, so the step can be captured in a CUDA graph over a static token buffer."""
        B = tokens.shape[0]
        ops.decode_advance(tokens, cache.len, cache.lo, cache.last_tok, self.doc_eos_id)
        h = ops.embedding(tokens.view(B, 1), self.tok_embeddings.weight)
        delta = None
        for i, layer in enumerate(self.layers):
            h, delta = layer(h, delta, cache.cos, cache.sin, self.attn_impl, None, cache.layer(i, decoding=True))
        x, _ = ops.add_rmsnorm(delta, h, self.norm.weight, self.args.norm_eps)
        return ops.linear(x.view(B, -1), self.output)

    def verify_step(self, tokens: torch.Tensor, cache) -> torch.Tensor:
        """The verify step of speculative decoding over a filled ``inference.KVCache``: ``tokens`` int64 [B, T], the next T tokens of
        every row → logits [B, T, V], those of query t predicting the token after tokens[:, t]. It computes what T decode steps would,
        in one forward at M = B·T: the cache state afterwards is theirs, and each query's document start is left in ``cache.lo_q``."""
        B, T = tokens.shape
        cache.lo_q = ops.verify_advance(tokens, cache.len, cache.lo, cache.last_tok, self.doc_eos_id)
        h = ops.embedding(tokens, self.tok_embeddings.weight)
        delta = None
        for i, layer in enumerate(self.layers):
            h, delta = layer(h, delta, cache.cos, cache.sin, self.attn_impl, None, cache.layer(i, verifying=True))
        x, _ = ops.add_rmsnorm(delta, h, self.norm.weight, self.args.norm_eps)
        return ops.linear(x.view(B * T, -1), self.output).view(B, T, -1)  # the LM head at M = B·T

    def loss(self, tokens: torch.Tensor, targets: torch.Tensor, *, grad_scale: float = 1.0, loss_acc: torch.Tensor | None = None) -> torch.Tensor:
        """Mean next-token loss; gradient (not value) is scaled by ``grad_scale``; call ``.backward()`` on it. ``loss_acc``: fp32
        scalar that additionally receives ``+= loss`` inside the loss kernel (the trainer's running sum over micro-batches)."""
        logits = self.forward(tokens)
        return ops.cross_entropy(logits, targets, grad_scale=grad_scale, unit_upstream=True, loss_acc=loss_acc)

    # ------------------------------------------------------------------ accounting
    def num_params(self, exclude_embedding: bool = False) -> int:
        n = sum(p.numel() for p in self.parameters())
        if exclude_embedding:
            n -= self.tok_embeddings.weight.numel()
        return n

    def flops_per_token(self, seq_len: int) -> float:
        """Training FLOPs/token (fwd+bwd): 6·N (matmul params) + causal attention 6·L·S·dim, times the share of the causal
        (query, key) pairs a sliding window W keeps: (W·S - W²/2) / (S²/2) = 1 - (1 - W/S)²."""
        a = self.args
        n_mm = self.num_params(exclude_embedding=True)
        kept = 1.0 if a.sliding_window is None else 1.0 - (1.0 - min(a.sliding_window, seq_len) / seq_len) ** 2
        return 6.0 * n_mm + 6.0 * a.n_layers * seq_len * a.dim * kept


# ---------------------------------------------------------------------- checkpoint naming interchange
def to_reference_state_dict(model: Transformer) -> dict[str, torch.Tensor]:
    a = model.args
    H, Hkv, D, hid = a.n_heads, a.kv_heads, a.head_dim, a.ffn_hidden
    out: dict[str, torch.Tensor] = {"tok_embeddings.weight": model.tok_embeddings.weight.detach()}
    for i, layer in enumerate(model.layers):
        p = f"layers.{i}."
        wqkv = layer.attention.wqkv.detach()
        out[p + "attention.wq.weight"] = wqkv[: H * D]
        out[p + "attention.wk.weight"] = wqkv[H * D : (H + Hkv) * D]
        out[p + "attention.wv.weight"] = wqkv[(H + Hkv) * D :]
        out[p + "attention.wo.weight"] = layer.attention.wo.detach()
        w13 = layer.feed_forward.w13.detach()
        out[p + "feed_forward.w1.weight"] = w13[:hid]
        out[p + "feed_forward.w3.weight"] = w13[hid:]
        out[p + "feed_forward.w2.weight"] = layer.feed_forward.w2.detach()
        out[p + "attention_norm.weight"] = layer.attention_norm.weight.detach()
        out[p + "ffn_norm.weight"] = layer.ffn_norm.weight.detach()
    out["norm.weight"] = model.norm.weight.detach()
    out["output.weight"] = model.output.detach()
    return out


@torch.no_grad()
def from_reference_state_dict(model: Transformer, sd: dict[str, torch.Tensor]) -> None:
    model.tok_embeddings.weight.copy_(sd["tok_embeddings.weight"])
    for i, layer in enumerate(model.layers):
        p = f"layers.{i}."
        layer.attention.wqkv.copy_(
            torch.cat([sd[p + "attention.wq.weight"], sd[p + "attention.wk.weight"], sd[p + "attention.wv.weight"]])
        )
        layer.attention.wo.copy_(sd[p + "attention.wo.weight"])
        layer.feed_forward.w13.copy_(torch.cat([sd[p + "feed_forward.w1.weight"], sd[p + "feed_forward.w3.weight"]]))
        layer.feed_forward.w2.copy_(sd[p + "feed_forward.w2.weight"])
        layer.attention_norm.weight.copy_(sd[p + "attention_norm.weight"])
        layer.ffn_norm.weight.copy_(sd[p + "ffn_norm.weight"])
    model.norm.weight.copy_(sd["norm.weight"])
    model.output.copy_(sd["output.weight"])


def build_model(name: str, type_model: str = "llama2", *, device="cpu", dtype=torch.bfloat16, seed: int | None = 0,
                **overrides) -> Transformer:  # fmt: skip
    args = get_model_args(name, type_model, **overrides)
    with torch.device(device):
        model = Transformer(args)
    model.to(dtype)
    model.init_weights(seed)
    return model
