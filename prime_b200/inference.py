"""Generation over a KV cache: prefill of ragged prompts, then one ``Transformer.decode_step`` per token, on the GPU replayed from a
CUDA graph.

The cache keeps, per layer, exactly the K|V columns of the fused QKV activation with K already rotated, so prefill fills it with one
strided copy per layer and a decode step appends one row per sequence (``ops.kv_append``) and runs split-KV attention over it
(``ops.decode_attention``). The per-row state (``len``, ``lo``: the first key the current query may see, ``last_tok``) lives on the
device, so a decode step depends on no host value that changes between tokens.
"""

from __future__ import annotations

from dataclasses import dataclass

import torch

from . import ops
from .models.llama import Transformer

PAD = 128  # prefill length and cache capacity granularity: the native attention kernels take S % 128 == 0


def _round_up(n: int, m: int) -> int:
    return (n + m - 1) // m * m


@dataclass
class LayerKV:
    """One layer's handle of a :class:`KVCache`, passed down to ``Attention.forward``."""

    cache: "KVCache"
    index: int
    decoding: bool

    @property
    def kv(self) -> torch.Tensor:
        return self.cache.kv[self.index]

    def store(self, qkv: torch.Tensor, k_col: int) -> None:
        """Prefill: copy the rotated K|V columns (from ``k_col`` on) of every position of qkv [B, S, ·] into the cache."""
        self.kv[:, : qkv.shape[1]].copy_(qkv[..., k_col:])


@dataclass
class KVCache:
    kv: torch.Tensor  # [L, B, capacity, 2·Hkv·D]
    len: torch.Tensor  # int32 [B]: valid cache rows
    lo: torch.Tensor  # int32 [B]: first key of the current query's document
    last_tok: torch.Tensor  # int64 [B]
    cos: torch.Tensor  # fp32 [>= capacity, D/2] RoPE tables, held here so a captured graph's pointers stay valid
    sin: torch.Tensor
    window: int | None  # ModelArgs.sliding_window

    @property
    def capacity(self) -> int:
        return self.kv.shape[2]

    def layer(self, i: int, decoding: bool = False) -> LayerKV:
        return LayerKV(self, i, decoding)

    @classmethod
    def allocate(cls, model: Transformer, batch: int, capacity: int, device) -> "KVCache":
        a = model.args
        dtype = model.output.dtype
        cos, sin = model.rope_tables(capacity, device)
        kv = torch.empty((a.n_layers, batch, capacity, 2 * a.kv_heads * a.head_dim), dtype=dtype, device=device)
        z32 = torch.zeros(batch, dtype=torch.int32, device=device)
        return cls(kv, z32, z32.clone(), torch.zeros(batch, dtype=torch.int64, device=device), cos, sin, a.sliding_window)


def cache_capacity(max_seq_len: int, prompt_lens: list[int], max_new: int) -> int:
    """The prompt length padded to 128, or min(max_seq_len, longest prompt + max_new) rounded up to 128, whichever is larger."""
    longest = max(prompt_lens)
    return max(_round_up(longest, PAD), _round_up(min(max_seq_len, longest + max_new), PAD))


@torch.no_grad()
def prefill(model: Transformer, prompts: list[list[int]], capacity: int) -> tuple[torch.Tensor, KVCache]:
    """Run the prompts (right-padded to one length, a multiple of 128 on CUDA) through ``forward_hidden`` while filling a new cache of
    ``capacity`` rows. Returns the logits [B, V] at each row's last prompt position and the cache, positioned after the prompts."""
    dev = model.output.device
    lens = [len(p) for p in prompts]
    if min(lens) < 1:
        raise ValueError("every prompt needs at least one token")
    S = _round_up(max(lens), PAD if dev.type == "cuda" else 1)
    if S > capacity:
        raise ValueError(f"prompts of {max(lens)} tokens need a cache of at least {S} rows, got {capacity}")
    B = len(prompts)
    tokens = torch.zeros((B, S), dtype=torch.int64)
    for b, p in enumerate(prompts):
        tokens[b, : len(p)] = torch.tensor(p, dtype=torch.int64)
    cache = KVCache.allocate(model, B, capacity, dev)
    # causal attention makes the right padding invisible to the prompt, and the cache rows it fills are overwritten before any
    # query reads them
    x = model.forward_hidden(tokens.to(dev), cache)
    last = torch.tensor(lens, device=dev) - 1
    logits = ops.linear(x[torch.arange(B, device=dev), last], model.output)  # the LM head at M = B
    eos = model.doc_eos_id
    lo = []
    for p in prompts:  # the document holding the last prompt token starts after the last EOS before it
        starts = [i + 1 for i in range(len(p) - 1) if eos is not None and p[i] == eos]
        lo.append(starts[-1] if starts else 0)
    cache.len.copy_(torch.tensor(lens, dtype=torch.int32))
    cache.lo.copy_(torch.tensor(lo, dtype=torch.int32))
    cache.last_tok.copy_(torch.tensor([p[-1] for p in prompts], dtype=torch.int64))
    return logits, cache


class GraphDecoder:
    """``model.decode_step`` captured once per (batch, capacity) in a CUDA graph over static token / logit buffers. A replay runs the
    same kernels on the same buffers as the eager step, so its logits are bitwise equal."""

    def __init__(self, model: Transformer, cache: KVCache):
        self.tokens = torch.zeros(cache.len.shape[0], dtype=torch.int64, device=cache.kv.device)
        state = [t.clone() for t in (cache.len, cache.lo, cache.last_tok)]
        # warm-up outside the capture (library load, kernel attributes); it advances the state and writes the next cache row, so the
        # state is restored afterwards, and that row is written again by the first real step
        side = torch.cuda.Stream(device=cache.kv.device)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            model.decode_step(self.tokens, cache)
        torch.cuda.current_stream().wait_stream(side)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.logits = model.decode_step(self.tokens, cache)
        for t, s in zip((cache.len, cache.lo, cache.last_tok), state):
            t.copy_(s)

    def __call__(self, tokens: torch.Tensor) -> torch.Tensor:
        self.tokens.copy_(tokens)
        self.graph.replay()
        return self.logits


def sample(logits: torch.Tensor, temperature: float, top_k: int, gen: torch.Generator) -> int:
    """Greedy (temperature 0) or top-k / temperature sampling of one fp32 CPU logit row."""
    if temperature <= 0:
        return int(logits.argmax())
    logits = logits / temperature
    if top_k > 0:
        kth = torch.topk(logits, min(top_k, logits.numel())).values[-1]
        logits = logits.masked_fill(logits < kth, float("-inf"))
    return int(torch.multinomial(torch.softmax(logits, -1), 1, generator=gen))


@torch.no_grad()
def generate_batch(model: Transformer, prompts: list[list[int]], *, max_new: int, temperature: float = 0.0, top_k: int = 0, seed: int = 0,
                   eos_id: int | None = None, graphs: bool | None = None) -> list[list[int]]:  # fmt: skip
    """Prompt + continuation of every prompt. A row stops at ``max_new`` new tokens, at ``model.args.max_seq_len`` tokens in all, or
    after ``eos_id``. Rows are sampled in order from one CPU generator seeded with ``seed``. ``graphs``: replay the decode step from
    a CUDA graph (default: on CUDA)."""
    model.eval()
    dev = model.output.device
    ids = [list(p) for p in prompts]
    limit = model.args.max_seq_len
    active = [len(p) < limit for p in ids]
    if max_new <= 0 or not any(active):
        return ids
    gen = torch.Generator(device="cpu").manual_seed(seed)
    logits, cache = prefill(model, ids, cache_capacity(limit, [len(p) for p in ids], max_new))
    if graphs if graphs is not None else dev.type == "cuda":
        step = GraphDecoder(model, cache)
    else:
        step = lambda t: model.decode_step(t, cache)  # noqa: E731
    for i in range(max_new):
        rows = logits.float().cpu()
        for b, row in enumerate(ids):
            if not active[b]:
                continue
            nxt = sample(rows[b], temperature, top_k, gen)
            row.append(nxt)
            active[b] = len(row) < limit and not (eos_id is not None and nxt == eos_id)
        if i == max_new - 1 or not any(active):
            break
        # finished rows keep feeding their last token; their logits are never read (and past the capacity nothing is written)
        logits = step(torch.tensor([row[-1] for row in ids], dtype=torch.int64, device=dev))
    return ids
