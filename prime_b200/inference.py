"""Generation over a KV cache: prefill of ragged prompts, then one ``Transformer.decode_step`` per token, on the GPU replayed from a
CUDA graph.

The cache keeps, per layer, exactly the K|V columns of the fused QKV activation with K already rotated, so prefill fills it with one
strided copy per layer and a decode step appends one row per sequence (``ops.kv_append``) and runs split-KV attention over it
(``ops.decode_attention``). With ``kv_dtype="fp8"`` the cache holds those values as e4m3 with one power-of-two scale per 32 columns
(the format of ``ops.kv_append``): 1 + 1/32 bytes per value instead of 2, so twice the context fits and the attention kernel, bound by
the bytes it reads, reads about half as many. The per-row state (``len``, ``lo``: the first key the current query may see, ``last_tok``) lives on the
device, so a decode step depends on no host value that changes between tokens.

``quantize_weights`` converts a model's projections to e4m3 (``ops.MXWeight``) for inference: every entry point here then runs
unchanged, the decode and verify steps reading about 1.03 bytes per weight instead of 2.

Sampling runs on the host (one CPU generator, the stream of earlier versions) or, with ``sampler="device"``, inside the step:
``ops.sample_tokens`` draws each row's next token from a Philox stream keyed by (seed, position), writes it into the step's static
input buffer and applies the stop rules on the device, so the captured graph runs step after step without the host.
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
    verifying: bool = False  # a speculative verify step: T tokens per row

    @property
    def kv(self) -> torch.Tensor:
        return self.cache.kv[self.index]

    @property
    def kv_scale(self) -> torch.Tensor | None:
        return None if self.cache.kv_scale is None else self.cache.kv_scale[self.index]

    def store(self, qkv: torch.Tensor, k_col: int) -> None:
        """Prefill: copy the rotated K|V columns (from ``k_col`` on) of every position of qkv [B, S, ·] into the cache, quantised
        (``ops.kv_quantize``) when the cache is e4m3."""
        if self.cache.kv_scale is not None:
            ops.kv_quantize(qkv[..., k_col:], self.kv, self.kv_scale)
        else:
            self.kv[:, : qkv.shape[1]].copy_(qkv[..., k_col:])


KV_DTYPES = ("bf16", "fp8")


def check_kv_dtype(model: Transformer, kv_dtype: str) -> None:
    """``kv_dtype`` is "bf16" (the model's dtype) or "fp8" (e4m3 with a scale per 32 columns, which needs head_dim % 32 == 0)."""
    if kv_dtype not in KV_DTYPES:
        raise ValueError(f"kv_dtype must be one of {KV_DTYPES}, got {kv_dtype!r}")
    if kv_dtype == "fp8" and model.args.head_dim % 32:
        raise ValueError(f"an fp8 KV cache needs head_dim % 32 == 0 (one scale per 32 columns of a head), got {model.args.head_dim}")


@dataclass
class KVCache:
    kv: torch.Tensor  # [L, B, capacity, 2·Hkv·D]: the model's dtype, or uint8 e4m3 bytes with kv_scale
    len: torch.Tensor  # int32 [B]: valid cache rows
    lo: torch.Tensor  # int32 [B]: first key of the current query's document
    last_tok: torch.Tensor  # int64 [B]
    cos: torch.Tensor  # fp32 [>= capacity, D/2] RoPE tables, held here so a captured graph's pointers stay valid
    sin: torch.Tensor
    window: int | None  # ModelArgs.sliding_window
    lo_q: torch.Tensor | None = None  # int32 [B, T]: each query's document start in the last verify step
    kv_scale: torch.Tensor | None = None  # uint8 [L, B, capacity, 2·Hkv·D/32]: UE8M0 exponents of an e4m3 cache (ops.kv_append)

    @property
    def capacity(self) -> int:
        return self.kv.shape[2]

    def layer(self, i: int, decoding: bool = False, verifying: bool = False) -> LayerKV:
        return LayerKV(self, i, decoding, verifying)

    @classmethod
    def allocate(cls, model: Transformer, batch: int, capacity: int, device, kv_dtype: str = "bf16") -> "KVCache":
        """``kv_dtype``: "bf16" keeps the model's dtype; "fp8" stores e4m3 bytes and one exponent byte per 32 values."""
        check_kv_dtype(model, kv_dtype)
        a = model.args
        dtype = model.output.dtype if kv_dtype == "bf16" else torch.uint8
        cos, sin = model.rope_tables(capacity, device)
        cols = 2 * a.kv_heads * a.head_dim
        kv = torch.empty((a.n_layers, batch, capacity, cols), dtype=dtype, device=device)
        scale = None if kv_dtype == "bf16" else torch.empty((a.n_layers, batch, capacity, cols // 32), dtype=torch.uint8, device=device)
        z32 = torch.zeros(batch, dtype=torch.int32, device=device)
        return cls(kv, z32, z32.clone(), torch.zeros(batch, dtype=torch.int64, device=device), cos, sin, a.sliding_window, kv_scale=scale)


def cache_capacity(max_seq_len: int, prompt_lens: list[int], max_new: int) -> int:
    """The prompt length padded to 128, or min(max_seq_len, longest prompt + max_new) rounded up to 128, whichever is larger."""
    longest = max(prompt_lens)
    return max(_round_up(longest, PAD), _round_up(min(max_seq_len, longest + max_new), PAD))


@torch.no_grad()
def prefill(model: Transformer, prompts: list[list[int]], capacity: int, kv_dtype: str = "bf16") -> tuple[torch.Tensor, KVCache]:
    """Run the prompts (right-padded to one length, a multiple of 128 on CUDA) through ``forward_hidden`` while filling a new cache of
    ``capacity`` rows (``kv_dtype``: see :meth:`KVCache.allocate`). Returns the logits [B, V] at each row's last prompt position and
    the cache, positioned after the prompts."""
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
    cache = KVCache.allocate(model, B, capacity, dev, kv_dtype)
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
    same kernels on the same buffers as the eager step, so its logits are bitwise equal.

    ``tokens``: use this int64 [B] buffer as the static input instead of a new one. ``then``: a function of the logits captured after
    the step, e.g. a sampler that writes the next step's tokens into ``tokens``, so :meth:`replay` runs step after step with no host
    work in between."""

    def __init__(self, model: Transformer, cache: KVCache, tokens: torch.Tensor | None = None, then=None):
        self.tokens = tokens if tokens is not None else torch.zeros(cache.len.shape[0], dtype=torch.int64, device=cache.kv.device)
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
            if then is not None:
                then(self.logits)
        for t, s in zip((cache.len, cache.lo, cache.last_tok), state):
            t.copy_(s)

    def __call__(self, tokens: torch.Tensor) -> torch.Tensor:
        self.tokens.copy_(tokens)
        self.graph.replay()
        return self.logits

    def replay(self) -> None:
        """One step on whatever the token buffer holds."""
        self.graph.replay()


def sample(logits: torch.Tensor, temperature: float, top_k: int, gen: torch.Generator, top_p: float = 1.0, min_p: float = 0.0) -> int:
    """Greedy (temperature 0) or temperature / top-k / top-p / min-p sampling of one fp32 CPU logit row, drawn by
    ``torch.multinomial`` from ``gen``. With top-p or min-p on, the keep-set is ``ops.reference.sample_keep``'s, the one the device
    sampler uses; with both off the draw is the one earlier versions made."""
    if temperature <= 0:
        return int(logits.argmax())
    if top_p < 1.0 or min_p > 0.0:
        keep = ops.reference.sample_keep(logits.view(1, -1), temperature, top_k, top_p, min_p)[0]
        logits = (logits / temperature).masked_fill(~keep, float("-inf"))
        return int(torch.multinomial(torch.softmax(logits, -1), 1, generator=gen))
    logits = logits / temperature
    if top_k > 0:
        kth = torch.topk(logits, min(top_k, logits.numel())).values[-1]
        logits = logits.masked_fill(logits < kth, float("-inf"))
    return int(torch.multinomial(torch.softmax(logits, -1), 1, generator=gen))


@dataclass
class SampleState:
    """Per-row bookkeeping of device-side generation, updated by ``ops.sample_tokens(state=...)`` (see its docstring)."""

    tokens: torch.Tensor  # int64 [B]: the next decode step's input; a finished row keeps its last token
    history: torch.Tensor  # int64 [B, max_new]: the new tokens
    n_out: torch.Tensor  # int32 [B]
    active: torch.Tensor  # bool [B]
    prompt_len: torch.Tensor  # int32 [B]
    max_seq_len: int
    eos_id: int | None

    @classmethod
    def allocate(cls, prompts: list[list[int]], max_new: int, max_seq_len: int, eos_id: int | None, device) -> "SampleState":
        lens = [len(p) for p in prompts]
        return cls(torch.tensor([p[-1] for p in prompts], dtype=torch.int64, device=device),
                   torch.zeros((len(prompts), max_new), dtype=torch.int64, device=device),
                   torch.zeros(len(prompts), dtype=torch.int32, device=device),
                   torch.tensor([n < max_seq_len for n in lens], dtype=torch.bool, device=device),
                   torch.tensor(lens, dtype=torch.int32, device=device), max_seq_len, eos_id)  # fmt: skip


CHECK_EVERY = 16  # device-sampled generation reads the "any row still active" flag once per this many steps


@torch.no_grad()
def generate_batch(model: Transformer, prompts: list[list[int]], *, max_new: int, temperature: float = 0.0, top_k: int = 0,
                   top_p: float = 1.0, min_p: float = 0.0, seed: int = 0, eos_id: int | None = None, graphs: bool | None = None,
                   sampler: str = "host", kv_dtype: str = "bf16") -> list[list[int]]:  # fmt: skip
    """Prompt + continuation of every prompt. A row stops at ``max_new`` new tokens, at ``model.args.max_seq_len`` tokens in all, or
    after ``eos_id`` (kept). ``graphs``: replay the decode step from a CUDA graph (default: on CUDA). ``kv_dtype``: "bf16" (default)
    or "fp8", the e4m3 cache of :meth:`KVCache.allocate`, with half the bytes per value.

    ``sampler`` picks the random stream as well as where sampling runs:

    * ``"host"`` (default): each step's logits are copied to the host and the rows are sampled in order from one CPU generator
      seeded with ``seed`` (:func:`sample`). It reproduces the seeded outputs of earlier versions.
    * ``"device"``: ``ops.sample_tokens`` draws on the device from a Philox stream keyed by ``seed + b`` for row b at each token's
      position, so a row's draws do not depend on the other rows. The first token comes from the prefill logits; on CUDA each later
      step (decode step, sampler and bookkeeping) is one CUDA graph replay writing its own next input, and the host reads a
      "still active" flag once every 16 steps and the tokens once at the end. Greedy tokens are the same under both samplers."""
    if sampler not in ("host", "device"):
        raise ValueError(f"sampler must be 'host' or 'device', got {sampler!r}")
    check_kv_dtype(model, kv_dtype)
    model.eval()
    dev = model.output.device
    ids = [list(p) for p in prompts]
    limit = model.args.max_seq_len
    active = [len(p) < limit for p in ids]
    if max_new <= 0 or not any(active):
        return ids
    use_graphs = graphs if graphs is not None else dev.type == "cuda"
    if sampler == "device":
        return _generate_device(model, ids, max_new, dict(temperature=temperature, top_k=top_k, top_p=top_p, min_p=min_p), seed,
                                eos_id, use_graphs, kv_dtype)  # fmt: skip
    gen = torch.Generator(device="cpu").manual_seed(seed)
    logits, cache = prefill(model, ids, cache_capacity(limit, [len(p) for p in ids], max_new), kv_dtype)
    if use_graphs:
        step = GraphDecoder(model, cache)
    else:
        step = lambda t: model.decode_step(t, cache)  # noqa: E731
    for i in range(max_new):
        rows = logits.float().cpu()
        for b, row in enumerate(ids):
            if not active[b]:
                continue
            nxt = sample(rows[b], temperature, top_k, gen, top_p, min_p)
            row.append(nxt)
            active[b] = len(row) < limit and not (eos_id is not None and nxt == eos_id)
        if i == max_new - 1 or not any(active):
            break
        # finished rows keep feeding their last token; their logits are never read (and past the capacity nothing is written)
        logits = step(torch.tensor([row[-1] for row in ids], dtype=torch.int64, device=dev))
    return ids


def _generate_device(model: Transformer, ids: list[list[int]], max_new: int, knobs: dict, seed: int, eos_id: int | None,
                     graphs: bool, kv_dtype: str = "bf16") -> list[list[int]]:  # fmt: skip
    """``generate_batch(sampler="device")``: sampling, the next step's input and the stop rules all stay on the device."""
    dev = model.output.device
    limit = model.args.max_seq_len
    logits, cache = prefill(model, ids, cache_capacity(limit, [len(p) for p in ids], max_new), kv_dtype)
    st = SampleState.allocate(ids, max_new, limit, eos_id, dev)
    seeds = torch.tensor([seed + b for b in range(len(ids))], dtype=torch.int64, device=dev)

    def draw(lg: torch.Tensor) -> None:  # the position of the token drawn is the row's cache length
        ops.sample_tokens(lg, **knobs, seeds=seeds, positions=cache.len, out=st.tokens, state=st)

    draw(logits)
    if max_new > 1:
        if graphs:
            advance = GraphDecoder(model, cache, tokens=st.tokens, then=draw).replay
        else:
            advance = lambda: draw(model.decode_step(st.tokens, cache))  # noqa: E731
        for i in range(max_new - 1):
            if i % CHECK_EVERY == 0 and not bool(st.active.any()):
                break
            advance()
    hist, n = st.history.cpu(), st.n_out.cpu()
    return [p + hist[b, : int(n[b])].tolist() for b, p in enumerate(ids)]


# ------------------------------------------------------------------------------------------------------------- e4m3 weights
def _projections(model: Transformer) -> list[tuple[torch.nn.Module, str]]:
    """(module, attribute) of every weight ``quantize_weights`` converts: each block's wqkv, wo, w13 and w2, then the LM head."""
    out = []
    for blk in model.layers:
        out += [(blk.attention, "wqkv"), (blk.attention, "wo"), (blk.feed_forward, "w13"), (blk.feed_forward, "w2")]
    return out + [(model, "output")]


@torch.no_grad()
def quantize_weights(model: Transformer) -> Transformer:
    """Convert, in place, ``wqkv``, ``wo``, ``w13`` and ``w2`` of every block and the LM head ``output`` to e4m3 ``ops.MXWeight``s
    (``ops.quantize_weight``: one power-of-two scale per 32 values along the contraction dimension) for inference. Each parameter is
    freed as soon as it is converted, so the peak stays near the model's own size. The embedding and the norms are left alone.

    Afterwards ``prefill``, ``generate_batch``, ``generate_speculative`` and ``eval.perplexity`` run as before: decode and verify steps
    read the e4m3 bytes in place (``ops.gemm_e4m3w``), prefill and full forwards run the bf16 kernels on the exactly dequantised
    weights, and on the CPU everything runs the reference on W̃. The model can no longer be trained. Returns ``model``.

    Raises ``ValueError`` for a contraction dimension that is not a multiple of 128, a model with MXFP8 training GEMMs on
    (``set_fp8(True)``), ZeRO-3-sharded parameters, or a model that is already quantised."""
    slots = _projections(model)
    if any(isinstance(getattr(m, n), ops.MXWeight) for m, n in slots):
        raise ValueError("the model's weights are already e4m3")
    if any(blk.attention.fp8 or blk.feed_forward.fp8 for blk in model.layers):
        raise ValueError("a model with MXFP8 training GEMMs (set_fp8(True)) cannot be converted; call set_fp8(False) first")
    if any(getattr(getattr(m, n), "z3", None) is not None for m, n in slots):
        raise ValueError("ZeRO-3-sharded weights cannot be converted to e4m3; assemble the full model first")
    for m, n in slots:
        w = getattr(m, n)
        if w.shape[1] % 128:
            raise ValueError(f"e4m3 weights need a contraction dimension % 128 == 0; {type(m).__name__}.{n} is {tuple(w.shape)}")
    for m, n in slots:
        mx = ops.quantize_weight(getattr(m, n))
        delattr(m, n)  # the parameter (and, once the caller holds no reference to it, its memory) goes here
        setattr(m, n, mx)
    return model


# ----------------------------------------------------------------------------------------------------------- speculative decoding
MAX_SPEC_K = 15  # drafts per round, the accept kernel's limit


@dataclass
class SpecResult:
    ids: list[list[int]]  # prompt + continuation of every prompt
    rounds: int  # rounds of the row that ran the most
    drafted: int  # draft tokens proposed, over all rows and rounds
    accepted: int  # of those, accepted by the target


@torch.no_grad()
def generate_speculative(model: Transformer, draft: Transformer, prompts: list[list[int]], *, k: int = 4, max_new: int,
                         temperature: float = 0.0, top_k: int = 0, top_p: float = 1.0, min_p: float = 0.0, seed: int = 0,
                         eos_id: int | None = None, graphs: bool | None = None, kv_dtype: str = "bf16") -> SpecResult:  # fmt: skip
    """Speculative decoding: ``draft`` proposes ``k`` tokens per round and ``model`` checks them in one verify step; the output has the
    distribution of ``generate_batch(sampler="device")`` with the same knobs, and greedy output is the target's greedy output.

    Both models are prefilled and the first token is drawn from the target's prefill logits with ``ops.sample_tokens``. Then, per
    round and row, with cache length L and the pending token x at index L:

    1. The draft runs k + 1 decode steps on x, d_1 .. d_k; after step i <= k it draws d_i (index L + i) with ``ops.sample_tokens``
       (the same knobs, Philox counter (L + i, 0, 0, 0)). The last step only puts d_k into the draft's cache.
    2. The target runs one verify step (:meth:`Transformer.verify_step`) on [x, d_1 .. d_k] at indices L .. L + k.
    3. ``ops.spec_accept`` accepts a prefix d_1 .. d_n by the exact rejection rule (Leviathan et al. 2023, Chen et al. 2023), draws
       y from the residual or, when all k are accepted, from p_{k+1}, and emits d_1 .. d_n, y through the stop rules of
       ``generate_batch`` (``max_new``, ``model.args.max_seq_len``, ``eos_id`` kept). Both caches keep the accepted prefix and y is
       pending. Document masking (``doc_eos_id``) and sliding windows keep their meaning inside the verify step.

    On CUDA (``graphs`` default) one whole round is one CUDA graph replay over static buffers; the host reads the "any row active"
    flag every 16 rounds and the history once at the end. Without graphs the same calls run eagerly; on the CPU through the
    reference ops. Each model keeps its own window, head dimension and GQA ratio; the vocabulary, device and ``doc_eos_id`` must
    match. ``kv_dtype`` ("bf16" or "fp8", see :meth:`KVCache.allocate`) applies to the target's and the draft's cache."""
    if draft.args.vocab_size != model.args.vocab_size:
        raise ValueError(f"draft vocabulary {draft.args.vocab_size} != target vocabulary {model.args.vocab_size}")
    if draft.output.device != model.output.device:
        raise ValueError(f"draft on {draft.output.device}, target on {model.output.device}")
    if draft.doc_eos_id != model.doc_eos_id:
        raise ValueError(f"draft doc_eos_id {draft.doc_eos_id} != target doc_eos_id {model.doc_eos_id}")
    if not 1 <= k <= MAX_SPEC_K:
        raise ValueError(f"k must be in [1, {MAX_SPEC_K}], got {k}")
    check_kv_dtype(model, kv_dtype)
    check_kv_dtype(draft, kv_dtype)
    ops.functional._sample_args(temperature, top_k, top_p, min_p)
    model.eval()
    draft.eval()
    dev = model.output.device
    ids = [list(p) for p in prompts]
    limit = model.args.max_seq_len
    if max_new <= 0 or not any(len(p) < limit for p in ids):
        return SpecResult(ids, 0, 0, 0)
    B = len(ids)
    cap = _round_up(cache_capacity(limit, [len(p) for p in ids], max_new) + k + 1, PAD)
    logits, cache = prefill(model, ids, cap, kv_dtype)
    _, dcache = prefill(draft, ids, cap, kv_dtype)
    st = SampleState.allocate(ids, max_new, limit, eos_id, dev)
    knobs = dict(temperature=temperature, top_k=top_k, top_p=top_p, min_p=min_p)
    seeds = torch.tensor([seed + b for b in range(B)], dtype=torch.int64, device=dev)
    xs = torch.zeros((k + 1, B), dtype=torch.int64, device=dev)  # the round's inputs: xs[0] = the pending token, xs[i] = d_i
    qbuf = torch.empty((k, B, model.args.vocab_size), dtype=logits.dtype, device=dev)
    drafted = torch.zeros(B, dtype=torch.int64, device=dev)
    accepted = torch.zeros(B, dtype=torch.int64, device=dev)
    ops.sample_tokens(logits, **knobs, seeds=seeds, positions=cache.len, out=xs[0], state=st)

    def round_() -> None:
        for i in range(k + 1):
            lg = draft.decode_step(xs[i], dcache)
            if i < k:
                qbuf[i].copy_(lg)
                ops.sample_tokens(qbuf[i], **knobs, seeds=seeds, positions=dcache.len, out=xs[i + 1])
        toks = xs.t().contiguous()
        p = model.verify_step(toks, cache)
        ops.spec_accept(p, qbuf, **knobs, seeds=seeds, tokens=toks, lo_q=cache.lo_q, target=cache, draft=dcache, state=st,
                        pending=xs[0], drafted=drafted, accepted=accepted)  # fmt: skip

    advance = round_
    if graphs if graphs is not None else dev.type == "cuda":
        advance = _capture(round_, [cache.len, cache.lo, cache.last_tok, dcache.len, dcache.lo, dcache.last_tok, xs, qbuf, drafted,
                                    accepted, st.history, st.n_out, st.active])  # fmt: skip
    for i in range(max_new - 1):  # every round emits at least one token per active row
        if i % CHECK_EVERY == 0 and not bool(st.active.any()):
            break
        advance()
    hist, n = st.history.cpu(), st.n_out.cpu()
    d = drafted.cpu()
    return SpecResult([p + hist[b, : int(n[b])].tolist() for b, p in enumerate(ids)], int(d.max()) // k, int(d.sum()),
                      int(accepted.sum()))  # fmt: skip


def _capture(fn, state: list[torch.Tensor]):
    """``fn`` captured in a CUDA graph; returns its replay. A warm-up run outside the capture (library load, kernel attributes)
    changes ``state``, so ``state`` is restored afterwards; the cache rows it wrote are written again by the first replay."""
    saved = [t.clone() for t in state]
    side = torch.cuda.Stream(device=state[0].device)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fn()
    for t, s in zip(state, saved):
        t.copy_(s)
    return graph.replay
