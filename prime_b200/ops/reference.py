"""Plain-PyTorch reference implementations of every hot op.

These are (a) the CPU/gloo execution path (BASELINE.json config 1) and (b) the
fp32 numerical oracle every sm_90a kernel is tested against
(``tests/test_kernels_gpu.py``).  Nothing here is ever selected on a CUDA
tensor by :mod:`prime_b200.ops.functional` — on the GPU the native kernels run
or the call fails loudly.
"""

from __future__ import annotations

import math

import torch
import torch.nn.functional as F


def rmsnorm(x: torch.Tensor, weight: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    xf = x.float()
    rstd = torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps)
    return (xf * rstd * weight.float()).to(x.dtype)


def add_rmsnorm(x: torch.Tensor, residual: torch.Tensor, weight: torch.Tensor, eps: float = 1e-5):
    """h = x + residual ; y = rmsnorm(h).  Returns (y, h)."""
    h = (x.float() + residual.float()).to(x.dtype)
    return rmsnorm(h, weight, eps), h


def linear(x: torch.Tensor, weight: torch.Tensor) -> torch.Tensor:
    return F.linear(x, weight)


def rope_tables(seq_len: int, head_dim: int, theta: float = 10000.0, device=None) -> tuple[torch.Tensor, torch.Tensor]:
    """cos/sin tables [seq, head_dim/2] (fp32), interleaved-pair convention (Llama reference)."""
    freqs = 1.0 / (theta ** (torch.arange(0, head_dim, 2, device=device, dtype=torch.float32) / head_dim))
    t = torch.arange(seq_len, device=device, dtype=torch.float32)
    ang = torch.outer(t, freqs)
    return ang.cos(), ang.sin()


def rope(x: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor) -> torch.Tensor:
    """x: [B, S, H, D]; rotates interleaved pairs (x[2i], x[2i+1])."""
    B, S, H, D = x.shape
    xf = x.float().reshape(B, S, H, D // 2, 2)
    c = cos[:S].view(1, S, 1, D // 2)
    s = sin[:S].view(1, S, 1, D // 2)
    x0, x1 = xf[..., 0], xf[..., 1]
    out = torch.stack((x0 * c - x1 * s, x0 * s + x1 * c), dim=-1)
    return out.reshape(B, S, H, D).to(x.dtype)


def swiglu(gate_up: torch.Tensor) -> torch.Tensor:
    """gate_up: [..., 2*F] = concat(gate, up) → silu(gate) * up."""
    g, u = gate_up.float().chunk(2, dim=-1)
    return (F.silu(g) * u).to(gate_up.dtype)


def document_bounds(tokens: torch.Tensor, eos_id: int | None, window: int | None = None) -> tuple[torch.Tensor, torch.Tensor]:
    """Documents of packed rows, tokens [B, S] → (doc_start, doc_end) int32 [B, S].

    Position s starts a document when s == 0 or tokens[b, s-1] == eos_id (the EOS belongs to the document it ends); ``eos_id``
    None = the whole row is one document. ``doc_start[b, s]`` is the first position of the document holding s, ``doc_end[b, s]``
    one past its last position. With a sliding ``window`` W, query s sees only the W most recent keys, itself included:
    doc_start = max(doc_start, s - W + 1) and doc_end = min(doc_end, s + W), one past the last query that sees key s."""
    B, S = tokens.shape
    is_eos = tokens == eos_id if eos_id is not None else torch.zeros((B, S), dtype=torch.bool, device=tokens.device)
    starts = torch.zeros((B, S), dtype=torch.bool, device=tokens.device)
    starts[:, 0] = True
    starts[:, 1:] = is_eos[:, :-1]
    pos = torch.arange(S, device=tokens.device).expand(B, S)
    doc_start = torch.where(starts, pos, 0).cummax(1).values  # latest start at or before s
    doc_end = torch.where(is_eos, pos + 1, S).flip(1).cummin(1).values.flip(1)  # first EOS at or after s, plus one
    if window is not None:
        doc_start = torch.maximum(doc_start, pos - window + 1)
        doc_end = torch.minimum(doc_end, pos + window)
    return doc_start.int(), doc_end.int()


def document_mask(doc_start: torch.Tensor) -> torch.Tensor:
    """Boolean [B, S, S] mask of document-masked causal attention: query q sees key k iff doc_start[b, q] <= k <= q."""
    B, S = doc_start.shape
    k = torch.arange(S, device=doc_start.device)
    return (k.view(1, 1, S) <= k.view(1, S, 1)) & (k.view(1, 1, S) >= doc_start.long().view(B, S, 1))


def attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, causal: bool = True, doc_start: torch.Tensor | None = None) -> torch.Tensor:
    """q: [B, S, H, D]; k/v: [B, S, Hkv, D] → [B, S, H, D].  ``doc_start`` [B, S]: document masking (implies causal)."""
    B, S, H, D = q.shape
    Hkv = k.shape[2]
    qf, kf, vf = (t.float().transpose(1, 2) for t in (q, k, v))
    if Hkv != H:
        kf = kf.repeat_interleave(H // Hkv, dim=1)
        vf = vf.repeat_interleave(H // Hkv, dim=1)
    scores = qf @ kf.transpose(-1, -2) / math.sqrt(D)
    if doc_start is not None:
        if not causal:
            raise ValueError("document masking implies causal attention")
        scores = scores.masked_fill(~document_mask(doc_start).unsqueeze(1), float("-inf"))
    elif causal:
        mask = torch.ones(S, S, dtype=torch.bool, device=q.device).tril()
        scores = scores.masked_fill(~mask, float("-inf"))
    out = scores.softmax(-1) @ vf
    return out.transpose(1, 2).to(q.dtype)


def rope_at(x: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor) -> torch.Tensor:
    """x: [B, heads, D] of one token per row; cos / sin: that token's table rows [B, D/2]. Interleaved pairs, as :func:`rope`."""
    B, Hh, D = x.shape
    xf = x.float().reshape(B, Hh, D // 2, 2)
    c, s = cos.view(B, 1, D // 2), sin.view(B, 1, D // 2)
    x0, x1 = xf[..., 0], xf[..., 1]
    return torch.stack((x0 * c - x1 * s, x0 * s + x1 * c), dim=-1).reshape(B, Hh, D).to(x.dtype)


def decode_attention(q: torch.Tensor, kv: torch.Tensor, length: torch.Tensor, lo: torch.Tensor | None = None,
                     window: int | None = None) -> torch.Tensor:  # fmt: skip
    """One query per row over a KV cache, in fp32: q [B, H, D] (rotated), kv [B, capacity, 2·Hkv·D] (rotated K heads, then V heads)
    → [B, H, D]. Row b sees keys max(lo[b], len[b] - window) <= k < len[b] (``lo`` None = 0, ``window`` None or 0 = none): the rule
    of :func:`document_bounds` for the query at position len[b] - 1. A row that sees no key gets zeros."""
    B, H, D = q.shape
    cap = kv.shape[1]
    Hkv = kv.shape[2] // (2 * D)
    kf = kv[..., : Hkv * D].float().reshape(B, cap, Hkv, D).repeat_interleave(H // Hkv, dim=2)
    vf = kv[..., Hkv * D :].float().reshape(B, cap, Hkv, D).repeat_interleave(H // Hkv, dim=2)
    L = length.long().clamp(max=cap).view(B, 1)
    start = torch.zeros_like(L) if lo is None else lo.long().view(B, 1)
    if window:
        start = torch.maximum(start, L - window)
    k = torch.arange(cap, device=q.device).view(1, cap)
    visible = (k >= start) & (k < L)
    scores = torch.einsum("bhd,bkhd->bhk", q.float(), kf) / math.sqrt(D)
    p = scores.masked_fill(~visible.unsqueeze(1), float("-inf")).softmax(-1).nan_to_num(0.0)
    # rows nobody may read (beyond len, or never written) can hold anything, NaN included: 0·NaN must not reach the output
    return torch.einsum("bhk,bkhd->bhd", p, vf.masked_fill(~visible.view(B, cap, 1, 1), 0.0))


def verify_attention(q: torch.Tensor, kv: torch.Tensor, length: torch.Tensor, lo_q: torch.Tensor | None = None,
                     window: int | None = None) -> torch.Tensor:  # fmt: skip
    """T queries per row over a KV cache, in fp32: q [B, T, H, D] (rotated) → [B, T, H, D]. Query t of row b sits at position
    pos = len[b] - T + t and sees keys max(lo_q[b, t], pos + 1 - window) <= k <= pos: :func:`decode_attention` of each query."""
    B, T, H, D = q.shape
    out = []
    for t in range(T):
        lo = None if lo_q is None else lo_q[:, t]
        out.append(decode_attention(q[:, t], kv, length - (T - 1 - t), lo, window))
    return torch.stack(out, dim=1)


# ----------------------------------------------------------------------------------------------------------- sampling
# The contract is stated in ``ops.sample_tokens``. Nothing below reads a value back to the host, so on CUDA the fallback can be
# captured in a CUDA graph like the native kernel.
MASS_UNIT = 2.0**40  # fixed-point scale of a token's mass p_i in [0, 1]: every mass sum is an exact int64 sum
_M32 = 0xFFFFFFFF


def _mulhilo32(a: int, b: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """(hi, lo) 32-bit words of the 64-bit product of the constant a and the uint32 values in int64 tensor b, without overflow."""
    p_lo = a * (b & 0xFFFF)  # < 2^48
    p_hi = a * (b >> 16)  # < 2^48
    t = p_lo + ((p_hi & 0xFFFF) << 16)
    return (p_hi >> 16) + (t >> 32), t & _M32


def philox4x32_10(key: torch.Tensor, counter: torch.Tensor) -> torch.Tensor:
    """Philox4x32-10 (Salmon et al., SC'11) in int64 arithmetic: key int64 [..., 2], counter int64 [..., 4] (uint32 words) → the
    four uint32 output words [..., 4]."""
    k0, k1 = key[..., 0] & _M32, key[..., 1] & _M32
    c0, c1, c2, c3 = (counter[..., i] & _M32 for i in range(4))
    for r in range(10):
        if r:
            k0, k1 = (k0 + 0x9E3779B9) & _M32, (k1 + 0xBB67AE85) & _M32
        hi0, lo0 = _mulhilo32(0xD2511F53, c0)
        hi1, lo1 = _mulhilo32(0xCD9E8D57, c2)
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
    return torch.stack((c0, c1, c2, c3), dim=-1)


def sample_uniform_bits(seeds: torch.Tensor, positions: torch.Tensor) -> torch.Tensor:
    """r = x0 >> 8 (24 bits, int64 [B]) of Philox4x32-10 with key = the 64-bit seed and counter = (position, 0, 0, 0); the draw's
    u = (r + 0.5)·2^-24."""
    s = seeds.long()
    key = torch.stack((s & _M32, (s >> 32) & _M32), dim=-1)
    z = torch.zeros_like(s)
    return philox4x32_10(key, torch.stack((positions.long() & _M32, z, z, z), dim=-1))[..., 0] >> 8


def _f32(x: float) -> float:
    return float(torch.tensor(x, dtype=torch.float32))


def sample_masses(logits: torch.Tensor, temperature: float) -> torch.Tensor:
    """Fixed-point masses int64 [B, V]: p_i = exp((l_i - l_max)·(1/T)) in fp64 (T the fp32 value), times 2^40, rounded."""
    lf = logits.float()
    x = (lf.double() - lf.amax(-1, keepdim=True).double()) * (1.0 / _f32(temperature))
    return (torch.exp(x) * MASS_UNIT).round().long()


def sample_keep(logits: torch.Tensor, temperature: float, top_k: int = 0, top_p: float = 1.0, min_p: float = 0.0,
                mass: torch.Tensor | None = None) -> torch.Tensor:  # fmt: skip
    """Keep-set bool [B, V] of temperature > 0 sampling: top-k, then top-p on the top-k set, then min-p, each an upper set of the
    logit order with tie groups kept whole (the contract of ``ops.sample_tokens``). Sort-based; masses from :func:`sample_masses`."""
    lf = logits.float()
    B, V = lf.shape
    if mass is None:
        mass = sample_masses(lf, temperature)
    lmax = lf.amax(-1, keepdim=True)
    keep = torch.ones((B, V), dtype=torch.bool, device=lf.device)
    if (top_k > 0 and top_k < V) or top_p < 1.0:
        ls, idx = lf.sort(dim=-1, descending=True, stable=True)
        t = torch.full_like(lmax, -math.inf)
        if top_k > 0 and top_k < V:
            t = ls[:, top_k - 1 : top_k]  # the k-th largest logit: its whole tie group stays
        if top_p < 1.0:
            in_s = ls >= t
            cum = torch.where(in_s, mass.gather(1, idx), 0).cumsum(-1)
            need = cum[:, -1:].double() * _f32(top_p)
            j = (cum.double() < need).sum(-1, keepdim=True)  # first sorted position whose inclusive mass reaches need
            t = torch.maximum(t, ls.gather(1, j.clamp(max=V - 1)))
        keep = lf >= t
    if min_p > 0.0:
        off = _f32(_f32(temperature) * math.log(_f32(min_p)))
        keep &= lf >= lmax + torch.tensor(off, dtype=torch.float32, device=lf.device)
    return keep


def sample_tokens(logits: torch.Tensor, temperature: float, top_k: int, top_p: float, min_p: float, seeds: torch.Tensor,
                  positions: torch.Tensor) -> torch.Tensor:  # fmt: skip
    """One token per row of logits [B, V] → int64 [B], by the contract of ``ops.sample_tokens``: fp32 logits, fp64 masses rounded to
    fixed point, int64 mass sums."""
    lf = logits.float()
    if temperature == 0:
        return lf.argmax(-1)
    B, V = lf.shape
    mass = sample_masses(lf, temperature)
    keep = sample_keep(lf, temperature, top_k, top_p, min_p, mass)
    cum = torch.where(keep, mass, 0).cumsum(-1)
    M = cum[:, -1]
    a = 2 * sample_uniform_bits(seeds.to(lf.device), positions.to(lf.device)) + 1  # u·M = (2r + 1)·M / 2^25, in int64
    target = a * (M >> 25) + ((a * (M & (2**25 - 1))) >> 25)
    tok = (cum <= target.view(B, 1)).sum(-1)
    last = torch.where(keep, torch.arange(V, device=lf.device), -1).amax(-1)
    return torch.where(tok < V, tok, last)


def sample_bookkeeping(tokens: torch.Tensor, out: torch.Tensor, history: torch.Tensor, n_out: torch.Tensor, active: torch.Tensor,
                       prompt_len: torch.Tensor, max_seq_len: int, eos_id: int | None) -> None:  # fmt: skip
    """The bookkeeping of ``ops.sample_tokens(state=...)``, in place: an active row writes its token to ``out`` and to
    ``history[b, n_out[b]]``, counts it, and stops at ``max_new`` tokens, at ``max_seq_len`` in all, or after ``eos_id``."""
    max_new = history.shape[1]
    act = active.bool()
    out.copy_(torch.where(act, tokens, out))
    col = n_out.long().clamp(max=max_new - 1).view(-1, 1)
    history.scatter_(1, col, torch.where(act.view(-1, 1), tokens.view(-1, 1), history.gather(1, col)))
    n_out.add_(act.to(n_out.dtype))
    stop = (n_out >= max_new) | (prompt_len + n_out >= max_seq_len)
    if eos_id is not None:
        stop |= tokens == eos_id
    active.copy_(act & ~stop)


def spec_masses(logits: torch.Tensor, temperature: float, top_k: int = 0, top_p: float = 1.0, min_p: float = 0.0) -> torch.Tensor:
    """The filtered distributions of ``ops.spec_accept``, int64 [N, V]: the kept fixed-point masses of ``ops.sample_tokens`` divided
    by their total, round(mass_j·2^40 / fp64(total)), in fp64 (every mass < 2^41 is exact in fp64, and so is its product with 2^40).
    Greedy (temperature 0): 2^40 at the argmax."""
    lf = logits.float()
    if temperature == 0:
        return F.one_hot(lf.argmax(-1), lf.shape[-1]).long() << 40
    mass = sample_masses(lf, temperature)
    kept = torch.where(sample_keep(lf, temperature, top_k, top_p, min_p, mass), mass, 0)
    total = kept.sum(-1, keepdim=True)
    return (kept.double() * MASS_UNIT / total.double()).round().long()


def _philox_r(seed: int, pos: int, word1: int) -> int:
    """The top 24 bits of Philox4x32-10 word x0 with key = seed and counter = (pos, word1, 0, 0)."""
    key = torch.tensor([seed & _M32, (seed >> 32) & _M32], dtype=torch.int64)
    return int(philox4x32_10(key, torch.tensor([pos & _M32, word1, 0, 0], dtype=torch.int64))[0]) >> 8


def spec_accept_row(P: torch.Tensor, Q: torch.Tensor, drafts: list[int], seed: int, L: int, greedy: bool) -> tuple[int, int]:
    """The accept rule of ``ops.spec_accept`` for one row: P [k+1, V] and Q [k, V] from :func:`spec_masses`, the k drafts, the seed
    and the cache length L before the round → (n accepted, y). Exact: the comparisons and the draw are in Python integers."""
    k = len(drafts)
    for i in range(1, k + 2):
        p = P[i - 1]
        if i <= k:
            d = drafts[i - 1]
            if greedy:
                if int(p.argmax()) == d:
                    continue
                return i - 1, int(p.argmax())
            r = _philox_r(seed, L + i, 1)
            if (2 * r + 1) * int(Q[i - 1, d]) < (1 << 25) * int(p[d]):
                continue
            w = (p - Q[i - 1]).clamp(min=0)
            if int(w.sum()) == 0:
                w = p
        elif greedy:
            return k, int(p.argmax())
        else:
            w = p
        total = int(w.sum())
        target = ((2 * _philox_r(seed, L + i, 2) + 1) * total) >> 25
        y = int((w.cumsum(0) <= target).sum())
        return i - 1, y
    raise AssertionError("unreachable")


def spec_accept(target_logits: torch.Tensor, draft_logits: torch.Tensor, temperature: float, top_k: int, top_p: float, min_p: float,
                seeds: torch.Tensor, tokens: torch.Tensor, lo_q: torch.Tensor, target, draft, state, pending: torch.Tensor,
                drafted: torch.Tensor, accepted: torch.Tensor) -> None:  # fmt: skip
    """``ops.spec_accept`` row by row on the host (the bit-exact oracle of the kernel); writes its outputs in place."""
    B, T, V = target_logits.shape
    k = T - 1
    max_new = state.history.shape[1]
    knobs = (temperature, top_k, top_p, min_p)
    act = state.active.cpu()
    for b in range(B):
        if not bool(act[b]):
            continue
        L = int(target.len[b]) - T
        P = spec_masses(target_logits[b], *knobs)
        Q = spec_masses(draft_logits[:, b], *knobs)
        toks = [int(x) for x in tokens[b].tolist()]
        n, y = spec_accept_row(P, Q, toks[1:], int(seeds[b]), L, temperature == 0)
        no = int(state.n_out[b])
        for tok in toks[1 : n + 1] + [y]:
            state.history[b, no] = tok
            no += 1
            if no >= max_new or int(state.prompt_len[b]) + no >= state.max_seq_len or tok == state.eos_id:
                state.active[b] = False
                break
        state.n_out[b] = no
        drafted[b] += k
        accepted[b] += n
        for c in (target, draft):
            c.len[b] = L + n + 1
            c.lo[b] = lo_q[b, n]
            c.last_tok[b] = toks[n]
        pending[b] = y


def cross_entropy(logits: torch.Tensor, targets: torch.Tensor, ignore_index: int = -100) -> torch.Tensor:
    return F.cross_entropy(logits.float().view(-1, logits.shape[-1]), targets.view(-1), ignore_index=ignore_index)


def adamw_step(
    p: torch.Tensor,
    g: torch.Tensor,
    m: torch.Tensor,
    v: torch.Tensor,
    *,
    lr: float,
    beta1: float,
    beta2: float,
    eps: float,
    weight_decay: float,
    step: int,
    grad_scale: float = 1.0,
) -> None:
    """In-place decoupled AdamW on fp32 master tensors (torch.optim.AdamW semantics)."""
    g = g.float() * grad_scale
    p.mul_(1.0 - lr * weight_decay)
    m.mul_(beta1).add_(g, alpha=1.0 - beta1)
    v.mul_(beta2).addcmul_(g, g, value=1.0 - beta2)
    bc1 = 1.0 - beta1**step
    bc2 = 1.0 - beta2**step
    denom = (v.sqrt() / math.sqrt(bc2)).add_(eps)
    p.addcdiv_(m, denom, value=-lr / bc1)


def quantize_int8_blockwise(x: torch.Tensor, block: int = 1024) -> tuple[torch.Tensor, torch.Tensor]:
    """Symmetric per-block int8: returns (q int8 [n], scales fp32 [ceil(n/block)])."""
    n = x.numel()
    nb = (n + block - 1) // block
    pad = nb * block - n
    xf = x.float().reshape(-1)
    if pad:
        xf = F.pad(xf, (0, pad))
    xb = xf.view(nb, block)
    amax = xb.abs().amax(dim=1)
    # tensor ÷ tensor: ``amax / 127.0`` (tensor ÷ Python scalar) is evaluated by torch as amax · (1/127), which differs from the
    # IEEE quotient the kernel computes by one ulp for some blocks — enough to round a tie the other way in a few elements per
    # million and make the fused-vs-reference comparison data dependent.
    # A subnormal scale divides instead of multiplying, as the kernel does: 1/scale overflows to inf below 2^-128 (0·inf = NaN).
    scale = torch.div(amax, torch.full_like(amax, 127.0))
    inv = torch.where(scale > 0, torch.ones_like(scale) / scale, torch.zeros_like(scale))
    divide = ((scale > 0) & (scale < torch.finfo(torch.float32).tiny))[:, None]
    y = torch.where(divide, xb / torch.where(divide, scale[:, None], torch.ones_like(scale[:, None])), xb * inv[:, None])
    q = torch.clamp(torch.round(y), -127, 127).to(torch.int8)
    return q.view(-1)[:n].contiguous(), scale


def dequantize_int8_blockwise(q: torch.Tensor, scale: torch.Tensor, block: int = 1024) -> torch.Tensor:
    n = q.numel()
    nb = scale.numel()
    pad = nb * block - n
    qf = q.float()
    if pad:
        qf = F.pad(qf, (0, pad))
    return (qf.view(nb, block) * scale[:, None]).view(-1)[:n]


def nesterov_outer_step(
    theta0: torch.Tensor,
    avg_pseudo_grad: torch.Tensor,
    momentum_buf: torch.Tensor,
    *,
    lr: float,
    momentum: float,
    nesterov: bool = True,
) -> None:
    """torch.optim.SGD(nesterov=True) semantics, in place on fp32 theta0 / momentum."""
    momentum_buf.mul_(momentum).add_(avg_pseudo_grad)
    step = avg_pseudo_grad + momentum * momentum_buf if nesterov else momentum_buf
    theta0.add_(step, alpha=-lr)


# ----------------------------------------------------------------------------------------------------------- MXFP8
def _mxfp8_sf_index(rows: int, k: int, device=None) -> torch.Tensor:
    """Byte offset of the scale of (row r, 32-block kb) in the tensor-core layout used by csrc/gemm_mxfp8_sm90.cu:
    [k/128][ceil(rows/128)+1] atoms of 512 bytes; inside an atom (r % 32) * 16 + ((r % 128) // 32) * 4 + kb % 4."""
    atoms = (rows + 127) // 128 + 1
    r = torch.arange(rows, device=device).view(-1, 1)
    kb = torch.arange(k // 32, device=device).view(1, -1)
    return ((kb >> 2) * atoms + (r >> 7)) * 512 + (r & 31) * 16 + ((r & 127) >> 5) * 4 + (kb & 3)


def _mx_e4m3(blocks: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """The MX e4m3 rule on fp32 blocks [..., 32]: the exponent e (int32 [...]) of the smallest power of two 2^(e-127) with
    amax / 2^(e-127) <= 448, e clamped to [1, 254], and the e4m3 bytes (uint8 [..., 32]) of x / 2^(e-127), rounded to nearest even
    with saturation (csrc/mx_common.cuh)."""
    amax = blocks.abs().amax(dim=-1)
    v = (amax * (1.0 / 448.0)).to(torch.float32)
    bits = v.view(torch.int32)
    e = (bits >> 23) & 0xFF
    e = torch.where((bits & 0x7FFFFF) != 0, e + 1, e).clamp(1, 254)
    inv = ((254 - e) << 23).to(torch.int32).view(torch.float32)
    return (blocks * inv.unsqueeze(-1)).clamp(-448.0, 448.0).to(torch.float8_e4m3fn).view(torch.uint8), e


def quantize_mxfp8(x: torch.Tensor, transpose: bool = False) -> tuple[torch.Tensor, torch.Tensor]:
    """OCP MX e4m3: per 32 contiguous contraction elements a power-of-two scale 2^e, the smallest with amax / 2^e <= 448."""
    xf = (x.t() if transpose else x).float().contiguous()
    rows, k = xf.shape
    assert k % 128 == 0
    q, e = _mx_e4m3(xf.view(rows, k // 32, 32))
    q = q.view(rows, k)
    sf = torch.full(((k // 128) * ((rows + 127) // 128 + 1) * 512,), 127, dtype=torch.uint8, device=x.device)
    sf[_mxfp8_sf_index(rows, k, x.device).reshape(-1)] = e.to(torch.uint8).reshape(-1)
    return q, sf


def dequantize_mxfp8(q: torch.Tensor, sf: torch.Tensor) -> torch.Tensor:
    rows, k = q.shape
    e = sf[_mxfp8_sf_index(rows, k, q.device).reshape(-1)].view(rows, k // 32).to(torch.int32)
    scale = (e << 23).view(torch.float32)
    return (q.view(torch.float8_e4m3fn).float().view(rows, k // 32, 32) * scale.unsqueeze(-1)).view(rows, k)


# ----------------------------------------------------------------------------------------------------------- e4m3 KV cache
def quantize_kv(x: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """Cache rows x [..., C] (C % 32 == 0; the values the bf16 cache would hold) → (e4m3 bytes uint8 [..., C], UE8M0 exponents
    uint8 [..., C / 32]): the MX rule of :func:`quantize_mxfp8` per 32 consecutive columns, the exponents stored dense."""
    C = x.shape[-1]
    assert C % 32 == 0, C
    q, e = _mx_e4m3(x.float().reshape(*x.shape[:-1], C // 32, 32))
    return q.reshape(x.shape), e.to(torch.uint8)


def dequantize_kv(q: torch.Tensor, e: torch.Tensor) -> torch.Tensor:
    """fp32 [..., C] of :func:`quantize_kv`'s output: every value e4m3 · 2^(e - 127), exact."""
    C = q.shape[-1]
    scale = (e.to(torch.int32) << 23).view(torch.float32)
    return (q.view(torch.float8_e4m3fn).float().reshape(*q.shape[:-1], C // 32, 32) * scale.unsqueeze(-1)).reshape(q.shape)
