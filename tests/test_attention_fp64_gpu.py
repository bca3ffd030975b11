"""The flash-attention kernels (``csrc/attention_sm90.cu``: forward, dK/dV, dQ, delta and document bounds) against an fp64 oracle,
element by element, on every templated instantiation and at the edges where tiles, masks and the online softmax meet.

The launchers are driven directly, so the test owns ``lse2`` (the forward's log2-domain log-sum-exp, which the backward reads) and
``delta`` and checks them too; every output buffer starts as NaN, so an element no kernel wrote fails. The oracle is plain torch in
fp64, one (b, head) at a time, on ``.double()`` of the exact bf16 ``qkv`` / ``dout`` the kernels read; ``delta`` and the gradients
use the kernel's own bf16 ``out``, as the kernels do. Every element obeys the rule of ``test_kernel_edges_gpu.py``:

    |got - ref| <= rtol·|ref| + allowance + 2^-100

``rtol`` is the final store; the allowance is a sum of tolerance constants (one rounding each, commented below) times the
magnitudes they act on: Σp·|v| for ``out``, scale·Σ|dO·out| for ``delta``, scale·Σ p·(|dP| + |δ|)·|K| for dQ (|Q| for dK),
Σ p·|dO| for dV, and the worst-case fp32 score error D·2^-24·Σ|q·k| per query row. Probes with Q = 0 make the kernels almost
exact: lse2[q] = log2 n(q) for the visible count n(q) of every query, and ``out`` the mean of 0/1 indicator channels of V over
the visible set. The CPU tests at the top apply one plausible kernel bug at a time and show that the same rule rejects it.

Coverage (pairwise, not a full product; every case runs the forward and the whole backward; ids of test_attention_matches_fp64):
- ``flash_fwd`` / ``bwd_dkdv`` / ``bwd_dq`` <D=128, kDoc=0>: causal S128 (minimum, one 128-row block), causal odd H = 5 sharp,
  1B causal + RoPE, non-causal GQA-4 rising, S8192 causal rising (a row crosses 128 key tiles)
- <D=64, kDoc=0>: non-causal S128 odd H = 3 sharp, 150M non-causal, GQA-4 S4096 causal rising, the autograd node (causal GQA-4)
- <D=128, kDoc=1>: W = 1 odd H = 3 GQA-3, group 16 EOS at 0 / S-1, W = S, W = 100 + mref documents, 1B documents at tile
  edges rising, 7B GQA-4 S4096 random documents + W = 100, the autograd node (RoPE + documents)
- <D=64, kDoc=1>: W > S + EOS at 0 / S-1, odd H = 5 group 5 tile-edge documents (mref), W = 65 + mref documents, group 8
  W = 63 sharp, 150M W = 64 sharp + RoPE, S8192 random documents + W = S - 1
- ``bwd_delta_kernel``: every case (odd H = 3 / 5 at both D leave lanes of the last warp step idle)
- ``doc_bounds_kernel``: S = 100, 128, 255 (idle threads), 256, 300, 1000 (S % 256 != 0), 32768 (128 positions per thread) ×
  every EOS layout and window, all-EOS rows, B = 3 rows that differ: test_doc_bounds_bitwise
- document starts at 63, 64, 65, 127, 128, 160, and 96 / 192 (32-row dK/dV tiles); one-token documents; EOS at 0 and S - 1;
  consecutive EOS: the "edges" and "ends" layouts; W ∈ {1, 63, 64, 65, 100, S-1, S, S+5}
- softmax regimes: plain randn·0.7, sharp (log2-domain scores to about ±60), rising (key magnitudes grow along the row: the
  running max moves on late tiles, so every tile rescales), mref (documents start inside a 64-row block: the block's first key
  tile is fully masked for its later rows, the kDoc mref = 0 path)
- fused inverse RoPE in the backward at D = 64 and 128, tables longer than S; autograd node at both D: test_autograd_node_*
- visible-set probes over every mask / boundary layout at both D, S up to 8192: test_visible_set_probe
"""

import math

import numpy as np
import pytest
import torch
from test_kernel_edges_gpu import ROPE_ATOL, U, U32, _gemm_atol, _rejects, assert_elementwise, rope64

from prime_b200.ops import reference as Rf

LOG2E = 1.0 / math.log(2.0)
LN2 = math.log(2.0)
EOS = 7

# -------------------------------------------------------------------------------------------------- tolerances, one per rounding
P_ROUND = U  # P (and dS) rounded to bf16 before the tensor-core P·V, Pᵀ·dO, dS·K, dSᵀ·Q products
EX2 = 2.0**-22  # ex2.approx.ftz.f32: relative error below 2^-22 (results under 2^-126 flush to 0, far below 2^-100 of any row)
SCORE_ROUND = 4 * U32  # s·scale_log2 in fp32: the product, and scale_log2 = fl(fl(1/√D)·fl(log2 e)) (relative, on |s|)
OUT_RTOL = U + 2.0**-22  # the bf16 store of out, after the fp32 reciprocal 1/l and the product o·(1/l)
LSE_RTOL = 2.0**-22  # log2f (1 ulp) and the fp32 add m + log2 l (1 ulp)
DELTA_RTOL = 2 * U32  # the fp32 scale (1/√D rounded) and the product acc·scale
DELTA_ATOL = 16 * U32  # 8 serial fp32 FMAs per lane and <= 4 shuffle adds over the D products dO·out
GRAD_RTOL = U  # the bf16 store of dQ / dK / dV (the store also rounds the kernel's own error: allowances carry a factor 1 + U)
PROBE_LSE_RTOL = 2.0**-23  # probe: s = 0 and l = n are exact, lse2 = 0 + log2f(n) is within 1 ulp
PROBE_LSE_ATOL = 2.0**-22  # probe: slack for one ex2.approx(0) ulp on l; log2 of n ± 1 differs from log2 n by more than 2^-14
PROBE_OUT_RTOL = U + 2.0**-22  # probe: o is an exact integer count; 1/l, o·(1/l) in fp32 and one bf16 store


def _acc(n: int) -> float:
    """fp32 tensor-core accumulation of n products (or n fp32 adds): <= n·2^-24 of Σ|terms|, doubled for the truncating
    alignment of partial sums (the GEMM rule of test_kernel_edges_gpu.py)."""
    return _gemm_atol(n)


def _l_rel(S: int) -> float:
    """Relative error of the softmax denominator l over S/64 key tiles: ex2.approx of each term and of each tile's corr factor,
    one fp32 rounding per corr product, and <= 16 serial adds per lane per tile + one per tile + 2 shuffle adds."""
    T = S // 64
    return EX2 + T * (EX2 + U32) + (T + 18) * U32


# -------------------------------------------------------------------------------------------------- fp64 oracle
def _mask(S, causal, lo_row, dev, diag=0):
    """[S, S] visible set of one row: k <= q + diag (causal) and k >= lo[q]."""
    i = torch.arange(S, device=dev)
    vis = i.view(1, S) <= i.view(S, 1) + diag if causal else torch.ones(S, S, dtype=torch.bool, device=dev)
    if lo_row is not None:
        vis = vis & (i.view(1, S) >= lo_row.to(dev).long().view(S, 1))
    return vis


def _fp32(x: float) -> float:
    return float(torch.tensor(x, dtype=torch.float32))


def attn64(qkv, H, Hkv, causal, lo=None, dout=None, out_k=None, rope=None, diag=0, head_of=None):
    """fp64 reference of every kernel output: {name: (ref, rtol, allowance)}. Forward: out [B, S, H·D], lse2 [B, H, S]. With
    ``dout`` and the kernel's bf16 ``out_k``: delta [B, H, S], dq [B, S, H, D], dk / dv [B, S, Hkv, D] (summed over the GQA group,
    dq / dk un-rotated by ``rope = (cos, sin)``). ``diag`` / ``head_of`` only serve the CPU mutants (a shifted causal edge, another
    head map)."""
    B, S, Wd = qkv.shape
    D = Wd // (H + 2 * Hkv)
    grp = H // Hkv
    dev = qkv.device
    scale = _fp32(1.0 / math.sqrt(D))  # the fp32 value the launcher receives
    x = qkv.view(B, S, H + 2 * Hkv, D)
    f64 = dict(dtype=torch.float64, device=dev)
    out, out_al = torch.zeros(B, S, H, D, **f64), torch.zeros(B, S, H, D, **f64)
    lse2, lse_al = torch.zeros(B, H, S, **f64), torch.zeros(B, H, S, **f64)
    bwd = dout is not None
    if bwd:
        do4, o4 = dout.view(B, S, H, D), out_k.view(B, S, H, D)
        delta, delta_al = torch.zeros(B, H, S, **f64), torch.zeros(B, H, S, **f64)
        dq, dq_al = torch.zeros(B, S, H, D, **f64), torch.zeros(B, S, H, D, **f64)
        dk, dk_al = torch.zeros(B, S, Hkv, D, **f64), torch.zeros(B, S, Hkv, D, **f64)
        dv, dv_al = torch.zeros(B, S, Hkv, D, **f64), torch.zeros(B, S, Hkv, D, **f64)
    for b in range(B):
        vis = _mask(S, causal, None if lo is None else lo[b], dev, diag)
        for h in range(H):
            hk = head_of(h) if head_of else h // grp
            q, k, v = (x[b, :, i].double() for i in (h, H + hk, H + Hkv + hk))
            z = (q @ k.t()) * scale
            za = (q.abs() @ k.abs().t()) * scale
            zm = z.masked_fill(~vis, -math.inf)
            m = zm.amax(-1, keepdim=True)
            e = torch.exp(zm - m)
            l_ = e.sum(-1, keepdim=True)
            p = e / l_
            out[b, :, h] = p @ v
            lse2[b, h] = (m + l_.log()).squeeze(-1) * LOG2E
            # worst-case error of one fp32 score in the log2 domain: the D-term tensor-core dot, then the scale product
            serr = (_acc(D) * za.masked_fill(~vis, 0).amax(-1) + SCORE_ROUND * z.abs().masked_fill(~vis, 0).amax(-1)) * LOG2E
            # out = Σ bf16(e)·v / Σ e: P's rounding, the relative error of each e (score, ex2), the P·V accumulation
            out_al[b, :, h] = (1 + U) * (P_ROUND + 2 * LN2 * serr + 2 * EX2 + _acc(2 * S)).view(S, 1) * (p @ v.abs())
            # worst case: on random data the fp32 dot errs ~√D below D·2^-24·Σ|q·k|; the Q = 0 probe holds lse2 to one ulp
            lse_al[b, h] = serr + _l_rel(S) * LOG2E
            if not bwd:
                continue
            do, o = do4[b, :, h].double(), o4[b, :, h].double()
            dsum = (do * o).sum(-1)
            dabs = (do * o).abs().sum(-1)
            delta[b, h] = scale * dsum
            delta_al[b, h] = DELTA_ATOL * scale * dabs
            d_err = DELTA_RTOL * scale * dsum.abs() + delta_al[b, h]
            # relative error of the backward's p = exp2(s·scale·log2e - lse2): its own score, the kernel's lse2, ex2.approx
            eps_p = (LN2 * (serr + lse_al[b, h]) + EX2).view(S, 1)
            dP = do @ v.t()
            mag = p * (scale * dP.abs() + (scale * dsum).abs().view(S, 1))  # the terms of dS = p·(scale·dP - delta)
            al_ds = (P_ROUND + eps_p) * mag + p * (scale * _acc(D) * (do.abs() @ v.abs().t()) + d_err.view(S, 1))
            dS = p * (scale * dP - (scale * dsum).view(S, 1))
            dq[b, :, h] = dS @ k
            dq_al[b, :, h] = (1 + U) * (al_ds @ k.abs() + _acc(S) * (mag @ k.abs()))
            dk[b, :, hk] += dS.t() @ q
            dk_al[b, :, hk] += (1 + U) * (al_ds.t() @ q.abs() + _acc(S * grp) * (mag.t() @ q.abs()))
            dv[b, :, hk] += p.t() @ do
            dv_al[b, :, hk] += (1 + U) * (((P_ROUND + eps_p + _acc(S * grp)) * p).t() @ do.abs())
    res = {"out": (out.reshape(B, S, H * D), OUT_RTOL, out_al.reshape(B, S, H * D)), "lse2": (lse2, LSE_RTOL, lse_al)}
    if not bwd:
        return res
    if rope is not None:
        dq, dq_al = _unrotate(dq, dq_al, rope)
        dk, dk_al = _unrotate(dk, dk_al, rope)
    res.update(delta=(delta, DELTA_RTOL, delta_al), dq=(dq, GRAD_RTOL, dq_al), dk=(dk, GRAD_RTOL, dk_al), dv=(dv, GRAD_RTOL, dv_al))
    return res


def _unrotate(g, al, rope):
    """Inverse RoPE of a gradient [B, S, heads, D] and its allowance: a rotated element mixes both errors of its pair, plus the
    fp32 rotation arithmetic."""
    cos, sin = rope
    B, S, Hh, D = g.shape
    ref, pair = rope64(g, cos, sin, -1.0)
    al_pair = al.reshape(B, S, Hh, D // 2, 2).sum(-1, keepdim=True).expand(B, S, Hh, D // 2, 2).reshape(B, S, Hh, D)
    return ref, al_pair + (1 + U) * ROPE_ATOL * pair


def check(got, entry, what, rtol=None, atol=None) -> float:
    """The rule for one output; ``rtol`` / ``atol`` replace the oracle's (probes: an exact rule with a constant floor)."""
    ref, r, allow = entry
    if rtol is None:
        return assert_elementwise(got, ref, r, 1.0, what, allow)
    return assert_elementwise(got, ref, rtol, atol, what, 1.0)


def _rejected(got, entry) -> bool:
    ref, r, allow = entry
    return _rejects(got, ref, r, 1.0, allow)


# -------------------------------------------------------------------------------------------------- inputs and masks
def _indicator(idx: torch.Tensor, D: int) -> torch.Tensor:
    """0/1 channels of an index: bit c of idx for c < 14, then (idx mod (c - 12)) == 0."""
    c = torch.arange(D)
    bits = (idx.view(-1, 1) >> c.clamp(max=13).view(1, -1)) & 1
    mods = (idx.view(-1, 1) % (c - 12).clamp(min=1).view(1, -1)) == 0
    return torch.where(c.view(1, -1) < 14, bits.bool(), mods).double()


def _inputs(B, S, H, Hkv, D, regime, seed):
    """bf16 (qkv, dout) on the CPU. plain: randn·0.7. sharp / mref: Q and K ×3.2, log2-domain scores to about ±60. rising: K grows
    along the row (×0.3 → ×3.3). probe: Q = 0, K random, V and dO 0/1 indicator channels of the key / query position."""
    g = torch.Generator().manual_seed(seed)
    nh = H + 2 * Hkv
    x = torch.randn(B, S, nh, D, generator=g, dtype=torch.float64)
    dout = torch.randn(B, S, H, D, generator=g, dtype=torch.float64)
    pos = torch.arange(S)
    if regime == "plain":
        x *= 0.7
    elif regime in ("sharp", "mref"):
        x[:, :, : H + Hkv] *= 3.2
    elif regime == "rising":
        x[:, :, H : H + Hkv] *= (0.3 + 3.0 * pos / S).view(1, S, 1, 1)
    elif regime == "probe":
        x[:, :, :H] = 0
        for hk in range(Hkv):
            x[:, :, H + Hkv + hk] = _indicator(pos + 1237 * hk, D)
        dout = _indicator(pos, D).view(1, S, 1, D).expand(B, S, H, D).clone()
    else:
        raise KeyError(regime)
    return x.reshape(B, S, nh * D).to(torch.bfloat16), dout.reshape(B, S, H * D).to(torch.bfloat16)


def _eos_positions(layout: str, S: int, b: int) -> list[int]:
    """EOS positions of row b. edges: documents start at 63, 64, 65, 127, 128, 160 (one-token documents at 63 and 64, consecutive
    EOS), odd rows shifted by 32 (starts on 32-row dK/dV tiles: 96, 160, 192). ends: EOS at 0, S - 1 and a consecutive pair.
    mref: documents start at 100, 164, 301 (inside 64-row blocks). random: lengths 1-300. all: every token is EOS."""
    if layout == "edges":
        pos = [62, 63, 64, 126, 127, 159] + ([S // 2 + 31] if S > 256 else [])
        pos = [p + 32 * (b % 2) for p in pos]
    elif layout == "ends":
        pos = [0, S // 3 + b, S // 3 + b + 1, S - 1]
    elif layout == "mref":
        pos = [99 + 64 * (b % 2), 163, 300]
    elif layout == "random":
        g = np.random.default_rng(1000 * b + S)
        pos, p = [], int(g.integers(0, 40))
        while p < S:
            pos.append(p)
            p += int(g.integers(1, 300))
    elif layout == "all":
        pos = list(range(S))
    elif layout == "none":
        pos = []
    else:
        raise KeyError(layout)
    return sorted({p for p in pos if 0 <= p < S})


def _tokens(layout: str | None, B: int, S: int) -> torch.Tensor:
    rows = []
    for b in range(B):
        row = np.random.default_rng(b).integers(8, 200, size=S)  # never EOS
        row[_eos_positions(layout or "none", S, b)] = EOS
        rows.append(row)
    return torch.tensor(np.stack(rows), dtype=torch.int64)


def _bounds(layout, window, B, S):
    """reference.document_bounds of the case's rows (None when the case has neither documents nor a window)."""
    if layout is None and window is None:
        return None
    return Rf.document_bounds(_tokens(layout, B, S), EOS if layout else None, window)


# -------------------------------------------------------------------------------------------------- CPU: the rule rejects bugs
def _rounded(res: dict) -> dict:
    """What a correct kernel stores: bf16 out and gradients, fp32 lse2 and delta."""
    dt = {"lse2": torch.float32, "delta": torch.float32}
    return {n: e[0].to(dt.get(n, torch.bfloat16)) for n, e in res.items()}


def _cpu_case(B=1, S=256, H=4, Hkv=2, D=64, causal=True, layout=None, window=None, regime="plain", rope=None, **bug):
    """(reference entries, what a kernel with ``bug`` would store) on random inputs; no bug = a correct kernel."""
    qkv, dout = _inputs(B, S, H, Hkv, D, regime, seed=S + D)
    b = _bounds(layout, window, B, S)
    lo = None if b is None else b[0]
    out_k = attn64(qkv, H, Hkv, causal, lo)["out"][0].to(torch.bfloat16)
    ref = attn64(qkv, H, Hkv, causal, lo, dout, out_k, rope)
    lo_bug = lo if "lo" not in bug else bug.pop("lo")
    out_bug = attn64(qkv, H, Hkv, causal, lo_bug, **bug)["out"][0].to(torch.bfloat16)
    got = _rounded(attn64(qkv, H, Hkv, causal, lo_bug, dout, out_bug, rope, **bug))
    return ref, got


def test_checker_accepts_a_correct_kernel():
    for kw in ({}, {"causal": False}, {"layout": "edges", "window": 65}, {"regime": "sharp", "layout": "mref"}):
        ref, got = _cpu_case(**kw)
        for n, e in ref.items():
            assert not _rejected(got[n], e), (kw, n)


@pytest.mark.parametrize("diag", [1, -1], ids=["sees_next_key", "misses_diagonal"])
def test_checker_rejects_causal_edge_off_by_one(diag):
    ref, got = _cpu_case(S=128, diag=diag)
    assert _rejected(got["out"], ref["out"]) and _rejected(got["dv"], ref["dv"])


@pytest.mark.parametrize("shift", [1, -1])
def test_checker_rejects_document_start_off_by_one(shift):
    ref, got = _cpu_case(layout="edges", lo=_bounds("edges", None, 1, 256)[0] + shift)
    assert _rejected(got["out"], ref["out"]) and _rejected(got["dk"], ref["dk"])


@pytest.mark.parametrize("dw", [1, -1])
def test_checker_rejects_window_off_by_one(dw):
    ref, got = _cpu_case(window=63, lo=_bounds(None, 63 + dw, 1, 256)[0])
    assert _rejected(got["out"], ref["out"]) and _rejected(got["dv"], ref["dv"])


def test_checker_rejects_gqa_head_map_modulo():
    ref, got = _cpu_case(H=4, Hkv=2, head_of=lambda h: h % 2)
    assert _rejected(got["out"], ref["out"])


def _flash64(z, v, vis, skip_corr_tile=None):
    """The forward's online softmax over 64-key tiles in fp64 (kDoc mref rule included); ``skip_corr_tile``: that tile's o is not
    rescaled by corr (l is)."""
    S = z.shape[0]
    m = torch.full((S, 1), -math.inf, dtype=torch.float64)
    l_ = torch.zeros(S, 1, dtype=torch.float64)
    o = torch.zeros(S, v.shape[1], dtype=torch.float64)
    for j in range(0, S, 64):
        zt = z[:, j : j + 64].masked_fill(~vis[:, j : j + 64], -math.inf)
        mx = torch.maximum(m, zt.amax(-1, keepdim=True))
        mref = torch.where(mx == -math.inf, torch.zeros_like(mx), mx)
        corr, e = torch.exp(m - mref), torch.exp(zt - mref)
        l_ = l_ * corr + e.sum(-1, keepdim=True)
        o = (o if j // 64 == skip_corr_tile else o * corr) + e @ v[j : j + 64]
        m = mx
    return o / l_


def test_checker_rejects_skipped_corr_rescale():
    S, D = 256, 64
    qkv, _ = _inputs(1, S, 1, 1, D, "rising", seed=3)
    ref = attn64(qkv, 1, 1, False)["out"]
    q, k, v = (t.double() for t in qkv.view(S, 3, D).unbind(1))
    z = (q @ k.t()) * _fp32(1.0 / math.sqrt(D))
    vis = torch.ones(S, S, dtype=torch.bool)
    assert not _rejected(_flash64(z, v, vis).view(1, S, D).to(torch.bfloat16), ref)
    assert _rejected(_flash64(z, v, vis, skip_corr_tile=2).view(1, S, D).to(torch.bfloat16), ref)


def test_checker_rejects_lse2_in_natural_log():
    ref, got = _cpu_case(regime="sharp")
    assert _rejected(got["lse2"] * LN2, ref["lse2"])


def test_checker_rejects_delta_missing_scale():
    ref, got = _cpu_case()
    assert _rejected(got["delta"] / _fp32(1.0 / 8.0), ref["delta"])


def test_checker_rejects_dkdv_dropping_the_last_query_tile():
    S, H, Hkv, D = 256, 4, 2, 64
    qkv, dout = _inputs(1, S, H, Hkv, D, "plain", seed=S + D)
    out_k = attn64(qkv, H, Hkv, True)["out"][0].to(torch.bfloat16)
    ref = attn64(qkv, H, Hkv, True, None, dout, out_k)
    cut = dout.clone()
    cut[:, S - 32 :] = 0  # the dK/dV loop stops one 32-query tile early: the last tile's dO (and so its dP, delta) never enter
    got = _rounded(attn64(qkv, H, Hkv, True, None, cut, out_k))
    assert _rejected(got["dv"], ref["dv"]) and _rejected(got["dk"], ref["dk"])


def test_checker_rejects_inverse_rope_with_forward_sign():
    S, D = 128, 64
    cos, sin = Rf.rope_tables(S + 40, D, 500000.0)
    ref, got = _cpu_case(S=S, rope=(cos, sin))
    _, fwd_sign = _cpu_case(S=S, rope=(cos, -sin))  # un-rotating by -sin rotates forward
    assert not _rejected(got["dq"], ref["dq"]) and not _rejected(got["dk"], ref["dk"])
    assert _rejected(fwd_sign["dq"], ref["dq"]) and _rejected(fwd_sign["dk"], ref["dk"])


def _probe_lse2(S, causal, lo, diag=0):
    """Probe forward: with Q = 0 every visible key scores 0, so lse2[q] = log2 n(q) of the visible count."""
    q = torch.arange(S, dtype=torch.float64)
    hi = torch.clamp(q + diag, max=S - 1) if causal else torch.full_like(q, S - 1)
    return torch.log2(hi - (lo.double() if lo is not None else 0) + 1)


@pytest.mark.parametrize("S", [4096, 8192])
def test_probe_rejects_off_by_one_visible_sets_at_long_rows(S):
    """At S >= 4096 one key more or less moves a random-input row by less than a bf16 ulp; the probe's lse2 = log2 n(q) does not
    miss it: a causal edge (rows up to S keys), a document start ("edges": documents of S/2 tokens) or a window of S/2 + 3 keys
    off by one, in either direction."""
    lo_doc = _bounds("edges", None, 1, S)[0][0]
    W = S // 2 + 3
    lo_win = _bounds(None, W, 1, S)[0][0]
    tol = (PROBE_LSE_RTOL, PROBE_LSE_ATOL, 1.0)
    good = {"causal": _probe_lse2(S, True, None), "doc": _probe_lse2(S, True, lo_doc), "win": _probe_lse2(S, True, lo_win)}
    for exact in good.values():
        assert not _rejects(exact.float(), exact, *tol)
    for d in (1, -1):
        assert _rejects(_probe_lse2(S, True, None, diag=d).float(), good["causal"], *tol)
        assert _rejects(_probe_lse2(S, True, lo_doc + d).float(), good["doc"], *tol)
        assert _rejects(_probe_lse2(S, True, _bounds(None, W + d, 1, S)[0][0]).float(), good["win"], *tol)


# -------------------------------------------------------------------------------------------------- GPU
def _dev():
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def native():
    from prime_b200.ops import _lib

    return _lib.load()  # a GPU box without the native library is a hard failure, never a silent fallback


def _launch(lib, qkv, dout, H, Hkv, causal, doc, rope):
    """pb_flash_attn_fwd then pb_flash_attn_bwd on NaN-filled outputs → {out, lse2, delta, dqkv}."""
    from prime_b200.ops import _lib
    from prime_b200.ops.functional import _ptr, _stream

    B, S, Wd = qkv.shape
    D = Wd // (H + 2 * Hkv)
    scale = 1.0 / math.sqrt(D)
    dev = qkv.device
    out = torch.full((B, S, H * D), math.nan, dtype=torch.bfloat16, device=dev)
    lse2 = torch.full((B, H, S), math.nan, dtype=torch.float32, device=dev)
    delta = torch.full((B, H, S), math.nan, dtype=torch.float32, device=dev)
    dqkv = torch.full_like(qkv, math.nan)
    ds, de = (None, None) if doc is None else (_ptr(doc[0]), _ptr(doc[1]))
    cos, sin = (None, None) if rope is None else (_ptr(rope[0]), _ptr(rope[1]))
    _lib.check(lib.pb_flash_attn_fwd(_ptr(qkv), _ptr(out), _ptr(lse2), ds, B, S, H, Hkv, D, scale, int(causal), _stream()), "fwd")
    _lib.check(lib.pb_flash_attn_bwd(_ptr(qkv), _ptr(out), _ptr(dout), _ptr(lse2), _ptr(delta), _ptr(dqkv), ds, de, B, S, H, Hkv, D,
                                     scale, int(causal), cos, sin, _stream()), "bwd")  # fmt: skip
    torch.cuda.synchronize()
    return {"out": out, "lse2": lse2, "delta": delta, "dqkv": dqkv}


def _native_bounds(native, layout, window, B, S):
    """pb_doc_bounds of the case's rows, asserted bit for bit against reference.document_bounds."""
    from prime_b200 import ops

    if layout is None and window is None:
        return None, None
    tok = _tokens(layout, B, S)
    doc = ops.document_bounds(tok.to(_dev()), EOS if layout else None, window)
    ref = Rf.document_bounds(tok, EOS if layout else None, window)
    assert torch.equal(doc[0].cpu(), ref[0]) and torch.equal(doc[1].cpu(), ref[1]), "pb_doc_bounds != reference.document_bounds"
    return doc, ref[0].to(_dev())


def _check_case(res, ref, H, Hkv, tag):
    B, S, _ = res["out"].shape
    g = res["dqkv"].view(B, S, H + 2 * Hkv, -1)
    got = {"out": res["out"], "lse2": res["lse2"], "delta": res["delta"], "dq": g[:, :, :H], "dk": g[:, :, H : H + Hkv],
           "dv": g[:, :, H + Hkv :]}  # fmt: skip
    return {n: check(got[n], ref[n], f"{n} {tag}") for n in got}


def _run_and_check(native, B, S, H, Hkv, D, causal, layout, window, regime, rope_len, tag):
    dev = _dev()
    qkv, dout = (t.to(dev) for t in _inputs(B, S, H, Hkv, D, regime, seed=S * 7 + H * 3 + D))
    doc, lo = _native_bounds(native, layout, window, B, S)
    rope = Rf.rope_tables(rope_len, D, 500000.0, device=dev) if rope_len else None
    res = _launch(native, qkv, dout, H, Hkv, causal, doc, rope)
    ref = attn64(qkv, H, Hkv, causal, lo, dout, res["out"], rope)
    return res, ref, _check_case(res, ref, H, Hkv, tag), (qkv, dout, doc, rope)


# id, B, S, H, Hkv, D, causal, EOS layout, window, regime, RoPE table length (0 = none)
CASES = [
    ("S128_causal_d128", 1, 128, 2, 1, 128, True, None, None, "plain", 0),
    ("S128_noncausal_oddH3_d64", 2, 128, 3, 3, 64, False, None, None, "sharp", 0),
    ("S128_w1_oddH3_d128", 1, 128, 3, 1, 128, True, None, 1, "plain", 0),
    ("S128_wgtS_ends_d64", 2, 128, 2, 2, 64, True, "ends", 133, "rising", 0),
    ("S256_oddH5_causal_d128", 1, 256, 5, 5, 128, True, None, None, "sharp", 0),
    ("S256_oddH5_g5_edges_mref_d64", 2, 256, 5, 1, 64, True, "edges", None, "mref", 0),
    ("S256_g16_ends_d128", 1, 256, 16, 1, 128, True, "ends", None, "plain", 0),
    ("S256_wS_d128", 1, 256, 2, 2, 128, True, None, 256, "plain", 0),
    ("S384_w65_mref_d64", 2, 384, 4, 2, 64, True, "mref", 65, "mref", 0),
    ("S512_g8_w63_sharp_d64", 2, 512, 8, 1, 64, True, None, 63, "sharp", 0),
    ("S512_w100_mref_d128", 1, 512, 4, 1, 128, True, "mref", 100, "sharp", 0),
    ("S512_noncausal_g4_rising_d128", 1, 512, 8, 2, 128, False, None, None, "rising", 0),
    ("S1024_1B_causal_rope_d128", 2, 1024, 16, 16, 128, True, None, None, "plain", 1100),
    ("S1024_1B_edges_rising_d128", 1, 1024, 16, 16, 128, True, "edges", None, "rising", 0),
    ("S1024_150M_noncausal_d64", 1, 1024, 16, 16, 64, False, None, None, "plain", 0),
    ("S1024_150M_w64_rope_d64", 1, 1024, 16, 16, 64, True, None, 64, "sharp", 1090),
    ("S4096_7B_g4_random_w100_d128", 1, 4096, 8, 2, 128, True, "random", 100, "plain", 0),
    ("S4096_g4_causal_rising_d64", 1, 4096, 4, 1, 64, True, None, None, "rising", 0),
    ("S8192_long_causal_rising_d128", 1, 8192, 2, 1, 128, True, None, None, "rising", 0),
    ("S8192_long_random_wSm1_d64", 1, 8192, 2, 2, 64, True, "random", 8191, "plain", 0),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_attention_matches_fp64(native, case):
    """Forward (out, lse2) and backward (delta, dQ, dK, dV) of one case, every element against the fp64 oracle."""
    tag, *args = case
    _run_and_check(native, *args, tag)


# id, B, S, H, Hkv, D, causal, EOS layout, window
PROBES = [
    ("S256_noncausal_d64", 1, 256, 2, 1, 64, False, None, None),
    ("S256_noncausal_d128", 1, 256, 2, 2, 128, False, None, None),
    ("S256_causal_d128", 2, 256, 2, 2, 128, True, None, None),
    ("S512_edges_d64", 2, 512, 2, 1, 64, True, "edges", None),
    ("S512_edges_d128", 2, 512, 4, 2, 128, True, "edges", None),
    ("S256_ends_d64", 2, 256, 3, 3, 64, True, "ends", None),
    ("S256_ends_d128", 2, 256, 2, 1, 128, True, "ends", None),
    ("S384_mref_w65_d64", 2, 384, 2, 1, 64, True, "mref", 65),
    ("S384_mref_d128", 2, 384, 2, 1, 128, True, "mref", None),
    ("S256_w1_d64", 1, 256, 2, 2, 64, True, None, 1),
    ("S256_w63_d128", 1, 256, 2, 1, 128, True, None, 63),
    ("S256_w64_d64", 1, 256, 2, 1, 64, True, None, 64),
    ("S256_w100_all_d128", 1, 256, 2, 1, 128, True, "all", 100),
    ("S256_wS_d64", 1, 256, 2, 1, 64, True, None, 256),
    ("S256_wgtS_d128", 1, 256, 2, 2, 128, True, None, 300),
    ("S4096_random_w100_d128", 1, 4096, 2, 1, 128, True, "random", 100),
    ("S8192_causal_d64", 1, 8192, 2, 1, 64, True, None, None),
    ("S8192_random_wSm1_d128", 1, 8192, 2, 1, 128, True, "random", 8191),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", PROBES, ids=[c[0] for c in PROBES])
def test_visible_set_probe(native, case):
    """Q = 0: lse2[q] = log2 n(q) to one ulp and out = the mean of V's 0/1 channels over the visible set to one bf16 rounding, for
    every query; dO = 0/1 channels of the query position, so dV[k] sums 1/n(q) over exactly the queries that see k (full rule)."""
    tag, B, S, H, Hkv, D, causal, layout, window = case
    res, ref, _, _ = _run_and_check(native, B, S, H, Hkv, D, causal, layout, window, "probe", 0, f"probe {tag}")
    check(res["lse2"], ref["lse2"], f"probe exact lse2 {tag}", PROBE_LSE_RTOL, PROBE_LSE_ATOL)
    check(res["out"], ref["out"], f"probe exact out {tag}", PROBE_OUT_RTOL, 0.0)


@pytest.mark.gpu
@pytest.mark.parametrize("S", [100, 128, 255, 256, 300, 1000, 32768])
def test_doc_bounds_bitwise(native, S):
    """pb_doc_bounds against reference.document_bounds bit for bit: B = 3 rows with different boundaries, every EOS layout (and an
    all-EOS row) × no window, W ∈ {1, 63, 64, 65, 100, S - 1, S, S + 5}."""
    from prime_b200 import ops

    for layout in ("none", "edges", "ends", "mref", "random", "all"):
        tok = _tokens(layout, 3, S)
        tok[2] = torch.from_numpy(np.random.default_rng(S).integers(0, 12, size=S))  # ~1 EOS in 12, runs of EOS
        for window in (None, 1, 63, 64, 65, 100, S - 1, S, S + 5):
            got = ops.document_bounds(tok.to(_dev()), EOS, window)
            ref = Rf.document_bounds(tok, EOS, window)
            assert torch.equal(got[0].cpu(), ref[0]), f"doc_start S={S} {layout} W={window}"
            assert torch.equal(got[1].cpu(), ref[1]), f"doc_end S={S} {layout} W={window}"


@pytest.mark.gpu
def test_autograd_node_d128_rope_documents(native):
    """ops.rope_attention_qkv(impl="native", pre_rotated=True) with documents: the autograd node's out and dQKV (inverse RoPE fused
    into the backward) equal the direct launches bit for bit, and those pass the fp64 rule."""
    from prime_b200 import ops

    B, S, H, Hkv, D = 1, 512, 4, 2, 128
    res, _, _, (qkv, dout, doc, rope) = _run_and_check(native, B, S, H, Hkv, D, True, "random", None, "plain", S + 64, "autograd d128")
    x = qkv.clone().requires_grad_(True)
    out = ops.rope_attention_qkv(x, rope[0], rope[1], H, Hkv, causal=True, impl="native", pre_rotated=True, doc=doc)
    out.backward(dout)
    torch.cuda.synchronize()
    assert torch.equal(out.detach(), res["out"]) and torch.equal(x.grad, res["dqkv"])


@pytest.mark.gpu
def test_autograd_node_d64_causal(native):
    """ops.attention_qkv(impl="native"), causal GQA at D = 64: out and dQKV equal the direct launches bit for bit."""
    from prime_b200 import ops

    B, S, H, Hkv, D = 2, 256, 4, 1, 64
    res, _, _, (qkv, dout, _, _) = _run_and_check(native, B, S, H, Hkv, D, True, None, None, "plain", 0, "autograd d64")
    x = qkv.clone().requires_grad_(True)
    out = ops.attention_qkv(x, H, Hkv, causal=True, impl="native")
    out.backward(dout)
    torch.cuda.synchronize()
    assert torch.equal(out.detach(), res["out"]) and torch.equal(x.grad, res["dqkv"])
