"""The per-token kernels (RMSNorm forward / backward, fused cross-entropy, SwiGLU, in-place RoPE, the MXFP8 quantiser and the fused
GEMM epilogues) against an fp64 oracle, on every dispatch branch of their launchers.

Every oracle is computed in plain torch from ``.double()`` of the exact tensors the kernel read; where a kernel rounds on purpose
the oracle takes the kernel's own rounded tensor (which is checked separately) or rounds at the same point. One per-element rule
decides, for every element:

    |got - ref| <= rtol·|ref| + atol_frac·scale + UNDERFLOW

``scale`` is max|ref| over the row unless a test passes the magnitude of the terms that cancel in that element (the sum of
|terms| of an fp32 reduction, |A|·|B|ᵀ of a GEMM, the gradient scale at the cross-entropy target). Each tolerance states the
rounding it covers. The CPU tests at the top apply one plausible kernel bug to a correct result and show that the same rule
with the same tolerances rejects it, so the GPU assertions are not vacuous.

Coverage of the launcher branches (test names below):
- ``rmsnorm_fwd_kernel`` MAXV = 1 / 2 / 4 / 8 and nvec < 32 (idle lanes, D = 64 / 200): test_rmsnorm_fwd_every_maxv
- ``rmsnorm_bwd_kernel`` R > pb_rmsnorm_bwd_grid (persistent rows with next-row prefetch), HAS_DRES, dw_accumulate = 1 into
  main_grad and the fresh-grad overwrite: test_rmsnorm_bwd_persistent_rows_into_main_grad
- ``cross_entropy_reg_kernel`` (V <= 32768, V = 8: one vector per row) and ``cross_entropy_kernel`` (V = 32776, 128256), targets
  at column 0 and V - 1, large logit spread, both ``unit_upstream`` values, ``loss_acc`` over two calls:
  test_cross_entropy_both_kernels; every target ignored: test_cross_entropy_all_targets_ignored
- ``swiglu_fwd/bwd_kernel`` with |gate| beyond the __expf overflow: test_swiglu_kernels_saturated_gate
- ``rope_inplace_kernel`` with a table longer than S, B = 3, GQA at D = 64: test_rope_inplace_long_table
- GEMM EPI = 2 / 3 with tail rows and FF = 64, and the ``_gemm_epi`` M <= 128 fallbacks: test_gemm_swiglu_epilogues_and_fallbacks
- GEMM EPI = 1 with ``rope_cols`` ending inside a 128-column tile: test_gemm_rope_epilogue_partial_tile
- ``_gemm_epi`` fallbacks reached from ``gemm_wgather`` (ZeRO-3, one rank): test_wgather_swiglu_fallbacks
- ``quantize_mxfp8[_t]_kernel`` all-zero, power-of-two, subnormal and negative-only blocks: test_quantize_mxfp8_edge_blocks
"""

import math

import pytest
import torch

from prime_b200.ops import reference as Rf

U = 2.0**-8  # bf16 unit roundoff: 8-bit significand, round to nearest
U32 = 2.0**-24  # fp32 unit roundoff
# absolute floor: below 2^-100 the kernels' exp-based formulas underflow (g / (1 + __expf(-g)) = g / inf = 0 for g < -88.7, where
# the exact silu(g) is < 2^-121); no trained quantity lives there
UNDERFLOW = 2.0**-100

# -------------------------------------------------------------------------------------------------- tolerances, one per output
RMS_Y = U + 2.0**-14  # one bf16 rounding; fp32 sum of squares over <= 64 serial terms + tree and rsqrtf: < 2^-17 relative
RMS_DX = U + 2.0**-14  # one bf16 rounding of g·rs - h·coef (+ dres), fp32 terms accurate to ~2^-22
RMS_DX_ATOL = 2.0**-14  # cancellation between g·rs and h·coef, whose fp32 error is ~2^-22 of terms that are O(max|dx_row|)
DW_RTOL = 2.0**-16  # the kernel's rstd (rsqrtf of an fp32 mean) is within ~2^-18 of the fp64 one; one fp32 add into main_grad
DW_ATOL = 128 * U32  # fp32 column sums, <= 32 rows per CTA + 66 partials per lane + 8 lanes + 1 serial adds, of Σ|dy·h·rstd|
CE_EXP = 2.0**-14  # fp32 exp arguments of logits up to |z| ~ 200: ex2.approx + argument rounding < 2^-16 relative
ROPE_RTOL = U  # one bf16 rounding of the rotated pair
ROPE_ATOL = 2.0**-22  # a·c - b·s in fp32 cancels: error <= 2^-23·(|a| + |b|) (c, s are read exactly from the fp32 table)
SWIGLU_RTOL = U + 2.0**-14  # one bf16 rounding; __expf / ex2.approx and the division are good to ~2^-20 for |g| <= 128
SILU_D_ATOL = 2.0**-20  # sg + silu·(1 - sg) cancels near g = -1.28: fp32 error ~2^-22 of |sg| + |silu·(1 - sg)|
MX_RTOL = 2.0**-4  # e4m3 has a 3-bit mantissa: round to nearest is within 2^-4 relative for normal values
# e4m3 subnormals are spaced 2^-9·s (abs error 2^-10·s); the kernel's fp32 amax·fl(1/448) may round up to the next power of two at
# an exact power-of-two boundary, doubling s relative to the exact fp64 scale
MX_ATOL = 2.0**-9


def _gemm_atol(K: int) -> float:
    """fp32 accumulation of K products: <= K·2^-24·Σ|a·b|, doubled for the tensor core's truncating alignment of partial sums."""
    return 2 * K * U32


def assert_elementwise(got, ref, rtol, atol_frac, what, scale=None) -> float:
    """|got - ref| <= rtol·|ref| + atol_frac·scale + UNDERFLOW for EVERY element (NaN fails). ``scale`` defaults to max|ref| over
    the last dimension. Returns the largest error as a fraction of its bound; on failure reports the worst element and the count."""
    g = got.detach().double()
    r = ref.detach().double().to(g.device)
    if scale is None:
        scale = r.abs().amax(dim=-1, keepdim=True) if r.dim() else r.abs()
    bound = rtol * r.abs() + atol_frac * torch.as_tensor(scale, dtype=torch.float64, device=g.device) + UNDERFLOW
    err = (g - r).abs()
    ok = err <= bound
    frac = torch.where(ok, err / bound, torch.full_like(err, math.inf))
    worst = float(frac.max()) if frac.numel() else 0.0
    if not bool(ok.all()):
        n = int((~ok).sum())
        i = int(torch.argmax(torch.where(ok, err / bound, torch.full_like(err, math.inf)).nan_to_num(math.inf)))
        idx = tuple(int(v) for v in torch.unravel_index(torch.tensor(i), g.shape)) if g.dim() else ()
        gi, ri, ei, bi = (float(t.reshape(-1)[i]) for t in (g, r, err, bound.expand_as(g)))
        raise AssertionError(f"{what}: {n} of {g.numel()} elements out of bound; worst at {idx}: got {gi!r} ref {ri!r} |err| {ei:.3e} "
                             f"> bound {bi:.3e}")
    print(f"[bound] {what}: max |err|/bound = {worst:.3f}")
    return worst


def _rejects(got, ref, rtol, atol_frac, scale=None) -> bool:
    try:
        assert_elementwise(got, ref, rtol, atol_frac, "mutant", scale)
    except AssertionError:
        return True
    return False


# -------------------------------------------------------------------------------------------------- fp64 oracles
def rmsnorm64(h, w, eps=1e-5):
    h, w = h.double(), w.double()
    return h * torch.rsqrt(h.pow(2).mean(-1, keepdim=True) + eps) * w


def rmsnorm_bwd64(h, w, dy, eps=1e-5):
    """(dh, dw, Σ_rows |dy·h·rstd| per column) in fp64 by autograd."""
    h64 = h.double().requires_grad_(True)
    w64 = w.double().requires_grad_(True)
    rmsnorm64(h64, w64, eps).backward(dy.double())
    rstd = torch.rsqrt(h.double().pow(2).mean(-1, keepdim=True) + eps)
    return h64.grad, w64.grad, (dy.double() * h.double() * rstd).abs().reshape(-1, h.shape[-1]).sum(0)


def rope64(x, cos, sin, sign=1.0):
    """Interleaved-pair rotation of x [..., S, heads, D] by the fp32 tables (read exactly, as the kernels do); sign -1 = inverse."""
    S, D = x.shape[-3], x.shape[-1]
    xf = x.double().reshape(*x.shape[:-1], D // 2, 2)
    c = cos[:S].double().view(S, 1, D // 2)
    s = sign * sin[:S].double().view(S, 1, D // 2)
    a, b = xf[..., 0], xf[..., 1]
    out = torch.stack((a * c - b * s, a * s + b * c), dim=-1).reshape(x.shape)
    pair = (a.abs() + b.abs()).unsqueeze(-1).expand(*a.shape, 2).reshape(x.shape)
    return out, pair


def swiglu64(gu):
    g, u = gu.double().chunk(2, dim=-1)
    return torch.nn.functional.silu(g) * u


def swiglu_bwd64(gu, dh):
    """(d_gate_up, scale of the cancelling terms of d_gate) for d_gate = dh·u·silu'(g), d_up = dh·silu(g)."""
    g, u = gu.double().chunk(2, dim=-1)
    dh = dh.double()
    sg = torch.sigmoid(g)
    silu = g * sg
    dg = dh * u * (sg + silu * (1 - sg))
    return torch.cat((dg, dh * silu), dim=-1), (dh * u).abs() * (sg.abs() + (silu * (1 - sg)).abs())


def cross_entropy64(z, tgt, ignore_index, grad_scale):
    """(mean loss, d(mean loss)/dz · grad_scale, magnitude entering the fp32 loss arithmetic) of bf16 logits z [R, V] in fp64."""
    z64 = z.double()
    valid = tgt != ignore_index
    n = int(valid.sum())
    lse = torch.logsumexp(z64, dim=-1)
    t = tgt.clamp(min=0)
    zt = z64.gather(1, t.view(-1, 1)).squeeze(1)
    loss = ((lse - zt) * valid).sum() / max(n, 1)
    p = torch.softmax(z64, dim=-1)
    p[torch.arange(z.shape[0], device=z.device)[valid], t[valid]] -= 1.0
    grad = p * valid.view(-1, 1) * (grad_scale / max(n, 1))
    mag = ((z64.amax(-1).abs() + zt.abs() + (lse - z64.amax(-1))) * valid).sum() / max(n, 1)
    return loss, grad, mag


def _ce_target_scale(z, tgt, ignore_index, s):
    """At the target column the kernel subtracts ``s`` from p_t·s: those two terms, not the row maximum, set the rounding floor."""
    sc = torch.zeros(z.shape, dtype=torch.float64, device=z.device)
    valid = tgt != ignore_index
    sc[torch.arange(z.shape[0], device=z.device)[valid], tgt[valid]] = s
    return sc


def _ce_tolerances(V: int, unit_upstream: bool) -> tuple[float, float]:
    """(rtol, target atol_frac) of the CE gradient. V <= 32768 runs cross_entropy_reg_kernel, which stores e = exp(z - max) back in
    bf16 before scaling (a second rounding, elementwise.cu pass 2); ``unit_upstream=False`` multiplies the bf16 gradient by the
    upstream value in bf16 (a third)."""
    reg = V // 8 <= 512 * 8
    rounds = 1 + int(reg) + int(not unit_upstream)
    return rounds * U + CE_EXP, (U if reg else 0.0) + CE_EXP


def _gemm_ref(a, b):
    """fp64 a·bᵀ and the rounding scale |a|·|b|ᵀ of its fp32 accumulation."""
    a64, b64 = a.double(), b.double()
    return a64 @ b64.t(), a64.abs() @ b64.abs().t()


def _quant_oracle(x, transpose):
    """Exact fp64 power-of-two scale per 32-block along the contraction dimension, broadcast over the block's elements."""
    xf = (x.t() if transpose else x).double()
    rows, k = xf.shape
    amax = xf.view(rows, k // 32, 32).abs().amax(-1)
    e = torch.where(amax > 0, torch.ceil(torch.log2(amax / 448.0)), torch.full_like(amax, -126.0)).clamp(min=-126.0)
    return xf, torch.exp2(e).repeat_interleave(32, dim=1)


# -------------------------------------------------------------------------------------------------- CPU: the rule rejects bugs
def test_checker_rejects_swapped_rows():
    torch.manual_seed(0)
    x = torch.randn(6, 64, dtype=torch.bfloat16) * 3
    w = (1 + 0.5 * torch.randn(64)).to(torch.bfloat16)
    ref = rmsnorm64(x, w)
    y = Rf.rmsnorm(x, w)
    assert not _rejects(y, ref, RMS_Y, 0.0)
    assert _rejects(y[[0, 2, 1, 3, 4, 5]], ref, RMS_Y, 0.0)


def test_checker_rejects_dropped_tail_row():
    torch.manual_seed(1)
    K = 64
    a = torch.randn(300, K, dtype=torch.bfloat16)
    b = torch.randn(192, K, dtype=torch.bfloat16)
    ref, sc = _gemm_ref(a, b)
    c = (a.float() @ b.float().t()).to(torch.bfloat16)
    assert not _rejects(c, ref, U, _gemm_atol(K), sc)
    for garbage in (torch.zeros_like(c[-1]), torch.empty_like(c[-1]).fill_(float("nan"))):
        bad = c.clone()
        bad[-1] = garbage
        assert _rejects(bad, ref, U, _gemm_atol(K), sc)


def test_checker_rejects_rope_position_shift():
    torch.manual_seed(2)
    S, D = 16, 64
    x = torch.randn(3, S, 2, D, dtype=torch.bfloat16)
    cos, sin = Rf.rope_tables(S + 1, D)
    ref, pair = rope64(x, cos, sin)
    assert not _rejects(Rf.rope(x, cos, sin), ref, ROPE_RTOL, ROPE_ATOL, pair)
    assert _rejects(Rf.rope(x, cos[1:], sin[1:]), ref, ROPE_RTOL, ROPE_ATOL, pair)


def test_checker_rejects_unnormalised_last_vector():
    torch.manual_seed(3)
    x = torch.randn(5, 200, dtype=torch.bfloat16) * 3
    w = (1 + 0.5 * torch.randn(200)).to(torch.bfloat16)
    ref = rmsnorm64(x, w)
    y = Rf.rmsnorm(x, w)
    assert not _rejects(y, ref, RMS_Y, 0.0)
    bad = y.clone()
    bad[:, -8:] = (x[:, -8:].float() * w[-8:].float()).to(torch.bfloat16)  # the c < nvec tail skipped by the rstd scaling
    assert _rejects(bad, ref, RMS_Y, 0.0)


def test_checker_rejects_scaled_dw():
    torch.manual_seed(4)
    h = torch.randn(700, 64, dtype=torch.bfloat16)
    w = (1 + 0.5 * torch.randn(64)).to(torch.bfloat16)
    dy = torch.randn(700, 64, dtype=torch.bfloat16)
    _, dw_ref, dw_sc = rmsnorm_bwd64(h, w, dy)
    dw = dw_ref.float()
    assert not _rejects(dw, dw_ref, DW_RTOL, DW_ATOL, dw_sc)
    assert _rejects(dw * (1 + 2.0**-7), dw_ref, DW_RTOL, DW_ATOL, dw_sc)


def test_checker_rejects_moved_cross_entropy_target():
    torch.manual_seed(5)
    V = 64
    z = (torch.randn(4, V) * 2).to(torch.bfloat16)
    tgt = torch.tensor([3, 0, V - 1, -100])
    _, gref, _ = cross_entropy64(z, tgt, -100, 0.5)
    s = 0.5 / 3
    rtol, atol = _ce_tolerances(V, True)
    sc = _ce_target_scale(z, tgt, -100, s)
    assert not _rejects(gref.to(torch.bfloat16), gref, rtol, atol, sc)
    bad = gref.clone()
    bad[0, 3] += s
    bad[0, 4] -= s
    assert _rejects(bad.to(torch.bfloat16), gref, rtol, atol, sc)


def test_checker_rejects_ue8m0_off_by_one():
    torch.manual_seed(6)
    x = (torch.randn(4, 128) * 5).to(torch.bfloat16)
    q, sf = Rf.quantize_mxfp8(x)
    ref, sc = _quant_oracle(x, False)
    assert not _rejects(Rf.dequantize_mxfp8(q, sf), ref, MX_RTOL, MX_ATOL, sc)
    i = int(Rf._mxfp8_sf_index(4, 128)[2, 1])
    for d in (1, -1):
        bad = sf.clone()
        bad[i] = int(bad[i]) + d
        assert _rejects(Rf.dequantize_mxfp8(q, bad), ref, MX_RTOL, MX_ATOL, sc)


# -------------------------------------------------------------------------------------------------- GPU
def _dev():
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def native():
    from prime_b200.ops import _lib

    return _lib.load()  # a GPU box without the native library is a hard failure, never a silent fallback


def _bf16(t):
    return t.to(torch.bfloat16)


# D: 64 / 200 (nvec < 32: idle lanes of the one warp), 2048 (MAXV 1), 4096 (2), 8192 (4), 12288 (8)
@pytest.mark.gpu
@pytest.mark.parametrize("residual", [False, True], ids=["plain", "add"])
@pytest.mark.parametrize("D", [64, 200, 2048, 4096, 8192, 12288])
def test_rmsnorm_fwd_every_maxv(native, D, residual):
    from prime_b200 import ops

    torch.manual_seed(D)
    dev = _dev()
    x = _bf16(torch.randn(67, D, device=dev) * 3)
    w = _bf16(1 + 0.5 * torch.randn(D, device=dev))
    if residual:
        r = _bf16(torch.randn(67, D, device=dev))
        y, h = ops.add_rmsnorm(x, r, w)
        # elementwise.cu:34 rounds x + res (an exact fp32 sum of two bf16 values) to bf16 and normalises that
        h_ref = _bf16((x.double() + r.double()).float())
        assert torch.equal(h, h_ref), "h != bf16(x + residual)"
    else:
        y, h_ref = ops.rmsnorm(x, w), x
    assert_elementwise(y, rmsnorm64(h_ref, w), RMS_Y, 0.0, f"rmsnorm y D={D} {'add' if residual else 'plain'}")


# R: 300 / 528 (one row per CTA, no loop), 529 (one CTA runs a second, prefetched row), 16384 (31-32 rows per CTA)
@pytest.mark.gpu
@pytest.mark.parametrize(
    "R,D,residual,fresh",
    [(300, 2048, False, False), (528, 2048, False, False), (529, 2048, False, False), (16384, 2048, False, False),
     (529, 64, False, False), (529, 200, True, False), (529, 4096, False, False), (529, 8192, True, False),
     (529, 12288, False, False), (16384, 12288, True, False), (16384, 4096, True, False), (2000, 2048, False, True)],
)  # fmt: skip
def test_rmsnorm_bwd_persistent_rows_into_main_grad(native, R, D, residual, fresh):
    """dx (and the residual gradient) per element; dw accumulated into main_grad (dw_accumulate = 1), or overwriting it when the
    engine armed ``_mg_fresh`` (dw_accumulate = 0)."""
    from prime_b200 import ops

    assert native.pb_rmsnorm_bwd_grid(R) == min(R, 528)
    torch.manual_seed(R + D)
    dev = _dev()
    x = _bf16(torch.randn(R, D, device=dev) * 3).requires_grad_(True)
    w = _bf16(1 + 0.5 * torch.randn(D, device=dev)).requires_grad_(True)
    before = torch.randn(D, device=dev) * 50 if not fresh else torch.full((D,), 1e30, device=dev)
    w.main_grad = before.clone()
    w._mg_fresh = fresh
    dy = _bf16(torch.randn(R, D, device=dev))
    if residual:
        r = _bf16(torch.randn(R, D, device=dev)).requires_grad_(True)
        dh = _bf16(torch.randn(R, D, device=dev))
        y, h = ops.add_rmsnorm(x, r, w)
        torch.autograd.backward([y, h], [dy, dh])
        h_in = h.detach()
        assert torch.equal(x.grad, r.grad)
    else:
        y = ops.rmsnorm(x, w)
        y.backward(dy)
        h_in = x.detach()
    torch.cuda.synchronize()
    assert w.grad is None
    dx_ref, dw_ref, dw_sc = rmsnorm_bwd64(h_in, w.detach(), dy)
    if residual:
        dx_ref = dx_ref + dh.double()
    tag = f"R={R} D={D}{' add' if residual else ''}{' fresh' if fresh else ''}"
    assert_elementwise(x.grad, dx_ref, RMS_DX, RMS_DX_ATOL, f"rmsnorm dx {tag}")
    expect = dw_ref if fresh else before.double() + dw_ref
    assert_elementwise(w.main_grad, expect, DW_RTOL, DW_ATOL, f"rmsnorm main_grad {tag}", dw_sc)


@pytest.mark.gpu
@pytest.mark.parametrize("unit_upstream", [True, False], ids=["unit", "upstream"])
@pytest.mark.parametrize("V", [8, 2048, 32000, 32768, 32776, 128256])
def test_cross_entropy_both_kernels(native, V, unit_upstream):
    """V <= 32768: cross_entropy_reg_kernel (V = 32768 fills every register slot, V = 8 is one vector per row); V >= 32776: the
    two-pass cross_entropy_kernel. Targets at columns 0 and V - 1, one ignored row, rows with a logit spread of ~±200 and a
    dominant target (p_t ≈ 1: the cancellation at p - 1). Loss, gradient with grad_scale ≠ 1, and loss_acc over two calls."""
    from prime_b200 import ops

    torch.manual_seed(V)
    dev = _dev()
    R_ = 256 if V > 32776 else 300
    gs = 0.375
    acc = torch.full((), 0.25, device=dev)
    acc_ref = 0.25
    for call in range(2):
        z = torch.randn(R_, V, device=dev) * 2
        z[3] *= 25  # spread ~±200: exp underflows for most of the row
        tgt = torch.randint(0, V, (R_,), device=dev)
        tgt[0], tgt[1], tgt[2] = 0, V - 1, -100
        z[4, tgt[4]] = 40.0  # dominant target
        z[5, tgt[5]] = 8.0
        z = _bf16(z)
        loss_ref, g_ref, mag = cross_entropy64(z, tgt, -100, gs)
        leaf = z.clone().requires_grad_(True)
        loss = ops.cross_entropy(leaf * 1.0, tgt, grad_scale=gs, unit_upstream=unit_upstream, loss_acc=acc)
        up = 1.0 if unit_upstream else 0.75
        (loss if unit_upstream else loss * up).backward()
        torch.cuda.synchronize()
        tag = f"V={V} {'unit' if unit_upstream else 'upstream'} call={call}"
        # loss: row sums of <= 256 serial fp32 terms + a tree (<= 2^-16 relative on Σe, so absolute on log Σe), lg2/ex2.approx
        # (~2^-21) and fp32 adds of max z, log Σe and z_t and of the mean: 2^-14 of the magnitudes that enter them
        assert_elementwise(loss, loss_ref, 2.0**-16, 2.0**-14, f"ce loss {tag}", mag)
        acc_ref += float(loss_ref)
        s = gs / (R_ - 1) * up
        rtol, atol = _ce_tolerances(V, unit_upstream)
        assert_elementwise(leaf.grad, g_ref * up, rtol, atol, f"ce grad {tag}", _ce_target_scale(z, tgt, -100, s))
    assert_elementwise(acc, torch.tensor(acc_ref, dtype=torch.float64), 2.0**-16, 2.0**-14, f"ce loss_acc V={V}", 2 * mag)


@pytest.mark.gpu
@pytest.mark.parametrize("V", [2048, 32776])
def test_cross_entropy_all_targets_ignored(native, V):
    """The native contract when no target counts: loss 0 and an all-zero gradient, loss_acc unchanged. (torch returns NaN here,
    0/0 of its mean; the kernel divides by max(n_valid, 1) so a fully padded micro-batch contributes nothing.)"""
    from prime_b200 import ops

    dev = _dev()
    torch.manual_seed(V)
    z = _bf16(torch.randn(64, V, device=dev) * 2).requires_grad_(True)
    tgt = torch.full((64,), -100, device=dev)
    acc = torch.full((), 1.5, device=dev)
    loss = ops.cross_entropy(z * 1.0, tgt, grad_scale=0.5, unit_upstream=True, loss_acc=acc)
    loss.backward()
    torch.cuda.synchronize()
    assert float(loss.detach()) == 0.0 and float(acc) == 1.5
    assert bool((z.grad == 0).all())


@pytest.mark.gpu
@pytest.mark.parametrize("FF", [200, 5632])
def test_swiglu_kernels_saturated_gate(native, FF):
    """Stand-alone swiglu_fwd/bwd_kernel with gates beyond ±88, where __expf(-g) overflows to inf or underflows to 0."""
    from prime_b200 import ops

    dev = _dev()
    torch.manual_seed(FF)
    M = 300
    g = torch.randn(M, FF, device=dev) * 3
    g[::7] = torch.empty(FF, device=dev).uniform_(-120, 120)  # every 7th row spans the saturated range
    g[:, 0], g[:, 1] = 88.5, -88.5
    gu = _bf16(torch.cat((g, torch.randn(M, FF, device=dev)), dim=1)).requires_grad_(True)
    h = ops.swiglu(gu)
    d = _bf16(torch.randn(M, FF, device=dev))
    h.backward(d)
    torch.cuda.synchronize()
    assert_elementwise(h, swiglu64(gu), SWIGLU_RTOL, 0.0, f"swiglu h FF={FF}")
    dgu, sc = swiglu_bwd64(gu, d)
    assert_elementwise(gu.grad[:, :FF], dgu[:, :FF], SWIGLU_RTOL, SILU_D_ATOL, f"swiglu d_gate FF={FF}", sc)
    assert_elementwise(gu.grad[:, FF:], dgu[:, FF:], SWIGLU_RTOL, 0.0, f"swiglu d_up FF={FF}")


@pytest.mark.gpu
@pytest.mark.parametrize("H,Hkv,D", [(8, 2, 64), (4, 4, 128), (6, 1, 128)])
def test_rope_inplace_long_table(native, H, Hkv, D):
    """rope_inplace_kernel on B = 3 sequences of S = 100 with a 160-row table: the position is token % S and the table stride is
    D/2, never S; V heads are left bit-identical; the backward rotates by -sin."""
    from prime_b200 import ops

    dev = _dev()
    torch.manual_seed(H * D)
    B, S = 3, 100
    nh = H + 2 * Hkv
    cos, sin = Rf.rope_tables(160, D, 500000.0, device=dev)
    qkv = _bf16(torch.randn(B, S, nh * D, device=dev) * 2)
    base = qkv.clone().requires_grad_(True)
    out = ops.rope_qkv(base * 1.0, cos, sin, H, Hkv)
    go = _bf16(torch.randn(B, S, nh * D, device=dev))
    out.backward(go.clone())
    torch.cuda.synchronize()
    for name, got, src, sign in (("fwd", out.detach(), qkv, 1.0), ("bwd", base.grad, go, -1.0)):
        g4, s4 = got.view(B, S, nh, D), src.view(B, S, nh, D)
        ref, pair = rope64(s4[:, :, : H + Hkv], cos, sin, sign)
        assert_elementwise(g4[:, :, : H + Hkv], ref, ROPE_RTOL, ROPE_ATOL, f"rope {name} H={H} Hkv={Hkv} D={D}", pair)
        assert torch.equal(g4[:, :, H + Hkv :], s4[:, :, H + Hkv :]), "V heads changed"


# M: 64 / 128 take the _gemm_epi fallbacks (plain GEMM + stand-alone SwiGLU kernel); 300 / 1000 end in a partial 128-row tile
# FF: 64 (the EPI = 3 tile is half empty), 192, 5632 (1B), 14336 (7B / 70B-class)
@pytest.mark.gpu
@pytest.mark.parametrize("FF", [64, 192, 5632, 14336])
@pytest.mark.parametrize("M", [64, 128, 300, 1000, 2048])
def test_gemm_swiglu_epilogues_and_fallbacks(native, M, FF):
    """Forward: gate_up = x·W13ᵀ and h = silu(gate)·up (EPI = 2 for M > 128). Backward: d_gate_up from dh = dy·W2 and the saved
    gate_up (EPI = 3 for M > 128, whose dh stays fp32; the fallback rounds dh to bf16 first)."""
    from prime_b200.ops import functional as Fn

    dev = _dev()
    torch.manual_seed(M + FF)
    K, Dm = 256, 384
    x = _bf16(torch.randn(M, K, device=dev))
    w13 = _bf16(torch.randn(2 * FF, K, device=dev) * K**-0.5 * 2)
    gu = torch.full((M, 2 * FF), float("nan"), dtype=torch.bfloat16, device=dev)
    h = torch.full((M, FF), float("nan"), dtype=torch.bfloat16, device=dev)
    Fn._gemm_epi(x, w13, gu, swiglu_h=h)
    dy = _bf16(torch.randn(M, Dm, device=dev))
    w2 = _bf16(torch.randn(Dm, FF, device=dev) * Dm**-0.5)
    dgu = torch.full((M, 2 * FF), float("nan"), dtype=torch.bfloat16, device=dev)
    Fn._gemm_epi(dy, w2, dgu, b_mn_major=True, swiglu_bwd_gu=gu)
    torch.cuda.synchronize()
    tag = f"M={M} FF={FF}"
    ref, sc = _gemm_ref(x, w13)
    assert_elementwise(gu, ref, U, _gemm_atol(K), f"swiglu gate_up {tag}", sc)
    # h is computed from the bf16-ROUNDED gate/up the kernel stores (gemm_sm90.cu:489): the oracle reads the same tensor
    assert_elementwise(h, swiglu64(gu), SWIGLU_RTOL, 0.0, f"swiglu h {tag}")
    dh, dh_sc = _gemm_ref(dy, w2.t())
    dref, _ = swiglu_bwd64(gu, dh)
    g, u = gu.double().chunk(2, dim=-1)
    sg = torch.sigmoid(g)
    d_gate_sc = u.abs() * (sg.abs() + (g * sg * (1 - sg)).abs()) * dh_sc  # |∂d_gate/∂dh|·(rounding scale of dh)
    d_up_sc = (g * sg).abs() * dh_sc
    # M <= 128: dh is rounded to bf16 before the stand-alone kernel (one more rounding); M > 128: EPI = 3 keeps dh in fp32
    rtol = SWIGLU_RTOL + (U if M <= 128 else 0.0)
    atol = _gemm_atol(Dm) + SILU_D_ATOL
    assert_elementwise(dgu[:, :FF], dref[:, :FF], rtol, atol, f"swiglu d_gate {tag}", d_gate_sc)
    assert_elementwise(dgu[:, FF:], dref[:, FF:], rtol, _gemm_atol(Dm), f"swiglu d_up {tag}", d_up_sc)


@pytest.mark.gpu
@pytest.mark.parametrize("H,Hkv,D,B,S", [(4, 1, 64, 3, 100), (8, 1, 64, 1, 64), (6, 1, 128, 2, 512)])
def test_gemm_rope_epilogue_partial_tile(native, H, Hkv, D, B, S):
    """EPI = 1: rope_cols = (H + Hkv)·D = 320 / 576 end inside a 128-column tile (896 at D = 128 ends on a boundary); M = B·S =
    300 / 64 end inside a 128-row tile; the table has more rows than S. Columns past rope_cols (V heads) are the plain product."""
    from prime_b200 import ops

    dev = _dev()
    torch.manual_seed(H * D + S)
    K = 256
    M, nh = B * S, H + 2 * Hkv
    x = _bf16(torch.randn(M, K, device=dev))
    w = _bf16(torch.randn(nh * D, K, device=dev) * K**-0.5)
    cos, sin = Rf.rope_tables(S + 37, D, 500000.0, device=dev)
    y = ops.gemm(x, w, rope=(cos, sin, S, (H + Hkv) * D, D))
    torch.cuda.synchronize()
    ref, sc = _gemm_ref(x, w)
    rot = (H + Hkv) * D
    r4 = ref.view(B, S, nh, D)
    rref, _ = rope64(r4[:, :, : H + Hkv], cos, sin)
    s4 = sc.view(B, S, nh, D)[:, :, : H + Hkv]
    # a rotated column mixes the accumulators of its pair: the rounding scale is the sum of both columns' |A|·|B|ᵀ
    pair_sc = (s4.reshape(B, S, H + Hkv, D // 2, 2).sum(-1, keepdim=True).expand(B, S, H + Hkv, D // 2, 2)).reshape(B, S, H + Hkv, D)
    tag = f"H={H} Hkv={Hkv} D={D} M={M}"
    y4 = y.view(B, S, nh, D)
    assert_elementwise(y4[:, :, : H + Hkv], rref, U, _gemm_atol(K) + ROPE_ATOL, f"rope epilogue rotated {tag}", pair_sc)
    assert_elementwise(y[:, rot:], ref[:, rot:], U, _gemm_atol(K), f"rope epilogue plain {tag}", sc[:, rot:])


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["small_m_swiglu", "small_m_swiglu_bwd", "resident_ff200"])
def test_wgather_swiglu_fallbacks(native, mode):
    """``gemm_wgather`` (ZeRO-3 weight, one-rank group) sends M <= 128 and a resident weight with FF % 64 != 0 through ``_gemm_epi``,
    which runs a plain GEMM and the stand-alone SwiGLU kernels."""
    import ctypes

    from prime_b200 import ops
    from prime_b200.parallel.fsdp import RowShard
    from prime_b200.parallel.symm import SymmetricHeap

    dev = _dev()
    heap = SymmetricHeap(64 << 20, 0, 1, lambda h: [h], dev)
    torch.manual_seed(23)
    K = 512

    def shard(W):
        rows, cols = W.shape
        sh = heap.alloc(rows * cols, torch.bfloat16).view(rows, cols)
        sh.copy_(W)
        full = torch.zeros(rows, cols, dtype=torch.bfloat16, device=dev)
        flags = torch.zeros(64, dtype=torch.int32, device=dev)
        peers = (ctypes.c_void_p * 1)(heap.peer_ptr(0, sh))
        return RowShard(rows, cols, 1, 0, rows, peers, full.data_ptr(), flags, sh, full=full)

    try:
        FF = 200 if mode == "resident_ff200" else 576
        W13 = _bf16(torch.randn(2 * FF, K, device=dev) * K**-0.5 * 2)
        z13 = shard(W13)
        if mode == "resident_ff200":
            warm = _bf16(torch.randn(64, K, device=dev))
            ops.gemm_wgather(warm, z13, out=torch.empty(64, 2 * FF, dtype=torch.bfloat16, device=dev),
                             swiglu_h=torch.empty(64, FF, dtype=torch.bfloat16, device=dev))  # fmt: skip
            assert ops.functional._resident(z13)
        M = 64 if mode.startswith("small_m") else 300
        x = _bf16(torch.randn(M, K, device=dev))
        gu = torch.empty(M, 2 * FF, dtype=torch.bfloat16, device=dev)
        h = torch.empty(M, FF, dtype=torch.bfloat16, device=dev)
        ops.gemm_wgather(x, z13, out=gu, swiglu_h=h)
        torch.cuda.synchronize()
        ref, sc = _gemm_ref(x, W13)
        assert_elementwise(gu, ref, U, _gemm_atol(K), f"wgather gate_up {mode}", sc)
        assert_elementwise(h, swiglu64(gu), SWIGLU_RTOL, 0.0, f"wgather h {mode}")
        if mode == "small_m_swiglu_bwd":
            W2 = _bf16(torch.randn(K, FF, device=dev) * K**-0.5)
            z2 = shard(W2)
            dy = _bf16(torch.randn(M, K, device=dev))
            dgu = ops.gemm_wgather(dy, z2, b_mn_major=True, swiglu_bwd_gu=gu)
            torch.cuda.synchronize()
            dh, dh_sc = _gemm_ref(dy, W2.t())
            dref, _ = swiglu_bwd64(gu, dh)
            g, u = gu.double().chunk(2, dim=-1)
            sg = torch.sigmoid(g)
            # dh is rounded to bf16 before the stand-alone backward kernel: two bf16 roundings
            assert_elementwise(dgu[:, :FF], dref[:, :FF], SWIGLU_RTOL + U, _gemm_atol(K) + SILU_D_ATOL, f"wgather d_gate {mode}",
                               u.abs() * (sg.abs() + (g * sg * (1 - sg)).abs()) * dh_sc)  # fmt: skip
            assert_elementwise(dgu[:, FF:], dref[:, FF:], SWIGLU_RTOL + U, _gemm_atol(K), f"wgather d_up {mode}", (g * sg).abs() * dh_sc)
        heap.check_errors()
    finally:
        ops.reset_gather_cache()
        heap.close()


def _mx_edge_matrix(rows: int, k: int, dev) -> torch.Tensor:
    """[rows, k] bf16 whose 32-element blocks along k cycle through: random magnitudes 2^-20..2^20, all zero, amax exactly
    448·2^j (amax/448 a power of two: the mantissa == 0 branch of ue8m0_for), bf16 subnormals (the e = 1 clamp), negative only,
    and amax 2^-125 (a normal input whose scale is clamped)."""
    nb = k // 32
    x = torch.randn(rows, nb, 32, device=dev)
    kind = (torch.arange(rows, device=dev).view(-1, 1) * 5 + torch.arange(nb, device=dev).view(1, -1)) % 6
    j = torch.randint(-20, 21, (rows, nb, 1), device=dev).float()
    out = x * torch.exp2(j)
    out = torch.where((kind == 1).unsqueeze(-1), torch.zeros_like(out), out)
    p2 = 448.0 * torch.exp2(torch.randint(-10, 11, (rows, nb, 1), device=dev).float())
    xs = x / x.abs().amax(-1, keepdim=True) * p2 * 0.99
    xs[..., 7] = torch.where(x[..., 7] < 0, -p2[..., 0], p2[..., 0])
    out = torch.where((kind == 2).unsqueeze(-1), xs, out)
    sub = torch.randint(-127, 128, (rows, nb, 32), device=dev).float() * 2.0**-133  # every bf16 subnormal spacing
    out = torch.where((kind == 3).unsqueeze(-1), sub, out)
    out = torch.where((kind == 4).unsqueeze(-1), -(x * torch.exp2(j)).abs(), out)
    tiny = x / x.abs().amax(-1, keepdim=True) * 2.0**-125
    out = torch.where((kind == 5).unsqueeze(-1), tiny, out)
    return _bf16(out.view(rows, k))


@pytest.mark.gpu
@pytest.mark.parametrize("transpose", [False, True], ids=["rows", "transposed"])
@pytest.mark.parametrize("rows,k", [(200, 384), (256, 1024), (1000, 2048)])
def test_quantize_mxfp8_edge_blocks(native, rows, k, transpose):
    """q and every UE8M0 byte bit for bit against reference.quantize_mxfp8, and the dequantised value against the fp64 input with
    the exact power-of-two scale. ``transposed`` quantises xᵀ [k, rows] along its rows (quantize_mxfp8_t_kernel)."""
    from prime_b200 import ops

    dev = _dev()
    torch.manual_seed(rows + k)
    m = _mx_edge_matrix(rows, k, dev)
    x = m.t().contiguous() if transpose else m
    q, sf = ops.quantize_mxfp8(x, transpose)
    q_ref, sf_ref = Rf.quantize_mxfp8(x, transpose)
    torch.cuda.synchronize()
    idx = Rf._mxfp8_sf_index(rows, k, dev).reshape(-1)
    bad = sf[idx] != sf_ref[idx]
    assert not bool(bad.any()), f"{int(bad.sum())} UE8M0 bytes differ, first at block {int(bad.nonzero()[0])}"
    assert torch.equal(q, q_ref), f"{int((q != q_ref).sum())} e4m3 values differ"
    ref, sc = _quant_oracle(x, transpose)
    assert_elementwise(Rf.dequantize_mxfp8(q, sf), ref, MX_RTOL, MX_ATOL, f"mxfp8 dequant {rows}x{k} t={transpose}", sc)
