"""The bf16 GEMM in both tile widths (128 × 128 and 128 × 256, forced with ``ops.set_gemm_tile``) against an fp64 oracle, with the
per-element rule of ``test_kernel_edges_gpu.py``, on every operand layout and every epilogue; each wide result also against the
narrow one, bit for bit wherever K is not split (both widths accumulate every output element over the same k16 steps in the same
order, so only a split, whose slices add through atomics, may reorder the sum).

Edge shapes: an odd number of 128-row tiles (M = 1152) and a partial one (M = 300, 328); N ≡ 128 (mod 256), a half-empty wide tile;
SwiGLU with FF % 128 = 64 (the last wide tile's gate and up halves each half past FF, zero-filled by the TMA unit); RoPE columns
ending inside a wide tile at D = 64 and D = 128; outputs padded inside a wider buffer, whose padding must stay untouched; fp32 +=
with a forced split-K.

The CPU tests check the automatic tile policy at the Llama-1B training shapes and at its boundaries, and that no GEMM
instantiation of the built library has a stack frame or spills (``cuobjdump --dump-resource-usage``)."""

import re
import shutil
import subprocess
from pathlib import Path

import pytest
import torch
from test_kernel_edges_gpu import (
    ROPE_ATOL,
    SILU_D_ATOL,
    SWIGLU_RTOL,
    U,
    U32,
    _gemm_atol,
    _gemm_ref,
    assert_elementwise,
    rope64,
    swiglu64,
    swiglu_bwd64,
)

from prime_b200.ops import reference as Rf

ROOT = Path(__file__).resolve().parent.parent
MODES = (128, 256)
PAD = 24  # padding columns of an output stored inside a wider buffer (keeps ldc a multiple of 8)
SENTINEL = 7.0  # the padding's value; exact in bf16 and fp32


# -------------------------------------------------------------------------------------------------- CPU: policy and resources
T, DIM, FF1B, VOCAB = 16384, 2048, 5632, 32000  # Llama-1B, 16 × 1024 tokens per micro-batch


@pytest.mark.parametrize(
    "what,M,N,K,epi,fp32,want",
    [
        ("fwd qkv+rope", T, 3 * DIM, DIM, 1, False, 256),
        ("fwd o", T, DIM, DIM, 0, False, 256),
        ("fwd w13+swiglu", T, 2 * FF1B, DIM, 2, False, 256),
        ("fwd w2", T, DIM, FF1B, 0, False, 256),
        ("fwd logits", T, VOCAB, DIM, 0, False, 256),
        ("dgrad w2+swiglu_bwd", T, FF1B, DIM, 3, False, 256),
        ("dgrad w13", T, DIM, 2 * FF1B, 0, False, 256),
        ("dgrad logits", T, DIM, VOCAB, 0, False, 256),
        ("wgrad qkv", 3 * DIM, DIM, T, 0, True, 256),
        ("wgrad o", DIM, DIM, T, 0, True, 256),
        ("wgrad w13", 2 * FF1B, DIM, T, 0, True, 256),
        ("wgrad w2", DIM, FF1B, T, 0, True, 256),
        ("wgrad output", VOCAB, DIM, T, 0, True, 256),
        # one row of tiles: the decode-step GEMMs (M = batch) stay narrow at any N
        ("decode M=1", 1, VOCAB, DIM, 0, False, 128),
        ("decode M=128", 128, 2 * FF1B, DIM, 0, False, 128),
        ("M=129", 129, VOCAB, DIM, 0, False, 256),
        # fewer narrow tiles than SMs: the wide grid would be no shorter and each tile twice as long
        ("one narrow round", 1024, 1024, 4096, 0, False, 128),
        # splits K under the narrow width (atomics): stays narrow so the result does not change
        ("split-K wgrad", 512, 512, T, 0, True, 128),
        # would split under the wide width only (40 wide tiles, 80 narrow ones): stays narrow, unsplit
        ("split only if wide", 1024, 1280, T, 0, True, 128),
    ],
)
def test_tile_policy(what, M, N, K, epi, fp32, want):
    from prime_b200 import ops

    assert ops.gemm_tile_policy(M, N, K, epilogue=epi, c_fp32=fp32, accumulate=fp32, num_sms=132) == want, what


def test_set_gemm_tile_rejects_unknown_width():
    from prime_b200 import ops

    with pytest.raises(ValueError):
        ops.set_gemm_tile(192)


@pytest.mark.skipif(shutil.which("cuobjdump") is None or shutil.which("nvcc") is None, reason="CUDA toolkit not installed")
def test_gemm_instantiations_have_no_stack_frame():
    """Every GEMM instantiation, local (narrow and wide) and collective: no stack frame, no local memory. The wide tile's 128
    accumulators per consumer thread fit only because the consumers take the producer warpgroup's registers (setmaxnreg)."""
    from prime_b200.ops import _lib

    lib = _lib.build()
    out = subprocess.run(["cuobjdump", "--dump-resource-usage", str(lib)], capture_output=True, text=True, check=True).stdout
    seen = {}
    lines = out.splitlines()
    for i, line in enumerate(lines):
        m = re.search(r"gemm_bf16_kernelILi(\d)ELi(\d)ELi(\d)ELi(\d)ELi(\d+)E", line)
        if m:
            usage = lines[i + 1]
            seen[m.groups()] = usage
            assert "STACK:0 " in usage and "LOCAL:0 " in usage, f"gemm_bf16_kernel<{', '.join(m.groups())}>: {usage.strip()}"
    assert len(seen) == 23, sorted(seen)  # local: 7 (layout, epilogue) variants × 2 widths; collective: 2 + 2 + 5 narrow
    assert {k[4] for k in seen} == {"128", "256"} and {k[3] for k in seen} == {"0", "1", "2", "3"}


# -------------------------------------------------------------------------------------------------- GPU
def _dev():
    return torch.device("cuda", 0)


@pytest.fixture
def tile():
    """Sets the forced tile mode for one test and restores the automatic policy (and split-K) afterwards."""
    from prime_b200 import ops

    yield ops.set_gemm_tile
    ops.set_gemm_tile(-1)
    ops.set_gemm_split_k(-1)


def _padded(M, N, dtype, dev):
    buf = torch.full((M, N + PAD), SENTINEL, dtype=dtype, device=dev)
    return buf, buf[:, :N]


def _check_padding(buf, N, what):
    assert bool((buf[:, N:] == SENTINEL).all()), f"{what}: the padding next to the output was written"


def _operands(M, N, K, a_mn, b_mn, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    a = torch.randn(M, K, device=dev, generator=g).to(torch.bfloat16)
    b = (torch.randn(N, K, device=dev, generator=g) * K**-0.5).to(torch.bfloat16)
    # stored as the kernel reads them: MN-major = the transpose made contiguous
    a_st = a.t().contiguous() if a_mn else a
    b_st = b.t().contiguous() if b_mn else b
    return a, b, a_st, b_st


@pytest.mark.gpu
# MN-major A is stored [K, M]: M is a multiple of 8 (16-byte rows) but not of 128
@pytest.mark.parametrize("M,N,K", [(1152, 640, 320), (328, 384, 200)], ids=["odd_mtiles_half_wide_tile", "partial_rows"])
@pytest.mark.parametrize("a_mn,b_mn", [(0, 0), (0, 1), (1, 0), (1, 1)], ids=["KK", "KM", "MK", "MM"])
def test_gemm_bf16_every_layout(tile, M, N, K, a_mn, b_mn):
    from prime_b200 import ops

    dev = _dev()
    a, b, a_st, b_st = _operands(M, N, K, a_mn, b_mn, dev, M + N + 2 * a_mn + b_mn)
    ref, sc = _gemm_ref(a, b)
    outs = {}
    for mode in MODES:
        tile(mode)
        buf, y = _padded(M, N, torch.bfloat16, dev)
        ops.gemm(a_st, b_st, a_mn_major=bool(a_mn), b_mn_major=bool(b_mn), out=y)
        torch.cuda.synchronize()
        what = f"tile {mode} M={M} N={N} K={K} a_mn={a_mn} b_mn={b_mn}"
        _check_padding(buf, N, what)
        assert_elementwise(y, ref, U, _gemm_atol(K), what, sc)
        outs[mode] = y.clone()
    assert torch.equal(outs[128], outs[256])


@pytest.mark.gpu
@pytest.mark.parametrize("split", [1, 3], ids=["nosplit", "split3"])
@pytest.mark.parametrize("M,N,K", [(1152, 640, 1024), (640, 384, 2048)])
def test_gemm_fp32_accumulate(tile, M, N, K, split):
    """Weight-gradient form: main_grad [M, N] += Aᵀ·B with both operands MN-major, into a padded fp32 buffer."""
    from prime_b200 import ops

    dev = _dev()
    a, b, a_st, b_st = _operands(M, N, K, 1, 1, dev, M + N + split)
    c0 = torch.randn(M, N, device=dev, dtype=torch.float64).float()
    ref, sc = _gemm_ref(a, b)
    ref = ref + c0.double()
    outs = {}
    for mode in MODES:
        tile(mode)
        ops.set_gemm_split_k(split if split > 1 else 0)
        buf, y = _padded(M, N, torch.float32, dev)
        y.copy_(c0)
        ops.gemm(a_st, b_st, a_mn_major=True, b_mn_major=True, out=y, accumulate=True)
        torch.cuda.synchronize()
        what = f"tile {mode} fp32 += M={M} N={N} K={K} split={split}"
        _check_padding(buf, N, what)
        # the product's fp32 accumulation, then one fp32 add per K slice into the buffer
        assert_elementwise(y, ref, (split + 1) * U32, _gemm_atol(K), what, sc + c0.double().abs())
        outs[mode] = y.clone()
    if split == 1:
        assert torch.equal(outs[128], outs[256])


@pytest.mark.gpu
@pytest.mark.parametrize("M,FF", [(300, 320), (1152, 448), (2048, 5632)])
def test_gemm_swiglu_epilogues(tile, M, FF):
    """EPI = 2 (gate_up and h) and EPI = 3 (d_gate_up); FF = 320 / 448: FF % 128 = 64, the last wide tile is half empty."""
    from prime_b200 import ops

    dev = _dev()
    torch.manual_seed(M + FF)
    K, Dm = 256, 384
    x = torch.randn(M, K, device=dev).to(torch.bfloat16)
    w13 = (torch.randn(2 * FF, K, device=dev) * K**-0.5 * 2).to(torch.bfloat16)
    dy = torch.randn(M, Dm, device=dev).to(torch.bfloat16)
    w2 = (torch.randn(Dm, FF, device=dev) * Dm**-0.5).to(torch.bfloat16)
    ref, sc = _gemm_ref(x, w13)
    dh, dh_sc = _gemm_ref(dy, w2.t())
    outs = {}
    for mode in MODES:
        tile(mode)
        gu_buf, gu = _padded(M, 2 * FF, torch.bfloat16, dev)
        h_buf, h = _padded(M, FF, torch.bfloat16, dev)
        ops.gemm(x, w13, out=gu, swiglu_h=h)
        dgu_buf, dgu = _padded(M, 2 * FF, torch.bfloat16, dev)
        ops.gemm(dy, w2, b_mn_major=True, out=dgu, swiglu_bwd_gu=gu)
        torch.cuda.synchronize()
        tag = f"tile {mode} M={M} FF={FF}"
        for buf, n, what in ((gu_buf, 2 * FF, "gate_up"), (h_buf, FF, "h"), (dgu_buf, 2 * FF, "d_gate_up")):
            _check_padding(buf, n, f"{what} {tag}")
        assert_elementwise(gu, ref, U, _gemm_atol(K), f"swiglu gate_up {tag}", sc)
        assert_elementwise(h, swiglu64(gu), SWIGLU_RTOL, 0.0, f"swiglu h {tag}")
        dref, _ = swiglu_bwd64(gu, dh)
        g, u = gu.double().chunk(2, dim=-1)
        sg = torch.sigmoid(g)
        d_gate_sc = u.abs() * (sg.abs() + (g * sg * (1 - sg)).abs()) * dh_sc
        d_up_sc = (g * sg).abs() * dh_sc
        assert_elementwise(dgu[:, :FF], dref[:, :FF], SWIGLU_RTOL, _gemm_atol(Dm) + SILU_D_ATOL, f"swiglu d_gate {tag}", d_gate_sc)
        assert_elementwise(dgu[:, FF:], dref[:, FF:], SWIGLU_RTOL, _gemm_atol(Dm), f"swiglu d_up {tag}", d_up_sc)
        outs[mode] = (gu.clone(), h.clone(), dgu.clone())
    for x128, x256 in zip(outs[128], outs[256]):
        assert torch.equal(x128, x256)


# rope_cols = (H + Hkv)·D: 320 (D = 64) and 384 (D = 128) end inside the second wide tile; M = B·S = 300 ends inside a row tile
@pytest.mark.gpu
@pytest.mark.parametrize("H,Hkv,D,B,S", [(4, 1, 64, 3, 100), (2, 1, 128, 2, 512)])
def test_gemm_rope_epilogue(tile, H, Hkv, D, B, S):
    from prime_b200 import ops

    dev = _dev()
    torch.manual_seed(H * D + S)
    K = 256
    M, nh = B * S, H + 2 * Hkv
    x = torch.randn(M, K, device=dev).to(torch.bfloat16)
    w = (torch.randn(nh * D, K, device=dev) * K**-0.5).to(torch.bfloat16)
    cos, sin = Rf.rope_tables(S + 37, D, 500000.0, device=dev)
    rot = (H + Hkv) * D
    ref, sc = _gemm_ref(x, w)
    rref, _ = rope64(ref.view(B, S, nh, D)[:, :, : H + Hkv], cos, sin)
    s4 = sc.view(B, S, nh, D)[:, :, : H + Hkv]
    pair_sc = (s4.reshape(B, S, H + Hkv, D // 2, 2).sum(-1, keepdim=True).expand(B, S, H + Hkv, D // 2, 2)).reshape(B, S, H + Hkv, D)
    outs = {}
    for mode in MODES:
        tile(mode)
        buf, y = _padded(M, nh * D, torch.bfloat16, dev)
        ops.gemm(x, w, out=y, rope=(cos, sin, S, rot, D))
        torch.cuda.synchronize()
        tag = f"tile {mode} H={H} Hkv={Hkv} D={D} M={M}"
        _check_padding(buf, nh * D, tag)
        y4 = y.reshape(B, S, nh, D)
        assert_elementwise(y4[:, :, : H + Hkv], rref, U, _gemm_atol(K) + ROPE_ATOL, f"rope rotated {tag}", pair_sc)
        assert_elementwise(y[:, rot:], ref[:, rot:], U, _gemm_atol(K), f"rope plain {tag}", sc[:, rot:])
        outs[mode] = y.clone()
    assert torch.equal(outs[128], outs[256])
