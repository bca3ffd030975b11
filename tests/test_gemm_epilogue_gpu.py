"""The staged epilogue of the local bf16 GEMM (shared-memory slots → TMA stores, and TMA loads of the saved gate_up for SwiGLU
backward), in both tile widths, against oracles that do not go through it:

- every layout: the bf16 output equals the fp32 output of the same product rounded with ``.to(torch.bfloat16)``, and the fp32
  output of ``+=`` (unsplit) equals ``c0 + product`` exactly, one fp32 add per element;
- SwiGLU: gate_up equals the plain GEMM's output and h the stand-alone SwiGLU kernel's result on it;
- SwiGLU backward: d_gate_up agrees to bf16 with the same formula evaluated in PyTorch on the fp32 product dh.

Edge shapes: a partial last row tile (M = 328 and, for SwiGLU, 300), N ≡ 128 (mod 256), FF % 128 = 64, and every output inside a wider buffer whose
padding must stay untouched."""

import pytest
import torch

from prime_b200.ops import functional as F

PAD = 24
SENTINEL = 7.0


def _dev():
    return torch.device("cuda", 0)


@pytest.fixture
def tile():
    from prime_b200 import ops

    yield ops.set_gemm_tile
    ops.set_gemm_tile(-1)
    ops.set_gemm_split_k(-1)


def _padded(M, N, dtype, dev, fill=SENTINEL):
    buf = torch.full((M, N + PAD), fill, dtype=dtype, device=dev)
    return buf, buf[:, :N]


def _untouched(buf, N, what):
    assert bool((buf[:, N:] == SENTINEL).all()), f"{what}: the padding next to the output was written"


def _rand(shape, dev, g, scale=1.0):
    return (torch.randn(*shape, device=dev, generator=g) * scale).to(torch.bfloat16)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [128, 256])
@pytest.mark.parametrize("M,N,K", [(328, 384, 192), (1152, 640, 256)], ids=["partial_rows", "half_wide_tile"])
@pytest.mark.parametrize("a_mn,b_mn", [(0, 0), (0, 1), (1, 0), (1, 1)], ids=["KK", "KM", "MK", "MM"])
def test_bf16_is_rounded_fp32_and_fp32_add_is_exact(tile, mode, M, N, K, a_mn, b_mn):
    from prime_b200 import ops

    dev = _dev()
    g = torch.Generator(device=dev).manual_seed(M + N + K + 2 * a_mn + b_mn)
    a = _rand((M, K), dev, g)
    b = _rand((N, K), dev, g, K**-0.5)
    a_st = a.t().contiguous() if a_mn else a
    b_st = b.t().contiguous() if b_mn else b
    tile(mode)
    ops.set_gemm_split_k(0)
    kw = dict(a_mn_major=bool(a_mn), b_mn_major=bool(b_mn))
    what = f"tile {mode} M={M} N={N} K={K} a_mn={a_mn} b_mn={b_mn}"

    fbuf, f = _padded(M, N, torch.float32, dev)
    ops.gemm(a_st, b_st, out=f, out_dtype=torch.float32, **kw)
    hbuf, h = _padded(M, N, torch.bfloat16, dev)
    ops.gemm(a_st, b_st, out=h, **kw)
    c0 = torch.randn(M, N, device=dev, generator=g)
    abuf, acc = _padded(M, N, torch.float32, dev)
    acc.copy_(c0)
    ops.gemm(a_st, b_st, out=acc, accumulate=True, **kw)
    torch.cuda.synchronize()
    for buf, name in ((fbuf, "fp32"), (hbuf, "bf16"), (abuf, "fp32 +=")):
        _untouched(buf, N, f"{what} {name}")
    assert torch.equal(h, f.to(torch.bfloat16)), what
    assert torch.equal(acc, c0 + f), what


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [128, 256])
@pytest.mark.parametrize("M,FF", [(300, 320), (1152, 448), (640, 512)])
def test_swiglu_epilogues_equal_the_standalone_kernels(tile, mode, M, FF):
    """SwiGLU: h equals the stand-alone forward kernel applied to the fused gate_up. SwiGLU backward (gate_up read by the TMA
    unit, from a wider buffer): d_gate_up against the formula on the fp32 product dh."""
    from prime_b200 import ops

    dev = _dev()
    g = torch.Generator(device=dev).manual_seed(M + FF)
    K = 256
    x = _rand((M, K), dev, g)
    w13 = _rand((2 * FF, K), dev, g, K**-0.5)
    tile(mode)
    what = f"tile {mode} M={M} FF={FF}"

    gubuf, gu = _padded(M, 2 * FF, torch.bfloat16, dev)
    hbuf, h = _padded(M, FF, torch.bfloat16, dev)
    ops.gemm(x, w13, out=gu, swiglu_h=h)
    gu_plain = ops.gemm(x, w13)
    h_ref = torch.empty(M, FF, dtype=torch.bfloat16, device=dev)
    F._launch("pb_swiglu_fwd", gu_plain.data_ptr(), h_ref.data_ptr(), M, FF, F._stream())
    torch.cuda.synchronize()
    _untouched(gubuf, 2 * FF, f"{what} gate_up")
    _untouched(hbuf, FF, f"{what} h")
    assert torch.equal(gu, gu_plain), what
    assert torch.equal(h, h_ref), what

    dy = _rand((M, K), dev, g)
    w2 = _rand((FF, K), dev, g, K**-0.5).t().contiguous()  # stored [K, FF]: the MN-major B of dh = dy·W2
    dbuf, dgu = _padded(M, 2 * FF, torch.bfloat16, dev)
    ops.gemm(dy, w2, b_mn_major=True, out=dgu, swiglu_bwd_gu=gu)
    dh = ops.gemm(dy, w2, b_mn_major=True, out_dtype=torch.float32)
    torch.cuda.synchronize()
    _untouched(dbuf, 2 * FF, f"{what} d_gate_up")
    # the fused epilogue computes from the fp32 accumulators: the same formula on the fp32 product, in PyTorch, agrees to bf16
    gf, uf = gu.float()[:, :FF], gu.float()[:, FF:]
    s = torch.sigmoid(gf)
    ref = torch.cat([dh * uf * s * (1 + gf * (1 - s)), dh * gf * s], dim=1)
    torch.testing.assert_close(dgu.float(), ref, rtol=2**-7, atol=1e-5, msg=what)
