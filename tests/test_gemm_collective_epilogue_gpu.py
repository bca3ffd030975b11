"""The collective bf16 GEMMs against the local one, bit for bit, on a one-rank group.

With one rank there is no rank rotation of the tiles or of the K loop, so every output element of the all-gather ⊕ GEMM (IO = 1),
the GEMM ⊕ reduce-scatter (IO = 2) and the parameter all-gather ⊕ GEMM (IO = 3) is accumulated over the same k16 steps, in the
same order, as in ``pb_gemm_bf16`` at the 128-wide tile. Their outputs, and the fused RoPE, SwiGLU and SwiGLU-backward epilogues
applied to them, must therefore equal the local GEMM's exactly. The reduce-scatter adds each fp32 element once into a zeroed
buffer, which is exact (``torch.equal`` counts 0 + (-0) as equal).

Edge shapes: a partial last row tile (M = 300, 328) for IO = 3, FF % 128 = 64, a weight whose last 128-row box is clipped
(1088 rows), and every output inside a wider buffer whose padding must stay untouched."""

import ctypes

import pytest
import torch

from prime_b200.ops import functional as F

PAD = 24  # padding columns (keeps every row stride a multiple of 8 elements)
SENTINEL = 7.0


def _dev():
    return torch.device("cuda", 0)


@pytest.fixture
def env():
    """A one-rank symmetric heap for the peer-mapped operands, with the local GEMM forced to the collective variants' tile."""
    from prime_b200 import ops
    from prime_b200.parallel.symm import SymmetricHeap

    dev = _dev()
    heap = SymmetricHeap(256 << 20, 0, 1, lambda h: [h], dev)
    ops.set_gemm_tile(128)
    try:
        yield heap
        torch.cuda.synchronize()
        heap.check_errors()
    finally:
        ops.set_gemm_tile(-1)
        ops.reset_gather_cache()
        heap.close()


def _padded(M, N, dtype, fill=SENTINEL):
    buf = torch.full((M, N + PAD), fill, dtype=dtype, device=_dev())
    return buf, buf[:, :N]


def _rand(shape, g, scale=1.0):
    return (torch.randn(*shape, device=_dev(), generator=g) * scale).to(torch.bfloat16)


def _on_heap(heap, t):
    s = heap.alloc(t.numel(), t.dtype).view(t.shape)
    s.copy_(t)
    return s


def _same(got_buf, want_buf, N, what):
    """Bit-for-bit equality of two padded outputs; the padding of ``got_buf`` must still be the sentinel."""
    assert bool((got_buf[:, N:] == SENTINEL).all()), f"{what}: the padding next to the output was written"
    got, want = got_buf[:, :N], want_buf[:, :N]
    if not torch.equal(got, want):
        ib = torch.int16 if got.dtype == torch.bfloat16 else torch.int32
        ulps = (got.view(ib).long() - want.view(ib).long()).abs().max().item()
        raise AssertionError(f"{what}: {int((got != want).sum())} elements differ, by up to {ulps} ulp")


class _Weight:
    """A weight W [rows, cols] sharded over the one-rank group: its shard on the heap and the local scratch the kernel gathers into."""

    def __init__(self, heap, W):
        self.W = W
        self.shard = _on_heap(heap, W)
        self.full = torch.zeros_like(W)
        self.flags = torch.zeros(64, dtype=torch.int32, device=W.device)
        self.peers = (ctypes.c_void_p * 1)(heap.peer_ptr(0, self.shard))


def _wgather(x, w, out, *, b_mn=False, own_resident=False, ahead=None, **epi):
    """``pb_gemm_wgather`` on one rank: out = x·Wᵀ (or x·W with ``b_mn``) with the epilogue of ``epi``."""
    rows, cols = w.W.shape
    F._launch(
        "pb_gemm_wgather", x.data_ptr(), w.peers, 1, 0, w.full.data_ptr(), w.flags.data_ptr(), out.data_ptr(), x.shape[0], rows, cols,
        x.stride(0), out.stride(0), int(b_mn), F._epilogue(epi.get("rope"), epi.get("swiglu_h"), epi.get("swiglu_bwd_gu")),
        int(own_resident), ahead.peers if ahead else None, ahead.full.data_ptr() if ahead else None,
        ahead.W.shape[0] if ahead else 0, ahead.W.shape[1] if ahead else 0, F._stream(),
    )  # fmt: skip


@pytest.mark.gpu
@pytest.mark.parametrize("M", [328, 300])
@pytest.mark.parametrize("mode", ["fwd", "dgrad", "ahead", "own_resident"])
def test_wgather_plain_equals_local_gemm(env, mode, M):
    from prime_b200 import ops

    g = torch.Generator(device=_dev()).manual_seed(M + len(mode))
    K, R = 512, 1088  # 1088 weight rows: the last 128-row box is clipped
    w = _Weight(env, _rand((R, K), g, 0.05))
    b_mn = mode == "dgrad"
    x = _rand((M, R if b_mn else K), g, 0.5)
    N = K if b_mn else R
    buf, out = _padded(M, N, torch.bfloat16)
    nxt = None
    if mode == "own_resident":
        w.full.copy_(w.W)
    if mode == "ahead":
        nxt = _Weight(env, _rand((640, R), g, 0.05))
    _wgather(x, w, out, b_mn=b_mn, own_resident=mode == "own_resident", ahead=nxt)
    rbuf, ref = _padded(M, N, torch.bfloat16)
    ops.gemm(x, w.W, b_mn_major=b_mn, out=ref)
    torch.cuda.synchronize()
    assert torch.equal(w.full, w.W)
    if nxt is not None:
        assert torch.equal(nxt.full, nxt.W)
    _same(buf, rbuf, N, f"wgather {mode} M={M}")


@pytest.mark.gpu
@pytest.mark.parametrize("H,Hkv,D,B,S", [(4, 1, 64, 3, 100), (2, 1, 128, 2, 164)], ids=["D64", "D128"])
def test_wgather_rope_equals_local_gemm(env, H, Hkv, D, B, S):
    from prime_b200 import ops
    from prime_b200.ops import reference as Rf

    g = torch.Generator(device=_dev()).manual_seed(H * D + S)
    K, M, nh = 256, B * S, H + 2 * Hkv
    w = _Weight(env, _rand((nh * D, K), g, K**-0.5))
    x = _rand((M, K), g)
    cos, sin = Rf.rope_tables(S + 37, D, 500000.0, device=_dev())
    rope = (cos, sin, S, (H + Hkv) * D, D)
    buf, out = _padded(M, nh * D, torch.bfloat16)
    _wgather(x, w, out, rope=rope)
    rbuf, ref = _padded(M, nh * D, torch.bfloat16)
    ops.gemm(x, w.W, out=ref, rope=rope)
    torch.cuda.synchronize()
    _same(buf, rbuf, nh * D, f"wgather rope D={D} M={M}")


@pytest.mark.gpu
@pytest.mark.parametrize("M", [328, 300])
def test_wgather_swiglu_equals_local_gemm(env, M):
    from prime_b200 import ops

    g = torch.Generator(device=_dev()).manual_seed(M)
    K, Dm, FF = 256, 384, 576  # FF % 128 = 64
    w13 = _Weight(env, _rand((2 * FF, K), g, K**-0.5 * 2))
    w2 = _Weight(env, _rand((Dm, FF), g, Dm**-0.5))  # dh = dy·W2: the input gradient of the down projection
    x, dy = _rand((M, K), g), _rand((M, Dm), g)

    gbuf, gu = _padded(M, 2 * FF, torch.bfloat16)
    hbuf, h = _padded(M, FF, torch.bfloat16)
    _wgather(x, w13, gu, swiglu_h=h)
    rgbuf, rgu = _padded(M, 2 * FF, torch.bfloat16)
    rhbuf, rh = _padded(M, FF, torch.bfloat16)
    ops.gemm(x, w13.W, out=rgu, swiglu_h=rh)
    torch.cuda.synchronize()
    _same(gbuf, rgbuf, 2 * FF, f"wgather swiglu gate_up M={M}")
    _same(hbuf, rhbuf, FF, f"wgather swiglu h M={M}")

    dbuf, dgu = _padded(M, 2 * FF, torch.bfloat16)
    _wgather(dy, w2, dgu, b_mn=True, swiglu_bwd_gu=gu)
    rdbuf, rdgu = _padded(M, 2 * FF, torch.bfloat16)
    ops.gemm(dy, w2.W, b_mn_major=True, out=rdgu, swiglu_bwd_gu=gu)
    torch.cuda.synchronize()
    _same(dbuf, rdbuf, 2 * FF, f"wgather swiglu backward M={M}")


@pytest.mark.gpu
@pytest.mark.parametrize("b_mn", [0, 1], ids=["K_major_B", "MN_major_B"])
def test_allgather_gemm_equals_local_gemm(env, b_mn):
    from prime_b200 import ops

    g = torch.Generator(device=_dev()).manual_seed(11 + b_mn)
    M, N, K = 384, 640, 320
    a = _on_heap(env, _rand((M, K), g))
    b = _rand((N, K), g, K**-0.5)
    b_st = b.t().contiguous() if b_mn else b
    full = torch.empty(M, K, dtype=torch.bfloat16, device=_dev())
    flags = torch.zeros(64, dtype=torch.int32, device=_dev())
    buf, out = _padded(M, N, torch.bfloat16)
    peers = (ctypes.c_void_p * 1)(env.peer_ptr(0, a))
    F._launch("pb_gemm_allgather", peers, 1, 0, b_st.data_ptr(), out.data_ptr(), full.data_ptr(), flags.data_ptr(), M, N, K,
              a.stride(0), b_st.stride(0), out.stride(0), b_mn, F._stream())  # fmt: skip
    rbuf, ref = _padded(M, N, torch.bfloat16)
    ops.gemm(a, b_st, b_mn_major=bool(b_mn), out=ref)
    torch.cuda.synchronize()
    _same(buf, rbuf, N, f"allgather b_mn={b_mn}")


@pytest.mark.gpu
@pytest.mark.parametrize("b_mn", [0, 1], ids=["K_major_B", "MN_major_B"])
def test_reduce_scatter_gemm_equals_local_gemm(env, b_mn):
    from prime_b200 import ops

    g = torch.Generator(device=_dev()).manual_seed(23 + b_mn)
    M, N, K = 384, 640, 320
    a = _rand((M, K), g)
    b = _rand((N, K), g, K**-0.5)
    b_st = b.t().contiguous() if b_mn else b
    buf = env.alloc(M * (N + PAD), torch.float32).view(M, N + PAD)
    buf.fill_(SENTINEL)
    out = buf[:, :N]
    out.zero_()
    peers = (ctypes.c_void_p * 1)(env.peer_ptr(0, buf))
    F._launch("pb_gemm_reduce_scatter", a.data_ptr(), b_st.data_ptr(), peers, 1, 0, M, N, K, a.stride(0), b_st.stride(0),
              buf.stride(0), b_mn, F._stream())  # fmt: skip
    rbuf, ref = _padded(M, N, torch.float32)
    ops.gemm(a, b_st, b_mn_major=bool(b_mn), out=ref, out_dtype=torch.float32)
    torch.cuda.synchronize()
    _same(buf, rbuf, N, f"reduce-scatter b_mn={b_mn}")
