"""The collective bf16 GEMMs at every group size P = 1, 2, 3, 4, 5, 8 on ONE GPU, against the local GEMM bit for bit and against
an fp64 oracle element by element.

The launchers take the other ranks' blocks as plain device addresses and build TMA maps from them, so a local allocation is as
valid a "peer" as an NVLink mapping; the readiness ``flags`` are local memory, zeroed by the launcher and published by the same
kernel's copier warps. One launch with ``rank = r`` therefore does exactly what rank r's GPU does, apart from the link the bytes
cross. At P = 1 the operands live on a one-rank symmetric heap; for P > 1 the other ranks' blocks are plain device tensors, and
every test loops over every rank r < P.

Each call is checked twice:
- bit for bit against ``pb_gemm_bf16`` at the 128-wide tile, which pins the order of the work:
  - all-gather ⊕ GEMM (IO = 1) and the forward parameter all-gather ⊕ GEMM (IO = 3, ``b_mn`` = 0: plain, RoPE, SwiGLU) only
    reorder whole tiles (``ag_tile`` / ``ag_next``, the output-column rotation ``tn_rot``), so they equal the local GEMM;
  - the IO = 3 input gradient (``b_mn`` = 1: plain, SwiGLU backward) starts its K loop at k-block ``kb_rot`` and wraps: it equals
    the local GEMM of both operands zero-padded to whole k-blocks and rolled by ``kb_rot`` (the kernel's TMA zero-fills the
    partial block too, and zero products do not change an fp32 sum);
  - GEMM ⊕ reduce-scatter (IO = 2), launched for ranks 0 … P-1 in turn into the same P zeroed fp32 buffers, leaves in buffer o
    the rank-ordered fp32 sum of the P local partial products' row block o;
- element by element against fp64 with the rule of ``test_kernel_edges_gpu.py`` (independent of the local GEMM).

Every output and every scratch the kernels write (the gathered weight ``w_full`` / ``next_full``, the gathered activations
``a_full``, the ``flags`` counters) lives inside a wider buffer filled with a sentinel that must stay bit-identical. After every
call the final counters are checked exactly: IO = 3 counts the {64 col, 128 row} boxes the copiers published per (rank block,
quarter), IO = 1 holds 1 for each remote tile row and 0 for the own rows, and a call that gathers nothing leaves them alone. In
``a_full`` every remote block equals its owner's block and the own block is not written.

A gated tile spins until its counter is complete and traps after 4 s, so a shape whose gate can never open would fault the GPU.
The CPU tests at the top model both schedules (the IO = 3 quarter arithmetic of ``gate_rows`` and the boxes ``gather_list``
publishes; the IO = 1 ``ag_tile`` / ``ag_next`` order) and check, for every (shape, P, rank) the GPU tests launch, that every tile
is produced once, every gate waits for exactly the count published to it, and every dependent all-gather tile waits only on a
gather tile of lower index; each GPU test runs the same check before it launches, and takes its expected counters from it. The
``test_checker_rejects_*`` tests show that the fp64 rule, at the GPU tests' own shapes, rejects plausible multi-rank bugs.

Edge shapes: weight rows 1080 (ragged rank blocks 540, 360, 270, 216, 135 rows, and a partial last k-block of the input
gradient; at P = 1 the last 128-row box is clipped), SwiGLU FF = 960 (FF % 128 = 64) with W2 [1080, 960], M = 300 / 328 (a partial last row tile), RoPE heads per P at D = 64 and 128, the
Llama-2 7B MLP at P = 2, 4, 8 (at P = 8 quarters of 6/6/6/4 chunk rows), all-gather N = 1000 and K = 200 (partial column tile and
k-block), and an all-gather with more gather tiles than SMs (the raster branch of ``ag_next``)."""

import ctypes

import pytest
import torch
from test_kernel_edges_gpu import (
    ROPE_ATOL,
    SILU_D_ATOL,
    SWIGLU_RTOL,
    U,
    _gemm_atol,
    _gemm_ref,
    _rejects,
    assert_elementwise,
    rope64,
    swiglu64,
    swiglu_bwd64,
)

from prime_b200.ops import functional as F
from prime_b200.ops import reference as Rf

GROUPS = (1, 2, 3, 4, 5, 8)  # 3 and 5: SwiGLU takes the plain gather order, and every shard below is ragged
PAD = 24  # padding columns (keeps every row stride a multiple of 8 elements)
GUARD = 64  # sentinel elements before and after every flat scratch (a multiple of 16 bytes)
SENTINEL = 7.0
FLAG_SENTINEL = 0x5EED5EED
SMS = 132  # H100 SXM: the grid of the schedule models on the CPU (the GPU tests use the device's own count)

# csrc/gemm_sm90.cu
BM = BN = 128
BK = 64
GROUP_M = 16  # kGroupM
GATHER_SUB = 4  # kGatherSub
AG_IDLE = 2  # kAgIdleRounds

# shapes of the GPU tests (the schedule checks below walk the same ones)
WG_ROWS, WG_COLS = 1080, 512  # rows / P = 540, 360, 270, 216, 135: every shard ragged; K = 1080 ends in a partial k-block
WG_MS = (328, 300)
WG_MODES = ("fwd", "dgrad", "ahead", "own_resident")
NEXT_SHAPE = (1080, 640)  # the gather-ahead weight
SW_K, SW_DM, SW_FF = 256, 1080, 960  # 2·FF = 1920 divides by every P; W2 [1080, 960]
LLAMA7B = dict(M=512, K=4096, Dm=4096, FF=11008)  # W13 [22016, 4096], W2 [4096, 11008]
LLAMA7B_GROUPS = (2, 4, 8)
ROPE_CASES = {"D64": (64, 3, 100), "D128": (128, 2, 164)}  # D, B, S: M = 300 / 328
ROPE_K = 256
# (H, Hkv) per (D, P): (H + 2·Hkv)·D divides by P
ROPE_HEADS = {
    64: {1: (4, 1), 2: (4, 1), 3: (4, 1), 4: (4, 1), 5: (3, 1), 8: (4, 1)},
    128: {1: (2, 1), 2: (2, 1), 3: (4, 1), 4: (2, 1), 5: (3, 1), 8: (2, 1)},
}
AG_N = 1000
AG_M_LOCAL = (128, 256)
AG_K = (320, 200)
AG_RASTER = dict(P=8, M_local=3072, N=256, K=64)  # 7 × 24 = 168 gather tiles > 132 SMs
RS_N, RS_K = 1000, 200  # K shard per rank
RS_ROWS = (128, 256)  # rows per rank: M = P·128, P·256


def _pid(P):
    return f"P{P}"


def _cdiv(a, b):
    return -(-a // b)


# -------------------------------------------------------------------------------------------------- schedule model (CPU)
def _tile_coords(tile, tiles_m, tiles_n):
    per_group = GROUP_M * tiles_n
    g = tile // per_group
    first_m = g * GROUP_M
    gsz = min(GROUP_M, tiles_m - first_m)
    r = tile - g * per_group
    return first_m + r % gsz, r // gsz


class _Gather:
    """What ``pb_gemm_wgather`` hands the kernel for a weight [rows, cols] at rank ``rank`` of ``P``: the rank block geometry,
    the copiers' block order and the tile / k-block rotation."""

    def __init__(self, rows, cols, P, rank, *, b_mn=False, kind=0, gate=True):
        assert rows % P == 0 and cols % 64 == 0
        self.P, self.rows = P, rows
        self.rpr = rows // P
        self.cpr = _cdiv(self.rpr, 128)  # 128-row chunk rows per rank block
        self.spc = _cdiv(self.cpr, GATHER_SUB)  # chunk rows per readiness counter
        self.col_chunks = cols // 64
        if kind == 2 and P % 2 == 0:  # SwiGLU: gate block g with up block g + P/2, own pair first
            h = P // 2
            g0 = rank % h
            pairs = [((g0 + t) % h, (g0 + t) % h + h) for t in range(h)]
            self.order = [b for gate_b, up_b in pairs for b in ((up_b, gate_b) if rank >= h else (gate_b, up_b))]
            start = g0 * self.rpr // 64
        else:
            self.order = [(rank + t) % P for t in range(P)]
            start = 0 if kind == 2 else rank * self.rpr // (BK if b_mn else BN)
        self.rot = start if gate else 0  # tn_rot (b_mn = 0) or kb_rot (b_mn = 1)

    def counter(self, owner, cr):
        return owner * GATHER_SUB + min(cr // self.spc, GATHER_SUB - 1)

    def boxes(self, grid, order=None):
        """(owner, chunk row, column chunk) of every box the copiers of a ``grid``-CTA launch fetch (``gather_list``)."""
        order = order or self.order
        cpb = self.cpr * self.col_chunks
        for cta in range(grid):
            for g in range(cta, cpb * self.P, grid):
                j, c = divmod(g, cpb)
                yield order[j], c // self.col_chunks, c % self.col_chunks

    def published(self, grid, order=None):
        """Boxes published to each counter; every box of the weight exactly once."""
        counts = [0] * (self.P * GATHER_SUB)
        seen = set()
        for owner, cr, cc in self.boxes(grid, order):
            assert (owner, cr, cc) not in seen, f"box {(owner, cr, cc)} fetched twice"
            seen.add((owner, cr, cc))
            counts[self.counter(owner, cr)] += 1
        assert len(seen) == self.P * self.cpr * self.col_chunks, "boxes left out of the gather"
        return counts

    def waits(self, r0, r1):
        """(counter, count it waits for) of every quarter block the producer's ``gate_rows(r0, r1)`` waits on."""
        out, x = [], r0
        while x <= r1:
            b = x // self.rpr
            cr = (x - b * self.rpr) >> 7
            q = min(cr // self.spc, GATHER_SUB - 1)
            cr_end = self.cpr if q == GATHER_SUB - 1 else min(self.cpr, (q + 1) * self.spc)
            out.append((b * GATHER_SUB + q, (cr_end - q * self.spc) * self.col_chunks))
            nx = b * self.rpr + min(self.rpr, cr_end * 128)
            assert nx > x, f"gate_rows makes no progress at row {x}"
            x = nx
        return out


def _preflight_wgather(M, rows, cols, P, rank, *, b_mn=False, kind=0, gate=True, ahead=None, grid=SMS):
    """The IO = 3 schedule of one launch: every output tile once, every k-block once per tile, every gate waiting for exactly
    the boxes published to its counter, every box of the weight (and of the gather-ahead weight) fetched once. Returns the
    plan; ``plan.flags`` are the final counters (None: the launch does not touch them)."""
    plan = _Gather(rows, cols, P, rank, b_mn=b_mn, kind=kind, gate=gate)
    N, K = (cols, rows) if b_mn else (rows, cols)
    ff = N // 2 if kind == 2 else 0
    tiles_m = _cdiv(M, BM)
    tiles_n = ff // 64 if kind == 2 else _cdiv(N, BN)
    num_kb = _cdiv(K, BK)
    grid = min(grid, tiles_m * tiles_n)
    tag = f"wgather rows={rows} cols={cols} b_mn={int(b_mn)} epi={kind} P={P} rank={rank}"
    published = plan.published(grid) if gate else None

    def check(r0, r1):
        for cid, expect in plan.waits(r0, r1):
            assert expect > 0 and expect == published[cid], f"{tag}: rows {r0}..{r1} wait for {expect} at counter {cid}, " \
                                                            f"which receives {published[cid]}"  # fmt: skip

    seen, gated = set(), set()
    for cta in range(grid):
        for tile in range(cta, tiles_m * tiles_n, grid):
            tm, tn = _tile_coords(tile, tiles_m, tiles_n)
            if not b_mn and plan.rot:
                tn = (tn + plan.rot) % tiles_n
            assert (tm, tn) not in seen, f"{tag}: tile {(tm, tn)} twice"
            seen.add((tm, tn))
            if gate and not b_mn and tn not in gated:
                gated.add(tn)
                if kind == 2:
                    check(tn * 64, min(tn * 64 + 64, rows) - 1)
                    check(ff + tn * 64, min(ff + tn * 64 + 64, rows) - 1)
                else:
                    check(tn * BN, min(tn * BN + BN, rows) - 1)
    assert len(seen) == tiles_m * tiles_n, f"{tag}: tiles left out"
    kbs = [(kbi + plan.rot) % num_kb for kbi in range(num_kb)] if b_mn else list(range(num_kb))
    assert sorted(kbs) == list(range(num_kb)), f"{tag}: the K loop is not a permutation of the k-blocks"
    if gate and b_mn:
        for kb in kbs:
            check(kb * BK, min(kb * BK + BK, rows) - 1)
    if ahead is not None:
        _Gather(*ahead, P, rank).published(grid, order=[(rank + 1 + t) % P for t in range(P)])
    plan.flags = published
    return plan


def _preflight_allgather(M_local, N, P, rank, grid=SMS):
    """The IO = 1 schedule of one launch (``ag_next`` over the CTAs, ``ag_tile``): every tile index and every output tile
    once, each CTA's indices increasing with its gather tiles first (its copier stops at the first other tile), every dependent
    tile behind the gather tile of its row block. Returns the final flags (None: untouched) and whether ``ag_next`` took the
    plain raster branch (more gather tiles than CTAs)."""
    tpr, tiles_n = M_local // BM, _cdiv(N, BN)
    num_tiles = P * tpr * tiles_n
    grid = min(grid, num_tiles)
    tag = f"allgather M_local={M_local} N={N} P={P} rank={rank}"
    if P == 1:
        assert {_tile_coords(t, tpr, tiles_n) for t in range(num_tiles)} == {(m, n) for m in range(tpr) for n in range(tiles_n)}
        return None, False
    G, L = (P - 1) * tpr, tpr * tiles_n

    def ag_tile(idx):
        if idx < G:
            return ((rank + 1 + idx % (P - 1)) % P) * tpr + idx // (P - 1), 0, 1
        if idx < G + L:
            j = idx - G
            return rank * tpr + j % tpr, j // tpr, 0
        j = idx - G - L
        g = j % G
        return ((rank + 1 + g % (P - 1)) % P) * tpr + g // (P - 1), 1 + j // G, 2

    def ag_next(it, cta):
        if G > grid:
            t = cta + it * grid
            return t if t < num_tiles else -2
        R = num_tiles - G
        if it == 0:
            if cta < G:
                return cta
            r = cta - G
        elif it <= AG_IDLE:
            if cta < G:
                return -1
            r = (grid - G) * it + (cta - G)
        else:
            r = (grid - G) * (AG_IDLE + 1) + (it - AG_IDLE - 1) * grid + cta
        return G + r if r < R else -2

    seen = set()
    for cta in range(grid):
        seq, it = [], 0
        while (t := ag_next(it, cta)) != -2:
            it += 1
            assert it <= num_tiles + AG_IDLE + 1, f"{tag}: CTA {cta} never finishes"
            if t >= 0:
                seq.append(t)
        assert seq == sorted(seq), f"{tag}: CTA {cta} takes its tiles out of order"
        kinds = [ag_tile(t)[2] for t in seq]
        assert kinds == sorted(kinds, key=lambda k: k != 1), f"{tag}: CTA {cta} has a gather tile behind another tile"
        for t in seq:
            assert t not in seen, f"{tag}: tile {t} twice"
            seen.add(t)
    assert seen == set(range(num_tiles)), f"{tag}: tiles left out"
    gather_of, coords = {}, set()
    for t in range(num_tiles):
        tm, tn, kind = ag_tile(t)
        remote = tm // tpr != rank
        assert kind == 0 or remote, f"{tag}: tile {t} gathers the own block"
        if kind == 1:
            assert tn == 0 and tm not in gather_of
            gather_of[tm] = t
        if kind == 2:
            assert gather_of.get(tm, num_tiles) < t, f"{tag}: dependent tile {t} waits on a later or missing gather tile"
        coords.add((tm, tn))
    assert len(coords) == num_tiles, f"{tag}: output tiles left out"
    return [int(tm // tpr != rank) for tm in range(P * tpr)], G > grid


def _preflight_reduce_scatter(M, P, rank):
    """IO = 2: the owner-interleaved row order ``rs_tile_row`` visits every tile row once."""
    tpr = M // P // BM
    rows = [((rank + 1 + t % P) % P) * tpr + t // P for t in range(P * tpr)]
    assert sorted(rows) == list(range(P * tpr)), f"reduce-scatter M={M} P={P} rank={rank}: rs_tile_row is not a permutation"


def _io3_launches(P):
    """Every IO = 3 launch the GPU tests make at group size P, as keyword arguments of ``_preflight_wgather``."""
    for mode in WG_MODES:
        for M in WG_MS:
            yield dict(M=M, rows=WG_ROWS, cols=WG_COLS, b_mn=mode == "dgrad", gate=mode != "own_resident",
                       ahead=NEXT_SHAPE if mode == "ahead" else None)  # fmt: skip
    for D, B, S in ROPE_CASES.values():
        H, Hkv = ROPE_HEADS[D][P]
        yield dict(M=B * S, rows=(H + 2 * Hkv) * D, cols=ROPE_K, kind=1)
    shapes = [(M, SW_K, SW_DM, SW_FF) for M in WG_MS]
    if P in LLAMA7B_GROUPS:
        shapes.append((LLAMA7B["M"], LLAMA7B["K"], LLAMA7B["Dm"], LLAMA7B["FF"]))
    for M, K, Dm, FF in shapes:
        yield dict(M=M, rows=2 * FF, cols=K, kind=2)
        yield dict(M=M, rows=Dm, cols=FF, b_mn=True, kind=3)


def _io1_launches(P):
    for M_local in AG_M_LOCAL:
        yield M_local, AG_N
    if P == AG_RASTER["P"]:
        yield AG_RASTER["M_local"], AG_RASTER["N"]


@pytest.mark.parametrize("P", GROUPS, ids=_pid)
def test_preflight_wgather_schedules(P):
    for launch in _io3_launches(P):
        for r in range(P):
            _preflight_wgather(P=P, rank=r, **launch)


@pytest.mark.parametrize("P", GROUPS, ids=_pid)
def test_preflight_allgather_schedules(P):
    for M_local, N in _io1_launches(P):
        for r in range(P):
            _preflight_allgather(M_local, N, P, r)


@pytest.mark.parametrize("P", GROUPS, ids=_pid)
def test_preflight_reduce_scatter_schedules(P):
    for rows in RS_ROWS:
        for r in range(P):
            _preflight_reduce_scatter(P * rows, P, r)


def test_preflight_counters_of_the_issue_examples():
    """The final counters: (128-row chunk rows of the quarter) × colsW / 64 per rank block, 0 where no box maps."""
    plan = _preflight_wgather(300, 1080, 512, 2, 0)
    assert plan.flags == [n * 8 for n in (2, 2, 1, 0)] * 2
    plan = _preflight_wgather(512, 22016, 4096, 8, 5, kind=2)
    assert plan.flags == [n * 64 for n in (6, 6, 6, 4)] * 8
    assert _preflight_wgather(300, 1080, 512, 2, 1, gate=False).flags is None
    flags, raster = _preflight_allgather(AG_RASTER["M_local"], AG_RASTER["N"], 8, 3)
    assert raster and flags == [int(b != 3) for b in range(8) for _ in range(24)]
    assert not _preflight_allgather(256, AG_N, 8, 3)[1]


def test_preflight_rejects_an_unreachable_gate(monkeypatch):
    """The model is not vacuous: copiers that split a rank block into proportional quarters (22 chunk rows → 6/5/6/5) while the
    gates wait for ceil-sized ones (6/6/6/4) leave a gate that never opens, and the check says so."""
    _preflight_wgather(512, 22016, 4096, 8, 0, kind=2)
    monkeypatch.setattr(_Gather, "counter", lambda self, owner, cr: owner * GATHER_SUB + cr * GATHER_SUB // self.cpr)
    with pytest.raises(AssertionError, match="wait for"):
        _preflight_wgather(512, 22016, 4096, 8, 0, kind=2)


# -------------------------------------------------------------------------------------------------- CPU: the rule rejects bugs
def _cpu_rand(shape, g, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).to(torch.bfloat16)


def _bf16_gemm(a, b):
    """a·bᵀ in fp32, rounded once to bf16: a correct result to mutate."""
    return (a.float() @ b.float().t()).to(torch.bfloat16)


@pytest.mark.parametrize("P", (2, 8), ids=_pid)
def test_checker_rejects_swapped_weight_blocks(P):
    """A wrong ``order[]``: the copiers store rank block 1's rows where block 0 belongs and the other way round."""
    g = torch.Generator().manual_seed(31)
    x, W = _cpu_rand((300, WG_COLS), g, 0.5), _cpu_rand((WG_ROWS, WG_COLS), g, 0.05)
    ref, sc = _gemm_ref(x, W)
    assert not _rejects(_bf16_gemm(x, W), ref, U, _gemm_atol(WG_COLS), sc)
    rpr = WG_ROWS // P
    bad = torch.cat((W[rpr : 2 * rpr], W[:rpr], W[2 * rpr :]))
    assert _rejects(_bf16_gemm(x, bad), ref, U, _gemm_atol(WG_COLS), sc)


@pytest.mark.parametrize("P", (2, 8), ids=_pid)
def test_checker_rejects_unclipped_ragged_tail(P):
    """The store of rank block 0's last chunk row not clipped at the block's end: block 1 lands behind the zero-filled rows."""
    g = torch.Generator().manual_seed(37)
    x, W = _cpu_rand((300, WG_COLS), g, 0.5), _cpu_rand((WG_ROWS, WG_COLS), g, 0.05)
    ref, sc = _gemm_ref(x, W)
    rpr = WG_ROWS // P
    tail = _cdiv(rpr, 128) * 128 - rpr
    assert tail > 0
    bad = torch.cat((W[:rpr], torch.zeros(tail, WG_COLS, dtype=W.dtype), W[rpr:]))[:WG_ROWS]
    assert _rejects(_bf16_gemm(x, bad), ref, U, _gemm_atol(WG_COLS), sc)
    # the input gradient over the same weight: the contraction runs over the shifted rows
    dy = _cpu_rand((300, WG_ROWS), g, 0.5)
    dref, dsc = _gemm_ref(dy, W.t())
    assert not _rejects(_bf16_gemm(dy, W.t()), dref, U, _gemm_atol(WG_ROWS), dsc)
    assert _rejects(_bf16_gemm(dy, bad.t()), dref, U, _gemm_atol(WG_ROWS), dsc)


@pytest.mark.parametrize("P", (2, 5), ids=_pid)
def test_checker_rejects_doubled_or_missing_partial(P):
    """The reduce-scatter adding one peer's partial product twice, or not at all, into an owner's rows."""
    g = torch.Generator().manual_seed(41)
    M = P * RS_ROWS[0]
    A = [_cpu_rand((M, RS_K), g) for _ in range(P)]
    B = [_cpu_rand((RS_N, RS_K), g, (P * RS_K) ** -0.5) for _ in range(P)]
    ref, sc = _gemm_ref(torch.cat(A, 1), torch.cat(B, 1))
    parts = [a.float() @ b.float().t() for a, b in zip(A, B)]
    atol = _gemm_atol(P * RS_K)
    assert not _rejects(sum(parts), ref, 0.0, atol, sc)
    assert _rejects(sum(parts) + parts[1], ref, 0.0, atol, sc)
    assert _rejects(sum(parts) - parts[1], ref, 0.0, atol, sc)


# -------------------------------------------------------------------------------------------------- GPU harness
def _dev():
    return torch.device("cuda", 0)


def _sms():
    return torch.cuda.get_device_properties(_dev()).multi_processor_count


@pytest.fixture
def env():
    """A one-rank symmetric heap for the P = 1 operands, with the local GEMM forced to the collective variants' tile."""
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


def _framed(n, dtype, fill):
    """``n`` elements inside a flat buffer with GUARD sentinel elements on either side: (buffer, the n-element view)."""
    buf = torch.full((n + 2 * GUARD,), fill, dtype=dtype, device=_dev())
    return buf, buf[GUARD : GUARD + n]


def _guards(buf, fill, what):
    for band in (buf[:GUARD], buf[-GUARD:]):
        assert bool((band == fill).all()), f"{what}: the guard band next to it was written"


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


def _blocks(heap, blocks):
    """The ranks' blocks as the kernels see them: on the one-rank heap at P = 1, plain device tensors otherwise."""
    if len(blocks) == 1:
        held = [_on_heap(heap, blocks[0])]
        ptrs = [heap.peer_ptr(0, held[0])]
    else:
        held = [b.contiguous() for b in blocks]
        ptrs = [b.data_ptr() for b in held]
    return held, (ctypes.c_void_p * len(ptrs))(*ptrs)


class _Weight:
    """A weight W [rows, cols] row-sharded over P ranks: the shards, and the local full-size scratch and counters the kernel
    gathers into, each inside a sentinel-filled buffer."""

    def __init__(self, heap, W, P):
        rows, cols = W.shape
        self.W, self.P = W, P
        self.shards, self.peers = _blocks(heap, list(W.chunk(P)))
        self.fbuf, full = _framed(rows * cols, torch.bfloat16, SENTINEL)
        self.full = full.view(rows, cols)
        self.gbuf, self.flags = _framed(P * GATHER_SUB, torch.int32, FLAG_SENTINEL)

    def reset(self, resident=False):
        """Before a call: the scratch holds the sentinel (or, ``resident``, the whole weight) and the counters garbage."""
        if resident:
            self.full.copy_(self.W)
        else:
            self.full.fill_(SENTINEL)
        self.flags.fill_(FLAG_SENTINEL)

    def check(self, flags, what):
        """After a call: the whole weight gathered, nothing written around it, the counters at ``flags`` (None: untouched)."""
        _guards(self.fbuf, SENTINEL, f"{what} w_full")
        _guards(self.gbuf, FLAG_SENTINEL, f"{what} flags")
        assert torch.equal(self.full, self.W), f"{what}: w_full is not the weight"
        want = [FLAG_SENTINEL] * (self.P * GATHER_SUB) if flags is None else flags
        assert self.flags.tolist() == want, f"{what}: counters {self.flags.tolist()}, want {want}"


def _wgather(x, w, out, rank, *, b_mn=False, own_resident=False, ahead=None, **epi):
    """``pb_gemm_wgather`` at rank ``rank`` of ``w.P``: out = x·Wᵀ (or x·W with ``b_mn``) with the epilogue of ``epi``."""
    rows, cols = w.W.shape
    F._launch(
        "pb_gemm_wgather", x.data_ptr(), w.peers, w.P, rank, w.full.data_ptr(), w.flags.data_ptr(), out.data_ptr(), x.shape[0], rows,
        cols, x.stride(0), out.stride(0), int(b_mn), F._epilogue(epi.get("rope"), epi.get("swiglu_h"), epi.get("swiglu_bwd_gu")),
        int(own_resident), ahead.peers if ahead else None, ahead.full.data_ptr() if ahead else None,
        ahead.W.shape[0] if ahead else 0, ahead.W.shape[1] if ahead else 0, F._stream(),
    )  # fmt: skip


def _rolled(x, W, kb_rot):
    """x [M, K] and W [K, N] zero-padded to whole k-blocks and rolled so that k-block ``kb_rot`` comes first: the local GEMM of
    the two accumulates in the order of the kernel's rotated K loop."""
    K, N = W.shape
    Kp = _cdiv(K, BK) * BK
    xp = torch.zeros(x.shape[0], Kp, dtype=x.dtype, device=x.device)
    wp = torch.zeros(Kp, N, dtype=W.dtype, device=W.device)
    xp[:, :K], wp[:K] = x, W
    return torch.roll(xp, -kb_rot * BK, 1).contiguous(), torch.roll(wp, -kb_rot * BK, 0).contiguous()


# -------------------------------------------------------------------------------------------------- GPU: IO = 3
@pytest.mark.gpu
@pytest.mark.parametrize("M", WG_MS)
@pytest.mark.parametrize("mode", WG_MODES)
@pytest.mark.parametrize("P", GROUPS, ids=_pid)
def test_wgather_plain_equals_local_gemm(env, P, mode, M):
    from prime_b200 import ops

    g = torch.Generator(device=_dev()).manual_seed(M + len(mode) + 100 * P)
    R, K = WG_ROWS, WG_COLS
    w = _Weight(env, _rand((R, K), g, 0.05), P)
    b_mn = mode == "dgrad"
    x = _rand((M, R if b_mn else K), g, 0.5)
    N = K if b_mn else R
    nxt = _Weight(env, _rand(NEXT_SHAPE, g, 0.05), P) if mode == "ahead" else None
    ref64, sc = _gemm_ref(x, w.W.t() if b_mn else w.W)
    rbuf, ref = _padded(M, N, torch.bfloat16)
    if not b_mn:
        ops.gemm(x, w.W, out=ref)  # the forward reference (the input gradient's is rolled per rank below)
    for r in range(P):
        tag = f"wgather {mode} P={P} rank={r} M={M}"
        plan = _preflight_wgather(M, R, K, P, r, b_mn=b_mn, gate=mode != "own_resident", ahead=NEXT_SHAPE if nxt else None,
                                  grid=_sms())  # fmt: skip
        w.reset(resident=mode == "own_resident")
        if nxt is not None:
            nxt.reset()
        buf, out = _padded(M, N, torch.bfloat16)
        _wgather(x, w, out, r, b_mn=b_mn, own_resident=mode == "own_resident", ahead=nxt)
        if b_mn:
            rbuf, ref = _padded(M, N, torch.bfloat16)
            ops.gemm(*_rolled(x, w.W, plan.rot), b_mn_major=True, out=ref)
        torch.cuda.synchronize()
        w.check(plan.flags, tag)
        if nxt is not None:
            _guards(nxt.fbuf, SENTINEL, f"{tag} next_full")
            assert torch.equal(nxt.full, nxt.W), f"{tag}: next_full is not the next weight"
        _same(buf, rbuf, N, tag)
        assert_elementwise(out, ref64, U, _gemm_atol(R if b_mn else K), tag, sc)


def _assert_rope(y, ref, sc, cos, sin, H, Hkv, D, B, S, K, what):
    """The RoPE epilogue against fp64: Q/K head columns rotated, V columns the plain product (test_kernel_edges_gpu.py)."""
    nh, rot = H + 2 * Hkv, (H + Hkv) * D
    rref, _ = rope64(ref.view(B, S, nh, D)[:, :, : H + Hkv], cos, sin)
    s4 = sc.view(B, S, nh, D)[:, :, : H + Hkv]
    pair_sc = s4.reshape(B, S, H + Hkv, D // 2, 2).sum(-1, keepdim=True).expand(B, S, H + Hkv, D // 2, 2).reshape(B, S, H + Hkv, D)
    y4 = y.view(B, S, nh, D)
    assert_elementwise(y4[:, :, : H + Hkv], rref, U, _gemm_atol(K) + ROPE_ATOL, f"{what} rotated", pair_sc)
    assert_elementwise(y[:, rot:], ref[:, rot:], U, _gemm_atol(K), f"{what} plain", sc[:, rot:])


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(ROPE_CASES))
@pytest.mark.parametrize("P", GROUPS, ids=_pid)
def test_wgather_rope_equals_local_gemm(env, P, case):
    from prime_b200 import ops

    D, B, S = ROPE_CASES[case]
    H, Hkv = ROPE_HEADS[D][P]
    g = torch.Generator(device=_dev()).manual_seed(H * D + S + 100 * P)
    K, M, nh = ROPE_K, B * S, H + 2 * Hkv
    w = _Weight(env, _rand((nh * D, K), g, K**-0.5), P)
    x = _rand((M, K), g)
    cos, sin = Rf.rope_tables(S + 37, D, 500000.0, device=_dev())
    rope = (cos, sin, S, (H + Hkv) * D, D)
    rbuf, ref = _padded(M, nh * D, torch.bfloat16)
    ops.gemm(x, w.W, out=ref, rope=rope)
    ref64, sc = _gemm_ref(x, w.W)
    for r in range(P):
        tag = f"wgather rope H={H} Hkv={Hkv} D={D} P={P} rank={r} M={M}"
        plan = _preflight_wgather(M, nh * D, K, P, r, kind=1, grid=_sms())
        w.reset()
        buf, out = _padded(M, nh * D, torch.bfloat16)
        _wgather(x, w, out, r, rope=rope)
        torch.cuda.synchronize()
        w.check(plan.flags, tag)
        _same(buf, rbuf, nh * D, tag)
        _assert_rope(out, ref64, sc, cos, sin, H, Hkv, D, B, S, K, tag)


def _swiglu_case(env, P, M, K, Dm, FF, seed):
    """SwiGLU forward (gate_up and h from W13 [2·FF, K]) and backward (d_gate_up from dy·W2, W2 [Dm, FF]) at every rank."""
    from prime_b200 import ops

    g = torch.Generator(device=_dev()).manual_seed(seed)
    w13 = _Weight(env, _rand((2 * FF, K), g, K**-0.5 * 2), P)
    w2 = _Weight(env, _rand((Dm, FF), g, Dm**-0.5), P)  # dh = dy·W2: the input gradient of the down projection
    x, dy = _rand((M, K), g), _rand((M, Dm), g)

    rgbuf, rgu = _padded(M, 2 * FF, torch.bfloat16)
    rhbuf, rh = _padded(M, FF, torch.bfloat16)
    ops.gemm(x, w13.W, out=rgu, swiglu_h=rh)
    ref64, sc = _gemm_ref(x, w13.W)
    dh, dh_sc = _gemm_ref(dy, w2.W.t())
    dref, _ = swiglu_bwd64(rgu, dh)
    gg, uu = rgu.double().chunk(2, dim=-1)
    sg = torch.sigmoid(gg)
    d_gate_sc = uu.abs() * (sg.abs() + (gg * sg * (1 - sg)).abs()) * dh_sc
    d_up_sc = (gg * sg).abs() * dh_sc
    torch.cuda.synchronize()
    assert_elementwise(rh, swiglu64(rgu), SWIGLU_RTOL, 0.0, f"swiglu h (local) FF={FF} M={M}")
    for r in range(P):
        tag = f"wgather swiglu FF={FF} P={P} rank={r} M={M}"
        plan = _preflight_wgather(M, 2 * FF, K, P, r, kind=2, grid=_sms())
        w13.reset()
        gbuf, gu = _padded(M, 2 * FF, torch.bfloat16)
        hbuf, h = _padded(M, FF, torch.bfloat16)
        _wgather(x, w13, gu, r, swiglu_h=h)
        torch.cuda.synchronize()
        w13.check(plan.flags, tag)
        _same(gbuf, rgbuf, 2 * FF, f"{tag} gate_up")
        _same(hbuf, rhbuf, FF, f"{tag} h")
        assert_elementwise(gu, ref64, U, _gemm_atol(K), f"{tag} gate_up", sc)

        tag = f"wgather swiglu backward FF={FF} P={P} rank={r} M={M}"
        plan = _preflight_wgather(M, Dm, FF, P, r, b_mn=True, kind=3, grid=_sms())
        w2.reset()
        dbuf, dgu = _padded(M, 2 * FF, torch.bfloat16)
        _wgather(dy, w2, dgu, r, b_mn=True, swiglu_bwd_gu=rgu)
        rdbuf, rdgu = _padded(M, 2 * FF, torch.bfloat16)
        ops.gemm(*_rolled(dy, w2.W, plan.rot), b_mn_major=True, out=rdgu, swiglu_bwd_gu=rgu)
        torch.cuda.synchronize()
        w2.check(plan.flags, tag)
        _same(dbuf, rdbuf, 2 * FF, tag)
        # the epilogue keeps dh in fp32 (test_gemm_swiglu_epilogues_and_fallbacks)
        assert_elementwise(dgu[:, :FF], dref[:, :FF], SWIGLU_RTOL, _gemm_atol(Dm) + SILU_D_ATOL, f"{tag} d_gate", d_gate_sc)
        assert_elementwise(dgu[:, FF:], dref[:, FF:], SWIGLU_RTOL, _gemm_atol(Dm), f"{tag} d_up", d_up_sc)


@pytest.mark.gpu
@pytest.mark.parametrize("M", WG_MS)
@pytest.mark.parametrize("P", GROUPS, ids=_pid)
def test_wgather_swiglu_equals_local_gemm(env, P, M):
    _swiglu_case(env, P, M, SW_K, SW_DM, SW_FF, seed=M + 100 * P)


@pytest.mark.gpu
@pytest.mark.parametrize("P", LLAMA7B_GROUPS, ids=_pid)
def test_wgather_swiglu_llama7b_mlp(env, P):
    """The Llama-2 7B MLP: W13 [22016, 4096] forward, W2 [4096, 11008] input gradient (at P = 8: rank blocks of 2752 rows,
    quarters of 6/6/6/4 chunk rows)."""
    c = LLAMA7B
    _swiglu_case(env, P, c["M"], c["K"], c["Dm"], c["FF"], seed=7 + P)


# -------------------------------------------------------------------------------------------------- GPU: IO = 1
def _allgather_case(env, P, M_local, N, K, b_mn, seed, raster=False):
    from prime_b200 import ops

    g = torch.Generator(device=_dev()).manual_seed(seed)
    M = P * M_local
    blocks = [_rand((M_local, K), g) for _ in range(P)]
    held, peers = _blocks(env, blocks)
    a = torch.cat(blocks)
    b = _rand((N, K), g, K**-0.5)
    b_st = b.t().contiguous() if b_mn else b
    rbuf, ref = _padded(M, N, torch.bfloat16)
    ops.gemm(a, b_st, b_mn_major=bool(b_mn), out=ref)
    ref64, sc = _gemm_ref(a, b)
    tpr = M_local // BM
    fbuf, full = _framed(M * K, torch.bfloat16, SENTINEL)
    full = full.view(M, K)
    gbuf, flags = _framed(P * tpr, torch.int32, FLAG_SENTINEL)
    for r in range(P):
        tag = f"allgather b_mn={b_mn} P={P} rank={r} M_local={M_local} K={K} N={N}"
        want_flags, took_raster = _preflight_allgather(M_local, N, P, r, grid=_sms())
        assert took_raster == raster, f"{tag}: the case takes the other branch of ag_next"
        full.fill_(SENTINEL)
        flags.fill_(FLAG_SENTINEL)
        buf, out = _padded(M, N, torch.bfloat16)
        F._launch("pb_gemm_allgather", peers, P, r, b_st.data_ptr(), out.data_ptr(), full.data_ptr(), flags.data_ptr(), M_local, N, K,
                  held[0].stride(0), b_st.stride(0), out.stride(0), b_mn, F._stream())  # fmt: skip
        torch.cuda.synchronize()
        _same(buf, rbuf, N, tag)
        assert_elementwise(out, ref64, U, _gemm_atol(K), tag, sc)
        _guards(fbuf, SENTINEL, f"{tag} a_full")
        _guards(gbuf, FLAG_SENTINEL, f"{tag} flags")
        for o in range(P):
            blk = full[o * M_local : (o + 1) * M_local]
            if o == r:  # the own block is read in place, never copied
                assert bool((blk == SENTINEL).all()), f"{tag}: the own block of a_full was written"
            else:
                assert torch.equal(blk, blocks[o]), f"{tag}: block {o} of a_full is not rank {o}'s block"
        want = [FLAG_SENTINEL] * (P * tpr) if want_flags is None else want_flags
        assert flags.tolist() == want, f"{tag}: flags {flags.tolist()}, want {want}"


@pytest.mark.gpu
@pytest.mark.parametrize("b_mn", [0, 1], ids=["K_major_B", "MN_major_B"])
@pytest.mark.parametrize("K", AG_K)
@pytest.mark.parametrize("M_local", AG_M_LOCAL)
@pytest.mark.parametrize("P", GROUPS, ids=_pid)
def test_allgather_gemm_equals_local_gemm(env, P, M_local, K, b_mn):
    _allgather_case(env, P, M_local, AG_N, K, b_mn, seed=11 + b_mn + K + M_local + 100 * P)


@pytest.mark.gpu
@pytest.mark.parametrize("b_mn", [0, 1], ids=["K_major_B", "MN_major_B"])
def test_allgather_gemm_raster_schedule(env, b_mn):
    """More gather tiles than CTAs: ``ag_next`` hands the tiles out in plain raster order."""
    c = AG_RASTER
    assert (c["P"] - 1) * c["M_local"] // BM > _sms()
    _allgather_case(env, c["P"], c["M_local"], c["N"], c["K"], b_mn, seed=13 + b_mn, raster=True)


# -------------------------------------------------------------------------------------------------- GPU: IO = 2
@pytest.mark.gpu
@pytest.mark.parametrize("b_mn", [0, 1], ids=["K_major_B", "MN_major_B"])
@pytest.mark.parametrize("rows", RS_ROWS)
@pytest.mark.parametrize("P", GROUPS, ids=_pid)
def test_reduce_scatter_gemm_equals_local_gemm(env, P, rows, b_mn):
    """Ranks 0 … P-1 in turn, each with its own K shard, into the same P zeroed fp32 buffers: buffer o ends up holding
    ((0 + P_0[o]) + P_1[o]) + …, the rank-ordered fp32 sum of the local partial products' row block o."""
    from prime_b200 import ops

    g = torch.Generator(device=_dev()).manual_seed(23 + b_mn + rows + 100 * P)
    M, N, K = P * rows, RS_N, RS_K
    A = [_rand((M, K), g) for _ in range(P)]
    B = [_rand((N, K), g, (P * K) ** -0.5) for _ in range(P)]
    B_st = [b.t().contiguous() if b_mn else b for b in B]
    if P == 1:
        bufs = [env.alloc(rows * (N + PAD), torch.float32).view(rows, N + PAD)]
        ptrs = [env.peer_ptr(0, bufs[0])]
    else:
        bufs = [torch.empty(rows, N + PAD, dtype=torch.float32, device=_dev()) for _ in range(P)]
        ptrs = [t.data_ptr() for t in bufs]
    for t in bufs:
        t.fill_(SENTINEL)
        t[:, :N].zero_()
    peers = (ctypes.c_void_p * P)(*ptrs)
    for s in range(P):
        _preflight_reduce_scatter(M, P, s)
        F._launch("pb_gemm_reduce_scatter", A[s].data_ptr(), B_st[s].data_ptr(), peers, P, s, M, N, K, A[s].stride(0),
                  B_st[s].stride(0), N + PAD, b_mn, F._stream())  # fmt: skip
    partials = [ops.gemm(a, b, b_mn_major=bool(b_mn), out_dtype=torch.float32) for a, b in zip(A, B_st)]
    ref64, sc = _gemm_ref(torch.cat(A, 1), torch.cat(B, 1))
    torch.cuda.synchronize()
    for o in range(P):
        tag = f"reduce-scatter b_mn={b_mn} P={P} owner={o} M={M}"
        wbuf, want = _padded(rows, N, torch.float32)
        want.zero_()
        for p in partials:
            want.copy_(want + p[o * rows : (o + 1) * rows])
        _same(bufs[o], wbuf, N, tag)
        blk = slice(o * rows, (o + 1) * rows)
        assert_elementwise(bufs[o][:, :N], ref64[blk], 0.0, _gemm_atol(P * K), tag, sc[blk])
