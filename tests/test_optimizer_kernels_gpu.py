"""The kernels that write the weights (csrc/comm.cu: gradient reduce-scatter, norm publication, fused AdamW + bf16 push, DiLoCo
pseudo-gradient quantiser and both outer Nesterov steps, cast + push; csrc/embedding.cu: peer all-gather copy and the row-sharded
embedding lookup) against an fp64 oracle or a bit-exact fp32 emulation, at every peer count, on ONE GPU.

Every one of these kernels takes its peers as plain device pointers (``PeerPtrs``, up to 8), and a local allocation is as valid a
"peer" for ``ld.relaxed.sys`` / ``st.release.sys`` / ``stg`` as a mapped one, so local tensors stand in for the other ranks and one
device runs every template instantiation and every peer count. A flag a kernel waits on always holds its epoch before the wait
starts (written by ``pb_signal`` / ``pb_norm_publish`` earlier in the same stream): no test reaches a spin timeout.

Every output lives inside a larger buffer filled with a sentinel, and the whole buffer is compared (the guard bands bit for bit);
the error word is checked after every call. Where a kernel's arithmetic is fixed (sums in rank order, an add followed by a
multiply, IEEE divisions feeding rint) the check is bitwise against a torch fp32 emulation; otherwise the per-element rule of
``test_kernel_edges_gpu.py`` applies, |got - ref| <= rtol·|ref| + atol·scale, with ``scale`` the magnitude of the terms that the
element's fp32 arithmetic rounds, and each tolerance names the roundings it covers. The CPU tests at the top show that the same
rules, at the GPU tests' own shapes and step numbers, reject each plausible bug, and that the launchers refuse impossible
arguments before touching the device.

Coverage (test names below):
- ``grad_reduce_kernel<4,1>``, ``<4,2>``, ``<2,4>`` (P = 3, 4) and ``<1,8>`` (P = 5, 8) through ``pb_grad_reduce``: one segment of one
  vector and one vector past whole grid-stride passes, every rank of the bucket, ``max_ctas`` 0 / 7, sum of squares over two
  buckets: test_grad_reduce_one_segment; 1 and 16 irregular segments and gaps, and none: test_grad_reduce_segments; the host-abort
  error word with the flags not yet signalled (the prologue the multicast instantiation shares; a multicast address needs two GPUs
  on an NVSwitch, tests/test_multigpu.py): test_grad_reduce_abort
- ``norm_publish_kernel``: test_norm_publish; ``adamw_push_kernel``: test_adamw_push; both through the engine at F = 1:
  test_engine_step_matches_fp64_adamw
- ``pseudograd_quant_kernel`` edge blocks (zero, ties, ±absmax at both ends, subnormal scale, scale 0, idle groups, grid-stride
  loop): test_pseudograd_quant
- ``outer_nesterov_kernel`` / ``outer_nesterov_f32_kernel``, W up to 8 workers, bucket tables with up to 37 entries, up to 8
  destinations, the host-abort error word: test_outer_nesterov_int8, test_outer_nesterov_f32
- ``cast_push_kernel``, ``allgather_copy_kernel``, ``embedding_fwd_kernel`` (row shards): test_cast_push, test_allgather_copy,
  test_embedding_fwd_row_shards
"""

import ctypes
import math

import pytest
import torch
from test_kernel_edges_gpu import U32, _rejects, assert_elementwise

from prime_b200.ops import _lib
from prime_b200.ops import reference as Rf

PEERS = (1, 2, 3, 4, 5, 8)  # P = 3 and 5 leave lanes of the <2,4> and <1,8> grad_reduce instantiations idle
GUARD = 64  # sentinel elements on either side of every output (a multiple of 16 bytes for every dtype used here)
SENT = {torch.float32: -1234.5, torch.bfloat16: 7.0, torch.int8: 90, torch.int32: 0, torch.int64: -5, torch.uint8: 0xA5}
EPOCH = 0x5EED
_INT = {torch.float32: torch.int32, torch.bfloat16: torch.int16, torch.int8: torch.int8, torch.int32: torch.int32,
        torch.int64: torch.int64, torch.uint8: torch.uint8}  # fmt: skip

# grid-stride pass lengths (elements) of the launchers: grid × threads × elements per thread and iteration
GR_GRID = 132 * 2


def _gr_pass(P: int) -> int:
    U = 4 if P <= 2 else 2 if P <= 4 else 1  # vectors per thread and iteration of the instantiation pb_grad_reduce picks
    return GR_GRID * 512 * 4 * U


ADAM_PASS = 264 * 512 * 8  # also cast_push
F32_PASS = 528 * 256 * 8  # outer_nesterov_f32
QBLK_PASS = 1056 * 4  # 1024-element blocks per pass of pseudograd_quant / outer_nesterov
AG_PASS = 528 * 512 * 16  # bytes per pass of allgather_copy


def _dev():
    return torch.device("cuda", 0)


# -------------------------------------------------------------------------------------------------- harness
def _launch(name, *args):
    from prime_b200.ops import functional as F

    F._launch(name, *args)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _pp(ts) -> _lib.PeerPtrs:
    """Local tensors standing in for the peers' buffers (rank order = list order)."""
    return _lib.PeerPtrs.of(t.data_ptr() for t in ts)


def _pref(pp):
    return ctypes.byref(pp)


class Out:
    """``n`` elements at ``t`` inside a buffer with GUARD sentinel elements on either side."""

    def __init__(self, n, dtype, init=None, device=None):
        self.dtype = dtype
        self.buf = torch.full((n + 2 * GUARD,), SENT[dtype], dtype=dtype, device=device or _dev())
        self.t = self.buf[GUARD : GUARD + n]
        if init is not None:
            self.t.copy_(init)

    def ptr(self):
        return self.t.data_ptr()

    def image(self, body):
        """The whole buffer as it must be: sentinels around ``body``."""
        want = torch.full_like(self.buf, SENT[self.dtype])
        want[GUARD : GUARD + self.t.numel()] = body
        return want

    def check_guards(self, what):
        for band in (self.buf[:GUARD], self.buf[GUARD + self.t.numel() :]):
            assert bitwise_equal(band, torch.full_like(band, SENT[self.dtype])), f"{what}: guard band overwritten"


def _err():
    return torch.zeros(2, dtype=torch.int32, device=_dev())


def _check_err(err, what):
    torch.cuda.synchronize()
    assert int(err.abs().sum()) == 0, f"{what}: error word {err.tolist()}"


def bitwise_equal(a, b) -> bool:
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.contiguous().view(_INT[a.dtype]), b.to(a.device).contiguous().view(_INT[b.dtype]))


def assert_bitwise(got, want, what):
    assert got.dtype == want.dtype and got.shape == want.shape, (what, got.dtype, want.dtype, got.shape, want.shape)
    a, b = got.contiguous().view(_INT[got.dtype]), want.to(got.device).contiguous().view(_INT[want.dtype])
    bad = a != b
    if bool(bad.any()):
        i = int(bad.reshape(-1).nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {got.numel()} elements differ bitwise; first at {i}: "
                             f"got {got.reshape(-1)[i].item()!r} want {want.reshape(-1)[i].item()!r}")  # fmt: skip
    print(f"[bitwise] {what}: identical ({got.numel()} elements)")


def _wide(n, lo, hi, seed, zeros=0.0):
    """fp32 values with random signs and magnitudes 2^U(lo, hi); a fraction ``zeros`` exact zeros (generated on the CPU)."""
    gen = torch.Generator().manual_seed(seed)
    e = torch.rand(n, generator=gen, dtype=torch.float64) * (hi - lo) + lo
    s = torch.where(torch.rand(n, generator=gen) < 0.5, -1.0, 1.0).double()
    x = (s * torch.exp2(e)).float()
    if zeros:
        x[torch.rand(n, generator=gen) < zeros] = 0.0
    return x


def _f32(x: float) -> float:
    return float(torch.tensor(x, dtype=torch.float32))


# -------------------------------------------------------------------------------------------------- reduce: emulation, data
def reduce_emulated(grads, off, n, scale, skip=None, twice=None):
    """fp32 ``acc = 0; acc = acc + g[p] (rank order); acc = acc * scale`` — the kernel's exact arithmetic (an add followed by a
    multiply cannot be contracted). ``skip`` / ``twice``: a peer left out / counted twice (mutants)."""
    acc = torch.zeros(n, dtype=torch.float32, device=grads[0].device)
    for p, g in enumerate(grads):
        for _ in range(0 if p == skip else 2 if p == twice else 1):
            acc = acc + g[off : off + n]
    return acc * torch.tensor(scale, dtype=torch.float32, device=acc.device)


def _reduce_case(P, size):
    shard = 4 if size == "vector" else _gr_pass(P) + 4
    start = 12  # 4-aligned bucket start
    grads = [_wide(start + P * shard + 8, -20, 4, seed=100 * P + p, zeros=0.05) for p in range(P)]
    return start, shard, grads, _f32(1.0 / P)


def _sumsq_bound(nvec_per_bucket, grid=GR_GRID):
    """Relative error of the fp32 sum of squares (positive terms): 4 serial terms per vector a thread owns in every bucket, the
    9-level block tree, one += per bucket, and a margin."""
    return (sum(4 * -(-nv // (grid * 512)) + 1 for nv in nvec_per_bucket) + 16) * U32


# -------------------------------------------------------------------------------------------------- AdamW: oracle, data
ADAM = dict(lr=1e-2, beta1=0.9, beta2=0.95, eps=1e-8, weight_decay=0.1)
NPARTS = GR_GRID  # sum-of-squares partials per rank, as the engine allocates them


def eps_clip(n_norm: int) -> float:
    """Relative error of the kernel's clip factor: fp32 sum of n_norm positive slots, sqrtf, + 1e-6, the division."""
    return (n_norm + 4) * U32


M_ATOL = 4 * U32  # m: g·clip, (1-β1)·gk, β1·m, the add — of Σ|terms|
V_ATOL = 6 * U32  # v: g·clip, gk·gk (doubles it), (1-β2)·gk², β2·v, the add — of v itself (all terms >= 0)
P_ATOL = 4 * U32  # p: fp32 decay = 1 - lr·wd, p·decay and the final subtraction — of |p|
# update: fp32 lr/bc1, m's error, sqrtf(v) with v's error halved, rsqrtf(bc2) (2 ulp = 4·2^-24), the product, + eps, step·m and the
# division — of step·Σ|m terms|/denom (m may cancel, so its term sum, not |m|, scales the update's error)
U_ATOL = 20 * U32


def adamw64(p, g, m, v, a, gn, n_clip_terms=1):
    """fp64 AdamW of the fp32 inputs with the fp32 hyper-parameters ``a`` the kernel read; ``gn`` = the global norm (None: no
    clip). Returns {p, m, v} and the scales of their per-element bounds."""
    p, g, m, v = (x.double() for x in (p, g, m, v))
    clip = 1.0 if gn is None or a.max_norm <= 0 else min(1.0, a.max_norm / (gn + 1e-6))
    gk = g * clip
    m_terms = (a.beta1 * m).abs() + ((1 - a.beta1) * gk).abs()
    m2 = a.beta1 * m + (1 - a.beta1) * gk
    v2 = a.beta2 * v + (1 - a.beta2) * gk * gk
    denom = v2.sqrt() / math.sqrt(a.bc2) + a.eps
    step = a.lr / a.bc1
    p2 = p * (1 - a.lr * a.weight_decay) - step * m2 / denom
    return dict(p=p2, m=m2, v=v2, m_terms=m_terms, u_terms=step * m_terms / denom, p_abs=p.abs(), clip=clip)


def check_adam(got, ref, ec, what, rejects=False):
    """The AdamW bounds; ``rejects``: return True if any of them fails instead of raising (mutation tests)."""
    checks = [
        (got["m"], ref["m"], M_ATOL + 2 * ec, ref["m_terms"], "m"),
        (got["v"], ref["v"], V_ATOL + 2 * ec, ref["v"], "v"),
        (got["p"], ref["p"], 1.0, P_ATOL * ref["p_abs"] + (U_ATOL + 2 * ec) * ref["u_terms"], "p"),
    ]
    if rejects:
        return any(_rejects(g, r, 0.0, atol, scale) for g, r, atol, scale, _ in checks)
    for g, r, atol, scale, name in checks:
        assert_elementwise(g, r, 0.0, atol, f"{what} {name}", scale=scale)
    return False


# (n, step, n_norm, clip regime, destinations)
ADAM_CASES = [
    (8, 1, 1, "clip<1", 1),
    (ADAM_PASS + 8, 1, 3, "clip<1", 2),
    (ADAM_PASS + 8, 1000, 8, "clip=1", 8),
    (ADAM_PASS + 8, 1000, 3, "clip<1", 8),
    (ADAM_PASS + 8, 1, 1, "max_norm=0", 1),
    (8 * 1000, 1000, 1, "no_slots", 2),
    (ADAM_PASS + 8, 1, 8, "clip=1", 1),
]


def _adam_id(c):
    return f"n{c[0]}-t{c[1]}-norm{c[2]}-{c[3]}-dst{c[4]}"


def adam_case(n, t, n_norm, regime):
    """(p, g, m, v, partials [n_norm, NPARTS], AdamArgs) on the CPU. Gradients span 2^-30..2^0 (eps dominates the denominator
    below ~2^-27) with 5 % exact zeros; half of |p| far above the update (lr = 1e-2), half far below; at t = 1000 m is random and
    v >= 0 comes from an earlier step."""
    seed = n + 7 * t + 31 * n_norm
    g = _wide(n, -30, 0, seed, zeros=0.05)
    big = torch.rand(n, generator=torch.Generator().manual_seed(seed + 1)) < 0.5
    p = torch.where(big, _wide(n, -1, 1, seed + 2), _wide(n, -24, -14, seed + 3))
    if t == 1:
        m, v = torch.zeros(n), torch.zeros(n)
    else:
        v = _wide(n, -30, 0, seed + 4).square()
        m = _wide(n, -1, 0, seed + 5) * v.sqrt()
    partials = torch.rand(n_norm, NPARTS, generator=torch.Generator().manual_seed(seed + 6)) * 0.01
    gn = math.sqrt(float(partials.double().sum()))
    max_norm = {"clip<1": 0.25 * gn, "clip=1": 10.0 * gn, "max_norm=0": 0.0, "no_slots": 0.25 * gn}[regime]
    bc1, bc2 = 1.0 - ADAM["beta1"] ** t, 1.0 - ADAM["beta2"] ** t
    a = _lib.AdamArgs(ADAM["lr"], ADAM["beta1"], ADAM["beta2"], ADAM["eps"], ADAM["weight_decay"], bc1, bc2, max_norm)
    return p, g, m, v, partials, a


def slots_emulated(partials):
    """What norm_publish leaves in the slots, to within its own bound (the CPU tests stand in for the kernel with this)."""
    return partials.double().sum(1).float()


# -------------------------------------------------------------------------------------------------- quantiser: emulation, data
def quant_emulated(d, trunc=False):
    """fp32 emulation of pseudograd_quant: IEEE am/127, 1/scale, rint(d·inv) (rint(d/scale) for a subnormal scale), clamp.
    ``trunc``: truncation instead of rint (mutant)."""
    db = d.view(-1, 1024)
    am = db.abs().amax(1)
    scale = torch.div(am, torch.full_like(am, 127.0))
    inv = torch.where(scale > 0, torch.ones_like(scale) / scale, torch.zeros_like(scale))
    sub = ((scale > 0) & (scale < 2.0**-126))[:, None]
    y = torch.where(sub, db / torch.where(sub, scale[:, None], torch.ones_like(scale[:, None])), db * inv[:, None])
    y = torch.trunc(y) if trunc else torch.round(y)
    return y.clamp(-127, 127).to(torch.int8).reshape(-1), scale


QUANT_BLOCKS = (1, 6, QBLK_PASS + 5)  # one block; not a multiple of 4 (idle groups in the last CTA); past one grid-stride pass


def quant_case(nblk):
    """(theta0, theta); the kernel quantises d = theta0 - theta. Block 0 has a subnormal scale (d[3] = 1e-37, d[5] = -2e-38,
    d[7] = 6e-39 — 7.6 steps, where rint and truncation differ — zeros elsewhere). With 6 or more blocks: an all-zero block,
    ties at ±1/2 step in every element, ±absmax at both ends, and scale 0 with non-zero data (absmax 2^-149). The rest are random
    blocks with magnitudes 2^-50..2^7 (theta = 0 in the edge blocks, so d is exactly the pattern)."""
    n = nblk * 1024
    theta = _wide(n, -8, 2, seed=nblk)
    d = _wide(n, -30, 4, seed=nblk + 1, zeros=0.02)
    d.view(nblk, 1024).mul_(torch.exp2(torch.randint(-20, 4, (nblk, 1), generator=torch.Generator().manual_seed(nblk))).float())
    theta0 = theta + d
    edges = [torch.zeros(1024) for _ in range(1 if nblk < 6 else 5)]
    edges[0][3], edges[0][5], edges[0][7] = 1e-37, -2e-38, 6e-39
    if nblk >= 6:
        s = 2.0**-10
        k = torch.randint(-126, 126, (1024,), generator=torch.Generator().manual_seed(5)).float()
        edges[2] = (k + 0.5) * s
        edges[2][0], edges[2][-1] = 127 * s, -127 * s  # absmax 127·s: scale = s exactly, every other d·inv = k + 1/2 exactly
        edges[3] = _wide(1024, -12, -2, seed=9)
        edges[3][0], edges[3][-1] = 0.75, -0.75  # ±absmax at both ends
        edges[4][17] = 2.0**-149  # scale = 2^-149/127 rounds to 0: the block is sent as zeros
    for i, blk in enumerate(edges):
        theta[i * 1024 : (i + 1) * 1024] = 0.0
        theta0[i * 1024 : (i + 1) * 1024] = blk
    return theta0, theta


def check_quant_invariant(q, scales, d, what):
    """fp64: |q - d/scale| <= 1/2 + 2^-15 wherever scale > 0 (1/scale and d·inv are each within 2^-24 relative, so d·inv is within
    127.5·2^-23 < 2^-15 of d/scale; the clamp at ±127 costs 127·2^-24); where scale = 0 every q is 0 and |d| <= 2^-142."""
    s = scales.double().repeat_interleave(1024)
    pos = s > 0
    assert_elementwise(q.double()[pos], d.double()[pos] / s[pos], 0.0, 0.5 + 2.0**-15, what, scale=1.0)
    flushed = d.double()[~pos]
    assert bool((q[~pos] == 0).all()) and (flushed.numel() == 0 or float(flushed.abs().max()) <= 2.0**-142)


# -------------------------------------------------------------------------------------------------- outer step: oracle, tables
OUTER = dict(lr=0.7, momentum=0.9)


def nesterov64(t0, m, gsum, gmag, a):
    """fp64 outer step on the average gsum·inv_workers. Returns (theta0', mom', scale of theta0's bound, scale of mom's bound):
    mom's error is that of the W-term fp32 dequant-sum (W roundings of Σ|terms|), ·inv_workers, and the FMA μ·m + g, of
    μ|m| + G; theta0's adds the FMAs g + μ·m' and t0 - lr·upd, of |t0| + lr·(G + μ·(μ|m| + G))."""
    t0, m = t0.double(), m.double()
    g, G = gsum * a.inv_workers, gmag * a.inv_workers
    mk = a.momentum * m + g
    upd = g + a.momentum * mk if a.nesterov else mk
    m_scale = a.momentum * m.abs() + G
    u_scale = G + a.momentum * m_scale if a.nesterov else m_scale
    return t0 - a.lr * upd, mk, t0.abs() + a.lr * u_scale, m_scale


def bucket_table(n, nb, seed, align=1024):
    """shard_start [nb + 1] (interior boundaries multiples of 1024, shard_start[nb] = n) and dst_start [nb]: the destination ranges
    in REVERSED bucket order with sentinel gaps (multiples of 8 elements) between them; and the destination buffer's length."""
    gen = torch.Generator().manual_seed(seed)
    cuts = sorted(torch.randperm((n - 1) // align, generator=gen)[: nb - 1].add(1).mul(align).tolist())
    starts = [0, *cuts, n]
    dst, pos = [0] * nb, 24
    for b in reversed(range(nb)):
        dst[b] = pos
        pos += starts[b + 1] - starts[b] + 8 * (1 + b % 5)
    return starts, dst, pos + 16


def writeback_image(theta0, starts, dst, total, device, shift=0):
    """The bf16 destination buffer as the write-back must leave it. ``shift``: table lookup one bucket off (mutant)."""
    img = torch.full((total,), SENT[torch.bfloat16], dtype=torch.bfloat16, device=device)
    st, ds = torch.tensor(starts, device=device), torch.tensor(dst, device=device)
    i = torch.arange(starts[-1], device=device)
    b = (torch.bucketize(i, st[1:-1], right=True) + shift).clamp(0, len(dst) - 1)  # last bucket whose start <= i (+ shift)
    pos = ds[b] + (i - st[b])
    ok = (pos >= 0) & (pos < total)
    img[pos[ok]] = theta0.to(device)[ok].to(torch.bfloat16)
    return img


# (workers, buckets, 1024-blocks, destinations, nesterov)
INT8_CASES = [(1, 1, 1, 1, 1), (2, 2, 6, 2, 1), (3, 5, QBLK_PASS + 1, 8, 1), (8, 37, QBLK_PASS + 1, 2, 1), (8, 5, 6, 8, 0),
              (3, 37, 40, 1, 1)]  # fmt: skip
# (workers, buckets, n, destinations, nesterov)
F32_CASES = [(1, 1, 8, 1, 1), (2, 2, 40 * 1024 + 8, 2, 1), (3, 5, F32_PASS + 8, 8, 1), (8, 37, F32_PASS + 8, 2, 1),
             (8, 5, 40 * 1024 + 8, 8, 0)]  # fmt: skip


def int8_case(W, nblk, seed):
    """Per-worker int8 payloads (random, 3 % zeros) and positive scales 2^U(-16, -10); theta0 ~ 2^U(-8, 1), momentum ~ 2^U(-14, -6)."""
    n = nblk * 1024
    gen = torch.Generator().manual_seed(seed)
    qs = [torch.randint(-127, 128, (n,), generator=gen, dtype=torch.int8) for _ in range(W)]
    for q in qs:
        q[torch.rand(n, generator=gen) < 0.03] = 0
    ss = [_wide(nblk, -16, -10, seed + 1 + w).abs() for w in range(W)]
    return qs, ss, _wide(n, -8, 1, seed + 20), _wide(n, -14, -6, seed + 21)


def int8_sum64(qs, ss):
    gsum = sum(q.double() * s.double().repeat_interleave(1024).to(q.device) for q, s in zip(qs, ss))
    gmag = sum((q.double() * s.double().repeat_interleave(1024).to(q.device)).abs() for q, s in zip(qs, ss))
    return gsum, gmag


# ================================================================================================== CPU: launcher contracts
def test_launchers_refuse_impossible_arguments_before_touching_the_device():
    try:
        lib = _lib.load()
    except Exception as e:  # noqa: BLE001
        pytest.skip(f"native library not loadable here: {e}")
    a = 1 << 20  # 16-byte aligned, never dereferenced: every call below is rejected first
    pp = _lib.PeerPtrs.of([a])
    none, nine = _lib.PeerPtrs(), _lib.PeerPtrs()
    nine.n = 9
    for i in range(8):
        nine.p[i] = a

    many = _lib.SegTable()
    many.nseg = 17  # the table holds 16
    for mc in (None, a):  # peer loads and the multicast instantiation check the same arguments
        def reduce(table):
            return lib.pb_grad_reduce(ctypes.byref(pp), mc, ctypes.byref(table), 1.0, a, a, None, 0, 0, a, 0, None)

        assert reduce(many) == -1
        for bad in ((2, 0, 8), (0, 6, 8), (0, 0, 6), (0, 0, 1022)):
            assert reduce(_lib.SegTable.of([(0, 0, 8), bad])) == -1  # every segment 4-aligned: float4 vectors

    args = _lib.AdamArgs(1e-3, 0.9, 0.95, 1e-8, 0.1, 0.1, 0.05, 1.0)

    def adamw(n=1024, dst_off=0):
        return lib.pb_adamw_push(a, a, a, a, n, ctypes.byref(args), None, 1, None, 0, 0, ctypes.byref(pp), dst_off, None, a, None, None)

    assert adamw(n=1020) == -1 and adamw(dst_off=4) == -1  # 16-byte bf16 stores
    assert lib.pb_cast_push(a, 1020, ctypes.byref(pp), 0, None) == -1 and lib.pb_cast_push(a, 1024, ctypes.byref(pp), 4, None) == -1

    def emb(w=pp, dim=64, rpr=16):
        return lib.pb_embedding_fwd(a, 4, ctypes.byref(w), rpr, dim, a, None)

    assert emb(w=none) == -1 and emb(w=nine) == -1 and emb(dim=60) == -1 and emb(rpr=0) == -1

    def gather(src=pp, nbytes=1024):
        return lib.pb_allgather_copy(ctypes.byref(src), nbytes, a, None)

    assert gather(src=none) == -1 and gather(src=nine) == -1 and gather(nbytes=1000) == -1


# ================================================================================================== CPU: the rules reject bugs
@pytest.mark.parametrize("case", [ADAM_CASES[1], ADAM_CASES[3]], ids=_adam_id)
def test_adam_bounds_reject_mutants(case):
    n, t, n_norm, regime, _ = case
    p, g, m, v, partials, a = adam_case(n, t, n_norm, regime)
    gn = math.sqrt(float(slots_emulated(partials).double().sum()))
    ec = eps_clip(n_norm)
    ref = adamw64(p, g, m, v, a, gn)
    assert ref["clip"] < 1.0
    as32 = {k: ref[k].float() for k in ("p", "m", "v")}
    assert not check_adam(as32, ref, ec, "", rejects=True)  # the exact result rounded to fp32 passes

    def mutant(**kw):
        p64, g64, m64, v64 = (x.double() for x in (p, g, m, v))
        clip = 1.0 if kw.get("stale_norm") else min(1.0, a.max_norm / (gn + 1e-6))
        gk = g64 * clip
        m2 = a.beta1 * m64 + (1 - a.beta1) * (g64 if kw.get("m_unclipped") else gk)
        v2 = a.beta2 * v64 + (1 - a.beta2) * gk * gk
        if kw.get("eps_inside"):
            denom = (v2 / a.bc2 + a.eps).sqrt()
        elif kw.get("bc2_outside"):
            denom = v2.sqrt() / a.bc2 + a.eps
        else:
            denom = v2.sqrt() / math.sqrt(a.bc2) + a.eps
        upd = a.lr / a.bc1 * m2 / denom
        decay = 1 - a.lr * a.weight_decay
        p2 = (p64 - upd) * decay if kw.get("decay_after") else p64 * decay - upd
        return {"p": p2.float(), "m": m2.float(), "v": v2.float()}

    for bug in ("decay_after", "eps_inside", "m_unclipped", "stale_norm") + (("bc2_outside",) if t == 1 else ()):
        assert check_adam(mutant(**{bug: True}), ref, ec, bug, rejects=True), f"the AdamW bounds accept the mutant {bug}"


@pytest.mark.parametrize("P", [2, 5, 8])
def test_reduce_rule_rejects_a_skipped_or_doubled_peer(P):
    start, shard, grads, scale = _reduce_case(P, "pass1")
    want = reduce_emulated(grads, start, shard, scale)
    assert bitwise_equal(reduce_emulated(grads, start, shard, scale), want)
    for kw in ({"skip": P - 1}, {"twice": 0}):
        assert not bitwise_equal(reduce_emulated(grads, start, shard, scale, **kw), want), kw


@pytest.mark.parametrize("nblk", QUANT_BLOCKS)
def test_quant_rules_reject_truncation_and_match_the_reference(nblk):
    theta0, theta = quant_case(nblk)
    d = theta0 - theta
    q, s = quant_emulated(d)
    rq, rs = Rf.quantize_int8_blockwise(d, 1024)
    assert bitwise_equal(q, rq) and bitwise_equal(s, rs)  # the emulation IS the reference's arithmetic
    check_quant_invariant(q, s, d, f"emulation nblk={nblk}")
    qt, _ = quant_emulated(d, trunc=True)
    assert not bitwise_equal(qt, q)
    pos = s.repeat_interleave(1024) > 0
    assert _rejects(qt.double()[pos], d.double()[pos] / s.double().repeat_interleave(1024)[pos], 0.0, 0.5 + 2.0**-15, 1.0)


def test_subnormal_scale_block_quantises_like_its_values():
    """absmax < 127·2^-128: 1/scale overflows to inf, and 0·inf = NaN must not become ±127."""
    d = torch.zeros(1024)
    d[3], d[5] = 1e-37, -2e-38
    q, s = Rf.quantize_int8_blockwise(d, 1024)
    assert 0 < float(s[0]) < 2.0**-126
    assert q[3] == 127 and int(q[5]) == round(-2e-38 / float(s[0])) and int((q != 0).sum()) == 2
    check_quant_invariant(q, s, d, "subnormal-scale block (reference)")


@pytest.mark.parametrize("case", [INT8_CASES[2], INT8_CASES[3]], ids=lambda c: f"W{c[0]}-nb{c[1]}-blk{c[2]}")
def test_outer_rules_reject_wrong_sign_and_table_off_by_one(case):
    W, nb, nblk, _, nesterov = case
    qs, ss, t0, mom = int8_case(W, nblk, seed=W * 100 + nb)
    a = _lib.OuterArgs(OUTER["lr"], OUTER["momentum"], 1.0 / W, nesterov)
    gsum, gmag = int8_sum64(qs, ss)
    t1, m1, ts, ms = nesterov64(t0, mom, gsum, gmag, a)
    assert not _rejects(t1.float(), t1, 0.0, (W + 5) * U32, ts)
    t1_bad, _, _, _ = nesterov64(t0, mom, -gsum, gmag, a)  # pseudo-gradient theta - theta0
    assert _rejects(t1_bad.float(), t1, 0.0, (W + 5) * U32, ts)
    starts, dst, total = bucket_table(nblk * 1024, nb, seed=nb)
    img = writeback_image(t1.float(), starts, dst, total, "cpu")
    for shift in (-1, 1):
        assert not bitwise_equal(writeback_image(t1.float(), starts, dst, total, "cpu", shift), img)


# ================================================================================================== GPU: reduce-scatter
@pytest.mark.gpu
@pytest.mark.parametrize("size", ["vector", "pass1"])
@pytest.mark.parametrize("P", PEERS)
def test_grad_reduce_one_segment(P, size):
    dev = _dev()
    start, shard, grads, scale = _reduce_case(P, size)
    grads = [g.to(dev) for g in grads]
    snap = [g.clone() for g in grads]
    err = _err()
    slot_base = 3
    flags = [Out(16, torch.int32) for _ in range(P)]
    for r in range(P):  # every rank signals its slot in every rank's flags (pb_signal, in stream order before the waits)
        _launch("pb_signal", _pref(_pp([f.t for f in flags])), slot_base + r, EPOCH, _stream())
    want_flags = torch.zeros(16, dtype=torch.int32, device=dev)
    want_flags[slot_base : slot_base + P] = EPOCH
    gp = _pp(grads)
    nvec = shard // 4

    def run(off, out, part, max_ctas, wait=None):
        table = _lib.SegTable.of([(off, 0, shard)])
        _launch("pb_grad_reduce", _pref(gp), None, ctypes.byref(table), scale, out.ptr(), part.ptr(), wait, slot_base, EPOCH,
                err.data_ptr(), max_ctas, _stream())  # fmt: skip
        _check_err(err, f"grad_reduce P={P}")

    for r in range(P):
        off = start + r * shard
        want = reduce_emulated(grads, off, shard, scale)
        out, part = Out(shard, torch.float32), Out(GR_GRID, torch.float32, torch.zeros(GR_GRID))
        run(off, out, part, 0, wait=flags[r].t.data_ptr())
        assert_bitwise(out.buf, out.image(want), f"grad_reduce P={P} rank {r} out")
        # sum of squares: += over a second bucket (the next rank's shard) into the same partials
        off_b = start + (r + 1) % P * shard
        out_b = Out(shard, torch.float32)
        run(off_b, out_b, part, 0)
        assert_bitwise(out_b.buf, out_b.image(reduce_emulated(grads, off_b, shard, scale)), f"grad_reduce P={P} bucket 2")
        part.check_guards("sumsq_partial")
        ss64 = out.t.double().square().sum() + out_b.t.double().square().sum()
        assert_elementwise(part.t.double().sum(), ss64, _sumsq_bound([nvec, nvec]), 0.0, f"grad_reduce P={P} sumsq over 2 buckets")
        # the same result from a 7-CTA grid, and on a repeated run: replicas stay bitwise identical
        out7, part7 = Out(shard, torch.float32), Out(GR_GRID, torch.float32, torch.zeros(GR_GRID))
        run(off, out7, part7, 7)
        assert_bitwise(out7.buf, out.buf, f"grad_reduce P={P} max_ctas=7")
        assert bool((part7.t[7:] == 0).all()), "a 7-CTA grid wrote partials past slot 6"
        assert_elementwise(part7.t.double().sum(), out.t.double().square().sum(), _sumsq_bound([nvec], grid=7), 0.0,
                           f"grad_reduce P={P} max_ctas=7 sumsq")  # fmt: skip
        again = Out(shard, torch.float32)
        run(off, again, Out(GR_GRID, torch.float32, torch.zeros(GR_GRID)), 0)
        assert_bitwise(again.buf, out.buf, f"grad_reduce P={P} repeated")
    for r, f in enumerate(flags):
        assert_bitwise(f.buf, f.image(want_flags), f"flags of rank {r}")
    for g, s in zip(grads, snap):
        assert bitwise_equal(g, s), "grad_reduce wrote its input"


def _segments(nseg, seed, P):
    """(src_off, dst_off, n) with irregular 4-aligned offsets, gaps between destinations; one segment one vector past a whole
    grid-stride pass of the instantiation that P peers select."""
    gen = torch.Generator().manual_seed(seed)
    lens = [_gr_pass(P) + 4] if nseg == 1 else [4 * int(x) for x in torch.randint(1, 3000, (nseg,), generator=gen)]
    if nseg > 1:
        lens[5] = _gr_pass(P) + 4
        lens[0], lens[9] = 4, 8
    segs, src, dst = [], 8, 4
    for n in lens:
        src += 4 * int(torch.randint(0, 50, (1,), generator=gen))
        dst += 4 * int(torch.randint(1, 10, (1,), generator=gen))
        segs.append((src, dst, n))
        src, dst = src + n, dst + n
    return segs, src + 12, dst + 12


def _segs_body(grads, segs, scale, dst_len):
    body = torch.full((dst_len,), SENT[torch.float32], device=grads[0].device)
    for s, d, n in segs:
        body[d : d + n] = reduce_emulated(grads, s, n, scale)
    return body


@pytest.mark.gpu
@pytest.mark.parametrize("nseg", [0, 1, 16])
@pytest.mark.parametrize("P", PEERS)
def test_grad_reduce_segments(P, nseg):
    dev = _dev()
    segs, src_len, dst_len = _segments(max(nseg, 1), seed=P * 17 + nseg, P=P)
    segs = segs[:nseg]
    grads = [_wide(src_len, -20, 4, seed=300 + 10 * P + p, zeros=0.05).to(dev) for p in range(P)]
    scale = _f32(1.0 / P)
    err = _err()
    out = Out(dst_len, torch.float32)
    part = Out(GR_GRID, torch.float32, torch.rand(GR_GRID))  # accumulates onto what earlier buckets left
    part0 = part.t.clone()
    table = _lib.SegTable.of(segs)
    _launch("pb_grad_reduce", _pref(_pp(grads)), None, ctypes.byref(table), scale, out.ptr(), part.ptr(), None, 0, 0, err.data_ptr(), 0,
            _stream())  # fmt: skip
    _check_err(err, f"grad_reduce P={P} nseg={nseg}")
    assert_bitwise(out.buf, out.image(_segs_body(grads, segs, scale, dst_len)), f"grad_reduce P={P} nseg={nseg} (gaps untouched)")
    part.check_guards("sumsq_partial")
    if nseg == 0:
        assert_bitwise(part.t, part0, "grad_reduce nseg=0 partials")
        return
    ss64 = sum(out.t[d : d + n].double().square().sum() for _, d, n in segs)
    # a thread's serial terms run through every segment; the partials it adds onto are >= 0 and part of the sum
    bound = (sum(4 * -(-n // 4 // (GR_GRID * 512)) for _, _, n in segs) + 16) * U32
    assert_elementwise(part.t.double().sum(), ss64 + part0.double().sum(), bound, 0.0, f"grad_reduce P={P} nseg={nseg} sumsq")


@pytest.mark.gpu
@pytest.mark.parametrize("P", PEERS)
def test_grad_reduce_abort(P):
    """With the host watchdog's abort value in the error word and the peers' flags not yet at the epoch, the flag wait gives up and
    the kernel returns before it reads or writes anything; once the flags are signalled and the word is cleared, the same call
    reduces."""
    dev = _dev()
    segs, src_len, dst_len = _segments(16, seed=P * 29, P=P)
    grads = [_wide(src_len, -20, 4, seed=700 + 10 * P + p, zeros=0.05).to(dev) for p in range(P)]
    scale = _f32(1.0 / P)
    slot_base = 2
    flags = Out(16, torch.int32)  # 0: below EPOCH
    out = Out(dst_len, torch.float32)
    part = Out(GR_GRID, torch.float32, torch.rand(GR_GRID))
    table = _lib.SegTable.of(segs)
    err = _err()

    def run():
        _launch("pb_grad_reduce", _pref(_pp(grads)), None, ctypes.byref(table), scale, out.ptr(), part.ptr(), flags.ptr(), slot_base,
                EPOCH, err.data_ptr(), 0, _stream())  # fmt: skip

    everything = [out.buf, part.buf, flags.buf, *grads]
    snap = [x.clone() for x in everything]
    err[0] = 2  # the host watchdog's abort value (a software flag), as SymmetricHeap.abort() writes it
    run()
    torch.cuda.synchronize()
    assert err.tolist() == [2, 0], f"grad_reduce P={P}: error word {err.tolist()}"
    for x, s in zip(everything, snap):
        assert bitwise_equal(x, s), f"grad_reduce P={P} wrote with the abort flag set"
    print(f"[bitwise] grad_reduce P={P} with err = 2: every buffer untouched")
    err.zero_()
    for r in range(P):
        _launch("pb_signal", _pref(_pp([flags.t])), slot_base + r, EPOCH, _stream())
    run()
    _check_err(err, f"grad_reduce P={P} after the abort")
    assert_bitwise(out.buf, out.image(_segs_body(grads, segs, scale, dst_len)), f"grad_reduce P={P} after the abort")
    for g, s in zip(grads, snap[3:]):
        assert bitwise_equal(g, s), "grad_reduce wrote its input"


# ================================================================================================== GPU: norm, AdamW
@pytest.mark.gpu
@pytest.mark.parametrize("nparts", [1, 37, NPARTS])
@pytest.mark.parametrize("P", PEERS)
def test_norm_publish(P, nparts):
    dev = _dev()
    my, flag_slot = P // 2, 5
    vals = _wide(nparts, -20, 6, seed=nparts).abs()
    part = Out(nparts, torch.float32, vals)
    slots = [Out(8, torch.float32) for _ in range(P)]
    flags = [Out(16, torch.int32) for _ in range(P)]
    _launch("pb_norm_publish", part.ptr(), nparts, _pref(_pp([s.t for s in slots])), _pref(_pp([f.t for f in flags])), my, flag_slot,
            EPOCH, _stream())  # fmt: skip
    torch.cuda.synchronize()
    assert_bitwise(part.buf, part.image(torch.zeros(nparts, device=dev)), f"norm_publish P={P} partials zeroed")
    # pairwise fp32 tree over positive terms: at most ceil(log2 nparts) non-trivial adds on any path, + margin
    bound = (math.ceil(math.log2(nparts)) + 2) * U32
    got = slots[0].t[my].clone()
    assert_elementwise(got.double(), vals.double().sum(), bound, 0.0, f"norm_publish P={P} nparts={nparts} slot")
    want_flags = torch.zeros(16, dtype=torch.int32, device=dev)
    want_flags[flag_slot + my] = EPOCH
    for p in range(P):
        body = torch.full((8,), SENT[torch.float32], device=dev)
        body[my] = got
        assert_bitwise(slots[p].buf, slots[p].image(body), f"norm slots of peer {p}")
        assert_bitwise(flags[p].buf, flags[p].image(want_flags), f"flags of peer {p}")


@pytest.mark.gpu
@pytest.mark.parametrize("case", ADAM_CASES, ids=_adam_id)
def test_adamw_push(case):
    n, t, n_norm, regime, ndst = case
    dev = _dev()
    p, g, m, v, partials, a = adam_case(n, t, n_norm, regime)
    P32, M, V = (Out(n, torch.float32, x) for x in (p, m, v))
    G = Out(n, torch.float32, g)
    dst_off = 24
    dsts = [Out(dst_off + n + 24, torch.bfloat16) for _ in range(ndst)]
    gnorm = Out(1, torch.float32)
    err = _err()
    slots, flags, flag_slot = Out(8, torch.float32), Out(16, torch.int32), 2
    with_slots = regime != "no_slots"
    if with_slots:  # every rank's norm_publish lands in this rank's slots and flags before adamw_push waits on them
        for i in range(n_norm):
            part = Out(NPARTS, torch.float32, partials[i])
            _launch("pb_norm_publish", part.ptr(), NPARTS, _pref(_pp([slots.t])), _pref(_pp([flags.t])), i, flag_slot, EPOCH, _stream())
    _launch("pb_adamw_push", P32.ptr(), G.ptr(), M.ptr(), V.ptr(), n, ctypes.byref(a), slots.ptr() if with_slots else None, n_norm,
            flags.ptr() if with_slots else None, flag_slot, EPOCH, _pref(_pp([d.t for d in dsts])), dst_off, gnorm.ptr(), err.data_ptr(),
            None, _stream())  # fmt: skip
    _check_err(err, "adamw_push")
    what = f"adamw_push {_adam_id(case)}"
    for o, name in ((P32, "p32"), (M, "m"), (V, "v")):
        o.check_guards(f"{what} {name}")
    assert_bitwise(G.buf, G.image(g.to(dev)), f"{what} gradient untouched")
    gn = None
    if with_slots:
        sl = slots.t[:n_norm].double()
        gn = math.sqrt(float(sl.sum()))
        # fp32 serial sum of n_norm positive slots, then sqrtf: (n_norm - 1)/2 + 1 units of 2^-24 (2^-22 up to n_norm = 7)
        assert_elementwise(gnorm.t.double(), torch.tensor([gn]), (n_norm / 2 + 1) * U32, 0.0, f"{what} gnorm_out")
        assert_elementwise(sl.sum(), partials.double().sum(), (math.ceil(math.log2(NPARTS)) + 2) * U32, 0.0, f"{what} slots")
    else:
        assert_bitwise(gnorm.buf, gnorm.image(torch.full((1,), SENT[torch.float32])), f"{what} gnorm_out untouched")
    ref = adamw64(p.to(dev), g.to(dev), m.to(dev), v.to(dev), a, gn)
    assert (ref["clip"] < 1.0) == (regime == "clip<1")
    check_adam({"p": P32.t, "m": M.t, "v": V.t}, ref, eps_clip(n_norm), what)
    for q, d in enumerate(dsts):
        body = torch.full((dst_off + n + 24,), SENT[torch.bfloat16], dtype=torch.bfloat16, device=dev)
        body[dst_off : dst_off + n] = P32.t.to(torch.bfloat16)
        assert_bitwise(d.buf, d.image(body), f"{what} bf16 destination {q}")


@pytest.mark.gpu
def test_engine_step_matches_fp64_adamw():
    """Two fused-engine steps at F = 1 (the first clipped, the second not) against the fp64 AdamW of the gradient the engine
    reduced, with the engine's own step count, lr and bias corrections."""
    from prime_b200.models.llama import build_model
    from prime_b200.parallel.fsdp import AdamHyper, ShardedEngine
    from prime_b200.parallel.mesh import WorldInfo, build_mesh
    from prime_b200.parallel.symm import SymmetricHeap

    dev = _dev()
    torch.manual_seed(0)
    model = build_model("debugmodel", device=dev, dtype=torch.bfloat16, seed=3)
    mesh = build_mesh(WorldInfo(), device=dev)
    heap = SymmetricHeap(256 << 20, 0, 1, lambda h: [h], dev)
    e = ShardedEngine(model, mesh, AdamHyper(lr=1e-2), backend="fused", heap=heap)
    V = model.args.vocab_size
    try:
        for step in range(2):
            tok = torch.randint(0, V, (2, 64), device=dev)
            e.zero_grad()
            e.set_micro_step(True)
            model.loss(tok, tok).backward()
            e.finish_backward()
            torch.cuda.synchronize()
            g = e.grad_flat.clone()
            before = {k: getattr(e, k).clone() for k in ("master", "exp_avg", "exp_avg_sq")}
            sumsq = sum(g[b.start : b.start + b.shard_size].double().square().sum() for b in e.buckets)
            gn64 = math.sqrt(float(sumsq))
            e.hyper.max_norm = 0.5 * gn64 if step == 0 else 100.0 * gn64
            e.step()
            torch.cuda.synchronize()
            heap.check_errors()
            h, t = e.hyper, e.step_count
            a = _lib.AdamArgs(h.lr, h.beta1, h.beta2, h.eps, h.weight_decay, 1.0 - h.beta1**t, 1.0 - h.beta2**t, h.max_norm)
            # relative error of the engine's norm: the per-bucket sums of squares, one += per bucket, norm_publish's tree, sqrtf
            rel_ss = _sumsq_bound([b.shard_size // 4 for b in e.buckets]) + 12 * U32
            assert_elementwise(e.last_grad_norm.double(), torch.tensor([gn64]), rel_ss / 2 + U32, 0.0, f"engine step {t} grad norm")
            ec = rel_ss / 2 + 3 * U32
            for b in e.buckets:
                sl = slice(b.shard_start, b.shard_start + b.shard_size)
                ref = adamw64(before["master"][sl], g[b.start : b.start + b.shard_size], before["exp_avg"][sl], before["exp_avg_sq"][sl], a,
                              gn64)  # fmt: skip
                assert (ref["clip"] < 1.0) == (step == 0)
                check_adam({"p": e.master[sl], "m": e.exp_avg[sl], "v": e.exp_avg_sq[sl]}, ref, ec, f"engine step {t} {b.name}")
                assert_bitwise(e.param_flat[b.pstart : b.pstart + b.shard_size], e.master[sl].to(torch.bfloat16), f"engine step {t} {b.name} bf16")
    finally:
        heap.close()


# ================================================================================================== GPU: DiLoCo outer step
@pytest.mark.gpu
@pytest.mark.parametrize("nblk", QUANT_BLOCKS)
def test_pseudograd_quant(nblk):
    dev = _dev()
    theta0, theta = (x.to(dev) for x in quant_case(nblk))
    n = nblk * 1024
    q, sc = Out(n, torch.int8), Out(nblk, torch.float32)
    _launch("pb_pseudograd_quant", theta0.data_ptr(), theta.data_ptr(), q.ptr(), sc.ptr(), n, _stream())
    torch.cuda.synchronize()
    d = theta0 - theta
    wq, ws = quant_emulated(d)
    assert_bitwise(sc.buf, sc.image(ws), f"pseudograd_quant nblk={nblk} scales")
    assert_bitwise(q.buf, q.image(wq), f"pseudograd_quant nblk={nblk} q")
    rq, rs = Rf.quantize_int8_blockwise(d, 1024)
    assert bitwise_equal(q.t, rq) and bitwise_equal(sc.t, rs), "kernel and reference.quantize_int8_blockwise disagree"
    assert 0 < float(sc.t[0]) < 2.0**-126  # block 0: subnormal scale
    check_quant_invariant(q.t, sc.t, d, f"pseudograd_quant nblk={nblk} |q - d/scale|")


def _outer_check(what, k, a, t0_in, mom_in, gsum, gmag, theta0, mom, theta_out, dsts, starts, dst, total):
    t1, m1, ts, ms = nesterov64(t0_in, mom_in, gsum, gmag, a)
    assert_elementwise(mom.t, m1, 0.0, (k + 2) * U32, f"{what} momentum", scale=ms)
    assert_elementwise(theta0.t, t1, 0.0, (k + 5) * U32, f"{what} theta0", scale=ts)
    assert_bitwise(theta_out.buf, theta_out.image(theta0.t), f"{what} theta = theta0")
    img = writeback_image(theta0.t, starts, dst, total, theta0.t.device)
    for q, d in enumerate(dsts):
        assert_bitwise(d.buf, d.image(img), f"{what} bf16 destination {q}")
    theta0.check_guards(what)
    mom.check_guards(what)


@pytest.mark.gpu
@pytest.mark.parametrize("case", INT8_CASES, ids=lambda c: f"W{c[0]}-nb{c[1]}-blk{c[2]}-dst{c[3]}-nest{c[4]}")
def test_outer_nesterov_int8(case):
    W, nb, nblk, ndst, nesterov = case
    dev = _dev()
    n = nblk * 1024
    qs, ss, t0, mom0 = int8_case(W, nblk, seed=W * 100 + nb)
    qs, ss = [q.to(dev) for q in qs], [s.to(dev) for s in ss]
    # worker 0's payload comes from the quantiser itself
    a0, b0 = _wide(n, -6, 0, seed=77).to(dev), _wide(n, -6, 0, seed=78).to(dev)
    _launch("pb_pseudograd_quant", a0.data_ptr(), b0.data_ptr(), qs[0].data_ptr(), ss[0].data_ptr(), n, _stream())
    starts, dst, total = bucket_table(n, nb, seed=nb)
    sh, ds = torch.tensor(starts, dtype=torch.int64, device=dev), torch.tensor(dst, dtype=torch.int64, device=dev)
    a = _lib.OuterArgs(OUTER["lr"], OUTER["momentum"], 1.0 / W, nesterov)
    theta0, mom = Out(n, torch.float32, t0), Out(n, torch.float32, mom0)
    theta_out = Out(n, torch.float32, torch.full((n,), 3.0))
    dsts = [Out(total, torch.bfloat16) for _ in range(ndst)]
    err = _err()

    def run():
        _launch("pb_outer_nesterov", _pref(_pp(qs)), _pref(_pp(ss)), theta0.ptr(), mom.ptr(), theta_out.ptr(), n, ctypes.byref(a),
                _pref(_pp([d.t for d in dsts])), sh.data_ptr(), ds.data_ptr(), nb, err.data_ptr(), _stream())  # fmt: skip

    everything = [theta0.buf, mom.buf, theta_out.buf, *[d.buf for d in dsts], *qs, *ss, sh, ds]
    snap = [x.clone() for x in everything]
    err[0] = 2  # the host watchdog's abort value (a software flag): the kernel must not read or write anything
    run()
    torch.cuda.synchronize()
    for x, s in zip(everything, snap):
        assert bitwise_equal(x, s), "outer_nesterov wrote with the abort flag set"
    print("[bitwise] outer_nesterov with err = 2: every buffer untouched")
    err.zero_()
    run()
    _check_err(err, "outer_nesterov")
    what = f"outer_nesterov W={W} nb={nb} nblk={nblk} dst={ndst}"
    for x, s in zip([*qs, *ss], snap[3 + ndst :]):
        assert bitwise_equal(x, s), f"{what}: an input payload or scale changed"
    gsum, gmag = int8_sum64(qs, ss)
    _outer_check(what, W, a, t0.to(dev), mom0.to(dev), gsum, gmag, theta0, mom, theta_out, dsts, starts, dst, total)


@pytest.mark.gpu
@pytest.mark.parametrize("case", F32_CASES, ids=lambda c: f"W{c[0]}-nb{c[1]}-n{c[2]}-dst{c[3]}-nest{c[4]}")
def test_outer_nesterov_f32(case):
    W, nb, n, ndst, nesterov = case
    dev = _dev()
    t0 = _wide(n, -8, 1, seed=n + W)
    mom0 = _wide(n, -14, -6, seed=n + W + 1)
    # the workers' inner masters: theta0 moved by a few inner steps (and one worker by nothing at all)
    thetas = [(t0 + _wide(n, -16, -6, seed=500 + w, zeros=0.1 if w else 1.0)).to(dev) for w in range(W)]
    snap_thetas = [x.clone() for x in thetas]
    starts, dst, total = bucket_table(n, nb, seed=nb + 1)
    sh, ds = torch.tensor(starts, dtype=torch.int64, device=dev), torch.tensor(dst, dtype=torch.int64, device=dev)
    a = _lib.OuterArgs(OUTER["lr"], OUTER["momentum"], 1.0 / W, nesterov)
    theta0, mom = Out(n, torch.float32, t0), Out(n, torch.float32, mom0)
    theta_new = Out(n, torch.float32, torch.full((n,), 3.0))
    dsts = [Out(total, torch.bfloat16) for _ in range(ndst)]
    err = _err()

    def run():
        _launch("pb_outer_nesterov_f32", _pref(_pp(thetas)), theta0.ptr(), mom.ptr(), theta_new.ptr(), n, ctypes.byref(a),
                _pref(_pp([d.t for d in dsts])), sh.data_ptr(), ds.data_ptr(), nb, err.data_ptr(), _stream())  # fmt: skip

    everything = [theta0.buf, mom.buf, theta_new.buf, *[d.buf for d in dsts], *thetas]
    snap = [x.clone() for x in everything]
    err[0] = 2
    run()
    torch.cuda.synchronize()
    for x, s in zip(everything, snap):
        assert bitwise_equal(x, s), "outer_nesterov_f32 wrote with the abort flag set"
    print("[bitwise] outer_nesterov_f32 with err = 2: every buffer untouched")
    err.zero_()
    run()
    _check_err(err, "outer_nesterov_f32")
    what = f"outer_nesterov_f32 W={W} nb={nb} n={n} dst={ndst}"
    for x, s in zip(thetas, snap_thetas):
        assert bitwise_equal(x, s), f"{what}: a peer master was written"
    t0d = t0.to(dev).double()
    gsum = sum(t0d - x.double() for x in thetas)
    gmag = sum((t0d - x.double()).abs() for x in thetas)
    # the fp32 pseudo-gradient: one subtraction and one add per worker
    _outer_check(what, 2 * W, a, t0.to(dev), mom0.to(dev), gsum, gmag, theta0, mom, theta_new, dsts, starts, dst, total)


# ================================================================================================== GPU: cast, gathers
def _specials(n):
    x = _wide(n, -140, 127, seed=n)  # fp32 subnormals up to the top of the range
    sp = torch.tensor([0.0, -0.0, 1e-40, -1e-41, 2.0**-149, 3.39e38, -3.3999e38, 3.4e38, float("inf"), float("-inf"), float("nan"),
                       1.0 + 2.0**-8, 1.0 + 3 * 2.0**-8, -(1.0 + 2.0**-8)])  # fmt: skip
    x[: sp.numel()] = sp
    x[-sp.numel() :] = sp
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("n", [16, ADAM_PASS + 8])
@pytest.mark.parametrize("ndst", [1, 2, 5, 8])
def test_cast_push(ndst, n):
    dev = _dev()
    src = _specials(n).to(dev)
    dst_off = 40
    dsts = [Out(dst_off + n + 8, torch.bfloat16) for _ in range(ndst)]
    _launch("pb_cast_push", src.data_ptr(), n, _pref(_pp([d.t for d in dsts])), dst_off, _stream())
    torch.cuda.synchronize()
    want = src.to(torch.bfloat16)
    nan = torch.isnan(src)
    for q, d in enumerate(dsts):
        got = d.t[dst_off : dst_off + n]
        assert bool((torch.isnan(got) == nan).all()), "NaN positions differ"
        body = torch.full((dst_off + n + 8,), SENT[torch.bfloat16], dtype=torch.bfloat16, device=dev)
        body[dst_off : dst_off + n] = torch.where(nan, got, want)  # NaN payloads compared with isnan above
        assert_bitwise(d.buf, d.image(body), f"cast_push n={n} destination {q}")
    j = n - 7  # the second copy of the specials ends the vector: 3.4e38 sits 7 from the end
    assert float(src[j]) == _f32(3.4e38) and bool(torch.isinf(dsts[0].t[dst_off + j])), "3.4e38 must round up to bf16 inf"


@pytest.mark.gpu
@pytest.mark.parametrize("nbytes", [48, 16 * 100_003])
@pytest.mark.parametrize("F", [1, 3, 8])
def test_allgather_copy(F, nbytes):
    assert nbytes % AG_PASS != 0
    dev = _dev()
    gen = torch.Generator().manual_seed(F + nbytes)
    shards = [torch.randint(0, 256, (nbytes,), generator=gen, dtype=torch.uint8).to(dev) for _ in range(F)]
    out = Out(F * nbytes, torch.uint8)
    _launch("pb_allgather_copy", _pref(_pp(shards)), nbytes, out.ptr(), _stream())
    torch.cuda.synchronize()
    assert_bitwise(out.buf, out.image(torch.cat(shards)), f"allgather_copy F={F} bytes/rank={nbytes}")


@pytest.mark.gpu
@pytest.mark.parametrize("F", [1, 2, 3, 8])
def test_embedding_fwd_row_shards(F):
    dev = _dev()
    rpr, dim = 37, 136
    V = F * rpr
    shards = [_wide(rpr * dim, -20, 4, seed=F * 10 + r).to(torch.bfloat16).to(dev) for r in range(F)]
    W_full = torch.cat(shards).view(V, dim)
    edge = [t for t in (0, rpr - 1, rpr, (F - 1) * rpr, V - 1) if t < V]
    tok = torch.cat([torch.tensor(edge), torch.randint(0, V, (301,), generator=torch.Generator().manual_seed(F))]).to(dev)
    T = tok.numel()
    out = Out(T * dim, torch.bfloat16)
    _launch("pb_embedding_fwd", tok.data_ptr(), T, _pref(_pp(shards)), rpr, dim, out.ptr(), _stream())
    torch.cuda.synchronize()
    assert_bitwise(out.buf, out.image(W_full[tok].reshape(-1)), f"embedding_fwd F={F} rows of {T} tokens")
