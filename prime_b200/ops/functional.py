"""Public op surface.  CUDA tensors → hand-written sm_90a kernels (required, loud failure);
CPU tensors → the torch reference in :mod:`prime_b200.ops.reference`.

Every CUDA op is a ``torch.autograd.Function`` whose forward/backward launch kernels from the
native library on the *current* torch stream (so they compose with streams and CUDA graphs).
``launch_count()`` reports how many native kernels were launched — bench.py's ``gpu_launches``.
"""

from __future__ import annotations

import math
from dataclasses import dataclass

import torch

from . import _lib, reference

_LAUNCHES = 0


def launch_count() -> int:
    return _LAUNCHES


def reset_launch_count() -> None:
    global _LAUNCHES
    _LAUNCHES = 0


def _count(n: int = 1) -> None:
    global _LAUNCHES
    _LAUNCHES += n


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: torch.Tensor | None) -> int | None:
    return None if t is None else t.data_ptr()


def _launch(name: str, *args, n: int = 1) -> None:
    """Call the native launcher ``name``, raise on a non-zero return code and count the ``n`` kernels it launches."""
    _lib.check(getattr(_lib.load(), name)(*args), name)
    _count(n)


def _rows(t: torch.Tensor) -> torch.Tensor:
    """``t`` as a 2-D [rows, last dim] matrix with unit strides (a view when the layout allows it)."""
    t2 = t.reshape(-1, t.shape[-1])
    return t2 if t2.is_contiguous() else t2.contiguous()


# --------------------------------------------------------------------------- GEMM


def gemm(
    a: torch.Tensor,
    b: torch.Tensor,
    *,
    a_mn_major: bool = False,
    b_mn_major: bool = False,
    out: torch.Tensor | None = None,
    out_dtype: torch.dtype = torch.bfloat16,
    accumulate: bool = False,
    rope: tuple | None = None,
    swiglu_h: torch.Tensor | None = None,
    swiglu_bwd_gu: torch.Tensor | None = None,
) -> torch.Tensor:
    """C[M,N] (+)= A·Bᵀ on the wgmma kernel.

    ``a``: [M,K] (K-major) or, if ``a_mn_major``, stored [K,M].
    ``b``: [N,K] (K-major) or, if ``b_mn_major``, stored [K,N].
    Both must be 2-D bf16 with unit inner stride.
    Fused epilogues (:func:`_epilogue`; K-major ``a``, bf16 output): ``rope`` rotates the Q/K head columns, ``swiglu_h`` receives
    silu(gate)·up of C = gate_up [M, 2·FF], ``swiglu_bwd_gu`` (MN-major ``b``, M > 128) turns the product dh [M, FF] into
    C = d_gate_up [M, 2·FF] from the saved gate_up.
    """
    assert a.dtype == torch.bfloat16 and b.dtype == torch.bfloat16
    assert a.dim() == 2 and b.dim() == 2 and a.stride(1) == 1 and b.stride(1) == 1
    if a_mn_major:
        K, M = a.shape
    else:
        M, K = a.shape
    if b_mn_major:
        Kb, N = b.shape
    else:
        N, Kb = b.shape
    assert K == Kb, f"contraction mismatch {K} vs {Kb}"
    out_n = 2 * N if swiglu_bwd_gu is not None else N
    if out is None:
        assert not accumulate
        out = torch.empty((M, out_n), dtype=out_dtype, device=a.device)
    else:
        assert out.shape == (M, out_n) and out.stride(1) == 1 and out.dtype in (torch.bfloat16, torch.float32)
    _launch(
        "pb_gemm_bf16", a.data_ptr(), b.data_ptr(), out.data_ptr(), M, N, K, a.stride(0), b.stride(0), out.stride(0),
        int(a_mn_major), int(b_mn_major), int(out.dtype == torch.float32), int(accumulate),
        _epilogue(rope, swiglu_h, swiglu_bwd_gu), _stream(),
    )  # fmt: skip
    return out


def _epilogue(rope: tuple | None, swiglu_h: torch.Tensor | None, swiglu_bwd_gu: torch.Tensor | None) -> _lib.GemmEpilogue | None:
    """The native epilogue descriptor of a GEMM launch, None for a plain GEMM. ``rope`` = (cos, sin, seq_len, rotated columns,
    head_dim) with fp32 [>= seq_len, head_dim/2] tables; ``swiglu_h`` = h [M, FF]; ``swiglu_bwd_gu`` = the saved gate_up [M, 2·FF]."""
    if swiglu_bwd_gu is not None:
        return _lib.GemmEpilogue(kind=3, aux=swiglu_bwd_gu.data_ptr(), ld_aux=swiglu_bwd_gu.stride(0))
    if swiglu_h is not None:
        return _lib.GemmEpilogue(kind=2, aux=swiglu_h.data_ptr(), ld_aux=swiglu_h.stride(0))
    if rope is not None:
        cos, sin, seq_len, rot_cols, head_dim = rope
        assert cos.dtype == torch.float32 and cos.is_contiguous() and sin.is_contiguous() and cos.shape[0] >= seq_len
        return _lib.GemmEpilogue(kind=1, rope_cos=cos.data_ptr(), rope_sin=sin.data_ptr(), rope_S=seq_len, rope_cols=rot_cols,
                                 rope_D=head_dim)  # fmt: skip
    return None


def set_gemm_split_k(mode: int) -> int:
    """Split-K policy of fp32 reduce-add GEMMs (weight gradients): -1 automatic, 0 off, n>1 force n slices. Returns the old mode."""
    return int(_lib.load().pb_gemm_set_split_k(int(mode)))


GEMM_TILE_MODES = (128, 256)  # tile widths of the local GEMM (128 x 128 and 128 x 256 tiles)


def set_gemm_tile(mode: int) -> int:
    """Tile width of :func:`gemm`: -1 automatic (the shape policy), 128 or 256 forced (testing). Returns the old mode."""
    if mode != -1 and mode not in GEMM_TILE_MODES:
        raise ValueError(f"GEMM tile mode must be -1 or one of {GEMM_TILE_MODES}, got {mode}")
    return int(_lib.load().pb_gemm_set_tile(int(mode)))


def gemm_tile_policy(M: int, N: int, K: int, *, epilogue: int = 0, c_fp32: bool = False, accumulate: bool = False, num_sms: int = 132) -> int:
    """The tile width (128 | 256) the automatic policy picks for C[M, N] = A·Bᵀ with contraction K; ``epilogue`` is the
    ``GemmEpilogue`` kind (2: SwiGLU, N = 2·FF). Host-side only: needs the library, not a GPU."""
    return int(_lib.load().pb_gemm_tile_policy(M, N, K, epilogue, int(c_fp32), int(accumulate), num_sms))


def _take_fresh(param: torch.Tensor) -> bool:
    """True exactly once per optimizer step and parameter (the sharded engine arms ``_mg_fresh`` in ``zero_grad``): the first
    gradient write of the step OVERWRITES main_grad, which is what lets the engine skip the 4·N-byte memset."""
    if getattr(param, "_mg_fresh", False):
        param._mg_fresh = False
        return True
    return False


def _wgrad(dy2: torch.Tensor, x2: torch.Tensor, weight: torch.Tensor) -> torch.Tensor | None:
    """dW = dyᵀ·x: fused fp32 accumulation into ``weight.main_grad`` when the engine attached one, else a bf16 gradient."""
    main_grad = getattr(weight, "main_grad", None)
    if main_grad is not None:
        gemm(dy2, x2, a_mn_major=True, b_mn_major=True, out=main_grad, accumulate=not _take_fresh(weight))
        return None
    return gemm(dy2, x2, a_mn_major=True, b_mn_major=True)


# Which weight currently sits, complete, in each gather scratch region: full_ptr → (id of the RowShard, shard version).
# Everything runs on one stream in program order, so "the kernel that gathers it has been enqueued" is all that needs tracking.
_RESIDENT: dict[int, tuple[int, int]] = {}


def reset_gather_cache() -> None:
    """Forget what the gather scratch holds (CUDA-graph capture: a captured micro-step must not depend on what an earlier
    micro-step happened to leave resident; engine construction / teardown)."""
    _RESIDENT.clear()


def _resident(z) -> bool:
    return z.full_ptr != 0 and _RESIDENT.get(z.full_ptr) == (id(z), z.ver[0])


def _mark_resident(z) -> None:
    _RESIDENT[z.full_ptr] = (id(z), z.ver[0])


def _full_weight(z, device) -> torch.Tensor:
    if z.full is not None:
        return z.full
    return torch.as_tensor(_RawBuffer(z.full_ptr, z.rows * z.cols * 2), device=device).view(torch.bfloat16).view(z.rows, z.cols)


def _gemm_epi(a: torch.Tensor, w: torch.Tensor, out: torch.Tensor, *, b_mn_major: bool = False, rope: tuple | None = None,
              swiglu_h: torch.Tensor | None = None, swiglu_bwd_gu: torch.Tensor | None = None) -> torch.Tensor:  # fmt: skip
    """The GEMM of :func:`gemm_wgather` and its epilogues on a local weight ``w`` [rows, cols]: C = a·wᵀ (``rope``, ``swiglu_h``) or,
    with ``b_mn_major``, C = a·w (``swiglu_bwd_gu``). SwiGLU runs as a stand-alone kernel after a plain GEMM where its fused
    epilogue does not apply (M <= 128, and for the forward hidden % 64 != 0)."""
    M = a.shape[0]
    if swiglu_bwd_gu is not None and M <= 128:
        dh = gemm(a, w, b_mn_major=True)
        _launch("pb_swiglu_bwd", swiglu_bwd_gu.data_ptr(), dh.data_ptr(), out.data_ptr(), M, w.shape[1], _stream())
    elif swiglu_h is not None and (M <= 128 or (w.shape[0] // 2) % 64 != 0):
        gemm(a, w, out=out)
        _launch("pb_swiglu_fwd", out.data_ptr(), swiglu_h.data_ptr(), M, w.shape[0] // 2, _stream())
    else:
        gemm(a, w, b_mn_major=b_mn_major, out=out, rope=rope, swiglu_h=swiglu_h, swiglu_bwd_gu=swiglu_bwd_gu)
    return out


def _matmul(a: torch.Tensor, weight: torch.Tensor, out: torch.Tensor, **epi) -> torch.Tensor:
    """:func:`_gemm_epi` on ``weight``, gathered from the peers' shards inside the GEMM when it is ZeRO-3 sharded (``weight.z3``).
    An e4m3 :class:`MXWeight` (forward only): at M <= :func:`gemm_e4m3w_m_max` the skinny kernel reads its bytes in place, with
    SwiGLU as the separate kernel (no RoPE epilogue: decode and verify rotate in the cache append); above it the weight is
    dequantised into a transient bf16 buffer and the bf16 GEMM runs with its epilogues, as it would on the bf16 model holding W̃."""
    if isinstance(weight, MXWeight):
        assert not epi.get("b_mn_major") and epi.get("swiglu_bwd_gu") is None, "e4m3 weights have no backward"
        M = a.shape[0]
        if M > gemm_e4m3w_m_max():
            return _gemm_epi(a, dequantize_weight(weight), out, rope=epi.get("rope"), swiglu_h=epi.get("swiglu_h"))
        assert epi.get("rope") is None, "the skinny e4m3 GEMM has no RoPE epilogue"
        gemm_e4m3w(a, weight, out=out)
        h = epi.get("swiglu_h")
        if h is not None:
            _launch("pb_swiglu_fwd", out.data_ptr(), h.data_ptr(), M, weight.shape[0] // 2, _stream())
        return out
    z = getattr(weight, "z3", None)
    if z is not None:
        return gemm_wgather(a, z, out=out, **epi)
    return _gemm_epi(a, weight, out, **epi)


def gemm_wgather(a: torch.Tensor, z, *, b_mn_major: bool = False, out: torch.Tensor | None = None, rope: tuple | None = None,
                 swiglu_h: torch.Tensor | None = None, swiglu_bwd_gu: torch.Tensor | None = None) -> torch.Tensor:  # fmt: skip
    """Parameter all-gather ⊕ GEMM (ZeRO-3): ``z`` is the ``RowShard`` of a weight W [rows, cols] sharded by rows over the FSDP group.

    ``b_mn_major=False``: C[M, rows] = a[M, cols]·Wᵀ (forward; ``rope`` = RoPE epilogue, ``swiglu_h`` = SwiGLU epilogue with W = W13,
    C = gate_up, ``swiglu_h`` = h).  ``b_mn_major=True``: C[M, cols] = a[M, rows]·W (input gradient; with ``swiglu_bwd_gu`` = the
    saved gate_up the epilogue turns dh into d_gate_up [M, 2·cols] on the fly).

    The peers' row blocks are pulled over NVLink by copier warps INSIDE the GEMM kernel (csrc/gemm_sm90.cu, IO = 3). The same
    kernel also gathers AHEAD the weight the next GEMM of the pass will consume (``z.next_fwd`` / ``z.next_bwd``), so in steady
    state a kernel finds its own operand already resident (no gating, full speed) and only carries the next one's transfer."""
    import ctypes

    assert a.dtype == torch.bfloat16 and a.dim() == 2 and a.stride(1) == 1
    M = a.shape[0]
    N = z.cols if b_mn_major else z.rows
    assert a.shape[1] == (z.rows if b_mn_major else z.cols)
    if out is None:
        out = torch.empty((M, 2 * N if swiglu_bwd_gu is not None else N), dtype=torch.bfloat16, device=a.device)
    own_resident = _resident(z)
    nz = z.next_bwd if b_mn_major else z.next_fwd
    if nz is not None and (nz.full_ptr == 0 or _resident(nz) or nz.n != z.n):
        nz = None
    if M <= 128 or (own_resident and nz is None):
        # operand complete in the local scratch (gathered ahead by the previous kernel), or tiny M (unit tests, debug models: explicit
        # gather by peer loads first): the plain kernels
        if not own_resident:
            pp = _lib.PeerPtrs.of(z.peer_ptrs[i] for i in range(z.n))
            _launch("pb_allgather_copy", ctypes.byref(pp), z.rpr * z.cols * 2, z.full_ptr, _stream())
            _mark_resident(z)
        return _gemm_epi(a, _full_weight(z, a.device), out, b_mn_major=b_mn_major, rope=rope, swiglu_h=swiglu_h, swiglu_bwd_gu=swiglu_bwd_gu)
    _launch(
        "pb_gemm_wgather", a.data_ptr(), z.peer_ptrs, z.n, z.rank, z.full_ptr, z.flags.data_ptr(), out.data_ptr(), M, z.rows, z.cols,
        a.stride(0), out.stride(0), int(b_mn_major), _epilogue(rope, swiglu_h, swiglu_bwd_gu),
        int(own_resident), nz.peer_ptrs if nz is not None else None, nz.full_ptr if nz is not None else None,
        nz.rows if nz is not None else 0, nz.cols if nz is not None else 0, _stream(), n=1 if own_resident else 2,
    )  # fmt: skip
    _mark_resident(z)
    if nz is not None:
        _mark_resident(nz)
    return out


class _RawBuffer:
    """Raw device pointer → torch (zero copy) through ``__cuda_array_interface__``."""

    def __init__(self, ptr: int, nbytes: int):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 3, "strides": None}


class _LinearFn(torch.autograd.Function):
    """y = x Wᵀ.  Weight gradient accumulates straight into ``weight.main_grad`` (fp32, fused in the GEMM
    epilogue) when the FSDP engine has attached one; otherwise a bf16 gradient is returned."""

    @staticmethod
    def forward(ctx, x: torch.Tensor, weight: torch.Tensor, rope: tuple | None = None) -> torch.Tensor:
        x2 = _rows(x)
        ctx.save_for_backward(x2, weight)
        ctx.x_shape = x.shape
        # allocate with the final shape: a Function output must not be a view (RoPE / the loss rotate / overwrite it in place)
        y = torch.empty((*x.shape[:-1], weight.shape[0]), dtype=x.dtype, device=x.device)
        # rope: fused QKV projection, the GEMM epilogue rotates the Q/K head columns while the tile is in registers. The consumer
        # (rope_attention_qkv(..., pre_rotated=True)) returns the gradient w.r.t. the UN-rotated activation, so backward below is the
        # plain linear backward.
        _matmul(x2, weight, y.view(-1, weight.shape[0]), rope=rope)
        return y

    @staticmethod
    def backward(ctx, dy: torch.Tensor):
        x2, weight = ctx.saved_tensors
        dy2 = _rows(dy)
        dx = dw = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty(ctx.x_shape, dtype=dy.dtype, device=dy.device)
            _matmul(dy2, weight, dx.view(-1, ctx.x_shape[-1]), b_mn_major=True)
        if ctx.needs_input_grad[1]:
            dw = _wgrad(dy2, x2, weight)
        return dx, dw, None


def linear(x: torch.Tensor, weight: torch.Tensor) -> torch.Tensor:
    """y = x Wᵀ; ``weight`` may be an e4m3 :class:`MXWeight` (inference only)."""
    if isinstance(weight, MXWeight):
        return _mx_linear(x, weight)
    if x.is_cuda:
        return _LinearFn.apply(x, weight)
    return reference.linear(x, weight)


# --------------------------------------------------------------------------- e4m3 inference weights


@dataclass(frozen=True, eq=False)
class MXWeight:
    """An inference weight W [N, K] held as e4m3: exactly what :func:`quantize_mxfp8` returns for it, the bytes ``q`` uint8 [N, K] and
    one UE8M0 exponent per 32 values along K in ``sf`` (the 512-byte atom layout of ``reference._mxfp8_sf_index``), about 1.03 bytes
    per weight. It stands for W̃ = ``reference.dequantize_mxfp8(q, sf)``, exact in fp32, and exact in bf16 for every block whose scale
    is above the bf16 subnormal edge. ``dtype`` is the dtype of the weight it was made from, the one its products are computed in.

    ``linear``, ``linear_qkv_rope``, ``linear_swiglu`` and ``mlp_swiglu`` take it in place of a weight tensor, forward only: a call that
    would need its gradient raises. On CUDA (``_matmul``) M <= :func:`gemm_e4m3w_m_max` runs :func:`gemm_e4m3w`; larger M runs the bf16
    GEMM on :func:`dequantize_weight`. On the CPU every op runs the reference on W̃ in the input's dtype."""

    q: torch.Tensor
    sf: torch.Tensor
    dtype: torch.dtype

    @property
    def shape(self) -> torch.Size:
        return self.q.shape

    @property
    def device(self) -> torch.device:
        return self.q.device


def quantize_weight(w: torch.Tensor) -> MXWeight:
    """W [N, K] (K % 128 == 0) → :class:`MXWeight`: :func:`quantize_mxfp8` of a bf16 CUDA weight, ``reference.quantize_mxfp8`` of a CPU
    weight of any float dtype, taken as stored."""
    if w.dim() != 2 or w.shape[1] % 128:
        raise ValueError(f"an e4m3 weight needs a 2-D [N, K] tensor with K % 128 == 0, got {tuple(w.shape)}")
    w = w.detach()
    if w.is_cuda:
        if w.dtype != torch.bfloat16:
            raise ValueError(f"a CUDA weight is quantised from bf16, got {w.dtype}")
        q, sf = quantize_mxfp8(w.contiguous())
    else:
        q, sf = reference.quantize_mxfp8(w)
    return MXWeight(q, sf, w.dtype)


def dequantize_weight(w: MXWeight, out: torch.Tensor | None = None) -> torch.Tensor:
    """W̃ of an :class:`MXWeight` in its ``dtype`` (``out``: [N, K] with unit column stride). On CUDA ``pb_dequantize_mxfp8``, bitwise
    equal to ``reference.dequantize_mxfp8(q, sf).to(torch.bfloat16)``."""
    N, K = w.shape
    if not w.q.is_cuda:
        full = reference.dequantize_mxfp8(w.q, w.sf).to(w.dtype)
        return full if out is None else out.copy_(full)
    if out is None:
        out = torch.empty((N, K), dtype=torch.bfloat16, device=w.device)
    assert out.shape == (N, K) and out.dtype == torch.bfloat16 and out.stride(1) == 1
    _launch("pb_dequantize_mxfp8", w.q.data_ptr(), w.sf.data_ptr(), out.data_ptr(), N, K, out.stride(0), _stream())
    return out


_E4M3W_M_MAX: list[int] = []
_SM_COUNT: dict = {}


def gemm_e4m3w_m_max() -> int:
    """The largest M :func:`gemm_e4m3w` takes (the native library's constant)."""
    if not _E4M3W_M_MAX:
        _E4M3W_M_MAX.append(int(_lib.load().pb_gemm_e4m3w_m_max()))
    return _E4M3W_M_MAX[0]


def gemm_e4m3w_splits(M: int, N: int, K: int, num_sms: int = 132) -> int:
    """The split-K count :func:`gemm_e4m3w` uses for C[M, N] with contraction K on ``num_sms`` SMs: a function of the shape only, so a
    captured step stays valid. Host-side only: needs the library, not a GPU."""
    n = int(_lib.load().pb_gemm_e4m3w_splits(M, N, K, num_sms))
    _lib.check(min(n, 0), "pb_gemm_e4m3w_splits")
    return n


def _num_sms(device: torch.device) -> int:
    n = _SM_COUNT.get(device)
    if n is None:
        n = _SM_COUNT[device] = torch.cuda.get_device_properties(device).multi_processor_count
    return n


def gemm_e4m3w(x: torch.Tensor, w: MXWeight, *, out: torch.Tensor | None = None, splits: int | None = None) -> torch.Tensor:
    """C[M, N] bf16 = x[M, K] · W̃ᵀ for 1 <= M <= :func:`gemm_e4m3w_m_max` on the native skinny kernel: each weight byte is read once,
    dequantised exactly in registers, and multiplied on bf16 MMAs with fp32 accumulation. ``out``: [M, N] with unit column stride (a
    strided view is fine; nothing outside its columns is written). ``splits``: the split-K count (None = :func:`gemm_e4m3w_splits`);
    the fp32 partials go to a workspace allocated here and are summed in a fixed order, so two calls are bitwise equal."""
    assert x.is_cuda and x.dtype == torch.bfloat16 and x.dim() == 2 and x.is_contiguous()
    M, K = x.shape
    N = w.shape[0]
    assert w.shape[1] == K, f"contraction mismatch {K} vs {w.shape[1]}"
    if out is None:
        out = torch.empty((M, N), dtype=torch.bfloat16, device=x.device)
    assert out.shape == (M, N) and out.dtype == torch.bfloat16 and out.stride(1) == 1
    if splits is None:
        splits = gemm_e4m3w_splits(M, N, K, _num_sms(x.device)) if 1 <= M <= gemm_e4m3w_m_max() else 1
    ws = torch.empty((splits, M, N), dtype=torch.float32, device=x.device) if splits > 1 else None
    _launch("pb_gemm_e4m3w", x.data_ptr(), w.q.data_ptr(), w.sf.data_ptr(), out.data_ptr(), _ptr(ws), M, N, K, out.stride(0) if M > 1 else N,
            splits, _stream(), n=1 if splits == 1 else 2)  # fmt: skip
    return out


def _mx_no_grad(x: torch.Tensor) -> None:
    if torch.is_grad_enabled() and x.requires_grad:
        raise RuntimeError("e4m3 weights (ops.MXWeight) are for inference only and have no gradient: run the forward under "
                           "torch.no_grad() or on inputs that do not require grad")  # fmt: skip


def _mx_linear(x: torch.Tensor, w: MXWeight, rope: tuple | None = None) -> torch.Tensor:
    """:func:`linear` (``rope``: :func:`linear_qkv_rope`) on an e4m3 weight; no autograd node, so nothing saves the weight."""
    _mx_no_grad(x)
    if not x.is_cuda:
        return reference.linear(x, dequantize_weight(w).to(x.dtype))
    x2 = _rows(x)
    y = torch.empty((*x.shape[:-1], w.shape[0]), dtype=x.dtype, device=x.device)
    _matmul(x2, w, y.view(-1, w.shape[0]), rope=rope)
    return y


# --------------------------------------------------------------------------- block-scaled fp8 (MXFP8)


def mxfp8_sf_bytes(rows: int, k: int) -> int:
    """Size of the scale-factor buffer of a [rows, k] MXFP8 operand: [k/128][ceil(rows/128)+1] atoms of 512 bytes."""
    return (k // 128) * ((rows + 127) // 128 + 1) * 512


def quantize_mxfp8(x: torch.Tensor, transpose: bool = False) -> tuple[torch.Tensor, torch.Tensor]:
    """bf16 [R, C] → (e4m3 values as uint8, UE8M0 scales in the tensor-core layout), one power-of-two scale per 32 elements.

    ``transpose=False``: values [R, C], blocks along C (operand contracted over C).
    ``transpose=True``:  values [C, R], blocks along R (the same matrix used with R as the contraction dimension)."""
    assert x.dim() == 2 and x.dtype == torch.bfloat16 and x.stride(1) == 1
    R, C = x.shape
    rows, k = (C, R) if transpose else (R, C)
    assert k % 128 == 0, f"MXFP8 contraction dimension must be a multiple of 128, got {k}"
    if not x.is_cuda:
        return reference.quantize_mxfp8(x, transpose)
    q = torch.empty((rows, k), dtype=torch.uint8, device=x.device)
    sf = torch.empty(mxfp8_sf_bytes(rows, k), dtype=torch.uint8, device=x.device)
    _launch("pb_quantize_mxfp8", x.data_ptr(), x.stride(0), q.data_ptr(), sf.data_ptr(), R, C, int(transpose), _stream())
    return q, sf


def gemm_mxfp8(aq: torch.Tensor, asf: torch.Tensor, bq: torch.Tensor, bsf: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
    """C[M,N] bf16 = dequant(A)·dequant(B)ᵀ with e4m3 tensor-core MMAs, scaled per 32-element block in registers."""
    M, K = aq.shape
    N, Kb = bq.shape
    assert K == Kb and aq.dtype == torch.uint8 and bq.dtype == torch.uint8 and aq.is_contiguous() and bq.is_contiguous()
    if not aq.is_cuda:
        c = reference.dequantize_mxfp8(aq, asf) @ reference.dequantize_mxfp8(bq, bsf).t()
        if out is None:
            return c.to(torch.bfloat16)
        out.copy_(c)
        return out
    if out is None:
        out = torch.empty((M, N), dtype=torch.bfloat16, device=aq.device)
    assert out.shape == (M, N) and out.dtype == torch.bfloat16 and out.stride(1) == 1
    _launch("pb_gemm_mxfp8", aq.data_ptr(), asf.data_ptr(), bq.data_ptr(), bsf.data_ptr(), out.data_ptr(), M, N, K, out.stride(0), _stream())
    return out


class _LinearMXFP8Fn(torch.autograd.Function):
    """y = x Wᵀ with the forward and the input-gradient GEMMs in block-scaled fp8; the weight gradient stays bf16 with fp32
    accumulation into ``main_grad`` (its contraction runs over tokens, where per-32 blocks along the token axis would need a
    third quantisation of both operands for the least precision-tolerant of the three GEMMs)."""

    @staticmethod
    def forward(ctx, x: torch.Tensor, weight: torch.Tensor) -> torch.Tensor:
        x2 = _rows(x)
        ctx.save_for_backward(x2, weight)
        ctx.x_shape = x.shape
        xq, xsf = quantize_mxfp8(x2)
        wq, wsf = quantize_mxfp8(weight)
        y = torch.empty((*x.shape[:-1], weight.shape[0]), dtype=x.dtype, device=x.device)
        gemm_mxfp8(xq, xsf, wq, wsf, out=y.view(-1, weight.shape[0]))
        return y

    @staticmethod
    def backward(ctx, dy: torch.Tensor):
        x2, weight = ctx.saved_tensors
        dy2 = _rows(dy)
        dx = dw = None
        if ctx.needs_input_grad[0]:
            dyq, dysf = quantize_mxfp8(dy2)                     # [M, N], blocks along N
            wtq, wtsf = quantize_mxfp8(weight, transpose=True)  # [K, N], blocks along N
            dx = torch.empty(ctx.x_shape, dtype=dy.dtype, device=dy.device)
            gemm_mxfp8(dyq, dysf, wtq, wtsf, out=dx.view(-1, ctx.x_shape[-1]))
        if ctx.needs_input_grad[1]:
            if x2.is_cuda:
                dw = _wgrad(dy2, x2, weight)
            else:
                dw = (dy2.float().t() @ x2.float()).to(weight.dtype)
        return dx, dw


def mxfp8_usable(x: torch.Tensor, weight: torch.Tensor) -> bool:
    """Both contraction dimensions (in for the forward, out for the input gradient) must be multiples of 128."""
    return weight.shape[0] % 128 == 0 and weight.shape[1] % 128 == 0 and x.dtype == torch.bfloat16


def linear_mxfp8(x: torch.Tensor, weight: torch.Tensor) -> torch.Tensor:
    """``linear`` with MXFP8 forward / input-gradient GEMMs (``train.precision = "mxfp8"``); falls back to bf16 for shapes the
    block format cannot express."""
    if not mxfp8_usable(x, weight):
        return linear(x, weight)
    return _LinearMXFP8Fn.apply(x, weight)


# A/B switch for measurements: PB_NO_EPILOGUE_FUSION=1 runs RoPE and SwiGLU as stand-alone kernels again
_NO_EPILOGUE_FUSION = bool(int(__import__("os").environ.get("PB_NO_EPILOGUE_FUSION", "0")))


def rope_fusable(x: torch.Tensor, n_heads: int, n_kv_heads: int, head_dim: int) -> bool:
    """Can the QKV projection rotate in its epilogue AND the native attention consume/undo it? (CUDA, [B,S,·] input, S%128==0)"""
    if _NO_EPILOGUE_FUSION or not (x.is_cuda and x.dim() == 3 and x.dtype == torch.bfloat16):
        return False
    from . import attention_native as native

    return native.supported_shape(x.shape[1], head_dim, n_heads, n_kv_heads)


def linear_qkv_rope(x: torch.Tensor, weight: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, n_heads: int, n_kv_heads: int) -> torch.Tensor:
    """Fused QKV projection ⊕ RoPE: [B,S,dim] → [B,S,(H+2Hkv)·D] with the Q and K heads already rotated (GEMM epilogue).
    Must be consumed by ``rope_attention_qkv(..., pre_rotated=True)``, whose backward undoes the rotation in its own epilogues."""
    head_dim = weight.shape[0] // (n_heads + 2 * n_kv_heads)
    rope = (cos, sin, x.shape[1], (n_heads + n_kv_heads) * head_dim, head_dim)
    if isinstance(weight, MXWeight):
        return _mx_linear(x, weight, rope)
    return _LinearFn.apply(x, weight, rope)


# --------------------------------------------------------------------------- embedding


class _EmbeddingFn(torch.autograd.Function):
    """Row gather out of the parameter (ZeRO-3: out of the peers' shards over NVLink) and a deterministic, sort-based scatter-add of
    the gradient into the fp32 ``main_grad`` (csrc/embedding.cu) — no torch indexing / radix-sort / atomics kernels."""

    @staticmethod
    def forward(ctx, tokens: torch.Tensor, weight: torch.Tensor) -> torch.Tensor:
        import ctypes

        V, dim = weight.shape
        t = tokens.reshape(-1)
        t = t if t.is_contiguous() else t.contiguous()
        assert t.dtype == torch.int64
        z = getattr(weight, "z3", None)
        if z is not None:
            pp, rpr = _lib.PeerPtrs.of(z.peer_ptrs[i] for i in range(z.n)), z.rpr
        else:
            assert weight.is_contiguous()
            pp, rpr = _lib.PeerPtrs.of([weight.data_ptr()]), V
        out = torch.empty((*tokens.shape, dim), dtype=weight.dtype, device=weight.device)
        _launch("pb_embedding_fwd", t.data_ptr(), t.numel(), ctypes.byref(pp), rpr, dim, out.data_ptr(), _stream())
        ctx.weight = weight
        ctx.sorted_ev = None
        if ctx.needs_input_grad[1]:  # (autograd runs forward() with grad mode off: needs_input_grad is the reliable signal)
            # the backward needs the positions sorted by token: a one-CTA kernel (~0.2 ms) that depends only on the token ids, so it
            # runs NOW on a side stream underneath the forward GEMMs instead of on the critical path at the end of the backward
            sorted_keys = torch.empty(t.numel(), dtype=torch.int64, device=weight.device)
            n_chunks = (t.numel() + 16383) // 16384
            if torch.cuda.is_current_stream_capturing():
                _launch("pb_embedding_sort", t.data_ptr(), t.numel(), sorted_keys.data_ptr(), _stream(), n=n_chunks)
            else:
                side = _side_stream(weight.device)
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    _launch("pb_embedding_sort", t.data_ptr(), t.numel(), sorted_keys.data_ptr(), side.cuda_stream, n=n_chunks)
                    ctx.sorted_ev = torch.cuda.Event()
                    ctx.sorted_ev.record(side)
                t.record_stream(side)
                sorted_keys.record_stream(side)
            ctx.save_for_backward(sorted_keys)
        return out

    @staticmethod
    def backward(ctx, dout: torch.Tensor):
        if not ctx.saved_tensors:
            return None, None
        (sorted_keys,) = ctx.saved_tensors
        weight = ctx.weight
        V, dim = weight.shape
        d2 = _rows(dout)
        main_grad = getattr(weight, "main_grad", None)
        if main_grad is not None:
            if _take_fresh(weight):
                main_grad.zero_()
            grad, ret = main_grad, None
        else:
            grad = torch.zeros((V, dim), dtype=torch.float32, device=dout.device)
            ret = grad
        if ctx.sorted_ev is not None:
            torch.cuda.current_stream().wait_event(ctx.sorted_ev)
        T = sorted_keys.numel()
        _launch("pb_embedding_scatter", sorted_keys.data_ptr(), T, d2.data_ptr(), grad.data_ptr(), dim, _stream(), n=(T + 16383) // 16384)
        return None, (None if ret is None else ret.to(weight.dtype))


_SIDE_STREAMS: dict = {}


def _side_stream(device: torch.device) -> "torch.cuda.Stream":
    s = _SIDE_STREAMS.get(device)
    if s is None:
        s = _SIDE_STREAMS[device] = torch.cuda.Stream(device=device)
    return s


def embedding(tokens: torch.Tensor, weight: torch.Tensor) -> torch.Tensor:
    """``weight[tokens]`` for a bf16 [V, dim] table (dim % 8 == 0)."""
    if weight.is_cuda and weight.dtype == torch.bfloat16 and weight.shape[1] % 8 == 0:
        return _EmbeddingFn.apply(tokens, weight)
    return torch.nn.functional.embedding(tokens, weight)


# --------------------------------------------------------------------------- RMSNorm


class _RMSNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, residual, weight, eps):
        x2 = _rows(x)
        R, D = x2.shape
        y = torch.empty(x.shape, dtype=x.dtype, device=x.device)
        rstd = torch.empty(R, dtype=torch.float32, device=x.device)
        if residual is not None:
            r2 = _rows(residual)
            h = torch.empty(x.shape, dtype=x.dtype, device=x.device)
        else:
            r2, h = None, x2
        _launch("pb_rmsnorm_fwd", _ptr(x2), _ptr(r2), _ptr(weight), _ptr(y), _ptr(h) if residual is not None else None,
                _ptr(rstd), R, D, float(eps), _stream())  # fmt: skip
        ctx.save_for_backward(h, weight, rstd)
        ctx.has_res = residual is not None
        ctx.shape = x.shape
        return y, (h if residual is not None else None)

    @staticmethod
    def backward(ctx, dy, dh):
        h, weight, rstd = ctx.saved_tensors
        dy2 = _rows(dy)
        R, D = dy2.shape
        dres = None if dh is None else _rows(dh)
        dx = torch.empty(ctx.shape, dtype=h.dtype, device=h.device)
        grid = _lib.load().pb_rmsnorm_bwd_grid(R)
        partial = torch.empty((grid, D), dtype=torch.float32, device=h.device)
        main_grad = getattr(weight, "main_grad", None)
        if main_grad is not None:
            dw32, acc = main_grad, 0 if _take_fresh(weight) else 1
        else:
            dw32, acc = torch.empty(D, dtype=torch.float32, device=h.device), 0
        _launch("pb_rmsnorm_bwd", _ptr(dy2), _ptr(h), _ptr(weight), _ptr(rstd), _ptr(dres), _ptr(dx), _ptr(partial),
                _ptr(dw32), acc, R, D, _stream(), n=2)  # fmt: skip
        dxv = dx
        dw = None if main_grad is not None else dw32.to(weight.dtype)
        # residual-add backward: gradient flows identically to x and residual
        return dxv, (dxv if ctx.has_res else None), dw, None


def rmsnorm(x: torch.Tensor, weight: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    if x.is_cuda:
        return _RMSNormFn.apply(x, None, weight, eps)[0]
    return reference.rmsnorm(x, weight, eps)


def add_rmsnorm(x: torch.Tensor, residual: torch.Tensor, weight: torch.Tensor, eps: float = 1e-5):
    """(rmsnorm(x + residual), x + residual) in one pass over HBM."""
    if x.is_cuda:
        return _RMSNormFn.apply(x, residual, weight, eps)
    return reference.add_rmsnorm(x, residual, weight, eps)


# --------------------------------------------------------------------------- RoPE (in place on fused QKV)


def _rope_inplace(qkv: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, n_heads: int, n_kv_heads: int, sign: float) -> None:
    """Rotate (``sign`` 1) or un-rotate (``sign`` -1) the Q and K heads of a contiguous fused [B,S,(H+2Hkv)·D] tensor in place."""
    total_heads = n_heads + 2 * n_kv_heads
    _launch("pb_rope_inplace", _ptr(qkv), _ptr(cos), _ptr(sin), qkv.numel() // qkv.shape[-1], qkv.shape[1], n_heads + n_kv_heads,
            total_heads, qkv.shape[-1] // total_heads, sign, _stream())  # fmt: skip


class _RopeQKVFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, qkv, cos, sin, n_heads, n_kv_heads):
        # qkv: [B, S, (H + 2*Hkv) * D] contiguous, produced by the QKV GEMM → rotate in place
        assert qkv.is_contiguous()
        _rope_inplace(qkv, cos, sin, n_heads, n_kv_heads, 1.0)
        ctx.mark_dirty(qkv)
        ctx.save_for_backward(cos, sin)
        ctx.meta = (n_heads, n_kv_heads)
        return qkv

    @staticmethod
    def backward(ctx, dqkv):
        cos, sin = ctx.saved_tensors
        # never rotate the incoming gradient in place: autograd may share that tensor with other consumers
        dqkv = dqkv.clone(memory_format=torch.contiguous_format)
        # rotation is orthogonal: the backward is the inverse rotation, applied in place on the incoming grad
        _rope_inplace(dqkv, cos, sin, *ctx.meta, -1.0)
        return dqkv, None, None, None, None


def rope_qkv(qkv: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, n_heads: int, n_kv_heads: int) -> torch.Tensor:
    """Rotate the Q and K heads of a fused [B,S,(H+2Hkv)·D] activation."""
    B, S, W = qkv.shape
    if qkv.is_cuda:
        return _RopeQKVFn.apply(qkv, cos, sin, n_heads, n_kv_heads)
    D = W // (n_heads + 2 * n_kv_heads)
    x = qkv.view(B, S, n_heads + 2 * n_kv_heads, D)
    rot = reference.rope(x[:, :, : n_heads + n_kv_heads], cos, sin)
    return torch.cat((rot, x[:, :, n_heads + n_kv_heads :]), dim=2).view(B, S, W)


# --------------------------------------------------------------------------- SwiGLU


class _SwiGLUFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, gate_up):
        gu = _rows(gate_up)
        M, FF = gu.shape[0], gu.shape[1] // 2
        out = torch.empty((*gate_up.shape[:-1], FF), dtype=gu.dtype, device=gu.device)
        _launch("pb_swiglu_fwd", _ptr(gu), _ptr(out), M, FF, _stream())
        ctx.save_for_backward(gu)
        ctx.shape = gate_up.shape
        return out

    @staticmethod
    def backward(ctx, dout):
        (gu,) = ctx.saved_tensors
        d2 = _rows(dout)
        dgu = torch.empty(ctx.shape, dtype=gu.dtype, device=gu.device)
        _launch("pb_swiglu_bwd", _ptr(gu), _ptr(d2), _ptr(dgu), gu.shape[0], gu.shape[1] // 2, _stream())
        return dgu


def swiglu(gate_up: torch.Tensor) -> torch.Tensor:
    if gate_up.is_cuda:
        return _SwiGLUFn.apply(gate_up)
    return reference.swiglu(gate_up)


class _LinearSwiGLUFn(torch.autograd.Function):
    """h = silu(x W1ᵀ) · (x W3ᵀ) with W13 = [W1; W3]: ONE GEMM whose epilogue emits both the bf16 gate/up activations (kept for
    the backward) and h — the separate SwiGLU pass over the 370 MB gate_up tensor disappears from the forward."""

    @staticmethod
    def forward(ctx, x: torch.Tensor, w13: torch.Tensor) -> torch.Tensor:
        x2 = _rows(x)
        M = x2.shape[0]
        FF = w13.shape[0] // 2
        gate_up = torch.empty((M, 2 * FF), dtype=x.dtype, device=x.device)
        h = torch.empty((*x.shape[:-1], FF), dtype=x.dtype, device=x.device)
        _matmul(x2, w13, gate_up, swiglu_h=h.view(M, FF))
        ctx.save_for_backward(x2, w13, gate_up)
        ctx.x_shape = x.shape
        return h

    @staticmethod
    def backward(ctx, dh: torch.Tensor):
        x2, w13, gate_up = ctx.saved_tensors
        M, FF = gate_up.shape[0], gate_up.shape[1] // 2
        d2 = _rows(dh)
        dgu = torch.empty_like(gate_up)
        _launch("pb_swiglu_bwd", _ptr(gate_up), _ptr(d2), _ptr(dgu), M, FF, _stream())
        dx = dw = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty(ctx.x_shape, dtype=dh.dtype, device=dh.device)
            _matmul(dgu, w13, dx.view(-1, ctx.x_shape[-1]), b_mn_major=True)
        if ctx.needs_input_grad[1]:
            dw = _wgrad(dgu, x2, w13)
        return dx, dw


class _MLPSwiGLUFn(torch.autograd.Function):
    """y = (silu(x W1ᵀ)·(x W3ᵀ)) W2ᵀ as ONE autograd node so that the backward can fuse across the two projections:
    the down-projection's input-gradient GEMM (dh = dy·W2) applies the SwiGLU derivative in its epilogue and writes d_gate_up
    directly (the SwiGLU-backward epilogue of ``pb_gemm_bf16``) — dh is never stored or re-read and the stand-alone swiglu_bwd
    pass is gone.
    Forward: gate/up GEMM with the SwiGLU epilogue, then the down projection. Saves exactly what the two separate nodes saved."""

    @staticmethod
    def forward(ctx, x: torch.Tensor, w13: torch.Tensor, w2: torch.Tensor) -> torch.Tensor:
        x2 = _rows(x)
        M = x2.shape[0]
        FF = w13.shape[0] // 2
        gate_up = torch.empty((M, 2 * FF), dtype=x.dtype, device=x.device)
        h = torch.empty((M, FF), dtype=x.dtype, device=x.device)
        _matmul(x2, w13, gate_up, swiglu_h=h)
        y = torch.empty((*x.shape[:-1], w2.shape[0]), dtype=x.dtype, device=x.device)
        _matmul(h, w2, y.view(M, -1))
        ctx.save_for_backward(x2, w13, w2, gate_up, h)
        ctx.x_shape = x.shape
        return y

    @staticmethod
    def backward(ctx, dy: torch.Tensor):
        x2, w13, w2, gate_up, h = ctx.saved_tensors
        dy2 = _rows(dy)
        dw2 = _wgrad(dy2, h, w2) if ctx.needs_input_grad[2] else None
        dgu = torch.empty_like(gate_up)
        _matmul(dy2, w2, dgu, b_mn_major=True, swiglu_bwd_gu=gate_up)
        dx = dw13 = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty(ctx.x_shape, dtype=dy.dtype, device=dy.device)
            _matmul(dgu, w13, dx.view(-1, ctx.x_shape[-1]), b_mn_major=True)
        if ctx.needs_input_grad[1]:
            dw13 = _wgrad(dgu, x2, w13)
        return dx, dw13, dw2


def mlp_swiglu(x: torch.Tensor, w13: torch.Tensor, w2: torch.Tensor) -> torch.Tensor:
    """SwiGLU MLP ``linear(swiglu(linear(x, w13)), w2)``; on CUDA one autograd node with the SwiGLU forward AND backward fused into
    GEMM epilogues (M > 128, hidden % 64 == 0), otherwise the composition of the separate ops. With e4m3 weights (:class:`MXWeight`,
    forward only) the composition, whose gate/up GEMM carries the SwiGLU epilogue wherever the bf16 path's does."""
    if isinstance(w13, MXWeight) or isinstance(w2, MXWeight):
        return linear(linear_swiglu(x, w13), w2)
    if (not _NO_EPILOGUE_FUSION and x.is_cuda and x.dtype == torch.bfloat16 and (w13.shape[0] // 2) % 64 == 0
            and x.numel() // x.shape[-1] > 128 and w2.stride(1) == 1 and w13.stride(1) == 1):  # fmt: skip
        return _MLPSwiGLUFn.apply(x, w13, w2)
    return linear(linear_swiglu(x, w13), w2)


def linear_swiglu(x: torch.Tensor, w13: torch.Tensor) -> torch.Tensor:
    """``swiglu(linear(x, w13))``; fused into one GEMM on CUDA when the shape allows it (M > 128, FF % 64 == 0)."""
    if isinstance(w13, MXWeight) and x.is_cuda and not _NO_EPILOGUE_FUSION:
        _mx_no_grad(x)
        x2 = _rows(x)
        M, FF = x2.shape[0], w13.shape[0] // 2
        h = torch.empty((*x.shape[:-1], FF), dtype=x.dtype, device=x.device)
        _matmul(x2, w13, torch.empty((M, 2 * FF), dtype=x.dtype, device=x.device), swiglu_h=h.view(M, FF))
        return h
    if not _NO_EPILOGUE_FUSION and x.is_cuda and x.dtype == torch.bfloat16 and (w13.shape[0] // 2) % 64 == 0 and x.numel() // x.shape[-1] > 128:
        return _LinearSwiGLUFn.apply(x, w13)
    return swiglu(linear(x, w13))


# --------------------------------------------------------------------------- cross entropy


class _CrossEntropyFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, targets, ignore_index, grad_scale, unit_upstream, loss_acc):
        V = logits.shape[-1]
        z = logits.reshape(-1, V)
        assert z.is_contiguous()
        t = targets.reshape(-1)
        t = t if t.is_contiguous() else t.contiguous()
        R = z.shape[0]
        work = torch.empty(R + 4, dtype=torch.float32, device=z.device)  # [0:2] scales, [2] loss, [4:] per-row losses
        # valid-target count → gradient scale, the fused row kernel (logits are overwritten with d(mean loss)/d(logits): nothing else
        # needs them afterwards) and a fixed-order sum of the row losses — three native launches, no framework kernel
        _launch("pb_cross_entropy_loss", _ptr(z), _ptr(t), work[4:].data_ptr(), work.data_ptr(), work[2:].data_ptr(), _ptr(loss_acc), R, V,
                ignore_index, float(grad_scale), _stream(), n=3)  # fmt: skip
        # NOTE: deliberately not mark_dirty(): the logits are consumed, not returned; their storage now holds the gradient
        ctx.save_for_backward(z)
        ctx.shape = logits.shape
        ctx.unit_upstream = unit_upstream
        return work[2].reshape(())

    @staticmethod
    def backward(ctx, dloss):
        (dz,) = ctx.saved_tensors
        # dz already holds the gradient for dloss == 1; rescale for loss scaling / grad accumulation
        if not ctx.unit_upstream:
            dz = dz * dloss.to(dz.dtype)
        return dz.view(ctx.shape), None, None, None, None, None


def cross_entropy(
    logits: torch.Tensor,
    targets: torch.Tensor,
    ignore_index: int = -100,
    *,
    grad_scale: float = 1.0,
    unit_upstream: bool = False,
    loss_acc: torch.Tensor | None = None,
) -> torch.Tensor:
    """Mean token cross-entropy.  On CUDA the logits buffer is consumed (overwritten with its gradient).

    ``grad_scale`` folds a gradient multiplier (e.g. 1/grad-accumulation-steps) into the fused kernel; the
    returned loss value is NOT scaled.  ``unit_upstream=True`` promises the loss is back-propagated with a
    unit upstream gradient, which removes one full pass over the logits gradient.  ``loss_acc``: optional fp32 scalar the
    (unscaled) loss is also added to, inside the finalising kernel — the trainer's per-step running sum.
    """
    if logits.is_cuda:
        return _CrossEntropyFn.apply(logits, targets, ignore_index, float(grad_scale), bool(unit_upstream), loss_acc)
    loss = reference.cross_entropy(logits, targets, ignore_index)
    if loss_acc is not None:
        loss_acc += loss.detach().float()
    if grad_scale != 1.0:
        # same contract on CPU: value unscaled, gradient scaled
        loss = loss.detach() + (loss - loss.detach()) * grad_scale
    return loss


# --------------------------------------------------------------------------- attention


def document_bounds(tokens: torch.Tensor, eos_id: int | None, window: int | None = None) -> tuple[torch.Tensor, torch.Tensor]:
    """Documents of packed token rows [B, S] → (doc_start, doc_end), int32 [B, S] each: the ``doc`` argument of the attention ops.
    Position s starts a document when s == 0 or tokens[b, s-1] == eos_id (None = no documents). ``window`` W (None = none): query q
    also sees only the W most recent keys, itself included, so q attends k iff max(doc_start, q - W + 1) <= k <= q (see
    :func:`reference.document_bounds`). One native kernel on CUDA; it reads only ``tokens``, so it can be captured in a CUDA graph
    over a static token buffer."""
    if window is not None and window < 1:
        raise ValueError(f"window must be >= 1 (or None for no window), got {window}")
    if tokens.is_cuda:
        from . import attention_native as native

        return native.document_bounds(tokens, eos_id, window)
    return reference.document_bounds(tokens, eos_id, window)


def attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, causal: bool = True, doc: tuple | None = None) -> torch.Tensor:
    """Unfused-layout attention, q [B,S,H,D], k/v [B,S,Hkv,D] → [B,S,H,D].  SDPA on CUDA (not a hot path: the models
    call :func:`attention_qkv`), torch reference on CPU. ``doc=(doc_start, doc_end)`` (:func:`document_bounds`): query q attends
    key k iff doc_start[b, q] <= k <= q; on CUDA this builds a boolean [B, 1, S, S] mask (O(S²) memory)."""
    if doc is not None and not causal:
        raise ValueError("document masking implies causal attention: causal=False with doc=(doc_start, doc_end) is not supported")
    if not q.is_cuda:
        return reference.attention(q, k, v, causal, doc_start=None if doc is None else doc[0])
    import torch.nn.functional as F

    H, Hkv = q.shape[2], k.shape[2]
    if doc is not None:
        out = F.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2),
                                             attn_mask=reference.document_mask(doc[0]).unsqueeze(1), enable_gqa=(H != Hkv))  # fmt: skip
        return out.transpose(1, 2)
    out = F.scaled_dot_product_attention(
        q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), is_causal=causal, enable_gqa=(H != Hkv)
    )
    return out.transpose(1, 2)


def attention_qkv(qkv: torch.Tensor, n_heads: int, n_kv_heads: int, causal: bool = True, impl: str = "auto",
                  doc: tuple | None = None) -> torch.Tensor:  # fmt: skip
    """Attention over the fused, RoPE-rotated QKV activation [B,S,(H+2Hkv)·D] → [B,S,H·D].

    ``impl``: "native" = the project's flash-attention kernels (error if the shape is unsupported); "sdpa" = library
    fallback; "auto" = native whenever supported. ``doc=(doc_start, doc_end)`` (:func:`document_bounds`): document masking.
    """
    B, S, W = qkv.shape
    D = W // (n_heads + 2 * n_kv_heads)
    if qkv.is_cuda and impl in ("auto", "native"):
        from . import attention_native as native

        if native.supported(qkv, n_heads, n_kv_heads):
            return native.flash_attention_qkv(qkv, n_heads, n_kv_heads, causal, doc)
        if impl == "native":
            raise RuntimeError(f"native flash attention does not support S={S}, D={D}, H={n_heads}, Hkv={n_kv_heads}")
    x = qkv.view(B, S, n_heads + 2 * n_kv_heads, D)
    q, k, v = x[:, :, :n_heads], x[:, :, n_heads : n_heads + n_kv_heads], x[:, :, n_heads + n_kv_heads :]
    return attention(q, k, v, causal, doc).reshape(B, S, n_heads * D)


def rope_attention_qkv(qkv: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, n_heads: int, n_kv_heads: int, causal: bool = True,
                       impl: str = "auto", pre_rotated: bool = False, doc: tuple | None = None) -> torch.Tensor:  # fmt: skip
    """RoPE on the Q/K heads of the fused QKV activation followed by attention → [B,S,H·D]. On the native path both run as one
    autograd node whose backward folds the inverse rotation into the dQ/dK epilogues. ``pre_rotated=True``: the producer
    (:func:`linear_qkv_rope`) already rotated in its GEMM epilogue; only the backward un-rotation is needed (native path only).
    ``doc=(doc_start, doc_end)``: document masking (see :func:`attention`); RoPE positions stay absolute."""
    if qkv.is_cuda and impl in ("auto", "native"):
        from . import attention_native as native

        if native.supported(qkv, n_heads, n_kv_heads):
            return native.rope_flash_attention_qkv(qkv, cos, sin, n_heads, n_kv_heads, causal, pre_rotated, doc)
    if pre_rotated:
        raise RuntimeError("pre_rotated=True needs the native attention path (its backward undoes the rotation)")
    return attention_qkv(rope_qkv(qkv, cos, sin, n_heads, n_kv_heads), n_heads, n_kv_heads, causal, impl, doc)


# --------------------------------------------------------------------------- KV-cache decoding


def _decode_native(qkv: torch.Tensor, kv: torch.Tensor, n_heads: int, n_kv_heads: int, kv_scale: torch.Tensor | None = None) -> bool:
    """Shapes and layouts the decode kernels (csrc/decode_sm90.cu) take: bf16, contiguous, D in {64, 128}, H % Hkv == 0; the cache
    bf16, or e4m3 (uint8) with its uint8 exponents (see :func:`kv_append`)."""
    if (kv.dtype == torch.uint8) != (kv_scale is not None):
        raise ValueError(f"an e4m3 cache is uint8 with a kv_scale tensor, a bf16 cache has none; got {kv.dtype} with kv_scale "
                         f"{'given' if kv_scale is not None else 'None'}")  # fmt: skip
    D = qkv.shape[-1] // (n_heads + 2 * n_kv_heads)
    cache = kv.dtype == torch.bfloat16 if kv_scale is None else kv_scale.dtype == torch.uint8 and kv_scale.is_contiguous()
    return (qkv.is_cuda and qkv.dtype == torch.bfloat16 and cache and qkv.is_contiguous() and kv.is_contiguous() and D in (64, 128)
            and n_heads % n_kv_heads == 0)  # fmt: skip


def _put_rows(kv: torch.Tensor, kv_scale: torch.Tensor | None, idx: torch.Tensor, ok: torch.Tensor, new: torch.Tensor) -> None:
    """Cache rows ``new`` [B, cols] into the flat rows ``idx`` of the cache where ``ok``, with no host synchronisation (no nonzero /
    item: on CUDA the fallbacks are captured in the decode step's graph as well). An e4m3 cache receives ``quantize_kv(new)``."""
    for dst, val in [(kv, new)] if kv_scale is None else zip((kv, kv_scale), reference.quantize_kv(new)):
        flat = dst.view(-1, dst.shape[-1])
        flat.index_copy_(0, idx, torch.where(ok.view(-1, 1), val, flat.index_select(0, idx)))


def _cache_values(kv: torch.Tensor, kv_scale: torch.Tensor | None) -> torch.Tensor:
    """The cache as the fallback attention reads it: the bf16 cache, or the e4m3 cache dequantised (exact, fp32)."""
    return kv if kv_scale is None else reference.dequantize_kv(kv, kv_scale)


def decode_attn_splits(batch: int, n_kv_heads: int, capacity: int) -> int:
    """The native split policy of :func:`decode_attention`: a function of the cache geometry only (never of the lengths), so one
    captured decode step stays valid at every position."""
    n = int(_lib.load().pb_decode_attn_splits(batch, n_kv_heads, capacity))
    _lib.check(min(n, 0), "pb_decode_attn_splits")
    return n


def decode_advance(tokens: torch.Tensor, length: torch.Tensor, lo: torch.Tensor, last_tok: torch.Tensor, eos_id: int | None) -> None:
    """Per-row bookkeeping at the start of a decode step, in place: pos = len; lo = pos if last_tok == eos_id; len = pos + 1;
    last_tok = tokens. ``tokens`` / ``last_tok`` int64 [B], ``length`` / ``lo`` int32 [B]; ``eos_id`` None = no documents."""
    if tokens.is_cuda:
        assert tokens.dtype == last_tok.dtype == torch.int64 and length.dtype == lo.dtype == torch.int32
        assert tokens.is_contiguous() and length.is_contiguous() and lo.is_contiguous() and last_tok.is_contiguous()
        _launch("pb_decode_advance", tokens.data_ptr(), -1 if eos_id is None else int(eos_id), length.data_ptr(), lo.data_ptr(),
                last_tok.data_ptr(), tokens.shape[0], _stream())  # fmt: skip
        return
    if eos_id is not None:
        lo.copy_(torch.where(last_tok == eos_id, length, lo))
    length.add_(1)
    last_tok.copy_(tokens)


def kv_append(qkv: torch.Tensor, kv: torch.Tensor, length: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, n_heads: int,
              n_kv_heads: int, kv_scale: torch.Tensor | None = None) -> torch.Tensor:  # fmt: skip
    """The new token of every row, un-rotated fused QKV [B, (H+2Hkv)·D], at position len[b] - 1: rotates its Q heads in place and
    writes its rotated K heads and its V heads into row len[b] - 1 of the layer's cache ``kv`` [B, capacity, 2·Hkv·D]. Rows whose
    position is outside the cache are left alone. Returns ``qkv``.

    The e4m3 cache (``kv`` uint8 with ``kv_scale``; CUDA: ``pb_kv_append_fp8``) has the same layout in bytes, and ``kv_scale`` uint8
    [B, capacity, 2·Hkv·D/32] holds one biased UE8M0 exponent e per 32 columns of a row (columns 32j .. 32j+31 → byte j; D % 32 ==
    0, so a block never straddles two heads): the value is e4m3 · 2^(e-127). The rule is MXFP8's (``reference.quantize_mxfp8``,
    csrc/mx_common.cuh): the smallest power of two s with amax / s <= 448, e clamped to [1, 254], then x / s rounded to nearest even
    with saturation. Its input is the value the bf16 cache would hold, the rotated K after its one bf16 rounding and V as is, so the
    e4m3 cache is ``reference.quantize_kv`` of the bf16 cache byte for byte, and every dequantised value is exact in fp32 and bf16.
    Queries stay bf16; rows past ``len`` are never read."""
    B = qkv.shape[0]
    H, Hkv = n_heads, n_kv_heads
    D = qkv.shape[-1] // (H + 2 * Hkv)
    cap = kv.shape[1]
    if _decode_native(qkv, kv, H, Hkv, kv_scale):
        assert length.dtype == torch.int32 and cos.dtype == torch.float32 and cos.is_contiguous() and sin.is_contiguous()
        assert cos.shape[0] >= cap and cos.shape[1] == D // 2
        if kv_scale is not None:
            _launch("pb_kv_append_fp8", qkv.data_ptr(), kv.data_ptr(), kv_scale.data_ptr(), length.data_ptr(), cos.data_ptr(),
                    sin.data_ptr(), B, 1, H, Hkv, D, cap, _stream())  # fmt: skip
            return qkv
        _launch("pb_kv_append", qkv.data_ptr(), kv.data_ptr(), length.data_ptr(), cos.data_ptr(), sin.data_ptr(), B, H, Hkv, D, cap,
                _stream())  # fmt: skip
        return qkv
    pos = length.long() - 1
    ok = (pos >= 0) & (pos < cap)
    p = pos.clamp(0, cap - 1)
    x = qkv.view(B, H + 2 * Hkv, D)
    rot = reference.rope_at(x[:, : H + Hkv], cos[p], sin[p])
    idx = torch.arange(B, device=kv.device) * cap + p
    new = torch.cat((rot[:, H:], x[:, H + Hkv :]), dim=1).reshape(B, -1)
    _put_rows(kv, kv_scale, idx, ok, new)
    x[:, :H] = torch.where(ok.view(B, 1, 1), rot[:, :H], x[:, :H])
    return qkv


def kv_quantize(src: torch.Tensor, kv: torch.Tensor, kv_scale: torch.Tensor) -> None:
    """Prefill of an e4m3 cache: the rows ``src`` [B, S, cols] (the rotated K|V columns of the fused QKV activation, a strided view
    with unit column stride) quantised into rows 0 .. S-1 of ``kv`` uint8 [B, capacity, cols] and ``kv_scale`` uint8 [B, capacity,
    cols / 32] by the rule of :func:`kv_append`. On CUDA the native ``pb_kv_quantize`` reads the strided bf16 rows once, with no
    temporaries."""
    B, S, cols = src.shape
    if src.is_cuda:
        assert src.dtype == torch.bfloat16 and kv.dtype == kv_scale.dtype == torch.uint8 and kv.is_contiguous() and kv_scale.is_contiguous()
        assert src.stride(2) == 1 and src.stride(0) == S * src.stride(1) and kv.shape[-1] == cols and kv_scale.shape[-1] == cols // 32
        _launch("pb_kv_quantize", src.data_ptr(), src.stride(1), kv.data_ptr(), kv_scale.data_ptr(), B, S, cols, kv.shape[1], _stream())
        return
    q, e = reference.quantize_kv(src)
    kv[:, :S].copy_(q)
    kv_scale[:, :S].copy_(e)


def decode_attention(qkv: torch.Tensor, kv: torch.Tensor, length: torch.Tensor, lo: torch.Tensor | None, window: int | None,
                     n_heads: int, n_kv_heads: int, splits: int | None = None, kv_scale: torch.Tensor | None = None) -> torch.Tensor:  # fmt: skip
    """Attention of the one (rotated) query per row in ``qkv`` [B, (H+2Hkv)·D] over the layer's cache ``kv`` [B, capacity, 2·Hkv·D]
    → [B, H·D]. Row b sees keys max(lo[b], len[b] - window) <= k < len[b] (``lo`` None = 0, ``window`` None = none). On CUDA the
    split-KV kernel (one launch, or two with the combine when ``splits`` > 1; None = :func:`decode_attn_splits`), else the fp32
    :func:`reference.decode_attention`. ``kv_scale``: the cache is e4m3 (:func:`kv_append`); the kernel computes the bf16 kernel's
    sums over the dequantised cache, and the fallback dequantises it."""
    B = qkv.shape[0]
    H, Hkv = n_heads, n_kv_heads
    D = qkv.shape[-1] // (H + 2 * Hkv)
    cap = kv.shape[1]
    if _decode_native(qkv, kv, H, Hkv, kv_scale):
        assert length.dtype == torch.int32 and (lo is None or lo.dtype == torch.int32)
        if splits is None:
            splits = decode_attn_splits(B, Hkv, cap)
        out = torch.empty((B, H * D), dtype=qkv.dtype, device=qkv.device)
        part = torch.empty((B, H, splits, D + 2), dtype=torch.float32, device=qkv.device) if splits > 1 else None
        fp8 = () if kv_scale is None else (kv_scale.data_ptr(),)
        _launch("pb_decode_attn" if kv_scale is None else "pb_decode_attn_fp8", qkv.data_ptr(), kv.data_ptr(), *fp8, length.data_ptr(),
                _ptr(lo), int(window or 0), out.data_ptr(), _ptr(part), B, H, Hkv, D, cap, splits, 1.0 / math.sqrt(D), _stream(),
                n=1 if splits == 1 else 2)  # fmt: skip
        return out
    q = qkv.view(B, H + 2 * Hkv, D)[:, :H]
    return reference.decode_attention(q, _cache_values(kv, kv_scale), length, lo, window).reshape(B, H * D).to(qkv.dtype)


# --------------------------------------------------------------------------- sampling


def _sample_args(temperature: float, top_k: int, top_p: float, min_p: float) -> None:
    if not (math.isfinite(temperature) and temperature >= 0):
        raise ValueError(f"temperature must be finite and >= 0, got {temperature}")
    if top_k < 0:
        raise ValueError(f"top_k must be >= 0 (0 = off), got {top_k}")
    if not 0 < top_p <= 1:
        raise ValueError(f"top_p must be in (0, 1] (1 = off), got {top_p}")
    if not 0 <= min_p <= 1:
        raise ValueError(f"min_p must be in [0, 1] (0 = off), got {min_p}")


def sample_tokens(logits: torch.Tensor, *, temperature: float = 0.0, top_k: int = 0, top_p: float = 1.0, min_p: float = 0.0,
                  seeds: torch.Tensor, positions: torch.Tensor, out: torch.Tensor | None = None, state=None) -> torch.Tensor:  # fmt: skip
    """One token per row of ``logits`` [B, V] → int64 [B] (``out`` if given).

    The contract, shared by the native kernel (csrc/sample_sm90.cu: CUDA bf16 logits with unit column stride) and
    :func:`reference.sample_tokens` (everything else; no host synchronisation, so a CUDA graph can capture it too):

    * Greedy: ``temperature == 0`` returns the argmax, the lowest index among tied maxima (``torch.argmax``); the other knobs are
      ignored.
    * Otherwise ``p_i ∝ exp((l_i − l_max) / T)``, and the filters apply in Hugging Face order, temperature → top-k → top-p → min-p.
      Each keeps an upper set of the logit order, tie groups (equal logits) whole, so the keep-set is ``{i : l_i >= t*}``:

      - top-k (``k > 0``): every token whose logit is at least the k-th largest (ties may keep more than k; ``k >= V`` keeps all).
      - top-p (``0 < p <= 1``, 1 = off): on the top-k set S, the largest threshold t with ``mass{i ∈ S : p_i >= t} >= p·mass(S)``;
        keeps ``S ∩ {p_i >= t}``, so the tie group that crosses p stays whole.
      - min-p (``0 <= m <= 1``, 0 = off): keeps ``p_i >= m·p_max``, i.e. ``l_i >= l_max + T·ln m``.
    * Draw: the inverse CDF in vocabulary index order over the kept set. With ``target = u·mass(kept)`` the token is the first kept
      index whose inclusive prefix mass exceeds ``target``, or, should rounding leave none, the last kept index.
    * Random stream: Philox4x32-10 with key = the row's 64-bit seed (``seeds`` int64 [B]: lo, hi words) and counter =
      ``(position, 0, 0, 0)`` (``positions`` int32 [B]: the index in its row of the token being drawn), so a draw depends on nothing
      but (seed, row position); ``u = ((x0 >> 8) + 0.5)·2^-24``.

    Both implementations compute ``p_i`` in fp64 (``exp((l_i − l_max)·(1/T))`` with T the fp32 value, ``p_max = 1``), round it to
    a 2^-40 fixed-point integer and sum masses in integers, so every sum (the top-p mass, the prefix of the draw) is exact in any
    order and the kernel is deterministic; ``p·mass(S)`` is compared in fp64 and the min-p bound is ``l_max + fp32(T·ln m)`` in fp32.
    They can differ only where two fp64 ``exp`` results round to different fixed-point integers.

    ``state``: bookkeeping of a generation loop (``inference.SampleState``). An inactive row (``state.active[b]`` false) writes
    nothing, so ``out`` keeps its last token; an active row writes its token to ``out`` and ``state.history[b, state.n_out[b]]``,
    increments ``n_out`` and goes inactive at ``history.shape[1]`` new tokens, at ``prompt_len + n_out == max_seq_len``, or after
    ``eos_id`` (kept in the output)."""
    if logits.dim() != 2:
        raise ValueError(f"logits must be [B, V], got {tuple(logits.shape)}")
    _sample_args(temperature, top_k, top_p, min_p)
    B, V = logits.shape
    if out is None:
        out = torch.empty(B, dtype=torch.int64, device=logits.device)
    if logits.is_cuda and logits.dtype == torch.bfloat16 and logits.stride(1) == 1:
        assert seeds.dtype == out.dtype == torch.int64 and positions.dtype == torch.int32
        assert seeds.is_contiguous() and positions.is_contiguous() and out.is_contiguous()
        book = [None] * 4
        max_new = max_seq = 0
        eos = -1
        if state is not None:
            assert state.history.dtype == torch.int64 and state.n_out.dtype == torch.int32 and state.active.dtype == torch.bool
            assert state.prompt_len.dtype == torch.int32 and state.history.is_contiguous()
            book = [state.history.data_ptr(), state.n_out.data_ptr(), state.active.data_ptr(), state.prompt_len.data_ptr()]
            max_new, max_seq = state.history.shape[1], state.max_seq_len
            eos = -1 if state.eos_id is None else int(state.eos_id)
        _launch("pb_sample_tokens", logits.data_ptr(), logits.stride(0) if B > 1 else V, B, V, float(temperature), int(top_k),
                float(top_p), float(min_p), seeds.data_ptr(), positions.data_ptr(), out.data_ptr(), *book, max_new, max_seq, eos,
                _stream())  # fmt: skip
        return out
    tok = reference.sample_tokens(logits, temperature, top_k, top_p, min_p, seeds, positions)
    if state is None:
        out.copy_(tok)
    else:
        reference.sample_bookkeeping(tok, out, state.history, state.n_out, state.active, state.prompt_len, state.max_seq_len,
                                     state.eos_id)  # fmt: skip
    return out


# --------------------------------------------------------------------------- speculative decoding


def verify_advance(tokens: torch.Tensor, length: torch.Tensor, lo: torch.Tensor, last_tok: torch.Tensor, eos_id: int | None) -> torch.Tensor:
    """:func:`decode_advance` for T tokens per row (``tokens`` int64 [B, T]), in place: the rule applied to the tokens in order, so
    the state afterwards is that of T decode steps. Returns each query's document start ``lo_q`` int32 [B, T]: an EOS among the
    tokens starts a new document for the queries after it."""
    B, T = tokens.shape
    lo_q = torch.empty((B, T), dtype=torch.int32, device=tokens.device)
    if tokens.is_cuda:
        assert tokens.dtype == last_tok.dtype == torch.int64 and length.dtype == lo.dtype == torch.int32
        assert tokens.is_contiguous() and length.is_contiguous() and lo.is_contiguous() and last_tok.is_contiguous()
        _launch("pb_verify_advance", tokens.data_ptr(), T, -1 if eos_id is None else int(eos_id), length.data_ptr(), lo.data_ptr(),
                lo_q.data_ptr(), last_tok.data_ptr(), B, _stream())  # fmt: skip
        return lo_q
    for t in range(T):
        if eos_id is not None:
            lo.copy_(torch.where(last_tok == eos_id, length + t, lo))
        lo_q[:, t] = lo
        last_tok.copy_(tokens[:, t])
    length.add_(T)
    return lo_q


def kv_append_tokens(qkv: torch.Tensor, kv: torch.Tensor, length: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, n_heads: int,
                     n_kv_heads: int, kv_scale: torch.Tensor | None = None) -> torch.Tensor:  # fmt: skip
    """:func:`kv_append` for T tokens per row: ``qkv`` [B, T, (H+2Hkv)·D], token t of row b at position len[b] - T + t. Positions
    outside the cache are left alone. Returns ``qkv``. ``kv_scale``: the cache is e4m3."""
    B, T = qkv.shape[:2]
    H, Hkv = n_heads, n_kv_heads
    D = qkv.shape[-1] // (H + 2 * Hkv)
    cap = kv.shape[1]
    if _decode_native(qkv, kv, H, Hkv, kv_scale):
        assert length.dtype == torch.int32 and cos.dtype == torch.float32 and cos.is_contiguous() and sin.is_contiguous()
        assert cos.shape[0] >= cap and cos.shape[1] == D // 2
        if kv_scale is not None:
            _launch("pb_kv_append_fp8", qkv.data_ptr(), kv.data_ptr(), kv_scale.data_ptr(), length.data_ptr(), cos.data_ptr(),
                    sin.data_ptr(), B, T, H, Hkv, D, cap, _stream())  # fmt: skip
            return qkv
        _launch("pb_kv_append_tokens", qkv.data_ptr(), kv.data_ptr(), length.data_ptr(), cos.data_ptr(), sin.data_ptr(), B, T, H, Hkv,
                D, cap, _stream())  # fmt: skip
        return qkv
    for t in range(T):  # token t is the one a decode step would append with len = len - T + t + 1
        kv_append(qkv[:, t], kv, length - (T - 1 - t), cos, sin, H, Hkv, kv_scale)
    return qkv


def verify_attention(qkv: torch.Tensor, kv: torch.Tensor, length: torch.Tensor, lo_q: torch.Tensor | None, window: int | None,
                     n_heads: int, n_kv_heads: int, splits: int | None = None, kv_scale: torch.Tensor | None = None) -> torch.Tensor:  # fmt: skip
    """Attention of T (rotated) queries per row, ``qkv`` [B, T, (H+2Hkv)·D], over the layer's cache → [B, T, H·D]. Query t of row b
    sits at position pos = len[b] - T + t and sees keys max(lo_q[b, t], pos + 1 - window) <= k <= pos. On CUDA the split-KV verify
    kernel with the split policy of :func:`decode_attn_splits` (at T = 1 bitwise equal to :func:`decode_attention`), else the fp32
    :func:`reference.verify_attention`. ``kv_scale``: the cache is e4m3, as in :func:`decode_attention`."""
    B, T = qkv.shape[:2]
    H, Hkv = n_heads, n_kv_heads
    D = qkv.shape[-1] // (H + 2 * Hkv)
    cap = kv.shape[1]
    if _decode_native(qkv, kv, H, Hkv, kv_scale):
        assert length.dtype == torch.int32 and (lo_q is None or (lo_q.dtype == torch.int32 and lo_q.is_contiguous()))
        if splits is None:
            splits = decode_attn_splits(B, Hkv, cap)
        out = torch.empty((B, T, H * D), dtype=qkv.dtype, device=qkv.device)
        part = torch.empty((B, T, H, splits, D + 2), dtype=torch.float32, device=qkv.device) if splits > 1 else None
        fp8 = () if kv_scale is None else (kv_scale.data_ptr(),)
        _launch("pb_verify_attn" if kv_scale is None else "pb_verify_attn_fp8", qkv.data_ptr(), kv.data_ptr(), *fp8, length.data_ptr(),
                _ptr(lo_q), int(window or 0), out.data_ptr(), _ptr(part), B, T, H, Hkv, D, cap, splits, 1.0 / math.sqrt(D), _stream(),
                n=1 if splits == 1 else 2)  # fmt: skip
        return out
    q = qkv.view(B, T, H + 2 * Hkv, D)[:, :, :H]
    return reference.verify_attention(q, _cache_values(kv, kv_scale), length, lo_q, window).reshape(B, T, H * D).to(qkv.dtype)


def spec_accept(target_logits: torch.Tensor, draft_logits: torch.Tensor, *, temperature: float = 0.0, top_k: int = 0, top_p: float = 1.0,
                min_p: float = 0.0, seeds: torch.Tensor, tokens: torch.Tensor, lo_q: torch.Tensor, target, draft, state,
                pending: torch.Tensor, drafted: torch.Tensor, accepted: torch.Tensor) -> None:  # fmt: skip
    """The accept step of one speculative round per row, in place (``inference.generate_speculative`` states the round in full).

    ``target_logits`` [B, k+1, V]: the verify step's logits p_1 .. p_{k+1}; ``draft_logits`` [k, B, V]: q_1 .. q_k; ``tokens`` int64
    [B, k+1]: the pending token x at index L, then the drafts d_1 .. d_k; ``lo_q``: :func:`verify_advance`'s; ``target`` / ``draft``:
    the two ``inference.KVCache`` (the target's len = L + k + 1); ``state``: an ``inference.SampleState``.

    * P_i / Q_i: the keep-set, temperature and fixed-point masses of :func:`sample_tokens` applied to p_i / q_i, normalised to 2^-40
      fixed point by one correctly rounded fp64 division per token, ``round(mass_j·2^40 / fp64(mass(kept)))``.
    * For i = 1 .. k: r = the top 24 bits of Philox word x0 at counter (L + i, 1, 0, 0); d_i is accepted iff
      ``(2r + 1)·Q_i[d_i] < 2^25·P_i[d_i]`` in exact integers. At the first rejection y is drawn from ``max(0, P_i − Q_i)`` (from P_i
      should that be all zero) by the inverse CDF of :func:`sample_tokens` in index order, with counter (L + i, 2, 0, 0); after k
      acceptances y is drawn from P_{k+1} with counter (L + k + 1, 2, 0, 0). Greedy (``temperature == 0``): d_i is accepted iff it
      is the argmax of p_i (lowest index among ties), and y is the argmax of the first p_i that rejects, or of p_{k+1}.
    * An active row emits d_1 .. d_n, y into the history through the stop rules of ``sample_tokens(state=...)``, adds k to
      ``drafted`` and n to ``accepted``, sets both caches to len = L + n + 1, lo = lo_q[b, n], last_tok = tokens[b, n], and writes y
      to ``pending``. An inactive row writes nothing.

    CUDA bf16 logits run the native kernel (csrc/sample_sm90.cu); everything else :func:`reference.spec_accept`, which reads values
    back to the host and so cannot be captured."""
    _sample_args(temperature, top_k, top_p, min_p)
    B, T, V = target_logits.shape
    k = T - 1
    if not 1 <= k <= 15:
        raise ValueError(f"k must be in [1, 15], got {k}")
    if tuple(draft_logits.shape) != (k, B, V) or tuple(tokens.shape) != (B, T):
        raise ValueError(f"draft logits {tuple(draft_logits.shape)} / tokens {tuple(tokens.shape)} do not match target [B={B}, k+1={T}, V]")
    eos = -1 if state.eos_id is None else int(state.eos_id)
    if target_logits.is_cuda and target_logits.dtype == draft_logits.dtype == torch.bfloat16:
        tl, dl = target_logits.reshape(B * T, V), draft_logits.reshape(k * B, V)
        assert tl.stride(1) == 1 and dl.stride(1) == 1 and state.active.dtype == torch.bool
        _launch("pb_spec_accept", tl.data_ptr(), tl.stride(0), dl.data_ptr(), dl.stride(0), B, k, V, float(temperature), int(top_k),
                float(top_p), float(min_p), seeds.data_ptr(), tokens.data_ptr(), lo_q.data_ptr(), target.len.data_ptr(),
                target.lo.data_ptr(), target.last_tok.data_ptr(), draft.len.data_ptr(), draft.lo.data_ptr(), draft.last_tok.data_ptr(),
                pending.data_ptr(), state.history.data_ptr(), state.n_out.data_ptr(), state.active.data_ptr(),
                state.prompt_len.data_ptr(), state.history.shape[1], state.max_seq_len, eos, drafted.data_ptr(), accepted.data_ptr(),
                _stream())  # fmt: skip
        return
    reference.spec_accept(target_logits, draft_logits, temperature, top_k, top_p, min_p, seeds, tokens, lo_q, target, draft, state,
                          pending, drafted, accepted)  # fmt: skip
