"""Build and load the native sm_90a kernel library (C ABI, ctypes).

The library is compiled in-tree (``prime_b200/_C/libprime_b200.so``) straight from
``prime_b200/csrc/*.cu`` with ``nvcc -gencode arch=compute_90a,code=sm_90a`` — no torch
headers, so a full rebuild takes seconds.  On a CUDA device every op in :mod:`prime_b200.ops.functional` requires this
library and raises if it is missing: there is no silent eager fallback on the GPU.
"""

from __future__ import annotations

import ctypes
import os
import shutil
import subprocess
import threading
from pathlib import Path

_ROOT = Path(__file__).resolve().parent.parent
CSRC = _ROOT / "csrc"
OUT_DIR = _ROOT / "_C"
LIB_PATH = OUT_DIR / "libprime_b200.so"
HASH_PATH = OUT_DIR / "build.hash"

NVCC_FLAGS = [
    "-gencode",
    "arch=compute_90a,code=sm_90a",
    "-lineinfo",
    "-O3",
    "-std=c++17",
    "-Xcompiler",
    "-fPIC",
    "-Xcompiler",
    "-fvisibility=hidden",
    "-shared",
]

_lock = threading.Lock()
_lib: ctypes.CDLL | None = None


def nvcc_path() -> str | None:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    return None


def sources() -> list[Path]:
    return sorted(CSRC.glob("*.cu"))


def source_hash() -> str:
    """Content hash of every kernel source + the flags (mtimes do not survive a copy of the tree)."""
    import hashlib

    h = hashlib.sha256(" ".join(NVCC_FLAGS).encode())
    for p in sorted(list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cuh"))):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    return h.hexdigest()


def needs_build() -> bool:
    if not LIB_PATH.exists() or not HASH_PATH.exists():
        return True
    return HASH_PATH.read_text().strip() != source_hash()


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile every ``.cu`` under ``csrc/`` into one shared library for sm_90a."""
    with _lock:
        if not force and not needs_build():
            return LIB_PATH
        nvcc = nvcc_path()
        if nvcc is None:
            raise RuntimeError("nvcc not found; cannot build prime_b200 native kernels")
        OUT_DIR.mkdir(parents=True, exist_ok=True)
        tmp = OUT_DIR / f".libprime_b200.{os.getpid()}.so"
        cmd = [nvcc, *NVCC_FLAGS, "-o", str(tmp), *[str(s) for s in sources()]]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        proc = subprocess.run(cmd, capture_output=True, text=True)
        if proc.returncode != 0:
            tmp.unlink(missing_ok=True)
            raise RuntimeError(f"nvcc failed ({proc.returncode}):\n{proc.stdout}\n{proc.stderr}")
        if verbose:
            print(proc.stderr)
        os.replace(tmp, LIB_PATH)  # atomic: concurrent ranks never see a half-written .so
        HASH_PATH.write_text(source_hash())
        return LIB_PATH


class PeerPtrs(ctypes.Structure):
    _fields_ = [("p", ctypes.c_void_p * 8), ("n", ctypes.c_int)]

    @classmethod
    def of(cls, ptrs) -> "PeerPtrs":
        s = cls()
        ptrs = list(ptrs)
        assert len(ptrs) <= 8, "at most 8 peers per NVSwitch box"
        for i, p in enumerate(ptrs):
            s.p[i] = int(p)
        s.n = len(ptrs)
        return s


class AdamArgs(ctypes.Structure):
    _fields_ = [(k, ctypes.c_float) for k in ("lr", "beta1", "beta2", "eps", "weight_decay", "bc1", "bc2", "max_norm")]


class SegTable(ctypes.Structure):
    """Up to 16 (src offset, dst offset, length) pieces that ``pb_grad_reduce`` (csrc/comm.cu) reduces: one for a flat bucket, one
    row block per parameter for a row-sharded one."""

    _fields_ = [("src_off", ctypes.c_int64 * 16), ("dst_off", ctypes.c_int64 * 16), ("n", ctypes.c_int64 * 16), ("nseg", ctypes.c_int)]

    @classmethod
    def of(cls, segs) -> "SegTable":
        segs = list(segs)
        assert len(segs) <= 16, "at most 16 row-sharded parameters per bucket"
        t = cls()
        for i, (src, dst, n) in enumerate(segs):
            t.src_off[i], t.dst_off[i], t.n[i] = int(src), int(dst), int(n)
        t.nseg = len(segs)
        return t


class OuterArgs(ctypes.Structure):
    _fields_ = [("lr", ctypes.c_float), ("momentum", ctypes.c_float), ("inv_workers", ctypes.c_float), ("nesterov", ctypes.c_int)]


class GemmEpilogue(ctypes.Structure):
    """Fused epilogue of ``pb_gemm_bf16`` / ``pb_gemm_wgather`` (csrc/gemm_sm90.cu). ``kind``: 0 plain, 1 RoPE, 2 SwiGLU (``aux`` = h,
    written), 3 SwiGLU backward (``aux`` = the saved gate_up, read)."""

    _fields_ = [("kind", ctypes.c_int), ("rope_cos", ctypes.c_void_p), ("rope_sin", ctypes.c_void_p), ("rope_S", ctypes.c_int),
                ("rope_cols", ctypes.c_int), ("rope_D", ctypes.c_int), ("aux", ctypes.c_void_p), ("ld_aux", ctypes.c_int)]  # fmt: skip


def _sigs() -> dict:
    """Argument types of every exported ``pb_*`` launcher (all return int)."""
    vp, i32, i64, f32, u32 = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float, ctypes.c_uint32
    PP = ctypes.POINTER(PeerPtrs)
    return {
        "pb_rmsnorm_fwd": [vp, vp, vp, vp, vp, vp, i64, i32, f32, vp],
        "pb_rmsnorm_bwd_grid": [i64],
        "pb_rmsnorm_bwd": [vp, vp, vp, vp, vp, vp, vp, vp, i32, i64, i32, vp],
        "pb_rope_inplace": [vp, vp, vp, i64, i32, i32, i32, i32, f32, vp],
        "pb_swiglu_fwd": [vp, vp, i64, i32, vp],
        "pb_swiglu_bwd": [vp, vp, vp, i64, i32, vp],
        "pb_cross_entropy_loss": [vp, vp, vp, vp, vp, vp, i64, i32, i64, f32, vp],
        "pb_gemm_bf16": [vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, i32, i32, i32, ctypes.POINTER(GemmEpilogue), vp],
        "pb_gemm_allgather": [vp, i32, i32, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, vp],
        "pb_gemm_reduce_scatter": [vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, i32, i32, vp],
        "pb_quantize_mxfp8": [vp, i64, vp, vp, i32, i32, i32, vp],
        "pb_gemm_mxfp8": [vp, vp, vp, vp, vp, i32, i32, i32, i32, vp],
        # e4m3 inference weights (csrc/gemm_e4m3w_sm90.cu)
        "pb_gemm_e4m3w": [vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, vp],
        "pb_gemm_e4m3w_splits": [i32, i32, i32, i32],
        "pb_gemm_e4m3w_m_max": [],
        "pb_dequantize_mxfp8": [vp, vp, vp, i32, i32, i64, vp],
        "pb_gemm_set_split_k": [i32],
        "pb_gemm_set_tile": [i32],
        "pb_gemm_tile_policy": [i32, i32, i32, i32, i32, i32, i32],
        "pb_flash_attn_fwd": [vp, vp, vp, vp, i32, i32, i32, i32, i32, f32, i32, vp],
        "pb_flash_attn_bwd": [vp, vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, f32, i32, vp, vp, vp],
        "pb_doc_bounds": [vp, i32, i32, i64, i32, vp, vp, vp],
        # KV-cache decoding (csrc/decode_sm90.cu)
        "pb_decode_advance": [vp, i64, vp, vp, vp, i32, vp],
        "pb_kv_append": [vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, vp],
        "pb_decode_attn": [vp, vp, vp, vp, i32, vp, vp, i32, i32, i32, i32, i32, i32, f32, vp],
        "pb_decode_attn_splits": [i32, i32, i32],
        "pb_verify_advance": [vp, i32, i64, vp, vp, vp, vp, i32, vp],
        "pb_kv_append_tokens": [vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, vp],
        "pb_verify_attn": [vp, vp, vp, vp, i32, vp, vp, i32, i32, i32, i32, i32, i32, i32, f32, vp],
        # the e4m3 KV cache (csrc/decode_sm90.cu)
        "pb_kv_append_fp8": [vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, vp],
        "pb_kv_quantize": [vp, i64, vp, vp, i32, i32, i32, i32, vp],
        "pb_decode_attn_fp8": [vp, vp, vp, vp, vp, i32, vp, vp, i32, i32, i32, i32, i32, i32, f32, vp],
        "pb_verify_attn_fp8": [vp, vp, vp, vp, vp, i32, vp, vp, i32, i32, i32, i32, i32, i32, i32, f32, vp],
        # token sampling (csrc/sample_sm90.cu)
        "pb_sample_tokens": [vp, i64, i32, i32, f32, i32, f32, f32, vp, vp, vp, vp, vp, vp, vp, i32, i32, i64, vp],
        "pb_spec_accept": [vp, i64, vp, i64, i32, i32, i32, f32, i32, f32, f32, *[vp] * 14, i32, i32, i64, vp, vp, vp],
        "pb_ipc_alloc": [ctypes.POINTER(vp), ctypes.c_size_t],
        "pb_ipc_free": [vp],
        "pb_ipc_handle_size": [],
        "pb_ipc_get_handle": [vp, vp],
        "pb_ipc_open_handle": [vp, ctypes.POINTER(vp)],
        "pb_ipc_close_handle": [vp],
        "pb_enable_peer_access": [i32],
        "pb_signal": [PP, i32, u32, vp],
        "pb_barrier": [PP, i32, i32, u32, vp, vp],
        "pb_grad_reduce_grid": [],
        "pb_grad_reduce": [PP, vp, ctypes.POINTER(SegTable), f32, vp, vp, vp, i32, u32, vp, i32, vp],
        "pb_norm_publish": [vp, i32, PP, PP, i32, i32, u32, vp],
        "pb_adamw_push": [vp, vp, vp, vp, i64, ctypes.POINTER(AdamArgs), vp, i32, vp, i32, u32, PP, i64, vp, vp, vp, vp],
        "pb_pseudograd_quant": [vp, vp, vp, vp, i64, vp],
        "pb_outer_nesterov": [PP, PP, vp, vp, vp, i64, ctypes.POINTER(OuterArgs), PP, vp, vp, i32, vp, vp],
        "pb_outer_nesterov_f32": [PP, vp, vp, vp, i64, ctypes.POINTER(OuterArgs), PP, vp, vp, i32, vp, vp],
        "pb_set_spin_timeout_ms": [ctypes.c_ulonglong],
        "pb_embedding_fwd": [vp, i64, PP, i32, i32, vp, vp],
        "pb_embedding_sort": [vp, i64, vp, vp],
        "pb_embedding_scatter": [vp, i64, vp, vp, i32, vp],
        "pb_allgather_copy": [PP, i64, vp, vp],
        "pb_gemm_wgather": [vp, ctypes.POINTER(vp), i32, i32, vp, vp, vp, i32, i32, i32, i32, i32, i32, ctypes.POINTER(GemmEpilogue), i32,
                            ctypes.POINTER(vp), vp, i32, i32, vp],
        "pb_cast_push": [vp, i64, PP, i64, vp],
        # NVLS: VMM allocations shared by fd and multicast objects (csrc/multicast.cu), the multimem all-reduce (csrc/comm.cu)
        "pb_mc_supported": [i32],
        "pb_vmm_granularity": [i32, i32, ctypes.c_size_t, ctypes.POINTER(ctypes.c_size_t)],
        "pb_vmm_create": [i32, ctypes.c_size_t, ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(i32)],
        "pb_vmm_import": [i32, ctypes.POINTER(ctypes.c_uint64)],
        "pb_vmm_map": [ctypes.c_uint64, ctypes.c_size_t, ctypes.c_size_t, i32, ctypes.POINTER(vp)],
        "pb_vmm_unmap": [vp, ctypes.c_size_t],
        "pb_vmm_release": [ctypes.c_uint64],
        "pb_mc_create": [i32, ctypes.c_size_t, ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(i32)],
        "pb_mc_add_device": [ctypes.c_uint64, i32],
        "pb_mc_bind": [ctypes.c_uint64, ctypes.c_uint64, ctypes.c_size_t],
        "pb_mc_unbind": [ctypes.c_uint64, i32, ctypes.c_size_t],
        "pb_mc_all_reduce_grid": [],
        "pb_mc_all_reduce": [vp, i64, i32, vp, vp, i32, i32, u32, vp, vp],
    }


def _declare(lib: ctypes.CDLL) -> None:
    for name, argtypes in _sigs().items():
        fn = getattr(lib, name)  # a declared launcher the library lacks is a stale build or a stale declaration: fail here
        fn.argtypes = argtypes
        fn.restype = ctypes.c_int


def load(build_if_missing: bool = True) -> ctypes.CDLL:
    """Return the loaded native library, building it first if sources are newer."""
    global _lib
    if _lib is not None:
        return _lib
    if build_if_missing and needs_build() and nvcc_path() is not None and os.environ.get("PRIME_B200_NO_BUILD") != "1":
        build()
    if not LIB_PATH.exists():
        raise RuntimeError(
            f"native kernel library missing: {LIB_PATH}. Run `python -c 'import __graft_entry__ as g; g.build()'` "
            "(needs nvcc). GPU execution has no eager fallback."
        )
    with _lock:
        if _lib is None:
            lib = ctypes.CDLL(str(LIB_PATH), mode=ctypes.RTLD_GLOBAL)
            _declare(lib)
            _lib = lib
    return _lib


def available() -> bool:
    try:
        load()
        return True
    except Exception:
        return False


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = f"{what} failed with code {rc}"
        if rc > 0:
            try:
                import torch

                msg += f" ({torch.cuda.cudart().cudaGetErrorString(rc) if hasattr(torch.cuda.cudart(), 'cudaGetErrorString') else 'cuda error'})"
            except Exception:
                pass
        raise RuntimeError(msg)
