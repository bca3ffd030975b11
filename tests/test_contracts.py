"""Driver contracts that must never rot: bench.py's reference arm, the JSON keys of the headline line, __graft_entry__ API,
metrics helpers."""

import json
import re
import shutil
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]


def test_bench_reference_arm_reports_unavailable():
    r = subprocess.run([sys.executable, "bench.py", "--impl", "reference", "--gpus", "1", "--steps", "2", "--warmup", "3"], cwd=ROOT,
                       capture_output=True, text=True, timeout=300)  # fmt: skip
    assert r.returncode == 0, r.stderr[-2000:]
    line = json.loads(r.stdout.strip().splitlines()[-1])
    assert line["impl"] == "reference" and "unavailable" in line and len(line["unavailable"]) > 20


def test_bench_source_declares_every_required_key():
    src = (ROOT / "bench.py").read_text()
    for key in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline", "dtype", "data",
                "config", "clocks", "e2e", "h2d_bytes_per_step", "d2h_bytes_per_step", "gpu_launches", "global_batch", "seq_len", "parallelism"):  # fmt: skip
        assert f'"{key}"' in src, key
    assert "--impl" in src and "--gpus" in src and "--steps" in src and "--warmup" in src


def test_graft_entry_exposes_build_and_smoke():
    sys.path.insert(0, str(ROOT))
    import __graft_entry__ as g

    assert callable(g.build) and callable(g.smoke)


def test_throughput_meter_and_sinks(tmp_path):
    from prime_b200.utils import JsonlSink, Throughput, peak_tflops

    m = Throughput(flops_per_token=6e9, n_gpus=2, window=3)
    for _ in range(5):
        m.update(1000, 0.5)
    assert m.tokens_per_s == 2000 and m.total_tokens == 5000
    assert abs(m.mfu - 2000 * 6e9 / (peak_tflops() * 1e12 * 2)) < 1e-12
    s = JsonlSink(tmp_path / "a" / "m.jsonl")
    s.write({"step": 1})
    s.write({"step": 2})
    s.close()
    assert [json.loads(x)["step"] for x in (tmp_path / "a" / "m.jsonl").read_text().splitlines()] == [1, 2]
    JsonlSink(None).write({"ignored": True})  # disabled sink is a no-op


def test_nvlink_counters_decode_and_delta():
    """NvlinkCounters against a fake NVML: aggregate scope, per-link fallback, KiB → bytes, per-step delta, graceful None."""
    from types import SimpleNamespace

    from prime_b200.utils.clocks import NvlinkCounters

    class FakeNvml:
        NVML_FI_DEV_NVLINK_THROUGHPUT_DATA_TX, NVML_FI_DEV_NVLINK_THROUGHPUT_DATA_RX = 138, 139

        def __init__(self, aggregate=True, links=4):
            self.aggregate, self.links, self.kib = aggregate, links, {l: [1000 * (l + 1), 500 * (l + 1)] for l in range(links)}

        def nvmlDeviceGetHandleByIndex(self, i):
            return "h"

        def nvmlDeviceGetFieldValues(self, h, ids):
            out = []
            for fid, scope in ids:
                col = 0 if fid == 138 else 1
                if scope == 0xFFFFFFFF:
                    ok, val = self.aggregate, sum(v[col] for v in self.kib.values())
                else:
                    ok, val = scope < self.links, self.kib.get(scope, [0, 0])[col]
                out.append(SimpleNamespace(nvmlReturn=0 if ok else 3, valueType=3, value=SimpleNamespace(ullVal=val)))
            return out

    for aggregate in (True, False):
        nv = FakeNvml(aggregate)
        c = NvlinkCounters(0, nvml=nv)
        a = c.read()
        assert a["tx_bytes"] == (1000 + 2000 + 3000 + 4000) * 1024 and a["rx_bytes"] == 5000 * 1024 and len(a["per_link"]) == 4
        for l in nv.kib:
            nv.kib[l][0] += 10 * 1024  # 10 MiB more on every link, transmit side
        d = NvlinkCounters.delta(a, c.read(), steps=4)
        assert d["tx_bytes_per_step"] == 4 * 10 * 1024 * 1024 // 4 and d["rx_bytes_per_step"] == 0 and d["links_active"] == 4
        assert d["per_link_bytes_per_step"][0] == [10 * 1024 * 1024 // 4, 0]
    assert NvlinkCounters(0, nvml=FakeNvml(aggregate=False, links=0)).read() is None  # no NVLink at all
    assert NvlinkCounters.delta(None, {"tx_bytes": 1, "rx_bytes": 1, "per_link": []}, 3) is None

    class Broken:
        def nvmlDeviceGetHandleByIndex(self, i):
            raise RuntimeError("no nvml")

    assert NvlinkCounters(0, nvml=Broken()).read() is None


def test_native_launchers_reject_impossible_arguments_before_touching_the_device():
    """The C-ABI launchers are called with shapes that come from user configs: impossible ones must come back as error codes, on any
    machine — the checks run before the first CUDA call, so this needs no GPU (the library itself loads wherever libcudart is)."""
    import ctypes

    from prime_b200.ops import _lib

    try:
        lib = _lib.load()
    except Exception as e:  # noqa: BLE001
        pytest.skip(f"native library not loadable here: {e}")
    peers = (ctypes.c_void_p * 8)()
    pp = _lib.PeerPtrs.of([0])
    oa = _lib.OuterArgs(0.7, 0.9, 1.0, 1)

    def wgather(n=2, rank=0, M=1024, rows=1024, cols=1024, lda=1024, ldc=1024, ldh=0, b_mn=0, epi=0, H=None):
        e = _lib.GemmEpilogue(kind=epi, aux=H, ld_aux=ldh)
        return lib.pb_gemm_wgather(None, peers, n, rank, None, None, None, M, rows, cols, lda, ldc, b_mn, e, 0, None, None, 0, 0, None)

    assert wgather(n=0) == -6 and wgather(n=9) == -6 and wgather(rank=2) == -6  # group size / rank out of range
    assert wgather(rows=1023) == -6 and wgather(cols=1000) == -6  # rows must divide over the ranks, columns come in 64-wide TMA boxes
    assert wgather(lda=1001) == -1  # 16-byte row pitch
    assert wgather(epi=1, b_mn=1) == -7 and wgather(epi=3, b_mn=0) == -7  # RoPE / SwiGLU epilogues are forward-only, SwiGLU-backward is dgrad-only
    assert wgather(epi=2, ldh=1024) == -5  # SwiGLU epilogue without an output for h
    assert wgather(epi=1) == -3  # RoPE without tables
    assert wgather(M=128) == -8  # below one CTA-pair tile: the host gathers explicitly instead

    aux = 1 << 20  # a 16-byte aligned address that is never dereferenced: every call below is rejected first

    def gemm(M=1024, N=1024, lda=1024, a_mn=0, b_mn=0, c_fp32=0, acc=0, epi=None):
        return lib.pb_gemm_bf16(None, None, None, M, N, 1024, lda, 1024, 1024, a_mn, b_mn, c_fp32, acc, epi, None)

    rope = _lib.GemmEpilogue(kind=1, rope_cos=aux, rope_sin=aux, rope_S=256, rope_cols=512, rope_D=128)
    swiglu = _lib.GemmEpilogue(kind=2, aux=aux, ld_aux=512)
    swiglu_bwd = _lib.GemmEpilogue(kind=3, aux=aux, ld_aux=2048)
    assert gemm(lda=1001) == -1  # 16-byte row pitch
    assert gemm(epi=_lib.GemmEpilogue(kind=1)) == -3  # RoPE without tables
    assert gemm(N=1088, epi=swiglu) == -5 and gemm(epi=_lib.GemmEpilogue(kind=2)) == -5  # SwiGLU: 64-feature tiles, an output for h
    assert gemm(M=128, b_mn=1, epi=swiglu_bwd) == -5  # the SwiGLU backward runs on training shapes only
    assert gemm(a_mn=1, epi=rope) == -7 and gemm(c_fp32=1, epi=rope) == -7  # RoPE / SwiGLU: K-major operands, bf16 output
    assert gemm(epi=swiglu_bwd) == -7  # SwiGLU backward: MN-major B (the input-gradient GEMM)
    assert gemm(epi=_lib.GemmEpilogue(kind=4)) == -7  # no such epilogue
    assert lib.pb_pseudograd_quant(None, None, None, None, 1000, None) == -1  # int8 blocks are 1024 elements
    assert lib.pb_outer_nesterov(ctypes.byref(pp), ctypes.byref(pp), None, None, None, 1000, ctypes.byref(oa), ctypes.byref(pp), None, None, 1, None, None) == -1
    assert lib.pb_outer_nesterov(ctypes.byref(pp), ctypes.byref(pp), None, None, None, 1024, ctypes.byref(oa), ctypes.byref(pp), None, None, 0, None, None) == -1  # no bucket table
    assert lib.pb_outer_nesterov_f32(ctypes.byref(pp), None, None, None, 1001, ctypes.byref(oa), ctypes.byref(pp), None, None, 1, None, None) == -1
    assert lib.pb_cast_push(None, 1001, ctypes.byref(pp), 0, None) == -1 and lib.pb_cast_push(None, 1024, ctypes.byref(pp), 3, None) == -1

    doc = ctypes.c_int(0)  # never read: every call below is rejected before a kernel could see it
    d = ctypes.addressof(doc)

    def attn_fwd(doc_start=None, S=256, causal=1):
        return lib.pb_flash_attn_fwd(None, None, None, doc_start, 1, S, 4, 2, 128, 0.1, causal, None)

    def attn_bwd(doc_start=None, doc_end=None, S=256, causal=1):
        return lib.pb_flash_attn_bwd(None, None, None, None, None, None, doc_start, doc_end, 1, S, 4, 2, 128, 0.1, causal, None, None, None)

    assert attn_fwd(doc_start=d, causal=0) == -1 and attn_bwd(doc_start=d, doc_end=d, causal=0) == -1  # document masking is causal
    assert attn_bwd(doc_start=d) == -1 and attn_bwd(doc_end=d) == -1  # the backward needs both bounds or neither
    assert attn_fwd(S=200) == -1 and attn_bwd(S=200) == -1  # 128-row query / key blocks


def test_ctypes_declarations_match_the_exported_prototypes():
    """Every exported ``pb_*`` launcher is declared in ``_lib`` and nothing else is, with as many ctypes argument types as its
    ``PB_EXPORT`` prototype has parameters: a declaration that drifts by one passes garbage into a kernel."""
    from prime_b200.ops import _lib

    if shutil.which("nm") is None:
        pytest.skip("nm not installed")
    try:
        _lib.load()
    except Exception as e:  # noqa: BLE001
        pytest.skip(f"native library not loadable here: {e}")
    nm = subprocess.run(["nm", "-D", "--defined-only", str(_lib.LIB_PATH)], capture_output=True, text=True, check=True).stdout
    exported = {line.split()[-1] for line in nm.splitlines() if line.split() and line.split()[-1].startswith("pb_")}
    sigs = _lib._sigs()
    assert exported == set(sigs), (sorted(exported - set(sigs)), sorted(set(sigs) - exported))
    protos = {}
    for src in sorted(_lib.CSRC.glob("*.cu")):
        for name, params in re.findall(r"PB_EXPORT\s+int\s+(pb_\w+)\s*\(([^)]*)\)", src.read_text()):
            params = params.strip()
            protos[name] = 0 if params in ("", "void") else params.count(",") + 1
    assert set(protos) == exported
    assert {n: len(a) for n, a in sigs.items()} == protos
