"""CPU-side guards on the BUILT library: the Hopper instruction paths must stay in the binary (cuobjdump needs no GPU).

If a refactor silently turns the wgmma GEMM into an `mma.sync` one, drops its TMA loads, or loses the peer / NVLS paths, these fail
here, before any GPU time is spent."""

import csv
import io
import shutil
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
LIB = ROOT / "prime_b200" / "_C" / "libprime_b200.so"

needs_toolchain = pytest.mark.skipif(shutil.which("cuobjdump") is None or shutil.which("nvcc") is None, reason="CUDA toolkit not installed")


@pytest.fixture(scope="module")
def sass() -> str:
    from prime_b200.ops import _lib

    _lib.build()  # no-op when the sources are unchanged
    return subprocess.run(["cuobjdump", "-sass", str(LIB)], capture_output=True, text=True, check=True).stdout


def _kernels(sass: str) -> dict[str, str]:
    out, cur = {}, None
    for line in sass.splitlines():
        if "Function :" in line:
            cur = line.split("Function :")[1].strip()
            out[cur] = ""
        elif cur is not None:
            out[cur] += line + "\n"
    return out


@needs_toolchain
def test_gemm_kernels_use_wgmma(sass):
    assert "arch = sm_90a" in sass
    gemms = {n: b for n, b in _kernels(sass).items() if "gemm_bf16_kernel" in n}
    assert gemms
    for n, b in gemms.items():
        assert "HGMMA" in b and "HMMA" not in b.replace("HGMMA", ""), f"{n} is not on the wgmma path"


@needs_toolchain
def test_hopper_instruction_paths_are_present(sass):
    k = _kernels(sass)

    def body(*needles):
        hits = [b for n, b in k.items() if all(x in n for x in needles)]
        assert hits, f"no kernel matching {needles}"
        return "\n".join(hits)

    gemm = body("gemm_bf16_kernel")
    assert "HGMMA" in gemm and "UTMALDG" in gemm and "UTMASTG" in gemm  # wgmma fed by TMA loads; TMA stores of the gather copiers
    assert "HMMA" in body("gemm_mxfp8_kernel")
    for name in ("flash_fwd_kernel", "bwd_dkdv_kernel", "bwd_dq_kernel"):
        a = body(name)
        assert "HMMA" in a and "LDSM" in a and "MUFU.EX2" in a, name  # tensor-core tiles fed by ldmatrix, exp2 softmax
    comm = body("adamw_push_kernel")
    assert "STG.E.128" in comm  # 128-bit peer stores
    assert "LD.E.STRONG.SYS" in body("outer_nesterov") or "STRONG.SYS" in body("outer_nesterov")
    # NVLS: the reduction is a multimem load (LDGMC), in f32 and in bf16 with fp32 accumulation in the switch; only the multicast
    # instantiation of the gradient reduce-scatter (MC = true) has it
    assert "LDGMC.E.ADD.F32x4" in body("grad_reduce_kernel", "Lb1E")
    assert "LDGMC" not in body("grad_reduce_kernel", "Lb0E") and "STRONG.SYS" in body("grad_reduce_kernel", "Lb0E")
    allred = body("mc_all_reduce_kernel")
    assert "LDGMC.E.ADD.F32x4" in allred and "BF16x8" in allred and "REDG.E.ADD.STRONG.SYS" in allred


def test_ncu_source_hotspots_condenses_runs(tmp_path, capsys):
    sys.path.insert(0, str(ROOT / "tools"))
    import ncu_source_hotspots as H

    buf = io.StringIO()
    w = csv.writer(buf)
    w.writerow(["Kernel Name", "void demo()"])
    w.writerow(["Address", "Source", "# Samples", "Instructions Executed"])
    rows = [("a", "      LDG.E R1, [R2]", 5, 100), ("b", "      FFMA R3, R1, R4, R5", 90, 100), ("c", "@P0   BRA 0x10", 4, 100),
            ("d", "      EXIT", 1, 1)]  # fmt: skip
    for a, s, n, e in rows:
        w.writerow([a, s, n, e])
    p = tmp_path / "src.csv"
    p.write_text(buf.getvalue())
    H.main(str(p), 2)
    out = capsys.readouterr().out
    assert "4 instructions, 100 stall samples" in out
    assert "exec       100" in out and "FFMA 90" in out and "(90.0 %)" in out
