"""Parameter all-gather ⊕ GEMM (ZeRO-3 hot path, IO = 3 of csrc/gemm_sm90.cu) against its roofline and against NCCL + GEMM.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 tools/wgather_bench.py --model 7B

For every weight of a Llama block (wqkv, wo, w13 with the SwiGLU epilogue, w2) and both uses (forward y = x·Wᵀ, input gradient
dx = dy·W): the fused kernel (weights sharded by rows over the ranks, gathered INSIDE the GEMM), the same GEMM on a resident
full weight (what the kernel would cost with no communication at all), and the baseline formulation
``dist.all_gather_into_tensor`` + GEMM.  Device-timed with CUDA events, max over ranks, median of 10, L2 flushed between
iterations; clocks sampled.  Roofline per the profiling recipe: the slower of FLOPs / measured sustained cuBLAS peak and
remote bytes / 770 GB/s (measured peer-copy bandwidth per direction; 900 nominal).
"""

import argparse
import ctypes
import json
import sys
from pathlib import Path

import torch
import torch.distributed as dist

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from prime_b200 import ops  # noqa: E402
from prime_b200.parallel.fsdp import RowShard  # noqa: E402
from prime_b200.parallel.mesh import init_distributed  # noqa: E402
from prime_b200.parallel.symm import SymmetricHeap, dist_exchange  # noqa: E402
from prime_b200.utils.clocks import ClockSampler  # noqa: E402

SHAPES = {"1B": dict(dim=2048, ff=5632, tokens=16384), "7B": dict(dim=4096, ff=11008, tokens=16384)}


def timeit(fn, flush, iters=10, warm=3):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(iters):
        flush.zero_()
        dist.barrier()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        t = torch.tensor([e0.elapsed_time(e1)], device="cuda")
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ts.append(float(t))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="7B")
    ap.add_argument("--tokens", type=int, default=0)
    a = ap.parse_args()
    w = init_distributed("nccl")
    dev = torch.device("cuda", w.device_index)
    n, r = w.world_size, w.rank
    sh = SHAPES[a.model]
    D, FF, T = sh["dim"], sh["ff"], a.tokens or sh["tokens"]
    heap = SymmetricHeap(3 << 30, r, n, dist_exchange(), dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    peaks = json.loads((ROOT / "MEASURED_PEAKS.json").read_text()) if (ROOT / "MEASURED_PEAKS.json").exists() else {}
    peak = float(peaks.get("bf16_tflops_sustained", 989.0)) * 1e12  # default: H100 SXM data-sheet dense bf16 (not a measured rate)
    link = 450e9  # H100 NVLink 4: 900 GB/s bidirectional per GPU = 450 GB/s per direction (data sheet)
    sampler = ClockSampler(torch.cuda.current_device())
    if r == 0:
        sampler.start()
    flags = torch.zeros(64, dtype=torch.int32, device=dev)
    rows = []

    def shard(rowsW, colsW):
        rpr = rowsW // n
        s = heap.alloc(rpr * colsW, torch.bfloat16).view(rpr, colsW)
        s.normal_(0, 0.05)
        full = torch.empty(rowsW, colsW, dtype=torch.bfloat16, device=dev)
        peers = (ctypes.c_void_p * n)(*[heap.peer_ptr(q, s) for q in range(n)])
        return RowShard(rowsW, colsW, n, r, rpr, peers, full.data_ptr(), flags, s), s, full

    def bench(name, rowsW, colsW, mode):
        z, s, full = shard(rowsW, colsW)
        zn, _, _ = shard(rowsW, colsW)  # a second weight of the same size: what the kernel gathers AHEAD for the next GEMM
        torch.cuda.synchronize()
        dist.barrier()
        kw = {}
        if mode == "fwd":
            x = (torch.randn(T, colsW, device=dev) * 0.5).to(torch.bfloat16)
            out = torch.empty(T, rowsW, dtype=torch.bfloat16, device=dev)
            local = lambda: ops.gemm(x, full, out=out)  # noqa: E731
        elif mode == "swiglu":
            x = (torch.randn(T, colsW, device=dev) * 0.5).to(torch.bfloat16)
            out = torch.empty(T, rowsW, dtype=torch.bfloat16, device=dev)
            h = torch.empty(T, rowsW // 2, dtype=torch.bfloat16, device=dev)
            kw = {"swiglu_h": h}
            local = lambda: ops.functional._gemm_epi(x, full, out, swiglu_h=h)  # noqa: E731
        else:  # dgrad: dx = dy · W
            x = (torch.randn(T, rowsW, device=dev) * 0.5).to(torch.bfloat16)
            out = torch.empty(T, colsW, dtype=torch.bfloat16, device=dev)
            kw = {"b_mn_major": True}
            local = lambda: ops.gemm(x, full, b_mn_major=True, out=out)  # noqa: E731

        def cold():  # first GEMM of a pass: nothing was gathered ahead, the tiles wait for the in-kernel gather of their own weight
            z.next_fwd = z.next_bwd = None
            z.ver[0] += 1
            ops.gemm_wgather(x, z, out=out, **kw)

        def steady():  # every other GEMM: own weight resident (gathered ahead by the previous kernel), carries the NEXT weight's gather
            z.next_fwd = z.next_bwd = zn
            zn.ver[0] += 1
            ops.gemm_wgather(x, z, out=out, **kw)

        def nccl():
            dist.all_gather_into_tensor(full, s)
            local()

        t_c = timeit(cold, flush)
        ops.gemm_wgather(x, z, out=out, **kw)  # leave z resident
        t_s, t_l, t_n = timeit(steady, flush), timeit(local, flush), timeit(nccl, flush)
        fl = 2.0 * T * rowsW * colsW
        remote = (n - 1) * (rowsW // n) * colsW * 2
        roof = max(fl / peak, remote / link)
        rows.append({"op": name, "mode": mode, "M": T, "W": [rowsW, colsW], "steady_ms (own resident + gather-ahead of the next weight)": round(t_s, 4),
                     "cold_ms (in-kernel gather of the own weight, first GEMM of a pass)": round(t_c, 4), "resident_weight_gemm_ms": round(t_l, 4),
                     "nccl_allgather_plus_gemm_ms": round(t_n, 4), "steady_tflops": round(fl / t_s / 1e9, 1),
                     "steady_cost_vs_resident": round(t_s / t_l, 3), "cold_cost_vs_resident": round(t_c / t_l, 3),
                     "steady_speedup_vs_nccl": round(t_n / t_s, 3), "cold_speedup_vs_nccl": round(t_n / t_c, 3),
                     "remote_MB": round(remote / 1e6, 1), "gather_GBps_needed_to_hide": round(remote / t_l / 1e6, 1),
                     "roofline_ms": round(roof * 1e3, 4), "steady_over_roofline": round(t_s / 1e3 / roof, 3), "cold_over_roofline": round(t_c / 1e3 / roof, 3)})  # fmt: skip
        del z, zn, s, full

    bench("wqkv", 3 * D, D, "fwd")
    bench("wo", D, D, "fwd")
    bench("w13+swiglu", 2 * FF // (64 * n) * (64 * n), D, "swiglu")
    bench("w2", D, FF, "fwd")
    bench("wqkv dgrad", 3 * D, D, "dgrad")
    bench("w13 dgrad", 2 * FF // (64 * n) * (64 * n), D, "dgrad")
    bench("w2 dgrad", D, FF, "dgrad")
    heap.check_errors()
    if r == 0:
        print(json.dumps({"n_gpus": n, "model": a.model, "tokens": T, "peak_tflops_sustained": peak / 1e12, "link_GBps": link / 1e9,
                          "clocks": sampler.finish(), "rows": rows}, indent=1))  # fmt: skip
    dist.barrier()
    heap.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
