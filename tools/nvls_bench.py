"""NVLS (multimem) collectives against NCCL and against the peer-load kernels they can replace.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 tools/nvls_bench.py [--out profiles/nvls_bench.json]

Per size: in-place all-reduce through the switch (f32, bf16) vs `dist.all_reduce` (NCCL, which may itself use NVLS — NCCL_DEBUG=INFO
says); gradient reduce-scatter by `multimem.ld_reduce` vs by F peer loads. Device-timed with CUDA events, max over ranks, median
of 10, inputs larger than L2 or L2 flushed in between. Bus bandwidth uses the usual 2(n-1)/n (all-reduce) and (n-1)/n (reduce-
scatter) factors so the numbers compare with nccl-tests; the roof is 900 GB/s per direction per GPU.
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
from prime_b200.ops import _lib  # noqa: E402
from prime_b200.parallel.mesh import init_distributed  # noqa: E402
from prime_b200.parallel.multicast import MulticastHeap, nvls_available  # noqa: E402
from prime_b200.parallel.symm import dist_exchange  # noqa: E402


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
    ap.add_argument("--out", default=None)
    ap.add_argument("--max-mib", type=int, default=1024)
    a = ap.parse_args()
    w = init_distributed("nccl")
    dev = torch.device("cuda", w.local_rank)
    n, r = w.world_size, w.rank
    if not nvls_available(w.local_rank):
        if r == 0:
            print(json.dumps({"unavailable": "multicast unsupported on this device/driver"}))
        dist.destroy_process_group()
        return
    heap = MulticastHeap((a.max_mib * 2 + 64) << 20, r, n, dist_exchange(), dev)
    lib = _lib.load()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    from prime_b200.utils.clocks import ClockSampler

    sampler = ClockSampler(torch.cuda.current_device(), period_s=0.05)
    if r == 0:
        sampler.start()
    stream = torch.cuda.current_stream().cuda_stream
    grid = lib.pb_grad_reduce_grid()
    rows = []
    mib = 1
    while mib <= a.max_mib:
        nbytes = mib << 20
        x32 = heap.alloc(nbytes // 4, torch.float32)
        ref = torch.empty(nbytes // 4, device=dev)
        x32.normal_()
        row = {"MiB": mib, "n_gpus": n}
        t = timeit(lambda: dist.all_reduce(ref), flush)
        row["nccl_allreduce_f32_ms"], row["nccl_busbw_GBs"] = round(t, 4), round(2 * (n - 1) / n * nbytes / t / 1e6, 1)
        t = timeit(lambda: heap.all_reduce_(x32), flush)
        row["nvls_allreduce_f32_ms"], row["nvls_busbw_GBs"] = round(t, 4), round(2 * (n - 1) / n * nbytes / t / 1e6, 1)
        xb = x32.view(torch.bfloat16)
        t = timeit(lambda: heap.all_reduce_(xb), flush)
        row["nvls_allreduce_bf16_ms"] = round(t, 4)
        # reduce-scatter of this rank's 1/n shard: switch-side sum vs n peer loads
        shard = (nbytes // 4) // n // 4 * 4
        out = torch.empty(shard, device=dev)
        ss = torch.zeros(grid, device=dev)
        pp = heap.peers(range(n), x32)
        table = _lib.SegTable.of([(r * shard, 0, shard)])
        for name, mc in (("p2p", None), ("nvls", heap.mc_ptr(x32))):
            t = timeit(lambda: _lib.check(lib.pb_grad_reduce(ctypes.byref(pp), mc, ctypes.byref(table), 1.0 / n, out.data_ptr(), ss.data_ptr(),
                                                             None, 0, 0, heap.err.data_ptr(), 0, stream), "pb_grad_reduce"), flush)  # fmt: skip
            row[f"{name}_reduce_scatter_ms"], row[f"{name}_rs_busbw_GBs"] = round(t, 4), round((n - 1) / n * nbytes / t / 1e6, 1)
        heap.check_errors()
        rows.append(row)
        if r == 0:
            print(json.dumps(row), flush=True)
        heap._cursor = heap.offset_of(x32)  # bump allocator: give the block back before the next size
        mib *= 4
    if r == 0 and a.out:
        Path(a.out).write_text(json.dumps({"rows": rows, "clocks": sampler.finish(),
                                           "note": "device-timed, max over ranks, median of 10, L2 flushed"}, indent=1))
    dist.barrier()
    heap.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
