"""Time the native flash-attention (fwd, bwd) against SDPA/cuDNN on the Llama shapes. CUDA events, median.

    python tools/attn_bench.py                                         # the default Llama shapes
    python tools/attn_bench.py --shape 4,4096,16,16,128 --doc-len 256  # + document-masked kernels, 256-token documents
    python tools/attn_bench.py --shape 4,8192,16,16,128 --window 1024  # + sliding-window attention over 1024 keys

``--doc-len N`` packs every row with documents of N tokens (EOS every N positions) and also times the document-masked kernels
(``native_doc_*``) in the same process, so masked and plain causal attention are compared on one shape in one invocation.
``--window W`` does the same for sliding-window attention (``native_win_*``) and reports the ratio of tiles the kernels visit,
counted from the bounds: key tiles of the forward / dQ kernels, query tiles of the dK/dV kernel."""

import argparse
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from prime_b200.ops import attention_native as A  # noqa: E402


def timeit(fn, iters=10, warm=3, flush=None):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        if flush is not None:
            flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


def tile_counts(lo: torch.Tensor, end: torch.Tensor) -> tuple[int, int]:
    """Tiles the kernels visit for int32 [B, S] bounds, summed over rows: (64-key tiles of the forward / dQ kernels, 32-query tiles
    of the dK/dV kernel). Per (b, head); the same loop bounds as Visibility::query_block / key_block in csrc/attention_sm90.cu."""
    blk = torch.arange(lo.shape[1] // 64, device=lo.device)
    fwd = (blk - lo[:, ::64].long() // 64 + 1).sum()
    dkdv = ((end[:, 63::64].long() + 31) // 32 - 2 * blk).sum()
    return int(fwd), int(dkdv)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--shape", action="append", default=None, metavar="B,S,H,Hkv,D", help="shape to time (repeatable); default: Llama shapes")
    ap.add_argument("--doc-len", type=int, default=0, help="also time document-masked attention with documents of this many tokens")
    ap.add_argument("--window", type=int, default=0, help="also time sliding-window attention over this many keys")
    a = ap.parse_args()
    shapes = [("1B mb16", 16, 1024, 16, 16, 128), ("7B-like", 8, 2048, 32, 32, 128), ("150M", 16, 1024, 16, 16, 64)]
    if a.shape:
        shapes = [(s, *map(int, s.split(","))) for s in a.shape]
    from prime_b200 import ops

    dev = torch.device("cuda", 0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    from prime_b200.utils.clocks import ClockSampler

    sampler = ClockSampler(0, period_s=0.05)
    sampler.start()
    rows = []
    for name, B, S, H, Hkv, D in shapes:
        W = (H + 2 * Hkv) * D
        qkv = (torch.randn(B, S, W, device=dev) * 0.5).to(torch.bfloat16).requires_grad_(True)
        out = A.flash_attention_qkv(qkv, H, Hkv, True)
        dout = torch.randn_like(out)
        fwd = timeit(lambda: A.flash_attention_qkv(qkv, H, Hkv, True), flush=flush)

        def fb():
            qkv.grad = None
            o = A.flash_attention_qkv(qkv, H, Hkv, True)
            o.backward(dout)

        both = timeit(fb, flush=flush)
        x = qkv.detach().view(B, S, H + 2 * Hkv, D)
        q = x[:, :, :H].transpose(1, 2).contiguous().requires_grad_(True)
        k = x[:, :, H : H + Hkv].transpose(1, 2).contiguous().requires_grad_(True)
        v = x[:, :, H + Hkv :].transpose(1, 2).contiguous().requires_grad_(True)
        sd = lambda: torch.nn.functional.scaled_dot_product_attention(q, k, v, is_causal=True, enable_gqa=H != Hkv)  # noqa: E731
        rfwd = timeit(sd, flush=flush)
        do2 = torch.randn(B, H, S, D, device=dev, dtype=torch.bfloat16)

        def rfb():
            q.grad = k.grad = v.grad = None
            sd().backward(do2)

        rboth = timeit(rfb, flush=flush)
        fl_f = 4.0 * B * H * S * S * D / 2
        rows.append({"shape": name, "B": B, "S": S, "H": H, "D": D, "native_fwd_ms": round(fwd, 4), "sdpa_fwd_ms": round(rfwd, 4),
                     "native_fwd_tflops": round(fl_f / fwd / 1e9, 1), "sdpa_fwd_tflops": round(fl_f / rfwd / 1e9, 1),
                     "native_bwd_ms": round(both - fwd, 4), "sdpa_bwd_ms": round(rboth - rfwd, 4),
                     "native_bwd_tflops_algorithmic": round(2.5 * fl_f / (both - fwd) / 1e9, 1),
                     "sdpa_bwd_tflops": round(2.5 * fl_f / (rboth - rfwd) / 1e9, 1)})  # fmt: skip
        if a.doc_len:
            tok = torch.full((B, S), 1, dtype=torch.int64, device=dev)
            tok[:, a.doc_len - 1 :: a.doc_len] = 0  # EOS (id 0) ends every document
            doc = ops.document_bounds(tok, 0)
            dfwd = timeit(lambda: A.flash_attention_qkv(qkv, H, Hkv, True, doc), flush=flush)

            def dfb():
                qkv.grad = None
                A.flash_attention_qkv(qkv, H, Hkv, True, doc).backward(dout)

            dboth = timeit(dfb, flush=flush)
            rows[-1].update({"doc_len": a.doc_len, "native_doc_fwd_ms": round(dfwd, 4), "native_doc_bwd_ms": round(dboth - dfwd, 4),
                             "doc_fwd_speedup": round(fwd / dfwd, 2), "doc_bwd_speedup": round((both - fwd) / (dboth - dfwd), 2)})  # fmt: skip
        if a.window:
            tok = torch.zeros((B, S), dtype=torch.int64, device=dev)
            win = ops.document_bounds(tok, None, a.window)
            wfwd = timeit(lambda: A.flash_attention_qkv(qkv, H, Hkv, True, win), flush=flush)

            def wfb():
                qkv.grad = None
                A.flash_attention_qkv(qkv, H, Hkv, True, win).backward(dout)

            wboth = timeit(wfb, flush=flush)
            (cf, cb), (wf, wb) = tile_counts(*ops.document_bounds(tok, None)), tile_counts(*win)
            rows[-1].update({"window": a.window, "native_win_fwd_ms": round(wfwd, 4), "native_win_bwd_ms": round(wboth - wfwd, 4),
                             "win_fwd_speedup": round(fwd / wfwd, 2), "win_bwd_speedup": round((both - fwd) / (wboth - wfwd), 2),
                             "win_fwd_tiles_per_bh": wf // B, "causal_fwd_tiles_per_bh": cf // B, "win_fwd_tile_ratio": round(cf / wf, 2),
                             "win_dkdv_tiles_per_bhkv": wb // B, "causal_dkdv_tiles_per_bhkv": cb // B,
                             "win_dkdv_tile_ratio": round(cb / wb, 2)})  # fmt: skip
        print(rows[-1], flush=True)
    (ROOT / "gpurun_out").mkdir(exist_ok=True)
    (ROOT / "gpurun_out" / "attn_bench.json").write_text(json.dumps({"rows": rows, "clocks": sampler.finish(),
                                                                      "timing": "CUDA events, median, 256 MB L2 flush between iterations; same process for both arms"}, indent=1))


if __name__ == "__main__":
    main()
