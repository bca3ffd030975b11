"""KV-cache decoding on one GPU: the split-KV decode-attention kernel against SDPA, end-to-end generation, and device sampling.

    python tools/decode_bench.py [--out results.json] [--skip-e2e] [--only-sampler]

Kernel section: ``ops.decode_attention`` (pb_decode_attn, split policy of pb_decode_attn_splits) at 1B heads (H = Hkv = 16) and
Llama-3-8B heads (H = 32, Hkv = 8), D = 128, B ∈ {1, 8, 32} × context ∈ {1 K, 8 K, 32 K}, plus one windowed case; every row sees
the whole context. CUDA events around one call, median of 20 with a 256 MB L2 flush before each. Bytes read = the visible K and V
rows (2·Hkv·D·2 bytes each) plus Q and the output; the share of bandwidth is against the 3.35 TB/s of the H100 SXM data sheet.
The comparison arm is ``F.scaled_dot_product_attention`` with a one-token query over the same cache (strided views, GQA), in the
same process.

End-to-end section: a random-init Llama-2 1B, prompt 512, 256 new tokens, greedy, B ∈ {1, 8}: tokens/s of cached generation with
CUDA graphs, cached generation eager, and the recompute loop (``eval._generate_recompute``, one row at a time). Also the share of
one eager decode step's kernel time spent in the M = B GEMMs (torch.profiler, a separate pass).

Sampler sections: ``ops.sample_tokens`` (pb_sample_tokens) alone at V ∈ {32000, 128256}, B ∈ {1, 8, 64}, greedy and T = 0.8 /
top_p = 0.9, timed like the kernel section (bytes = the logits read once); then 1B generation with ``sampler="device"`` next to
``"host"`` at B ∈ {1, 8}, greedy and T = 0.8 / top_p = 0.9, the two alternating in one process, with the sampler's share of one
device-loop step's kernel time (torch.profiler).

    python tools/decode_bench.py --only-sampler

Speculative section (``--speculative``, alone): a random-init Llama-2 1B target with a random-init 150M draft, prompt 512,
B ∈ {1, 8}, k ∈ {2, 4, 8}. CUDA events around graph replays, median of 20: one target decode step, one verify step at T = k + 1,
one draft decode step, and the accept kernel alone. The break-even acceptance rate α is where the expected tokens per round,
(1 − α^{k+1}) / (1 − α), equals the round's time over one decode step's. Then greedy generation of 256 new tokens: tokens/s and
acceptance of ``generate_speculative`` with the target as its own draft (the overhead ceiling) and with the independent draft (the
floor, random weights agree rarely), next to ``generate_batch(sampler="device")``.

    python tools/decode_bench.py --speculative

fp8 KV-cache section (``--kv-fp8``, alone): decode attention over the bf16 cache and over the e4m3 cache (``kv_dtype="fp8"``) at the
shapes of the kernel section, timed the same way, with GB/s counted from the bytes each must read (bf16: 2 bytes per value; fp8: 1
byte per value plus one scale byte per 32). Then a random-init Llama-2 1B at B = 8 with a 16 K-token prompt, device sampler, CUDA
graphs: decode tokens/s with either cache (the time of 129 new tokens minus that of 1, so the prefill cancels). Last, a random-init
Llama-2 7B at B = 4 and 32 K context (``max_seq_len`` = 32768): the cache bytes of both dtypes from the shapes, and decode tokens/s
with the fp8 cache only, since the bf16 one does not fit next to the weights.

    python tools/decode_bench.py --kv-fp8

fp8-weight section (``--weights-fp8``, alone). Kernel table: every projection shape (QKV, O, W13, W2, head) of Llama-2 1B, Llama-2
7B and Llama-3 8B at M ∈ {1, 8, 16, 32, 64, M_MAX + 1}: ``ops.linear`` on the e4m3 weight (``pb_gemm_e4m3w`` up to M_MAX; above it
the dequantise-then-bf16 path) next to ``ops.linear`` on the bf16 W̃, timed like the kernel section, with GB/s of the bytes each
must read (weights at 1 + 1/32 or 2 bytes per value, plus x and C), their share of 3.35 TB/s and the split count. Steps: graph-replay
times of a decode step and of a verify step at k = 4 (T = 5), bf16 against fp8 weights, random-init Llama-2 1B and 7B at B ∈ {1, 8},
prompt 512. End to end: decode tokens/s (``_decode_tok_s``, 129 new tokens) and peak allocated memory for the same models.

    python tools/decode_bench.py --weights-fp8
"""

from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

import torch
import torch.nn.functional as F

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

from prime_b200 import eval as ev  # noqa: E402
from prime_b200 import inference, ops  # noqa: E402
from prime_b200.models.llama import build_model  # noqa: E402

HBM_BPS = 3.35e12


def card() -> dict:
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()  # fmt: skip
        out["power_limit"], out["max_sm_clock"] = (x.strip() for x in q.split(","))
    except Exception as e:  # noqa: BLE001
        out["power_limit"] = f"unread: {e}"
    return out


def timed(fn, flush: torch.Tensor, reps: int = 20) -> float:
    """Median ms of ``fn`` over ``reps`` calls, each after an L2 flush, CUDA events around the call only."""
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def kernel_section(flush) -> list[dict]:
    rows = []
    D = 128
    cases = [(H, Hkv, B, ctx, None) for (H, Hkv) in ((16, 16), (32, 8)) for B in (1, 8, 32) for ctx in (1024, 8192, 32768)]
    cases.append((32, 8, 8, 32768, 4096))
    for H, Hkv, B, ctx, window in cases:
        dev = torch.device("cuda", 0)
        kv = torch.randn(B, ctx, 2 * Hkv * D, device=dev, dtype=torch.bfloat16)
        qkv = torch.randn(B, (H + 2 * Hkv) * D, device=dev, dtype=torch.bfloat16)
        length = torch.full((B,), ctx, dtype=torch.int32, device=dev)
        ms = timed(lambda: ops.decode_attention(qkv, kv, length, None, window, H, Hkv), flush)
        vis = min(ctx, window or ctx)
        nbytes = B * vis * 2 * Hkv * D * 2 + 2 * B * H * D * 2
        r = {"heads": f"{H}/{Hkv}", "B": B, "context": ctx, "window": window, "splits": ops.decode_attn_splits(B, Hkv, ctx), "ms": round(ms, 4),
             "bytes": nbytes, "GB_s": round(nbytes / ms / 1e6, 1), "share_of_3.35TB_s": round(nbytes / ms / 1e-3 / HBM_BPS, 3)}  # fmt: skip
        q = qkv[:, : H * D].view(B, H, 1, D)
        k = kv[..., : Hkv * D].view(B, ctx, Hkv, D).transpose(1, 2)
        v = kv[..., Hkv * D :].view(B, ctx, Hkv, D).transpose(1, 2)
        mask = None
        if window:
            mask = torch.zeros(1, 1, 1, ctx, dtype=torch.bool, device=dev)
            mask[..., ctx - window :] = True
        try:
            sd = timed(lambda: F.scaled_dot_product_attention(q, k, v, attn_mask=mask, enable_gqa=H != Hkv), flush)
            r["sdpa_ms"] = round(sd, 4)
            r["speedup_vs_sdpa"] = round(sd / ms, 2)
        except Exception as e:  # noqa: BLE001
            r["sdpa_ms"] = f"failed: {type(e).__name__}"
        print(json.dumps(r), flush=True)
        rows.append(r)
        del kv, qkv
        torch.cuda.empty_cache()
    return rows


def e2e_section(prompt_len: int = 512, new: int = 256) -> list[dict]:
    model = build_model("1B", device="cuda", dtype=torch.bfloat16, seed=0).eval()
    g = torch.Generator().manual_seed(0)
    rows = []
    for B in (1, 8):
        prompts = [torch.randint(0, model.args.vocab_size, (prompt_len,), generator=g).tolist() for _ in range(B)]
        r = {"B": B, "prompt": prompt_len, "new_tokens": new}
        for name, graphs in (("cached_graphs", True), ("cached_eager", False)):
            ev.generate_batch(model, prompts, max_new=8, graphs=graphs)  # warm-up: library, kernel attributes
            torch.cuda.synchronize()
            t = time.perf_counter()
            out = ev.generate_batch(model, prompts, max_new=new, graphs=graphs)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t
            r[f"{name}_tok_s"] = round(sum(len(o) - prompt_len for o in out) / dt, 1)
        if B == 1:
            ev._generate_recompute(model, prompts[0], max_new=4)
            torch.cuda.synchronize()
            t = time.perf_counter()
            out = ev._generate_recompute(model, prompts[0], max_new=new)
            torch.cuda.synchronize()
            r["recompute_tok_s"] = round((len(out) - prompt_len) / (time.perf_counter() - t), 1)
        r["gemm_share_of_decode_step"] = gemm_share(model, prompts, prompt_len + new)
        print(json.dumps(r), flush=True)
        rows.append(r)
    return rows


@torch.no_grad()
def gemm_share(model, prompts, capacity: int) -> float:
    """Share of one eager decode step's CUDA kernel time in the GEMM kernels (QKV, output, gate/up, down projections, LM head)."""
    from torch.profiler import ProfilerActivity, profile

    _, cache = inference.prefill(model, prompts, inference.cache_capacity(model.args.max_seq_len, [len(p) for p in prompts], capacity))
    tok = torch.zeros(len(prompts), dtype=torch.int64, device="cuda")
    for _ in range(3):
        model.decode_step(tok, cache)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            model.decode_step(tok, cache)
        torch.cuda.synchronize()
    tot = gemm = 0.0
    for e in prof.key_averages():
        t = e.device_time_total
        tot += t
        if "gemm" in e.key.lower():
            gemm += t
    return round(gemm / tot, 3) if tot else float("nan")


SAMPLE_KNOBS = {"greedy": dict(temperature=0.0), "T0.8_p0.9": dict(temperature=0.8, top_p=0.9)}


def sampler_kernel_section(flush) -> list[dict]:
    rows = []
    dev = torch.device("cuda", 0)
    for V in (32000, 128256):
        for B in (1, 8, 64):
            logits = (torch.randn(B, V, device=dev) * 3).to(torch.bfloat16)
            seeds = torch.arange(B, dtype=torch.int64, device=dev)
            pos = torch.full((B,), 600, dtype=torch.int32, device=dev)
            out = torch.empty(B, dtype=torch.int64, device=dev)
            for name, knobs in SAMPLE_KNOBS.items():
                ms = timed(lambda: ops.sample_tokens(logits, **knobs, seeds=seeds, positions=pos, out=out), flush)
                nbytes = B * V * 2
                r = {"sampler": name, "V": V, "B": B, "us": round(ms * 1e3, 1), "bytes": nbytes, "GB_s": round(nbytes / ms / 1e6, 1)}
                print(json.dumps(r), flush=True)
                rows.append(r)
    return rows


def sampler_e2e_section(prompt_len: int = 512, new: int = 256, rounds: int = 2) -> list[dict]:
    model = build_model("1B", device="cuda", dtype=torch.bfloat16, seed=0).eval()
    g = torch.Generator().manual_seed(0)
    rows = []
    for B in (1, 8):
        prompts = [torch.randint(0, model.args.vocab_size, (prompt_len,), generator=g).tolist() for _ in range(B)]
        for name, knobs in SAMPLE_KNOBS.items():
            r = {"B": B, "sampling": name, "prompt": prompt_len, "new_tokens": new, "card": card()}
            best = {}
            for sampler in ("host", "device"):
                ev.generate_batch(model, prompts, max_new=8, sampler=sampler, **knobs)  # warm-up
            for _ in range(rounds):  # alternate, keep each arm's best
                for sampler in ("host", "device"):
                    torch.cuda.synchronize()
                    t = time.perf_counter()
                    out = ev.generate_batch(model, prompts, max_new=new, sampler=sampler, **knobs)
                    torch.cuda.synchronize()
                    tok_s = sum(len(o) - prompt_len for o in out) / (time.perf_counter() - t)
                    best[sampler] = max(best.get(sampler, 0.0), tok_s)
            r["host_tok_s"], r["device_tok_s"] = round(best["host"], 1), round(best["device"], 1)
            r["device_over_host"] = round(best["device"] / best["host"], 3)
            r["sampler_share_of_device_step"] = sampler_share(model, prompts, prompt_len + new, knobs)
            print(json.dumps(r), flush=True)
            rows.append(r)
    return rows


@torch.no_grad()
def sampler_share(model, prompts, capacity: int, knobs: dict) -> float:
    """Share of one device-loop step's CUDA kernel time (decode step + sample_tokens, eager) spent in the sampling kernel."""
    from torch.profiler import ProfilerActivity, profile

    logits, cache = inference.prefill(model, prompts, inference.cache_capacity(model.args.max_seq_len, [len(p) for p in prompts], capacity))
    B = len(prompts)
    tok = torch.zeros(B, dtype=torch.int64, device="cuda")
    seeds = torch.arange(B, dtype=torch.int64, device="cuda")

    def step():
        ops.sample_tokens(model.decode_step(tok, cache), **knobs, seeds=seeds, positions=cache.len, out=tok)

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            step()
        torch.cuda.synchronize()
    tot = samp = 0.0
    for e in prof.key_averages():
        t = e.device_time_total
        tot += t
        if "sample_tokens" in e.key:
            samp += t
    return round(samp / tot, 4) if tot else float("nan")


def _replay_ms(replay, state: list[torch.Tensor], reps: int = 20) -> float:
    """Median ms of one graph replay (CUDA events), the state restored after every replay so every call sees the same lengths."""
    saved = [t.clone() for t in state]
    ts = []
    for _ in range(reps + 1):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        replay()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
        for t, v in zip(state, saved):
            t.copy_(v)
    return statistics.median(ts[1:])


def _break_even(ratio: float, k: int) -> float | None:
    """α with (1 − α^{k+1}) / (1 − α) = ratio (bisection); None if even α = 1 (k + 1 tokens per round) does not pay."""
    if ratio > k + 1:
        return None
    lo, hi = 0.0, 1.0
    for _ in range(60):
        mid = (lo + hi) / 2
        if sum(mid**j for j in range(k + 1)) < ratio:
            lo = mid
        else:
            hi = mid
    return round(hi, 3)


def speculative_section(prompt_len: int = 512, new: int = 256) -> list[dict]:
    dev = torch.device("cuda")
    target = build_model("1B", device=dev, seed=0)
    draft = build_model("150M", device=dev, seed=1)
    V = target.args.vocab_size
    rows = []
    for B in (1, 8):
        g = torch.Generator().manual_seed(B)
        prompts = torch.randint(1, V, (B, prompt_len), generator=g).tolist()
        cap = prompt_len + 1024
        _, tc = inference.prefill(target, prompts, cap)
        _, dc = inference.prefill(draft, prompts, cap)
        t_state, d_state = [tc.len, tc.lo, tc.last_tok], [dc.len, dc.lo, dc.last_tok]
        tok = torch.ones(B, dtype=torch.int64, device=dev)
        decode_ms = _replay_ms(inference.GraphDecoder(target, tc, tokens=tok).replay, t_state)
        draft_ms = _replay_ms(inference.GraphDecoder(draft, dc, tokens=tok).replay, d_state)
        for k in (2, 4, 8):
            T = k + 1
            toks = torch.ones(B, T, dtype=torch.int64, device=dev)
            verify_ms = _replay_ms(inference._capture(lambda: target.verify_step(toks, tc), t_state), t_state)
            tl = (torch.randn(B, T, V, device=dev) * 2).to(torch.bfloat16)
            dl = (torch.randn(k, B, V, device=dev) * 2).to(torch.bfloat16)
            st = inference.SampleState.allocate(prompts, new, 4096, None, dev)
            z = [torch.zeros(B, dtype=torch.int64, device=dev) for _ in range(3)]
            lo_q = torch.zeros(B, T, dtype=torch.int32, device=dev)
            tc.len.add_(T)
            acc_state = t_state + d_state + [st.history, st.n_out, st.active, *z]
            accept_ms = _replay_ms(lambda: ops.spec_accept(tl, dl, temperature=0.8, top_p=0.9, seeds=z[0], tokens=toks, lo_q=lo_q,
                                                           target=tc, draft=dc, state=st, pending=z[0], drafted=z[1],
                                                           accepted=z[2]), acc_state)  # fmt: skip
            tc.len.sub_(T)
            round_ms = T * draft_ms + verify_ms + accept_ms
            r = {"B": B, "k": k, "decode_ms": round(decode_ms, 3), "verify_ms": round(verify_ms, 3),
                 "verify_over_decode": round(verify_ms / decode_ms, 2), "draft_step_ms": round(draft_ms, 3),
                 "accept_ms": round(accept_ms, 3), "round_ms": round(round_ms, 3),
                 "break_even_acceptance": _break_even(round_ms / decode_ms, k)}  # fmt: skip
            for name, dr in (("self", target), ("independent", draft)):
                inference.generate_speculative(target, dr, prompts, k=k, max_new=8)  # warm-up
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                res = inference.generate_speculative(target, dr, prompts, k=k, max_new=new)
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                r[f"{name}_tok_s"] = round(sum(len(x) - prompt_len for x in res.ids) / dt, 1)
                r[f"{name}_acceptance"] = round(res.accepted / max(res.drafted, 1), 3)
            inference.generate_batch(target, prompts, max_new=8, sampler="device")
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = inference.generate_batch(target, prompts, max_new=new, sampler="device")
            torch.cuda.synchronize()
            r["baseline_tok_s"] = round(sum(len(x) - prompt_len for x in out) / (time.perf_counter() - t0), 1)
            print(json.dumps(r), flush=True)
            rows.append(r)
    return rows


def _kv_fp8_kernel_rows(flush) -> list[dict]:
    rows = []
    D = 128
    dev = torch.device("cuda", 0)
    cases = [(H, Hkv, B, ctx, None) for (H, Hkv) in ((16, 16), (32, 8)) for B in (1, 8, 32) for ctx in (1024, 8192, 32768)]
    cases.append((32, 8, 8, 32768, 4096))
    for H, Hkv, B, ctx, window in cases:
        cols = 2 * Hkv * D
        kv = torch.randn(B, ctx, cols, device=dev, dtype=torch.bfloat16)
        kv8 = torch.empty(B, ctx, cols, dtype=torch.uint8, device=dev)
        sc = torch.empty(B, ctx, cols // 32, dtype=torch.uint8, device=dev)
        ops.kv_quantize(kv, kv8, sc)
        qkv = torch.randn(B, (H + 2 * Hkv) * D, device=dev, dtype=torch.bfloat16)
        length = torch.full((B,), ctx, dtype=torch.int32, device=dev)
        vis = min(ctx, window or ctx)
        r = {"heads": f"{H}/{Hkv}", "B": B, "context": ctx, "window": window, "splits": ops.decode_attn_splits(B, Hkv, ctx)}
        for name, args, per_value in (("bf16", (kv, None), 2.0), ("fp8", (kv8, sc), 1.0 + 1.0 / 32)):
            ms = timed(lambda: ops.decode_attention(qkv, args[0], length, None, window, H, Hkv, kv_scale=args[1]), flush)
            nbytes = B * vis * cols * per_value + 2 * B * H * D * 2
            r[f"{name}_ms"] = round(ms, 4)
            r[f"{name}_GB_s"] = round(nbytes / ms / 1e6, 1)
        r["fp8_speedup"] = round(r["bf16_ms"] / r["fp8_ms"], 2)
        print(json.dumps(r), flush=True)
        rows.append(r)
        del kv, kv8, sc, qkv
        torch.cuda.empty_cache()
    return rows


def _decode_tok_s(model, prompts, new: int, kv_dtype: str) -> float:
    """Decode tokens/s of generate_batch(sampler="device", graphs on): (new − 1)·B tokens over the time of ``new`` new tokens
    minus that of 1 (the prefill and the first token cancel)."""

    def run(n):
        torch.cuda.synchronize()
        t = time.perf_counter()
        inference.generate_batch(model, prompts, max_new=n, sampler="device", kv_dtype=kv_dtype)
        torch.cuda.synchronize()
        return time.perf_counter() - t

    run(8)  # warm-up
    return (new - 1) * len(prompts) / (run(new) - run(1))


def kv_fp8_section(flush) -> dict:
    out = {"kernel": _kv_fp8_kernel_rows(flush)}
    g = torch.Generator().manual_seed(0)
    model = build_model("1B", device="cuda", dtype=torch.bfloat16, seed=0, max_seq_len=16384 + 256).eval()
    prompts = torch.randint(1, model.args.vocab_size, (8, 16384), generator=g).tolist()
    r = {"model": "llama2 1B", "B": 8, "prompt": 16384, "new_tokens": 128}
    for kv_dtype in ("bf16", "fp8"):
        r[f"{kv_dtype}_tok_s"] = round(_decode_tok_s(model, prompts, 129, kv_dtype), 1)
    r["fp8_over_bf16"] = round(r["fp8_tok_s"] / r["bf16_tok_s"], 3)
    print(json.dumps(r), flush=True)
    out["e2e_1b"] = r
    del model
    torch.cuda.empty_cache()
    model = build_model("7B", device="cuda", dtype=torch.bfloat16, seed=0, max_seq_len=32768).eval()
    a = model.args
    B, ctx, new = 4, 32768, 64
    per_row = a.n_layers * ctx * 2 * a.kv_heads * a.head_dim
    r = {"model": "llama2 7B", "B": B, "context": ctx, "weights_GB": round(sum(p.numel() for p in model.parameters()) * 2 / 1e9, 2),
         "cache_GiB_bf16": round(B * per_row * 2 / 2**30, 2), "cache_GiB_fp8": round(B * per_row * (1 + 1 / 32) / 2**30, 2),
         "new_tokens": new}  # fmt: skip
    prompts = torch.randint(1, a.vocab_size, (B, ctx - new), generator=g).tolist()
    try:
        r["fp8_tok_s"] = round(_decode_tok_s(model, prompts, new, "fp8"), 1)
        r["peak_allocated_GB"] = round(torch.cuda.max_memory_allocated() / 1e9, 2)
    except torch.cuda.OutOfMemoryError as e:
        r["fp8_tok_s"] = f"out of memory: {str(e).splitlines()[0]}"
    print(json.dumps(r), flush=True)
    out["7b_32k"] = r
    return out


def _weight_shapes() -> list[tuple[str, str, int, int]]:
    """(model, projection, N, K) of every projection of Llama-2 1B, Llama-2 7B and Llama-3 8B."""
    from prime_b200.models.llama import get_model_args

    out = []
    for label, name, kind in (("llama2 1B", "1B", "llama2"), ("llama2 7B", "7B", "llama2"), ("llama3 8B", "7B", "llama3")):
        a = get_model_args(name, kind)
        qkv = (a.n_heads + 2 * a.kv_heads) * a.head_dim
        out += [(label, "qkv", qkv, a.dim), (label, "o", a.dim, a.n_heads * a.head_dim), (label, "w13", 2 * a.ffn_hidden, a.dim),
                (label, "w2", a.dim, a.ffn_hidden), (label, "head", a.vocab_size, a.dim)]  # fmt: skip
    return out


@torch.no_grad()
def _weights_fp8_kernel_rows(flush) -> list[dict]:
    rows = []
    dev = torch.device("cuda", 0)
    m_max = ops.gemm_e4m3w_m_max()
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    for label, proj, N, K in _weight_shapes():
        mx = ops.quantize_weight((torch.randn(N, K, device=dev) * 0.02).to(torch.bfloat16))
        wt = ops.dequantize_weight(mx)
        for M in (1, 8, 16, 32, 64, m_max + 1):
            x = torch.randn(M, K, device=dev, dtype=torch.bfloat16)
            io = M * K * 2 + M * N * 2
            r = {"model": label, "proj": proj, "M": M, "N": N, "K": K,
                 "path": "gemm_e4m3w" if M <= m_max else "dequantize + bf16 GEMM",
                 "splits": ops.gemm_e4m3w_splits(M, N, K, sms) if M <= m_max else None}  # fmt: skip
            for name, w, per_value in (("fp8", mx, 1.0 + 1.0 / 32), ("bf16", wt, 2.0)):
                ms = timed(lambda: ops.linear(x, w), flush)
                nbytes = N * K * per_value + io
                r[f"{name}_ms"] = round(ms, 4)
                r[f"{name}_GB_s"] = round(nbytes / ms / 1e6, 1)
                r[f"{name}_share"] = round(nbytes / ms / 1e-3 / HBM_BPS, 3)
            r["fp8_speedup"] = round(r["bf16_ms"] / r["fp8_ms"], 2)
            print(json.dumps(r), flush=True)
            rows.append(r)
        del mx, wt
        torch.cuda.empty_cache()
    return rows


@torch.no_grad()
def weights_fp8_section(flush) -> dict:
    out = {"kernel": _weights_fp8_kernel_rows(flush), "steps": [], "e2e": []}
    dev = torch.device("cuda")
    for name in ("1B", "7B"):
        model = build_model(name, device=dev, dtype=torch.bfloat16, seed=0).eval()
        V = model.args.vocab_size
        res = {}
        for wdt in ("bf16", "fp8"):
            if wdt == "fp8":
                inference.quantize_weights(model)
                torch.cuda.empty_cache()
            for B in (1, 8):
                prompts = torch.randint(1, V, (B, 512), generator=torch.Generator().manual_seed(B)).tolist()
                _, c = inference.prefill(model, prompts, 2048)
                state = [c.len, c.lo, c.last_tok]
                tok = torch.ones(B, dtype=torch.int64, device=dev)
                toks = torch.ones(B, 5, dtype=torch.int64, device=dev)
                decode_ms = _replay_ms(inference.GraphDecoder(model, c, tokens=tok).replay, state)
                verify_ms = _replay_ms(inference._capture(lambda: model.verify_step(toks, c), state), state)
                del c
                torch.cuda.reset_peak_memory_stats()
                tok_s = _decode_tok_s(model, prompts, 129, "bf16")
                res[(wdt, B)] = (decode_ms, verify_ms, tok_s, torch.cuda.max_memory_allocated() / 1e9)
        for B in (1, 8):
            b, f = res[("bf16", B)], res[("fp8", B)]
            r = {"model": f"llama2 {name}", "B": B, "decode_ms_bf16": round(b[0], 3), "decode_ms_fp8": round(f[0], 3),
                 "decode_speedup": round(b[0] / f[0], 2), "verify_k4_ms_bf16": round(b[1], 3), "verify_k4_ms_fp8": round(f[1], 3),
                 "verify_speedup": round(b[1] / f[1], 2)}  # fmt: skip
            e = {"model": f"llama2 {name}", "B": B, "prompt": 512, "new_tokens": 128, "tok_s_bf16": round(b[2], 1),
                 "tok_s_fp8": round(f[2], 1), "fp8_over_bf16": round(f[2] / b[2], 3), "peak_allocated_GB_bf16": round(b[3], 2),
                 "peak_allocated_GB_fp8": round(f[3], 2)}  # fmt: skip
            print(json.dumps(r), flush=True)
            print(json.dumps(e), flush=True)
            out["steps"].append(r)
            out["e2e"].append(e)
        del model
        torch.cuda.empty_cache()
    return out


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    ap.add_argument("--skip-e2e", action="store_true")
    ap.add_argument("--only-sampler", action="store_true", help="run only the two sampler sections")
    ap.add_argument("--speculative", action="store_true", help="run only the speculative-decoding section")
    ap.add_argument("--kv-fp8", action="store_true", help="run only the fp8 KV-cache section")
    ap.add_argument("--weights-fp8", action="store_true", help="run only the fp8-weight section")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("decode_bench needs a CUDA device")
    info = card()
    print(json.dumps({"card": info}), flush=True)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    res = {"card": info}
    if a.speculative or a.kv_fp8 or a.weights_fp8:
        if a.weights_fp8:
            res["weights_fp8"] = weights_fp8_section(flush)
        if a.speculative:
            res["speculative"] = speculative_section()
        if a.kv_fp8:
            res["kv_fp8"] = kv_fp8_section(flush)
        if a.out:
            Path(a.out).parent.mkdir(parents=True, exist_ok=True)
            Path(a.out).write_text(json.dumps(res, indent=1))
        return
    if not a.only_sampler:
        res["kernel"] = kernel_section(flush)
    res["sampler_kernel"] = sampler_kernel_section(flush)
    if not a.skip_e2e:
        if not a.only_sampler:
            res["e2e"] = e2e_section()
        res["sampler_e2e"] = sampler_e2e_section()
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
