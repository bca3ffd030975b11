"""The e4m3 KV cache on an H100: the append and prefill quantisers bit for bit against ``reference.quantize_kv`` of the bf16 cache, the
decode and verify kernels against fp64 attention over the dequantised cache, the quantisation error against an analytic bound,
CUDA-graph replay, speculative rounds, and the model-level effect on 1B-shape models (reported)."""

import math

import pytest
import torch
from test_kv_cache import DEC_ATOL, DEC_RTOL, LENS, _doc_seq, _model, assert_elementwise, decode64

from prime_b200 import inference, ops
from prime_b200.models.llama import build_model
from prime_b200.ops import reference as Rf


def _dev():
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def native():
    from prime_b200.ops import _lib

    return _lib.load()  # a GPU box without the native library is a hard failure, never a silent fallback


def _blocky_cache(B, cap, cols, seed, dev):
    """bf16 cache rows whose 32-column blocks span magnitudes 2^-4 .. 2^4, and their e4m3 quantisation (the exponents differ)."""
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(B, cap, cols // 32, 32, device=dev, generator=g)
    x *= 2.0 ** torch.randint(-4, 5, (B, cap, cols // 32, 1), device=dev, generator=g).float()
    kv = x.view(B, cap, cols).to(torch.bfloat16)
    q, e = Rf.quantize_kv(kv)
    return q, e, Rf.dequantize_kv(q, e).to(torch.bfloat16)  # the dequantised cache is exact in bf16


# ------------------------------------------------------------------------------------------------------------ exact quantisation
@pytest.mark.gpu
@pytest.mark.parametrize("T", [1, 3, 9])
@pytest.mark.parametrize("D", [64, 128])
def test_append_fp8_is_quantize_of_the_bf16_append(native, D, T):
    dev = _dev()
    g = torch.Generator(device=dev).manual_seed(D + T)
    B, H, Hkv, cap = 4, 8, 2, 384
    cols = 2 * Hkv * D
    cos, sin = Rf.rope_tables(cap, D, 500000.0, device=dev)
    qkv = torch.randn(B, T, (H + 2 * Hkv) * D, device=dev, generator=g).to(torch.bfloat16) * 3
    length = torch.tensor([T, 130, 300 + T, cap + 2], dtype=torch.int32, device=dev)  # ragged; row 3 partly past the capacity
    kv = torch.zeros(B, cap, cols, dtype=torch.bfloat16, device=dev)
    kv8 = torch.full((B, cap, cols), 0x5A, dtype=torch.uint8, device=dev)
    sc = torch.full((B, cap, cols // 32), 0x33, dtype=torch.uint8, device=dev)
    q1, q2 = qkv.clone(), qkv.clone()
    if T == 1:  # the decode step's append
        ops.kv_append(q1.view(B, -1), kv, length, cos, sin, H, Hkv)
        ops.kv_append(q2.view(B, -1), kv8, length, cos, sin, H, Hkv, kv_scale=sc)
    else:
        ops.kv_append_tokens(q1, kv, length, cos, sin, H, Hkv)
        ops.kv_append_tokens(q2, kv8, length, cos, sin, H, Hkv, kv_scale=sc)
    assert torch.equal(q1, q2)  # Q rotated in place exactly as the bf16 append rotates it
    pos = length.long().view(B, 1) - T + torch.arange(T, device=dev).view(1, T)
    written = torch.zeros(B, cap, dtype=torch.bool, device=dev)
    for b in range(B):
        for p in pos[b].tolist():
            if 0 <= p < cap:
                written[b, p] = True
    rq, re = Rf.quantize_kv(kv[written])
    assert torch.equal(kv8[written], rq) and torch.equal(sc[written], re)
    assert bool((kv8[~written] == 0x5A).all()) and bool((sc[~written] == 0x33).all())  # every other row left alone


@pytest.mark.gpu
@pytest.mark.parametrize("D,Hkv", [(64, 2), (128, 2), (128, 4)])
def test_prefill_fp8_cache_is_quantize_of_the_bf16_cache(native, D, Hkv):
    model = _model(D, Hkv, None)
    prompts = [list(range(5, 205)), list(range(9, 40)), [3] * 257]  # ragged: S = 384 after padding
    _, c16 = inference.prefill(model, prompts, 512)
    _, c8 = inference.prefill(model, prompts, 512, kv_dtype="fp8")
    S = 384
    q, e = Rf.quantize_kv(c16.kv[:, :, :S])
    assert torch.equal(c8.kv[:, :, :S], q) and torch.equal(c8.kv_scale[:, :, :S], e)
    # strided source, rows straight from ops.kv_quantize: the K|V columns of a fused [B, S, (H + 2Hkv)·D] activation
    H = 512 // D
    qkv = torch.randn(3, S, (H + 2 * Hkv) * D, device=_dev()).to(torch.bfloat16)
    kv8 = torch.empty(3, 640, 2 * Hkv * D, dtype=torch.uint8, device=_dev())
    sc = torch.empty(3, 640, 2 * Hkv * D // 32, dtype=torch.uint8, device=_dev())
    ops.kv_quantize(qkv[..., H * D :], kv8, sc)
    q, e = Rf.quantize_kv(qkv[..., H * D :])
    assert torch.equal(kv8[:, :S], q) and torch.equal(sc[:, :S], e)


# ------------------------------------------------------------------------------------------------------------------- attention
@pytest.mark.gpu
@pytest.mark.parametrize("with_lo", [False, True], ids=["nolo", "lo"])
@pytest.mark.parametrize("window", [0, 1, 100, 1024])
@pytest.mark.parametrize("G", [1, 4, 6, 8, 16])
@pytest.mark.parametrize("D", [64, 128])
def test_decode_attn_fp8_matches_fp64_over_the_dequantised_cache(native, D, G, window, with_lo):
    dev = _dev()
    Hkv = 2
    H, B, cap = G * Hkv, len(LENS), 32768
    q8, e, kvd = _blocky_cache(B, cap, 2 * Hkv * D, D + G + window, dev)
    g = torch.Generator().manual_seed(7)
    q = torch.randn(B, H, D, generator=g).to(dev, torch.bfloat16)
    length = torch.tensor(LENS, dtype=torch.int32, device=dev)
    lo = torch.tensor([int(torch.randint(0, L, (1,), generator=g)) for L in LENS], dtype=torch.int32, device=dev) if with_lo else None
    qkv = torch.cat((q.reshape(B, -1), torch.randn(B, 2 * Hkv * D, device=dev).to(torch.bfloat16)), dim=1).contiguous()
    ref, sc = decode64(q, kvd, length, lo, window)
    policy = ops.decode_attn_splits(B, Hkv, cap)
    for splits in (1, policy, cap // 64 + 3):  # one launch; the policy; more splits than key tiles (the tail splits are empty)
        out = ops.decode_attention(qkv, q8, length, lo, window or None, H, Hkv, splits=splits, kv_scale=e)
        assert_elementwise(out.view(B, H, D), ref, DEC_RTOL, DEC_ATOL, sc, f"splits={splits}")


def _verify64(q, kv, length, lo_q, window):
    """fp64 attention of q [B, T, H, D] by the verify rule, and max|v| over each query's visible keys [B, T, H, 1]."""
    B, T, H, D = q.shape
    cap = kv.shape[1]
    Hkv = kv.shape[2] // (2 * D)
    kf = kv[..., : Hkv * D].double().reshape(B, cap, Hkv, D).repeat_interleave(H // Hkv, dim=2)
    vf = kv[..., Hkv * D :].double().reshape(B, cap, Hkv, D).repeat_interleave(H // Hkv, dim=2)
    pos = length.long().view(B, 1) - T + torch.arange(T, device=q.device).view(1, T)
    start = torch.zeros_like(pos) if lo_q is None else lo_q.long()
    if window:
        start = torch.maximum(start, pos + 1 - window)
    k = torch.arange(cap, device=q.device).view(1, 1, cap)
    vis = (k >= start.unsqueeze(-1)) & (k <= pos.unsqueeze(-1))  # [B, T, cap]
    s = torch.einsum("bthd,bkhd->bthk", q.double(), kf) / math.sqrt(D)
    p = s.masked_fill(~vis.unsqueeze(2), -math.inf).softmax(-1)
    vmax = torch.where(vis.unsqueeze(-1), vf.abs().amax(-1).unsqueeze(1), 0.0).amax(2)  # [B, T, H]
    return torch.einsum("bthk,bkhd->bthd", p, vf), vmax.unsqueeze(-1)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["plain", "window", "lo", "eos"])
@pytest.mark.parametrize("T", [1, 2, 5, 16])
@pytest.mark.parametrize("G", [1, 4, 8, 16])
@pytest.mark.parametrize("D", [64, 128])
def test_verify_attn_fp8_matches_fp64_and_decode_at_t1(native, D, G, T, mode):
    dev = _dev()
    Hkv, cap = 2, 2048
    H = G * Hkv
    lens = [T, T + 1, 64 + T, 700, 2048]
    B = len(lens)
    q8, e, kvd = _blocky_cache(B, cap, 2 * Hkv * D, D * 1000 + G * 10 + T, dev)
    g = torch.Generator(device=dev).manual_seed(T)
    qkv = torch.randn(B, T, (H + 2 * Hkv) * D, device=dev, generator=g).to(torch.bfloat16)
    length = torch.tensor(lens, dtype=torch.int32, device=dev)
    window = 100 if mode == "window" else 0
    lo_q = None
    if mode == "lo":
        lo_q = torch.tensor([0, 1, 30, 500, 1000], dtype=torch.int32, device=dev).view(B, 1).expand(B, T).contiguous()
    elif mode == "eos":  # an EOS among the drafts at t0 - 1 opens a document at the query of t0
        t0 = T // 2
        lo_q = torch.zeros(B, T, dtype=torch.int32, device=dev)
        lo_q[:, t0:] = (length - T + t0).view(B, 1)
    ref, sc = _verify64(qkv.view(B, T, H + 2 * Hkv, D)[:, :, :H], kvd, length, lo_q, window)
    for splits in (1, None, cap // 64 + 3):
        out = ops.verify_attention(qkv, q8, length, lo_q, window, H, Hkv, splits=splits, kv_scale=e)
        assert_elementwise(out.view(B, T, H, D), ref, DEC_RTOL, DEC_ATOL, sc, f"splits={splits}")
        if T == 1:
            dec = ops.decode_attention(qkv.view(B, -1), q8, length, None if lo_q is None else lo_q[:, 0].contiguous(), window, H, Hkv,
                                       splits=splits, kv_scale=e)  # fmt: skip
            assert torch.equal(out.view(B, -1), dec)


@pytest.mark.gpu
@pytest.mark.parametrize("D,G", [(64, 1), (128, 1), (128, 4), (128, 8)])
def test_fp8_error_against_bf16_cache_within_the_analytic_bound(native, D, G):
    """One layer's attention over the e4m3 cache against the bf16 cache it was quantised from, same q.

    e4m3 keeps 3 mantissa bits: a normal value is rounded with relative error <= 2^-4 and a subnormal one (|x| < 2^-6·s) with
    absolute error <= 2^-10·s, s the block's scale. So |Δk_j| <= max(2^-4·|k_j|, 2^-10·s_j) =: r_j, and the score of key i moves by
    at most δ_i = Σ_j |q_j|·r_ij / sqrt(D); let δ = max_i δ_i over the visible keys. Every softmax weight then moves by a factor in
    [e^-2δ, e^2δ] (numerator and normaliser each by at most e^δ), so Σ_i |p'_i − p_i| <= e^2δ − 1 and the output moves by at most
    (e^2δ − 1)·max|v|. V's own rounding adds at most max_i |Δv_i| <= 2^-4·max|v| (as 2^-10·s < 2^-4·amax of the block, s <= amax /
    224). Both kernels then round their output to bf16 and carry the fp32 error of ``test_kv_cache.py``'s rule, twice:

        |out_fp8 − out_bf16| <= (e^2δ − 1 + 2^-4)·max|v| + 2·(DEC_RTOL·|out_bf16| + DEC_ATOL·max|v|)
    """
    dev = _dev()
    Hkv, cap = 4, 8192
    H, lens = G * Hkv, [1, 100, 4000, 8192]
    B = len(lens)
    cols = 2 * Hkv * D
    g = torch.Generator(device=dev).manual_seed(D + G)
    kv = (torch.randn(B, cap, cols, device=dev, generator=g) * 2).to(torch.bfloat16)
    q8, e = Rf.quantize_kv(kv)
    qkv = torch.randn(B, (H + 2 * Hkv) * D, device=dev, generator=g).to(torch.bfloat16)
    length = torch.tensor(lens, dtype=torch.int32, device=dev)
    a16 = ops.decode_attention(qkv, kv, length, None, None, H, Hkv).view(B, H, D).double()
    a8 = ops.decode_attention(qkv, q8, length, None, None, H, Hkv, kv_scale=e).view(B, H, D).double()
    s = (e.to(torch.int32) - 127).double().exp2().repeat_interleave(32, dim=-1)  # [B, cap, cols]
    kd = kv.double()
    r = torch.maximum(2.0**-4 * kd.abs(), 2.0**-10 * s)[..., : Hkv * D].reshape(B, cap, Hkv, 1, D)
    q = qkv.view(B, H + 2 * Hkv, D)[:, :H].double().abs().view(B, 1, Hkv, G, D)
    vis = (torch.arange(cap, device=dev).view(1, cap) < length.view(B, 1)).view(B, cap, 1, 1)
    delta = torch.where(vis, (q * r).sum(-1) / math.sqrt(D), 0.0).amax(1).reshape(B, H, 1)  # [B, H, 1]
    vmax = torch.where(vis, kd[..., Hkv * D :].abs().reshape(B, cap, Hkv, D).amax(-1, keepdim=True), 0.0).amax(1)  # [B, Hkv, 1]
    vmax = vmax.repeat_interleave(G, dim=1)
    bound = (torch.expm1(2 * delta) + 2.0**-4) * vmax + 2 * (DEC_RTOL * a16.abs() + DEC_ATOL * vmax)
    err = (a8 - a16).abs()
    print(f"[fp8 vs bf16 cache] D={D} G={G}: max δ = {float(delta.max()):.3f}, max|Δ| / bound = {float((err / bound).max()):.3f}")
    assert bool((err <= bound).all())


# -------------------------------------------------------------------------------------------------------------------- graphs
@pytest.mark.gpu
@torch.no_grad()
def test_graph_replay_with_fp8_cache_is_bitwise_eager_and_deterministic(native):
    dev = _dev()
    model = _model(128, 2, 64)
    model.doc_eos_id = 7
    prompts = [list(range(3, 100)), list(range(5, 30)) + [7, 8, 9]]
    g = torch.Generator().manual_seed(0)
    feed = torch.randint(0, 2048, (70, 2), generator=g)
    feed[10, 0] = feed[20, 1] = 7

    def run(graph: bool):
        _, cache = inference.prefill(model, prompts, 256, kv_dtype="fp8")
        step = inference.GraphDecoder(model, cache) if graph else (lambda t: model.decode_step(t, cache))
        return [step(feed[i].to(dev)).clone() for i in range(feed.shape[0])]

    eager, replay, eager2 = run(False), run(True), run(False)
    for i in range(feed.shape[0]):
        assert torch.equal(eager[i], replay[i]), f"step {i}"
        assert torch.equal(eager[i], eager2[i]), f"step {i}"


@pytest.mark.gpu
@pytest.mark.parametrize("sampler", ["host", "device"])
def test_generate_fp8_on_cuda_uses_graphs_and_matches_eager(native, sampler):
    model = _model(64, 2, None)
    prompts = [list(range(3, 40)), [11, 12]]
    a = inference.generate_batch(model, prompts, max_new=40, sampler=sampler, kv_dtype="fp8")
    b = inference.generate_batch(model, prompts, max_new=40, graphs=False, sampler=sampler, kv_dtype="fp8")
    assert a == b and all(len(r) == len(p) + 40 for r, p in zip(a, prompts))


def _spec_pair(dev):
    t = build_model("debugmodel", device=dev, seed=1, n_heads=4)  # D = 64: the native kernels
    d = build_model("debugmodel", device=dev, seed=2, n_heads=4, n_layers=1)
    return t, d


@pytest.mark.gpu
@pytest.mark.parametrize("knobs", [dict(temperature=0.0), dict(temperature=1.0, top_p=0.9)], ids=["greedy", "topp"])
def test_captured_round_with_fp8_caches_equals_eager_round(native, knobs):
    t, d = _spec_pair(_dev())
    t.doc_eos_id = d.doc_eos_id = 17
    prompts = [[5, 17, 9, 4], [3] * 20, [17, 17, 2]]
    a = inference.generate_speculative(t, d, prompts, k=3, max_new=40, graphs=True, seed=9, kv_dtype="fp8", **knobs)
    b = inference.generate_speculative(t, d, prompts, k=3, max_new=40, graphs=False, seed=9, kv_dtype="fp8", **knobs)
    assert a == b


@pytest.mark.gpu
@pytest.mark.parametrize("temperature,floor", [(0.0, 0.98), (1.0, 0.95)])
def test_self_draft_with_fp8_caches_accepts_nearly_everything(native, temperature, floor):
    t, _ = _spec_pair(_dev())
    prompts = [[1 + (7 * b + j) % 2000 for j in range(5 + 3 * b)] for b in range(8)]
    r = inference.generate_speculative(t, t, prompts, k=4, max_new=64, temperature=temperature, seed=3, kv_dtype="fp8")
    assert r.accepted >= floor * r.drafted, (r.accepted, r.drafted)


# ------------------------------------------------------------------------------------------------------- model level, reported
@pytest.mark.gpu
@torch.no_grad()
@pytest.mark.parametrize("type_model", ["llama2", "llama3"])
def test_fp8_cache_on_1b_shape_models_reported(native, type_model):
    """Teacher forcing through prefill (1024 tokens) and 128 decode steps of a random-init 1B-shape model (llama2: 16 heads MHA;
    llama3: 16 query heads over 8 KV heads), fp8 cache against bf16 cache: the logit error and the greedy-token agreement.
    Recorded in DESIGN.md §1.5; asserted only loosely."""
    dev = _dev()
    model = build_model("1B", type_model, device=dev, seed=0, **({"n_kv_heads": 8} if type_model == "llama3" else {})).eval()
    seq = _doc_seq(2, 1024 + 128, model.args.vocab_size, None, seed=5).to(dev)
    P = 1024

    def run(kv_dtype):
        logits, cache = inference.prefill(model, [seq[b, :P].tolist() for b in range(2)], P + 128, kv_dtype)
        got = [logits.float()]
        for t in range(P, seq.shape[1] - 1):
            got.append(model.decode_step(seq[:, t].contiguous(), cache).float())
        return torch.stack(got, dim=1)

    a16, a8 = run("bf16"), run("fp8")
    err = float((a8 - a16).abs().max() / a16.abs().max())
    agree = float((a8.argmax(-1) == a16.argmax(-1)).float().mean())
    print(f"[fp8 cache, 1B {type_model}] max|Δlogit| / max|logit| = {err:.3e}, greedy agreement = {agree:.4f}")
    assert math.isfinite(err) and err < 0.25 and agree > 0.5
