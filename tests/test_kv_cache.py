"""KV-cache generation: the decode kernels (``csrc/decode_sm90.cu``) against an fp64 oracle, prefill and decode steps against the full
forward, CUDA-graph replay, and ``eval.generate`` against the recompute loop it replaced.

Decode attention is checked element by element with one rule, as in ``test_kernel_edges_gpu.py``:

    |got - ref| <= rtol·|ref| + atol_frac·scale

where ``ref`` is fp64 attention computed from the exact bf16 cache and query the kernel read, and ``scale`` is max|v| over the keys
the row sees (the output is a convex combination of those V rows). The CPU tests at the top apply one plausible kernel bug to a
correct result and show that the same rule rejects it.
"""

import math

import pytest
import torch

from prime_b200 import eval as ev
from prime_b200 import inference, ops
from prime_b200.models.llama import ModelArgs, Transformer, build_model
from prime_b200.ops import reference as Rf

U = 2.0**-8  # bf16 unit roundoff
# one bf16 rounding of the output, plus fp32 relative error of the final division and the exp2 of the split / warp merges
DEC_RTOL = U + 2.0**-16
# fp32 accumulation of sum(p·v) and sum(p): at most 4096 serial terms per lane group (32768 keys in one split over 8 lane groups),
# <= 4096·2^-24 = 2^-12 of max|v|; doubled for ex2.approx and the rounding of the fp32 scores (q pre-scaled by scale·log2 e)
DEC_ATOL = 2.0**-11
ROPE_RTOL = U  # one bf16 rounding of the rotated pair
ROPE_ATOL = 2.0**-22  # a·c - b·s in fp32 cancels: error <= 2^-23·(|a| + |b|)


def decode64(q, kv, length, lo, window):
    """fp64 oracle: q [B, H, D], kv [B, cap, 2·Hkv·D] → (out [B, H, D], scale [B, H, 1] = max|v| over the visible keys)."""
    B, H, D = q.shape
    Hkv = kv.shape[2] // (2 * D)
    G = H // Hkv
    out = torch.zeros((B, H, D), dtype=torch.float64, device=q.device)
    scale = torch.zeros((B, H, 1), dtype=torch.float64, device=q.device)
    for b in range(B):
        L = int(length[b])
        s = max(int(lo[b]) if lo is not None else 0, L - window if window else 0, 0)
        if s >= L:
            continue
        k = kv[b, s:L, : Hkv * D].double().view(-1, Hkv, D)
        v = kv[b, s:L, Hkv * D :].double().view(-1, Hkv, D)
        qq = q[b].double().view(Hkv, G, D)
        p = (torch.einsum("kgd,nkd->kgn", qq, k) / math.sqrt(D)).softmax(-1)
        out[b] = torch.einsum("kgn,nkd->kgd", p, v).reshape(H, D)
        scale[b] = v.abs().amax(dim=(0, 2)).repeat_interleave(G).view(H, 1)
    return out, scale


def assert_elementwise(got, ref, rtol, atol_frac, scale, what):
    g, r = got.double(), ref.double().to(got.device)
    bound = rtol * r.abs() + atol_frac * scale.to(got.device)
    err = (g - r).abs()
    ok = err <= bound
    if not bool(ok.all()):
        i = int(torch.argmax(torch.where(ok, torch.zeros_like(err), err / bound).nan_to_num(math.inf)))
        idx = tuple(int(v) for v in torch.unravel_index(torch.tensor(i), g.shape))
        raise AssertionError(f"{what}: {int((~ok).sum())} of {g.numel()} out of bound; worst at {idx}: got {float(g.reshape(-1)[i])!r} "
                             f"ref {float(r.reshape(-1)[i])!r} bound {float(bound.expand_as(g).reshape(-1)[i]):.3e}")


def _rejects(got, ref, rtol, atol, scale) -> bool:
    try:
        assert_elementwise(got, ref, rtol, atol, scale, "mutant")
    except AssertionError:
        return True
    return False


def rope64_rows(x, pos, cos, sin):
    """x [B, heads, D] rotated at per-row positions, fp64, and the |a| + |b| pair magnitudes."""
    B, Hh, D = x.shape
    xf = x.double().reshape(B, Hh, D // 2, 2)
    c, s = cos[pos].double().view(B, 1, D // 2), sin[pos].double().view(B, 1, D // 2)
    a, b = xf[..., 0], xf[..., 1]
    out = torch.stack((a * c - b * s, a * s + b * c), dim=-1).reshape(x.shape)
    pair = (a.abs() + b.abs()).unsqueeze(-1).expand(*a.shape, 2).reshape(x.shape)
    return out, pair


def _cache(B, cap, H, Hkv, D, lens, dev, seed=0, dtype=torch.bfloat16):
    g = torch.Generator(device="cpu").manual_seed(seed)
    q = torch.randn(B, H, D, generator=g).to(dev, dtype)
    kv = torch.randn(B, cap, 2 * Hkv * D, generator=g).to(dev, dtype)
    return q, kv, torch.tensor(lens, dtype=torch.int32, device=dev)


# -------------------------------------------------------------------------------------------------- CPU: reference and model
@pytest.mark.parametrize("window,eos", [(3, None), (None, 9), (4, 9), (1, 9), (50, None), (50, 9)],
                         ids=["window", "docs", "window+docs", "w1", "w>=len", "w>=len+docs"])  # fmt: skip
def test_reference_decode_attention_is_full_attention_at_the_last_query(window, eos):
    torch.manual_seed(0)
    H, Hkv, D = 4, 2, 16
    tokens = torch.tensor([[1, 2, 9, 4, 5, 6, 9, 8, 3, 2, 1, 7], [9, 3, 3, 3, 9, 9, 1, 2, 3, 4, 5, 6], [5] * 12])
    B, S = tokens.shape
    q, k, v = (torch.randn(B, S, h, D) for h in (H, Hkv, Hkv))
    doc_start, _ = Rf.document_bounds(tokens, eos, window)
    full = Rf.attention(q, k, v, causal=True, doc_start=doc_start)
    kv = torch.cat((k.reshape(B, S, -1), v.reshape(B, S, -1)), dim=-1)
    for L in (1, 5, 8, S):
        lo, _ = Rf.document_bounds(tokens[:, :L], eos)  # documents only: the window is the decode op's own argument
        got = Rf.decode_attention(q[:, L - 1], kv, torch.full((B,), L), lo[:, L - 1], window)
        torch.testing.assert_close(got, full[:, L - 1], rtol=1e-5, atol=1e-6)


def _teacher_forced(model, seq, P, dev):
    """(max |logit error| / max |logit|) of prefill + decode_step against model.forward over the whole sequence."""
    full = model(seq.to(dev)).float()
    B, T = seq.shape
    logits, cache = inference.prefill(model, [seq[b, :P].tolist() for b in range(B)], inference.cache_capacity(4096, [P], T))
    got = [logits.float()]
    for t in range(P, T):
        got.append(model.decode_step(seq[:, t].to(dev), cache).float())
    got = torch.stack(got, dim=1)
    return float((got - full[:, P - 1 :]).abs().max() / full.abs().max())


def _doc_seq(B, T, V, eos, seed):
    g = torch.Generator().manual_seed(seed)
    seq = torch.randint(0, V, (B, T), generator=g)
    if eos is not None:
        seq[seq == eos] = eos + 1
        seq[0, 5] = seq[1, 3] = eos  # inside the prompt
        seq[0, T - 12] = seq[1, T - 5] = eos  # inside the continuation
    return seq


@pytest.mark.parametrize("variant", ["debugmodel", "gqa_window_docs"])
def test_teacher_forced_decode_matches_full_forward_cpu(variant):
    kw = {} if variant == "debugmodel" else dict(n_kv_heads=2, sliding_window=6)
    model = build_model("debugmodel", device="cpu", dtype=torch.float32, **kw)
    eos = None if variant == "debugmodel" else 7
    model.doc_eos_id = eos
    seq = _doc_seq(2, 40, model.args.vocab_size, eos, seed=1)
    assert _teacher_forced(model, seq, 12, "cpu") <= 1e-4


def test_greedy_generate_equals_recompute_and_batch_rows_equal_single_runs():
    model = build_model("debugmodel", device="cpu", dtype=torch.float32)
    prompts = [[5, 9, 100, 3], [7] * 11, [1, 2]]
    one = ev.generate(model, prompts[0], max_new=24)
    assert one == ev._generate_recompute(model, prompts[0], max_new=24)
    batch = ev.generate_batch(model, prompts, max_new=24)
    assert batch == [ev._generate_recompute(model, p, max_new=24) for p in prompts]
    assert batch == [ev.generate(model, p, max_new=24) for p in prompts]


def test_generate_stop_rules_match_recompute():
    model = build_model("debugmodel", device="cpu", dtype=torch.float32, max_seq_len=20)
    prompts = [[5, 9, 100, 3], [7] * 17]
    batch = ev.generate_batch(model, prompts, max_new=30)
    assert [len(r) for r in batch] == [20, 20]
    assert batch == [ev._generate_recompute(model, p, max_new=30) for p in prompts]
    first = ev._generate_recompute(model, prompts[0], max_new=30)[4]
    assert ev.generate(model, prompts[0], max_new=30, eos_id=first) == prompts[0] + [first]


def test_seeded_sampling_is_reproducible_and_equals_recompute():
    model = build_model("debugmodel", device="cpu", dtype=torch.float32)
    p = [5, 9, 100, 3]
    kw = dict(max_new=20, temperature=0.8, top_k=40, seed=11)
    a = ev.generate(model, p, **kw)
    assert a == ev.generate(model, p, **kw) == ev._generate_recompute(model, p, **kw)
    assert a != ev.generate(model, p, **{**kw, "seed": 12})


def test_decode_launchers_reject_impossible_arguments_before_touching_the_device():
    from prime_b200.ops import _lib

    try:
        lib = _lib.load()
    except Exception as e:  # noqa: BLE001
        pytest.skip(f"native library not loadable here: {e}")
    a = 1 << 20  # 16-byte aligned, never dereferenced: every call below is rejected first
    odd = a + 2

    def adv(tokens=a, len_=a, lo=a, last=a, B=4):
        return lib.pb_decode_advance(tokens, -1, len_, lo, last, B, None)

    assert adv(tokens=None) == -1 and adv(last=None) == -1 and adv(B=0) == -3 and adv(last=odd) == -6

    def app(qkv=a, kv=a, len_=a, cos=a, B=2, H=8, Hkv=2, D=128, cap=256):
        return lib.pb_kv_append(qkv, kv, len_, cos, a, B, H, Hkv, D, cap, None)

    assert app(kv=None) == -1 and app(cos=None) == -1 and app(D=96) == -2 and app(H=6, Hkv=4) == -3 and app(cap=0) == -3
    assert app(qkv=odd) == -6 and app(len_=a + 1) == -6

    def attn(qkv=a, kv=a, len_=a, lo=None, window=0, out=a, part=None, H=8, Hkv=2, D=64, cap=256, splits=1):
        return lib.pb_decode_attn(qkv, kv, len_, lo, window, out, part, 2, H, Hkv, D, cap, splits, 0.125, None)

    assert attn(len_=None) == -1 and attn(out=None) == -1 and attn(splits=2) == -1  # a split needs the partials workspace
    assert attn(D=32) == -2 and attn(H=6, Hkv=4) == -3 and attn(Hkv=0) == -3 and attn(window=-1) == -4 and attn(splits=0) == -5
    assert attn(kv=odd) == -6 and attn(lo=a + 1) == -6 and attn(out=odd) == -6
    assert lib.pb_decode_attn_splits(0, 8, 1024) == -3 and lib.pb_decode_attn_splits(1, 8, 0) == -3
    assert lib.pb_decode_attn_splits(1, 8, 32768) * 8 >= 132  # one sequence fills the machine at long capacity
    assert lib.pb_decode_attn_splits(32, 8, 128) == 1


# -------------------------------------------------------------------------------------------------- CPU: the rule rejects bugs
def test_checker_rejects_append_rope_position_off_by_one():
    torch.manual_seed(1)
    B, D, heads = 3, 64, 4
    cos, sin = Rf.rope_tables(64, D)
    x = torch.randn(B, heads, D).to(torch.bfloat16)
    pos = torch.tensor([0, 17, 40])
    ref, pair = rope64_rows(x, pos, cos, sin)
    assert not _rejects(Rf.rope_at(x, cos[pos], sin[pos]), ref, ROPE_RTOL, ROPE_ATOL, pair)
    assert _rejects(Rf.rope_at(x, cos[pos + 1], sin[pos + 1]), ref, ROPE_RTOL, ROPE_ATOL, pair)


def _attn_case():
    B, H, Hkv, D, cap = 3, 8, 2, 128, 1024
    q, kv, length = _cache(B, cap, H, Hkv, D, [1000, 300, 777], "cpu", seed=2)
    lo = torch.tensor([0, 120, 500], dtype=torch.int32)
    return q, kv, length, lo


def _rounded(q, kv, length, lo, window):
    return Rf.decode_attention(q, kv, length, lo, window).to(torch.bfloat16)


def test_checker_rejects_window_bound_off_by_one():
    q, kv, length, lo = _attn_case()
    ref, sc = decode64(q, kv, length, lo, 100)
    assert not _rejects(_rounded(q, kv, length, lo, 100), ref, DEC_RTOL, DEC_ATOL, sc)
    assert _rejects(_rounded(q, kv, length, lo, 101), ref, DEC_RTOL, DEC_ATOL, sc)
    assert _rejects(_rounded(q, kv, length, lo, 99), ref, DEC_RTOL, DEC_ATOL, sc)


def test_checker_rejects_combine_dropping_the_last_split():
    q, kv, length, lo = _attn_case()
    ref, sc = decode64(q, kv, length, lo, None)
    assert not _rejects(_rounded(q, kv, length, lo, None), ref, DEC_RTOL, DEC_ATOL, sc)
    # splits of 256 keys: the last split of each row holds its keys from floor((len - 1) / 256) * 256 on
    last_split = (length - 1) // 256 * 256
    assert _rejects(_rounded(q, kv, torch.maximum(last_split, lo + 1), lo, None), ref, DEC_RTOL, DEC_ATOL, sc)


def test_checker_rejects_row_reading_another_rows_length():
    q, kv, length, lo = _attn_case()
    ref, sc = decode64(q, kv, length, lo, None)
    wrong = length[[0, 2, 1]]  # rows 1 and 2 swap lengths
    assert _rejects(_rounded(q, kv, wrong, lo, None), ref, DEC_RTOL, DEC_ATOL, sc)


# -------------------------------------------------------------------------------------------------- GPU
def _dev():
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def native():
    from prime_b200.ops import _lib

    return _lib.load()  # a GPU box without the native library is a hard failure, never a silent fallback


LENS = [1, 2, 63, 64, 65, 127, 128, 129, 1000, 4096, 32768]


@pytest.mark.gpu
@pytest.mark.parametrize("with_lo", [False, True], ids=["nolo", "lo"])
@pytest.mark.parametrize("window", [0, 1, 100, 1024])
# G = 6: one chunk of 8 heads with two zeroed padding heads; G = 16: two chunks of 8 (h0 = hk·G + c·8)
@pytest.mark.parametrize("G", [1, 4, 6, 8, 16])
@pytest.mark.parametrize("D", [64, 128])
def test_decode_attn_matches_fp64(native, D, G, window, with_lo):
    dev = _dev()
    Hkv = 2
    H, B, cap = G * Hkv, len(LENS), 32768
    q, kv, length = _cache(B, cap, H, Hkv, D, LENS, dev, seed=D + G + window)
    g = torch.Generator().manual_seed(7)
    lo = torch.tensor([int(torch.randint(0, L, (1,), generator=g)) for L in LENS], dtype=torch.int32, device=dev) if with_lo else None
    qkv = torch.cat((q.reshape(B, -1), torch.randn(B, 2 * Hkv * D, device=dev).to(torch.bfloat16)), dim=1).contiguous()
    ref, sc = decode64(q, kv, length, lo, window)
    policy = ops.decode_attn_splits(B, Hkv, cap)
    for splits in (1, policy, cap // 64 + 3):  # one launch; the policy; more splits than key tiles (the tail splits are empty)
        out = ops.decode_attention(qkv, kv, length, lo, window or None, H, Hkv, splits=splits)
        assert_elementwise(out.view(B, H, D), ref, DEC_RTOL, DEC_ATOL, sc, f"splits={splits}")


@pytest.mark.gpu
@pytest.mark.parametrize("D", [64, 128])
def test_kv_append_rotates_at_ragged_positions(native, D):
    dev = _dev()
    B, H, Hkv, cap = 5, 8, 2, 384
    cos, sin = Rf.rope_tables(cap, D, 500000.0, device=dev)
    length = torch.tensor([1, 2, 129, 300, cap], dtype=torch.int32, device=dev)
    qkv = torch.randn(B, (H + 2 * Hkv) * D, device=dev).to(torch.bfloat16)
    kv = torch.randn(B, cap, 2 * Hkv * D, device=dev).to(torch.bfloat16)
    qkv0, kv0 = qkv.clone(), kv.clone()
    ops.kv_append(qkv, kv, length, cos, sin, H, Hkv)
    pos = length.long() - 1
    x = qkv0.view(B, H + 2 * Hkv, D)
    ref, pair = rope64_rows(x[:, : H + Hkv], pos, cos, sin)
    rows = torch.arange(B, device=dev)
    assert_elementwise(qkv.view(B, -1, D)[:, :H], ref[:, :H], ROPE_RTOL, ROPE_ATOL, pair[:, :H], "q")
    assert_elementwise(kv[rows, pos, : Hkv * D].view(B, Hkv, D), ref[:, H:], ROPE_RTOL, ROPE_ATOL, pair[:, H:], "k")
    assert torch.equal(kv[rows, pos, Hkv * D :], x[:, H + Hkv :].reshape(B, -1))  # V copied
    assert torch.equal(qkv.view(B, -1, D)[:, H:], x[:, H:])  # K / V of the activation untouched
    untouched = torch.ones(B, cap, dtype=torch.bool, device=dev)
    untouched[rows, pos] = False
    assert torch.equal(kv[untouched], kv0[untouched])


@pytest.mark.gpu
def test_decode_advance_bookkeeping_across_eos(native):
    dev = _dev()
    eos = 3
    steps = torch.tensor([[5, 3, 7, 8], [3, 3, 1, 2], [9, 9, 9, 3]])
    length, lo, last = [4, 1, 7], [2, 0, 0], [3, 6, 3]
    gpu = [torch.tensor(length, dtype=torch.int32, device=dev), torch.tensor(lo, dtype=torch.int32, device=dev), torch.tensor(last, device=dev)]
    for t in range(steps.shape[1]):
        ops.decode_advance(steps[:, t].to(dev), *gpu, eos)
        for b in range(3):  # the token after an EOS starts a document at its own position
            lo[b] = length[b] if last[b] == eos else lo[b]
            length[b] += 1
            last[b] = int(steps[b, t])
        assert gpu[0].tolist() == length and gpu[1].tolist() == lo and gpu[2].tolist() == last
    # rows 0 and 2 start after an EOS; row 0's EOS at step 1 and row 1's at steps 0 and 1 move lo one step later; row 2's EOS at
    # the last step has not moved it yet
    assert lo == [6, 3, 7]


def _model(D, Hkv, window, seed=0):
    args = ModelArgs(dim=512, n_layers=2, n_heads=512 // D, n_kv_heads=Hkv, vocab_size=2048, max_seq_len=1024, sliding_window=window)
    with torch.device(_dev()):
        m = Transformer(args)
    m.to(torch.bfloat16)
    m.init_weights(seed)
    return m.eval()


@pytest.mark.gpu
@torch.no_grad()
def test_prefill_is_forward_hidden_bitwise(native):
    dev = _dev()
    model = _model(128, 2, None)
    prompts = [list(range(5, 205)), list(range(9, 40)), list(range(1, 257))]
    S = 256
    tokens = torch.zeros((3, S), dtype=torch.int64, device=dev)
    for b, p in enumerate(prompts):
        tokens[b, : len(p)] = torch.tensor(p)
    seen = []
    hooks = [layer.attention.register_forward_hook(lambda mod, inp, out: seen.append(inp[0].clone())) for layer in model.layers]
    cache = inference.KVCache.allocate(model, 3, 512, dev)
    h_cache = model.forward_hidden(tokens, cache)
    for h in hooks:
        h.remove()
    h_plain = model.forward_hidden(tokens)
    assert torch.equal(h_cache, h_plain)
    a = model.args
    cos, sin = model.rope_tables(S, dev)
    for i, x in enumerate(seen):
        qkv = ops.linear_qkv_rope(x, model.layers[i].attention.wqkv, cos, sin, a.n_heads, a.kv_heads)
        assert torch.equal(cache.kv[i][:, :S], qkv[..., a.n_heads * a.head_dim :])
    logits, _ = inference.prefill(model, prompts, 512)
    full = model(tokens).float()
    ref = full[torch.arange(3), torch.tensor([len(p) - 1 for p in prompts])]
    # the LM head runs at M = 3 instead of M = 768: the fp32 sums may round to the neighbouring bf16 value
    assert_elementwise(logits.float(), ref, 2.0**-7, 2.0**-12, ref.abs().amax(-1, keepdim=True), "prefill logits")


# bf16 through two layers: flash attention rounds P to bf16 before P·V while decode attention keeps it in fp32, and the difference
# is carried through the residual stream and the LM head; 2^-5 of max|logit| is about eight bf16 roundings of the largest logit
TEACHER_TOL = 2.0**-5


@pytest.mark.gpu
@pytest.mark.parametrize("D,window,eos", [(64, None, None), (128, None, None), (64, 48, 7), (128, 48, 7)],
                         ids=["d64", "d128", "d64-window-docs", "d128-window-docs"])  # fmt: skip
def test_teacher_forced_decode_matches_forward_bf16(native, D, window, eos):
    model = _model(D, 2, window)
    model.doc_eos_id = eos
    seq = _doc_seq(2, 256, 2048, eos, seed=D)
    with torch.no_grad():
        err = _teacher_forced(model, seq, 150, _dev())
    print(f"[teacher forcing] D={D} window={window} eos={eos}: max|err| / max|logit| = {err:.2e}")
    assert err <= TEACHER_TOL


@pytest.mark.gpu
@torch.no_grad()
def test_graph_replay_is_bitwise_eager_and_deterministic(native):
    dev = _dev()
    model = _model(128, 2, 64)
    model.doc_eos_id = 7
    prompts = [list(range(3, 100)), list(range(5, 30)) + [7, 8, 9]]
    g = torch.Generator().manual_seed(0)
    feed = torch.randint(0, 2048, (70, 2), generator=g)
    feed[10, 0] = feed[20, 1] = 7

    def run(graph: bool):
        _, cache = inference.prefill(model, prompts, 256)
        step = inference.GraphDecoder(model, cache) if graph else (lambda t: model.decode_step(t, cache))
        return [step(feed[i].to(dev)).clone() for i in range(feed.shape[0])]

    eager, replay, eager2 = run(False), run(True), run(False)
    for i in range(feed.shape[0]):
        assert torch.equal(eager[i], replay[i]), f"step {i}"
        assert torch.equal(eager[i], eager2[i]), f"step {i}"


@pytest.mark.gpu
def test_generate_on_cuda_uses_graphs_and_matches_eager(native):
    model = _model(64, 2, None)
    prompts = [list(range(3, 40)), [11, 12]]
    a = ev.generate_batch(model, prompts, max_new=40)
    b = ev.generate_batch(model, prompts, max_new=40, graphs=False)
    assert a == b and all(len(r) == len(p) + 40 for r, p in zip(a, prompts))


@pytest.mark.gpu
def test_generate_on_cuda_with_head_dim_the_kernels_do_not_take(native):
    """debugmodel (D = 32) on CUDA: append and decode attention take the plain-torch fallbacks, which must be capturable too."""
    model = build_model("debugmodel", device="cuda", dtype=torch.bfloat16).eval()
    assert model.args.head_dim == 32
    prompts = [list(range(3, 40)), [11, 12]]
    a = ev.generate_batch(model, prompts, max_new=24)
    assert a == ev.generate_batch(model, prompts, max_new=24, graphs=False)
    assert a[1] == ev.generate(model, prompts[1], max_new=24)
    # the first token comes from the prompt's logits, computed by the same kernels as the recompute loop's (the LM head at another M)
    assert [r[len(p)] for r, p in zip(a, prompts)] == [ev._generate_recompute(model, p, max_new=1)[-1] for p in prompts]
    seq = _doc_seq(2, 200, model.args.vocab_size, None, seed=3)
    with torch.no_grad():
        err = _teacher_forced(model, seq, 130, _dev())
    print(f"[teacher forcing] debugmodel D=32 (fallback ops): max|err| / max|logit| = {err:.2e}")
    assert err <= TEACHER_TOL
