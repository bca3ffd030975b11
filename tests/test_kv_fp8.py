"""The e4m3 KV cache on the CPU: the quantiser against the MXFP8 one, the checker of ``test_kv_cache.py`` against plausible fp8 bugs,
generation, speculative decoding and the CLI with ``kv_dtype="fp8"``, and bad input refused before any device work."""

import pytest
import torch
from test_kv_cache import DEC_ATOL, DEC_RTOL, _doc_seq, _rejects, decode64

from prime_b200 import eval as ev
from prime_b200 import inference
from prime_b200.models.llama import build_model
from prime_b200.ops import reference as Rf


def _blocky(shape, seed, spread=4):
    """Random values whose 32-column blocks have different magnitudes (powers of two in 2^-spread .. 2^spread), so that the blocks'
    exponents differ and a scale taken from the wrong block changes the result."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(*shape, generator=g)
    mag = 2.0 ** torch.randint(-spread, spread + 1, (*shape[:-1], shape[-1] // 32, 1), generator=g).float()
    return (x.view(*shape[:-1], -1, 32) * mag).view(shape)


# ------------------------------------------------------------------------------------------------------------- the quantiser
def test_quantize_kv_is_the_mxfp8_rule():
    x = _blocky((300, 512), seed=0).to(torch.bfloat16)
    q, e = Rf.quantize_kv(x)
    qm, sf = Rf.quantize_mxfp8(x)
    assert q.dtype == e.dtype == torch.uint8 and e.shape == (300, 16)
    assert torch.equal(q, qm)
    assert torch.equal(e, sf[Rf._mxfp8_sf_index(300, 512).reshape(-1)].view(300, 16))
    assert torch.equal(Rf.dequantize_kv(q, e), Rf.dequantize_mxfp8(qm, sf))


def test_dequantized_values_round_trip_through_bf16():
    x = _blocky((4, 64, 256), seed=1, spread=20) * 1e3  # a wide exponent range
    q, e = Rf.quantize_kv(x)
    d = Rf.dequantize_kv(q, e)
    assert torch.equal(d.to(torch.bfloat16).float(), d)
    assert bool(((d - x).abs() <= 2.0**-4 * x.view(4, 64, 8, 32).abs().amax(-1, keepdim=True).expand(4, 64, 8, 32).reshape(x.shape)).all())


def test_all_zero_block_gets_exponent_one():
    x = torch.randn(2, 96)
    x[0, 32:64] = 0
    q, e = Rf.quantize_kv(x)
    assert int(e[0, 1]) == 1 and int(q[0, 32:64].abs().sum()) == 0
    assert bool((e[0, [0, 2]] > 1).all())


# ------------------------------------------------------------------------------------------------- the checker rejects fp8 bugs
def _fp8_case():
    B, H, Hkv, D, cap = 3, 8, 2, 128, 1024
    g = torch.Generator().manual_seed(5)
    q = torch.randn(B, H, D, generator=g).to(torch.bfloat16)
    kv = _blocky((B, cap, 2 * Hkv * D), seed=6)
    kv[..., Hkv * D :] *= 8  # V blocks larger than K blocks: K's exponents are wrong for V
    qb, e = Rf.quantize_kv(kv)
    length = torch.tensor([1000, 300, 777], dtype=torch.int32)
    lo = torch.tensor([0, 120, 500], dtype=torch.int32)
    return q, qb, e, length, lo


def _attn(q, qb, e, length, lo):
    return Rf.decode_attention(q, Rf.dequantize_kv(qb, e), length, lo, None).to(torch.bfloat16)


@pytest.mark.parametrize("bug", ["neighbour_block_scale", "k_scale_on_v", "scale_off_by_one"])
def test_checker_rejects_fp8_scale_bugs(bug):
    q, qb, e, length, lo = _fp8_case()
    ref, sc = decode64(q, Rf.dequantize_kv(qb, e).to(torch.bfloat16), length, lo, None)  # the dequantised cache is exact in bf16
    assert not _rejects(_attn(q, qb, e, length, lo), ref, DEC_RTOL, DEC_ATOL, sc)
    half = e.shape[-1] // 2
    if bug == "neighbour_block_scale":
        bad = e.roll(1, dims=-1)
    elif bug == "k_scale_on_v":
        bad = torch.cat((e[..., :half], e[..., :half]), dim=-1)
    else:
        bad = e + 1
    assert _rejects(_attn(q, qb, bad, length, lo), ref, DEC_RTOL, DEC_ATOL, sc)


# ----------------------------------------------------------------------------------------------------------------- generation
VARIANTS = {"debugmodel": ({}, None), "gqa_window_docs": (dict(n_kv_heads=2, sliding_window=6), 7)}
# fp8 K and V (relative rounding 2^-4) against the full fp32 forward, through two layers of a random-init debugmodel; measured
# 6.3e-4 and 2.0e-3 of max|logit| for the two variants
FP8_TEACHER_TOL = 2.0**-6


def _teacher_forced_fp8(model, seq, P):
    full = model(seq).float()
    B, T = seq.shape
    logits, cache = inference.prefill(model, [seq[b, :P].tolist() for b in range(B)], inference.cache_capacity(4096, [P], T), "fp8")
    got = [logits.float()]
    for t in range(P, T):
        got.append(model.decode_step(seq[:, t], cache).float())
    return float((torch.stack(got, dim=1) - full[:, P - 1 :]).abs().max() / full.abs().max())


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_fp8_generation_on_the_cpu(variant):
    kw, eos = VARIANTS[variant]
    model = build_model("debugmodel", device="cpu", dtype=torch.float32, **kw)
    model.doc_eos_id = eos
    prompts = [[5, 9, 100, 3], [7] * 11, [1, 2]]
    for sampler in ("host", "device"):
        out = inference.generate_batch(model, prompts, max_new=12, temperature=0.8, top_k=40, seed=3, sampler=sampler, kv_dtype="fp8")
        assert [len(r) for r in out] == [len(p) + 12 for p in prompts] and all(r[: len(p)] == p for r, p in zip(out, prompts))
    cache = inference.KVCache.allocate(model, 2, 128, "cpu", kv_dtype="fp8")
    assert cache.kv.dtype == cache.kv_scale.dtype == torch.uint8
    assert (cache.kv.numel() + cache.kv_scale.numel()) / cache.kv.numel() == 1 + 1 / 32
    with torch.no_grad():
        err = _teacher_forced_fp8(model, _doc_seq(2, 40, model.args.vocab_size, eos, seed=1), 12)
    print(f"[fp8 teacher forcing] {variant}: max|err| / max|logit| = {err:.2e}")
    assert err <= FP8_TEACHER_TOL


def test_greedy_speculation_with_fp8_caches_equals_greedy_generation():
    t = build_model("debugmodel", dtype=torch.float32, seed=1)
    d = build_model("debugmodel", dtype=torch.float32, seed=2, n_layers=1)
    prompts = [[1, 2, 3, 4, 5], [7, 8, 9], [10] * 12, [300]]
    ref = inference.generate_batch(t, prompts, max_new=20, sampler="device", kv_dtype="fp8")
    for k in (1, 3):
        for draft in (d, t):
            assert inference.generate_speculative(t, draft, prompts, k=k, max_new=20, kv_dtype="fp8").ids == ref


def test_eval_generate_kv_dtype_fp8_cli(tmp_path):
    from prime_b200.models import hf

    hf.save_hf_dir(build_model("debugmodel", dtype=torch.float32, seed=4), tmp_path / "m")
    hf.save_hf_dir(build_model("debugmodel", dtype=torch.float32, seed=5, n_layers=1), tmp_path / "d")
    base = ["generate", "--hf", str(tmp_path / "m"), "--prompt-ids", "5,9,100,3", "--max-new", "6", "--device", "cpu"]
    out = ev.main(base + ["--kv-dtype", "fp8"])["ids"]
    assert len(out) == 10 and out[:4] == [5, 9, 100, 3]
    spec = ev.main(base + ["--kv-dtype", "fp8", "--sampler", "device", "--draft-hf", str(tmp_path / "d"), "--spec-k", "2"])
    assert spec["ids"] == ev.main(base + ["--kv-dtype", "fp8", "--sampler", "device"])["ids"]  # greedy: the target's own output
    with pytest.raises(SystemExit):
        ev.main(base + ["--kv-dtype", "int8"])


# ------------------------------------------------------------------------------------------------------------------ bad input
def test_bad_kv_dtype_and_head_dim_are_refused():
    m = build_model("debugmodel", dtype=torch.float32)
    with pytest.raises(ValueError, match="kv_dtype"):
        inference.generate_batch(m, [[1, 2]], max_new=2, kv_dtype="fp16")
    with pytest.raises(ValueError, match="kv_dtype"):
        inference.generate_speculative(m, m, [[1, 2]], max_new=2, kv_dtype="e5m2")
    d48 = build_model("debugmodel", dtype=torch.float32, dim=384)  # 8 heads of 48
    assert d48.args.head_dim == 48
    with pytest.raises(ValueError, match="head_dim % 32"):
        inference.generate_batch(d48, [[1, 2]], max_new=2, kv_dtype="fp8")
    with pytest.raises(ValueError, match="head_dim % 32"):
        inference.KVCache.allocate(d48, 1, 128, "cpu", kv_dtype="fp8")
    assert inference.generate_batch(d48, [[1, 2]], max_new=2) is not None  # the bf16 cache takes any head_dim


def test_fp8_launchers_reject_impossible_arguments_before_touching_the_device():
    from prime_b200.ops import _lib

    try:
        lib = _lib.load()
    except Exception as e:  # noqa: BLE001
        pytest.skip(f"native library not loadable here: {e}")
    a = 1 << 20  # 16-byte aligned, never dereferenced: every call below is rejected first

    def app(qkv=a, kv=a, sc=a, B=2, T=3, H=8, Hkv=2, D=128, cap=256):
        return lib.pb_kv_append_fp8(qkv, kv, sc, a, a, a, B, T, H, Hkv, D, cap, None)

    assert app(sc=None) == -1 and app(kv=None) == -1 and app(D=96) == -2 and app(T=0) == -3 and app(H=6, Hkv=4) == -3
    assert app(qkv=a + 8) == -6 and app(kv=a + 4) == -6 and app(sc=a + 2) == -6 and app(sc=a + 1) == -6

    def quant(src=a, ld=1536, kv=a, sc=a, B=2, S=128, cols=512, cap=256):
        return lib.pb_kv_quantize(src, ld, kv, sc, B, S, cols, cap, None)

    assert quant(sc=None) == -1 and quant(src=None) == -1
    assert quant(S=300) == -3 and quant(cols=48) == -3 and quant(ld=256) == -3 and quant(B=0) == -3
    assert quant(src=a + 8) == -6 and quant(ld=1540) == -6 and quant(kv=a + 4) == -6 and quant(sc=a + 2) == -6

    def attn(sc=a, kv=a, lo=None, window=0, out=a, part=None, H=8, Hkv=2, D=64, cap=256, splits=1):
        return lib.pb_decode_attn_fp8(a, kv, sc, a, lo, window, out, part, 2, H, Hkv, D, cap, splits, 0.125, None)

    assert attn(sc=None) == -1 and attn(out=None) == -1 and attn(splits=2) == -1 and attn(D=32) == -2 and attn(H=6, Hkv=4) == -3
    assert attn(window=-1) == -4 and attn(splits=0) == -5 and attn(sc=a + 1) == -6 and attn(kv=a + 4) == -6 and attn(lo=a + 1) == -6

    def ver(sc=a, kv=a, T=5, D=64, splits=1, part=None, window=0):
        return lib.pb_verify_attn_fp8(a, kv, sc, a, None, window, a, part, 2, T, 8, 2, D, 256, splits, 0.125, None)

    assert ver(sc=None) == -1 and ver(splits=2) == -1 and ver(D=48) == -2 and ver(T=0) == -3 and ver(window=-1) == -4
    assert ver(splits=0) == -5 and ver(sc=a + 2) == -6 and ver(kv=a + 2) == -6
