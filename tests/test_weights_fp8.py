"""e4m3 inference weights on the CPU: what ``inference.quantize_weights`` converts and refuses, exact equality of a quantised model
with the model holding W̃ through prefill, both samplers, both cache dtypes and speculation, the inference-only guard, the
launchers' argument checks, and the CLI."""

import copy
import json

import pytest
import torch

from prime_b200 import eval as ev
from prime_b200 import inference, ops
from prime_b200.models.llama import build_model
from prime_b200.ops import reference as Rf


def _pair(seed=0, **kw):
    """A quantised fp32 debugmodel and a copy whose projections hold W̃ (exact in fp32)."""
    q = build_model("debugmodel", dtype=torch.float32, seed=seed, **kw).eval()
    ref = copy.deepcopy(q)
    inference.quantize_weights(q)
    with torch.no_grad():
        for (m, n), (rm, _) in zip(inference._projections(q), inference._projections(ref)):
            getattr(rm, n).copy_(ops.dequantize_weight(getattr(m, n)))
    return q, ref


PROMPTS = [[1, 2, 3, 4, 5], [7, 8, 9], [100 + j for j in range(20)]]


def test_quantize_weights_replaces_exactly_the_projections():
    m = build_model("debugmodel", dtype=torch.float32, seed=0)
    before = {n: p.detach().clone() for n, p in m.named_parameters()}
    inference.quantize_weights(m)
    after = dict(m.named_parameters())
    assert set(after) == {n for n in before if n == "tok_embeddings.weight" or n.endswith("norm.weight")}
    for n, p in after.items():
        assert torch.equal(p, before[n]), n
    kinds = {"attention.wqkv", "attention.wo", "feed_forward.w13", "feed_forward.w2"}
    for i, blk in enumerate(m.layers):
        for k in kinds:
            mod, attr = k.split(".")
            w = getattr(getattr(blk, mod), attr)
            assert isinstance(w, ops.MXWeight) and w.dtype == torch.float32
            q, sf = Rf.quantize_mxfp8(before[f"layers.{i}.{k}"])
            assert torch.equal(w.q, q) and torch.equal(w.sf, sf)
    assert isinstance(m.output, ops.MXWeight) and m.output.shape == before["output"].shape and m.output.device.type == "cpu"


def test_quantize_weights_refuses_what_it_cannot_convert():
    with pytest.raises(ValueError, match="128"):
        inference.quantize_weights(build_model("10M", dtype=torch.float32, seed=0, vocab_size=256))
    m = build_model("debugmodel", dtype=torch.float32, seed=0)
    m.set_fp8(True)
    with pytest.raises(ValueError, match="set_fp8"):
        inference.quantize_weights(m)
    m = build_model("debugmodel", dtype=torch.float32, seed=0)
    m.layers[0].attention.wo.z3 = object()
    with pytest.raises(ValueError, match="ZeRO-3"):
        inference.quantize_weights(m)
    m = build_model("debugmodel", dtype=torch.float32, seed=0)
    inference.quantize_weights(m)
    with pytest.raises(ValueError, match="already"):
        inference.quantize_weights(m)


def test_prefill_logits_equal_the_model_holding_the_dequantised_weights():
    q, ref = _pair()
    a, ca = inference.prefill(q, PROMPTS, 64)
    b, cb = inference.prefill(ref, PROMPTS, 64)
    S = max(len(p) for p in PROMPTS)  # rows past the prompts are not written yet
    assert torch.equal(a, b) and torch.equal(ca.kv[:, :, :S], cb.kv[:, :, :S])
    tok = torch.tensor([PROMPTS[2]])
    with torch.no_grad():
        assert torch.equal(q(tok), ref(tok))


@pytest.mark.parametrize("kv_dtype", ["bf16", "fp8"])
@pytest.mark.parametrize("sampler", ["host", "device"])
@pytest.mark.parametrize("knobs", [dict(), dict(temperature=0.9, top_k=20), dict(temperature=0.8, top_p=0.9)], ids=["greedy", "topk", "topp"])
def test_generate_batch_equals_the_model_holding_the_dequantised_weights(kv_dtype, sampler, knobs):
    q, ref = _pair()
    a = inference.generate_batch(q, PROMPTS, max_new=12, seed=5, sampler=sampler, kv_dtype=kv_dtype, **knobs)
    b = inference.generate_batch(ref, PROMPTS, max_new=12, seed=5, sampler=sampler, kv_dtype=kv_dtype, **knobs)
    assert a == b


def test_greedy_speculation_equals_the_model_holding_the_dequantised_weights():
    q, ref = _pair()
    dq, dref = _pair(seed=3, n_layers=1)
    a = inference.generate_speculative(q, dq, PROMPTS, k=3, max_new=12)
    b = inference.generate_speculative(ref, dref, PROMPTS, k=3, max_new=12)
    assert a == b
    assert a.ids == inference.generate_batch(q, PROMPTS, max_new=12, sampler="device")


def test_grad_enabled_forward_of_a_quantised_model_raises():
    q, _ = _pair()
    with pytest.raises(RuntimeError, match="inference only"):
        q(torch.tensor([PROMPTS[0]]))
    with torch.no_grad():
        q(torch.tensor([PROMPTS[0]]))
    x = torch.randn(3, 256, requires_grad=True)
    with pytest.raises(RuntimeError, match="inference only"):
        ops.linear(x, q.output)
    assert ops.linear(x.detach(), q.output).shape == (3, 2048)


def test_quantize_weight_rejects_a_contraction_dimension_not_a_multiple_of_128():
    with pytest.raises(ValueError, match="128"):
        ops.quantize_weight(torch.randn(64, 96))


def test_e4m3w_launchers_reject_impossible_arguments_before_touching_the_device():
    from prime_b200.ops import _lib

    try:
        lib = _lib.load()
    except Exception as e:  # noqa: BLE001
        pytest.skip(f"native library not loadable here: {e}")
    a = 1 << 20  # 16-byte aligned, never dereferenced: every call below is rejected first
    odd = a + 2

    def gemm(x=a, q=a, sf=a, c=a, ws=a, M=4, N=256, K=512, ldc=256, splits=2):
        return lib.pb_gemm_e4m3w(x, q, sf, c, ws, M, N, K, ldc, splits, None)

    assert gemm(x=None) == -1 and gemm(q=None) == -1 and gemm(sf=None) == -1 and gemm(c=None) == -1 and gemm(ws=None) == -1
    assert gemm(K=200) == -2 and gemm(K=0) == -2
    assert gemm(M=0) == -3 and gemm(M=65) == -3 and gemm(N=0) == -3 and gemm(ldc=255) == -3
    assert gemm(splits=0) == -5 and gemm(splits=5) == -5  # K = 512 holds 4 chunks of 128
    assert gemm(K=1280, splits=7) == -5  # 10 chunks in 7 splits would leave one empty
    assert gemm(x=odd) == -6 and gemm(q=odd) == -6 and gemm(sf=a + 1) == -6
    assert lib.pb_gemm_e4m3w_m_max() == ops.gemm_e4m3w_m_max() == 64

    def deq(q=a, sf=a, out=a, N=256, K=512, ldo=512):
        return lib.pb_dequantize_mxfp8(q, sf, out, N, K, ldo, None)

    assert deq(q=None) == -1 and deq(sf=None) == -1 and deq(out=None) == -1
    assert deq(K=100) == -2 and deq(N=0) == -3 and deq(ldo=500) == -3 and deq(out=odd) == -6 and deq(ldo=514) == -6

    sp = lib.pb_gemm_e4m3w_splits
    assert sp(0, 2048, 2048, 132) == -3 and sp(65, 2048, 2048, 132) == -3 and sp(1, 2048, 100, 132) == -3 and sp(1, 2048, 2048, 0) == -3
    for M in (1, 8, 33, 64):
        for N, K in ((2048, 2048), (6144, 2048), (32000, 4096), (4096, 14336), (128256, 4096)):
            s = sp(M, N, K, 132)
            chunks = K // 128
            cps = (chunks + s - 1) // s
            assert 1 <= s <= chunks and (chunks + cps - 1) // cps == s, (M, N, K, s)
    assert sp(1, 2048, 2048, 132) > 1  # a small projection at M = 1 is split to fill the machine
    assert sp(64, 128256, 4096, 132) == 1  # the LM head fills it on its own


def _ckpt_free_model(monkeypatch):
    """The eval CLI's model loader, returning a random-init debugmodel."""
    monkeypatch.setattr(ev, "load_model", lambda a, device, prefix="": build_model("debugmodel", dtype=torch.float32, seed=0 if not prefix else 1))


def test_cli_generate_and_ppl_with_fp8_weights(monkeypatch, tmp_path, capsys):
    _ckpt_free_model(monkeypatch)
    out = ev.main(["generate", "--ckpt", "x", "--device", "cpu", "--prompt-ids", "1,2,3", "--max-new", "6", "--weight-dtype", "fp8"])
    q, _ = _pair()
    assert out["ids"] == inference.generate_batch(q, [[1, 2, 3]], max_new=6)[0]
    out = ev.main(["generate", "--ckpt", "x", "--device", "cpu", "--prompt-ids", "1,2,3", "--max-new", "6", "--weight-dtype", "fp8",
                   "--draft-ckpt", "y", "--sampler", "device", "--spec-k", "2"])  # fmt: skip
    assert out["ids"] == inference.generate_batch(q, [[1, 2, 3]], max_new=6, sampler="device")[0]
    import numpy as np

    np.arange(4096, dtype=np.uint16).__mod__(2048).astype(np.uint16).tofile(tmp_path / "val_000.bin")
    out = ev.main(["ppl", "--ckpt", "x", "--device", "cpu", "--data", str(tmp_path / "val_000.bin"), "--seq", "64", "--batches", "2",
                   "--batch-size", "2", "--weight-dtype", "fp8"])  # fmt: skip
    assert out["tokens"] == 256 and out["loss"] > 0
    assert json.loads(capsys.readouterr().out.strip().splitlines()[-1]) == out
