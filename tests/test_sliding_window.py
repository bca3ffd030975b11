"""Sliding-window causal attention, alone and composed with document masking: bounds, the fp32 oracle against transformers'
Mistral, export, checkpoints, the native sm_90a kernels, the model, the trainer.

Query q of row b attends key k iff max(doc_start[b, q], q - W + 1) <= k <= q: the W most recent keys, q itself included, and
never a key of another document."""

import json
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from prime_b200 import ops
from prime_b200.models.llama import ModelArgs, Transformer, build_model
from prime_b200.ops import reference as R

ROOT = Path(__file__).resolve().parents[1]
EOS = 7


def _window_mask(S: int, W: int) -> torch.Tensor:
    k = torch.arange(S)
    return (k.view(1, S) <= k.view(S, 1)) & (k.view(1, S) > k.view(S, 1) - W)


def _end_of(mask: torch.Tensor) -> list[int]:
    """One past the last query that sees each key of a [S, S] (query, key) mask."""
    S = mask.shape[0]
    return [max(q for q in range(S) if mask[q, k]) + 1 for k in range(S)]


def test_reference_bounds_window_only():
    t = torch.tensor([[3, 1, 4, 1, 5, 9, 2, 6]])
    ds, de = R.document_bounds(t, None, 3)
    assert ds.dtype == torch.int32 and de.dtype == torch.int32
    assert ds.tolist() == [[0, 0, 0, 1, 2, 3, 4, 5]]
    assert de.tolist() == [[3, 4, 5, 6, 7, 8, 8, 8]]
    assert torch.equal(R.document_mask(ds)[0], _window_mask(8, 3))
    # without documents and without a window every query sees its whole prefix
    ds, de = R.document_bounds(t, None)
    assert ds.tolist() == [[0] * 8] and de.tolist() == [[8] * 8]


def test_reference_bounds_window_and_documents_is_the_and_of_both_masks():
    t = torch.tensor([[5, EOS, 9, EOS, EOS, 3, 4, EOS]])
    ds, de = R.document_bounds(t, EOS, 2)
    assert ds.tolist() == [[0, 0, 2, 2, 4, 5, 5, 6]]
    assert de.tolist() == [[2, 2, 4, 4, 5, 7, 8, 8]]
    g = np.random.default_rng(0)
    for S, W in [(8, 2), (64, 5), (64, 17), (200, 33)]:
        rows = torch.tensor(g.integers(0, 12, size=(3, S)))  # EOS (7) about once in 12 tokens
        ds, de = R.document_bounds(rows, EOS, W)
        dd, _ = R.document_bounds(rows, EOS)
        want = R.document_mask(dd) & _window_mask(S, W)
        assert torch.equal(R.document_mask(ds), want)
        for b in range(3):
            assert de[b].tolist() == _end_of(want[b])  # end is the matching upper bound
        assert torch.equal(ops.document_bounds(rows, EOS, W)[0], ds)  # the CPU op is the reference


def test_reference_bounds_window_at_least_s_is_no_window():
    rows = torch.tensor(np.random.default_rng(1).integers(0, 12, size=(2, 50)))
    for eos in (EOS, None):
        plain = R.document_bounds(rows, eos)
        for W in (50, 51, 1000):
            got = R.document_bounds(rows, eos, W)
            assert torch.equal(got[0], plain[0]) and torch.equal(got[1], plain[1])


def test_reference_bounds_window_one_is_the_diagonal():
    rows = torch.tensor(np.random.default_rng(2).integers(0, 12, size=(2, 40)))
    for eos in (EOS, None):
        ds, de = R.document_bounds(rows, eos, 1)
        assert ds.tolist() == [list(range(40))] * 2 and de.tolist() == [list(range(1, 41))] * 2
        assert torch.equal(R.document_mask(ds)[0], torch.eye(40, dtype=torch.bool))


def test_document_bounds_refuses_a_window_below_one():
    t = torch.zeros((1, 8), dtype=torch.int64)
    for W in (0, -3):
        with pytest.raises(ValueError, match="window"):
            ops.document_bounds(t, None, W)


def test_native_doc_bounds_rejects_a_negative_window_before_touching_the_device():
    """Same contract as the other launchers: an impossible window comes back as -1 before the first CUDA call (no GPU needed)."""
    from prime_b200.ops import _lib

    try:
        lib = _lib.load()
    except Exception as e:  # noqa: BLE001
        pytest.skip(f"native library not loadable here: {e}")
    assert lib.pb_doc_bounds(None, 1, 256, EOS, -1, None, None, None) == -1
    assert lib.pb_doc_bounds(None, 2, 256, -1, -1024, None, None, None) == -1


# ------------------------------------------------------------------------------------------------ transformers' Mistral
def test_window_model_matches_transformers_mistral():
    """A tiny MistralForCausalLM (eager, GQA, window 8) loaded into a Transformer with the same window is the same function; full
    attention agrees with it only on the first 8 positions."""
    transformers = pytest.importorskip("transformers")
    from prime_b200.models import hf

    cfg = transformers.MistralConfig(vocab_size=512, hidden_size=64, intermediate_size=176, num_hidden_layers=2, num_attention_heads=4,
                                     num_key_value_heads=2, head_dim=16, max_position_embeddings=128, rms_norm_eps=1e-5,
                                     rope_theta=10000.0, sliding_window=8, tie_word_embeddings=False, attn_implementation="eager")  # fmt: skip
    torch.manual_seed(3)
    ref = transformers.MistralForCausalLM(cfg).eval()
    args = ModelArgs(dim=64, n_layers=2, n_heads=4, n_kv_heads=2, vocab_size=512, intermediate_size=176, max_seq_len=128, sliding_window=8)
    m = Transformer(args).float()
    hf.load_hf_state_dict(m, ref.state_dict())
    tok = torch.randint(0, 512, (2, 48))
    with torch.no_grad():
        want = ref(tok).logits
        got = m(tok)
        full = Transformer(ModelArgs(**{**args.__dict__, "sliding_window": None})).float()
        full.load_state_dict(m.state_dict())
        plain = full(tok)
    torch.testing.assert_close(got, want, rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(plain[:, :8], want[:, :8], rtol=1e-4, atol=1e-4)
    assert (plain[:, 8:] - want[:, 8:]).abs().amax(-1).min() > 1e-3  # every later position differs


def test_window_model_exports_as_mistral(tmp_path):
    transformers = pytest.importorskip("transformers")
    pytest.importorskip("safetensors")
    from prime_b200.models import hf

    m = build_model("debugmodel", dtype=torch.float32, seed=11, n_kv_heads=4, sliding_window=8)
    hf.save_hf_dir(m, tmp_path)
    cfg = json.loads((tmp_path / "config.json").read_text())
    assert cfg["model_type"] == "mistral" and cfg["architectures"] == ["MistralForCausalLM"] and cfg["sliding_window"] == 8
    tok = torch.randint(0, m.args.vocab_size, (1, 40))
    loaded = transformers.AutoModelForCausalLM.from_pretrained(tmp_path, torch_dtype=torch.float32, attn_implementation="eager").eval()
    assert type(loaded).__name__ == "MistralForCausalLM"
    with torch.no_grad():
        torch.testing.assert_close(loaded(tok).logits, m(tok), rtol=1e-4, atol=1e-4)
    # without a window the export is the Llama one, with no window key
    plain = hf.hf_config_from_args(build_model("debugmodel", dtype=torch.float32).args)
    assert plain["model_type"] == "llama" and "sliding_window" not in plain


def test_receptive_field_is_layers_times_window():
    """After L layers position q depends only on tokens q - L·(W - 1) .. q: perturbing every earlier token leaves its fp32 logits
    bit for bit unchanged, and perturbing the first token inside that range changes them."""
    W, S = 5, 64
    m = build_model("debugmodel", dtype=torch.float32, seed=5, sliding_window=W)
    L = m.args.n_layers
    g = torch.Generator().manual_seed(0)
    tok = torch.randint(0, 2048, (1, S), generator=g)
    with torch.no_grad():
        base = m(tok)
        for q in (L * (W - 1), 30, S - 1):
            first = q - L * (W - 1)
            t2 = tok.clone()
            t2[0, :first] = torch.randint(0, 2048, (first,), generator=g)
            assert torch.equal(m(t2)[0, q], base[0, q]), q
            t2[0, first] = (tok[0, first] + 1) % 2048
            assert not torch.equal(m(t2)[0, q], base[0, q]), q


def test_flops_per_token_counts_the_attended_pairs():
    plain = build_model("debugmodel", dtype=torch.float32)
    attn = 6.0 * plain.args.n_layers * 1024 * plain.args.dim
    for W, kept in [(1024, 1.0), (4096, 1.0), (512, 0.75), (256, 1 - 0.75**2)]:
        m = build_model("debugmodel", dtype=torch.float32, sliding_window=W)
        assert m.flops_per_token(1024) == pytest.approx(plain.flops_per_token(1024) - attn * (1 - kept), rel=1e-12)


# ---------------------------------------------------------------------------------------------- config, checkpoints, eval
def test_config_sliding_window_default_and_validation():
    from pydantic import ValidationError

    from prime_b200.config import Config, load_config

    assert Config().sliding_window is None
    assert load_config(["--sliding_window", "16"]).sliding_window == 16
    for bad in (0, -1):
        with pytest.raises(ValidationError):
            Config(sliding_window=bad)
        with pytest.raises(SystemExit):
            load_config(["--sliding_window", str(bad)])


def _losses(p: Path) -> dict[int, float]:
    return {r["step"]: r["loss"] for r in map(json.loads, p.read_text().splitlines())}


BASE = ["--name_model", "debugmodel", "--sliding_window", "8", "--data.seq_length", "32", "--optim.batch_size", "4", "--train.micro_bs", "2",
        "--optim.warmup_steps", "2", "--optim.total_steps", "12", "--optim.optim.lr", "3e-3", "--diloco.inner_steps", "4"]  # fmt: skip


def test_trainer_sliding_window_cpu_run_and_exact_resume(tmp_path):
    from prime_b200 import checkpoint as ck
    from prime_b200.config import load_config
    from prime_b200.train import train

    a, b = tmp_path / "a", tmp_path / "b"
    out = train(load_config(BASE + ["--monitor.jsonl_path", str(a / "log.jsonl")]))
    straight = _losses(a / "log.jsonl")
    assert out["step"] == 12 and all(np.isfinite(list(straight.values())))
    assert straight[12] < straight[1] - 0.5
    train(load_config(BASE + ["--ckpt.path", str(b), "--ckpt.interval", "4", "--monitor.jsonl_path", str(b / "l1.jsonl")]), max_steps=4)
    assert ck.list_steps(b) == [4]
    train(load_config(BASE + ["--ckpt.path", str(b), "--ckpt.interval", "4", "--ckpt.resume", "latest", "--monitor.jsonl_path", str(b / "l2.jsonl")]))
    assert {**_losses(b / "l1.jsonl"), **_losses(b / "l2.jsonl")} == straight
    # the option reaches the model: the same run with full attention computes a different first loss
    train(load_config(BASE + ["--sliding_window", "none", "--monitor.jsonl_path", str(tmp_path / "plain.jsonl")]), max_steps=1)
    assert _losses(tmp_path / "plain.jsonl")[1] != straight[1]


def _tokenize(tmp_path: Path) -> Path:
    sys.path.insert(0, str(ROOT))
    from tools.tokenize_corpus import main as tokenize

    words = ["alpha", "beta", "gamma", "delta", "epsilon", "zeta", "eta", "theta"]
    docs = [" ".join(words[(i + j) % len(words)] for j in range(3 + (i * 7) % 23)) + "." for i in range(60)]
    (tmp_path / "docs.jsonl").write_text("\n".join(json.dumps({"text": d}) for d in docs))
    tokenize([str(tmp_path / "docs.jsonl"), "--tokenizer", "bytes", "--out", str(tmp_path / "ds")])
    return tmp_path / "ds"


def test_window_survives_checkpoint_assembly_eval_and_export(tmp_path):
    import shutil

    from prime_b200 import checkpoint as ck
    from prime_b200 import eval as ev
    from prime_b200.config import load_config
    from prime_b200.models import hf
    from prime_b200.train import train

    root = tmp_path / "ckpt"
    train(load_config(BASE + ["--ckpt.path", str(root), "--ckpt.interval", "4", "--monitor.jsonl_path", str(tmp_path / "l.jsonl")]), max_steps=4)
    step = ck.step_dir(root, 4)
    m = ck.assemble_full_model(step, "debugmodel")
    assert m.args.sliding_window == 8
    # a checkpoint written before the option existed has no key: it is rebuilt with full attention, as before
    old = tmp_path / "old"
    shutil.copytree(step, old)
    meta = json.loads((old / "meta.json").read_text())
    del meta["config"]["sliding_window"]
    (old / "meta.json").write_text(json.dumps(meta))
    m_old = ck.assemble_full_model(old, "debugmodel")
    assert m_old.args.sliding_window is None
    for (k, p), (_, p_old) in zip(m.named_parameters(), m_old.named_parameters()):
        assert torch.equal(p, p_old), k
    # eval rebuilds the windowed model from the checkpoint: its loss differs from the same weights with full attention
    ds = _tokenize(tmp_path)

    def ppl(ckpt):
        return ev.main(["ppl", "--ckpt", str(ckpt), "--model", "debugmodel", "--data", str(ds), "--seq", "64", "--batches", "2",
                        "--batch-size", "2", "--device", "cpu"])["loss"]  # fmt: skip

    windowed = ppl(step)
    assert windowed == ev.perplexity(m, ev.MemmapTokenDataset(str(ds), 64, vocab_size=m.args.vocab_size, shuffle=False), batches=2,
                                     batch_size=2, device="cpu")["loss"]  # fmt: skip
    assert windowed != ppl(old)
    # and the export is a Mistral directory with the window
    hf.main(["export", "--ckpt", str(step), "--model", "debugmodel", "--out", str(tmp_path / "hf"), "--dtype", "float32"])
    cfg = json.loads((tmp_path / "hf" / "config.json").read_text())
    assert cfg["model_type"] == "mistral" and cfg["sliding_window"] == 8


# ====================================================================================================================== GPU
def _dev():
    return torch.device("cuda", 0)


def _rel_err(a: torch.Tensor, b: torch.Tensor) -> float:
    return float((a.detach().float() - b.detach().float()).norm() / (b.detach().float().norm() + 1e-12))


def _rows(layout: str, B: int, S: int) -> torch.Tensor:
    """int64 [B, S] CUDA token rows: "none" has no EOS; "mixed" has documents of 1 to 300 tokens, its own boundaries per row."""
    rows = []
    for b in range(B):
        g = np.random.default_rng(100 * b + S)
        row = [int(x) for x in g.integers(8, 200, size=S)]  # never EOS
        if layout == "mixed":
            p = int(g.integers(0, 40))
            while p < S:
                row[p] = EOS
                p += int(g.integers(1, 300))
        rows.append(row)
    return torch.tensor(rows, device=_dev())


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["none", "mixed"])
@pytest.mark.parametrize("S", [256, 1000, 4096])
def test_native_window_bounds_match_reference(S, layout):
    tok = _rows(layout, 3, S)
    eos = EOS if layout == "mixed" else None
    for W in (1, 17, 64, 100, 1000, S, S + 7):
        got = ops.document_bounds(tok, eos, W)
        want = R.document_bounds(tok.cpu(), eos, W)
        assert torch.equal(got[0].cpu(), want[0]) and torch.equal(got[1].cpu(), want[1]), W
    # documents only, and no documents with a negative EOS id: the same kernel
    for e in (EOS, None):
        got, want = ops.document_bounds(tok, e), R.document_bounds(tok.cpu(), e)
        assert torch.equal(got[0].cpu(), want[0]) and torch.equal(got[1].cpu(), want[1])


GPU_SHAPES = [(2, 256, 4, 4, 128), (2, 256, 8, 2, 64), (2, 1024, 4, 1, 128), (3, 1024, 4, 2, 64), (2, 4096, 2, 2, 128), (1, 4096, 4, 1, 64)]


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["none", "mixed"])
@pytest.mark.parametrize("W", [1, 63, 100, 1024])
@pytest.mark.parametrize("B,S,H,Hkv,D", GPU_SHAPES)
def test_native_window_attention_matches_reference(B, S, H, Hkv, D, W, layout):
    from prime_b200.ops import attention_native as A

    torch.manual_seed(S + H + D + W)
    doc = ops.document_bounds(_rows(layout, B, S), EOS if layout == "mixed" else None, W)
    Wd = (H + 2 * Hkv) * D
    qkv = (torch.randn(B, S, Wd, device=_dev()) * 0.7).to(torch.bfloat16).requires_grad_(True)
    out = A.flash_attention_qkv(qkv, H, Hkv, True, doc)
    dout = torch.randn_like(out)
    out.backward(dout)
    torch.cuda.synchronize()
    ref_in = qkv.detach().float().requires_grad_(True)
    x = ref_in.view(B, S, H + 2 * Hkv, D)
    ref = R.attention(x[:, :, :H], x[:, :, H : H + Hkv], x[:, :, H + Hkv :], True, doc_start=doc[0]).reshape(B, S, H * D)
    ref.backward(dout.float())
    assert torch.isfinite(out).all() and torch.isfinite(qkv.grad).all()
    assert _rel_err(out, ref) < 2e-2, f"fwd rel err {_rel_err(out, ref)}"
    g, gr = qkv.grad.view(B, S, H + 2 * Hkv, D), ref_in.grad.view(B, S, H + 2 * Hkv, D)
    assert _rel_err(g[:, :, H + Hkv :], gr[:, :, H + Hkv :]) < 3e-2, f"dV rel err {_rel_err(g[:, :, H + Hkv :], gr[:, :, H + Hkv :])}"
    if W == 1:
        # every query sees only itself: softmax is exactly 1, so the exact dQ and dK are 0 and a relative error is undefined; the
        # kernels' are rounding noise of dP - delta, far below the gradients that flow
        scale = float(gr[:, :, H + Hkv :].abs().max())
        assert float(g[:, :, : H + Hkv].abs().max()) < 1e-2 * scale
        return
    assert _rel_err(g[:, :, :H], gr[:, :, :H]) < 3e-2, f"dQ rel err {_rel_err(g[:, :, :H], gr[:, :, :H])}"
    assert _rel_err(g[:, :, H : H + Hkv], gr[:, :, H : H + Hkv]) < 3e-2, f"dK rel err {_rel_err(g[:, :, H : H + Hkv], gr[:, :, H : H + Hkv])}"


@pytest.mark.gpu
@pytest.mark.parametrize("B,S,H,Hkv,D", [(2, 512, 4, 2, 128), (1, 1024, 8, 8, 64), (3, 384, 2, 2, 64)])
def test_window_covering_the_row_is_bitwise_causal(B, S, H, Hkv, D):
    """W >= S without documents: output, lse2 and dQKV of the bounded kernels equal the plain causal kernels' bit for bit."""
    import math

    from prime_b200.ops import _lib
    from prime_b200.ops import attention_native as A
    from prime_b200.ops.functional import _ptr, _stream

    lib = _lib.load()
    torch.manual_seed(11)
    Wd = (H + 2 * Hkv) * D
    qkv = (torch.randn(B, S, Wd, device=_dev()) * 0.7).to(torch.bfloat16)
    dout = torch.randn(B, S, H * D, device=_dev()).to(torch.bfloat16)
    scale = 1.0 / math.sqrt(D)
    o1 = torch.empty(B, S, H * D, dtype=torch.bfloat16, device=_dev())
    l1 = torch.empty(B, H, S, dtype=torch.float32, device=_dev())
    _lib.check(lib.pb_flash_attn_fwd(_ptr(qkv), _ptr(o1), _ptr(l1), None, B, S, H, Hkv, D, scale, 1, _stream()), "fwd")
    x = qkv.clone().requires_grad_(True)
    A.flash_attention_qkv(x, H, Hkv, True).backward(dout)
    for W in (S, 4 * S):
        doc = ops.document_bounds(_rows("none", B, S), None, W)
        o2, l2 = torch.empty_like(o1), torch.empty_like(l1)
        _lib.check(lib.pb_flash_attn_fwd(_ptr(qkv), _ptr(o2), _ptr(l2), _ptr(doc[0]), B, S, H, Hkv, D, scale, 1, _stream()), "fwd win")
        y = qkv.clone().requires_grad_(True)
        A.flash_attention_qkv(y, H, Hkv, True, doc).backward(dout)
        torch.cuda.synchronize()
        assert torch.equal(o1, o2) and torch.equal(l1, l2) and torch.equal(x.grad, y.grad), W


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["none", "mixed"])
@pytest.mark.parametrize("pre_rotated", [False, True])
def test_rope_attention_with_window(pre_rotated, layout):
    """RoPE ⊕ windowed attention as one autograd node; ``pre_rotated`` = the rotation ran in the QKV GEMM epilogue."""
    torch.manual_seed(5)
    B, S, dim, H, Hkv, D = 2, 512, 512, 8, 2, 64
    Wd = (H + 2 * Hkv) * D
    doc = ops.document_bounds(_rows(layout, B, S), EOS if layout == "mixed" else None, 100)
    x = (torch.randn(B, S, dim, device=_dev()) * 0.5).to(torch.bfloat16).requires_grad_(True)
    w = (torch.randn(Wd, dim, device=_dev()) * 0.05).to(torch.bfloat16).requires_grad_(True)
    cos, sin = R.rope_tables(S, D, device=_dev())
    qkv = ops.linear_qkv_rope(x, w, cos, sin, H, Hkv) if pre_rotated else ops.linear(x, w)
    out = ops.rope_attention_qkv(qkv, cos, sin, H, Hkv, causal=True, impl="native", pre_rotated=pre_rotated, doc=doc)
    dout = torch.randn_like(out)
    out.backward(dout)
    torch.cuda.synchronize()
    xr = x.detach().float().requires_grad_(True)
    wr = w.detach().float().requires_grad_(True)
    q4 = (xr @ wr.t()).view(B, S, H + 2 * Hkv, D)
    rot = R.rope(q4[:, :, : H + Hkv], cos, sin)
    ref = R.attention(rot[:, :, :H], rot[:, :, H:], q4[:, :, H + Hkv :], True, doc_start=doc[0]).reshape(B, S, H * D)
    ref.backward(dout.float())
    assert _rel_err(out, ref) < 2e-2
    assert _rel_err(x.grad, xr.grad) < 4e-2, _rel_err(x.grad, xr.grad)
    assert _rel_err(w.grad, wr.grad) < 4e-2, _rel_err(w.grad, wr.grad)


@pytest.mark.gpu
@pytest.mark.parametrize("W", [16, 100])
def test_window_model_bf16_native_matches_fp32_cpu(W):
    """The bf16 model on the native kernels against the fp32 CPU model with the same window; and its receptive field in bf16: keys
    outside a query's window are skipped or get P = 0 exactly, so tokens before q - L·(W - 1) cannot change the logits at q."""
    import copy

    cpu = build_model("debugmodel", dtype=torch.float32, seed=3, n_heads=4, sliding_window=W)  # head size 64 for the native kernels
    gpu = copy.deepcopy(cpu).to(device=_dev(), dtype=torch.bfloat16)
    gpu.attn_impl = "native"
    g = torch.Generator().manual_seed(0)
    tok = torch.randint(0, cpu.args.vocab_size, (2, 512), generator=g)
    with torch.no_grad():
        want = cpu(tok)
        got = gpu(tok.to(_dev())).float().cpu()
        assert _rel_err(got, want) < 2e-2, _rel_err(got, want)
        for q in (300, 511):
            first = q - cpu.args.n_layers * (W - 1)
            t2 = tok.clone()
            t2[:, :first] = torch.randint(0, cpu.args.vocab_size, (2, first), generator=g)
            assert torch.equal(gpu(t2.to(_dev()))[:, q].cpu(), gpu(tok.to(_dev()))[:, q].cpu()), q
            t2[:, first] = (tok[:, first] + 1) % cpu.args.vocab_size
            assert not torch.equal(gpu(t2.to(_dev()))[:, q].cpu(), gpu(tok.to(_dev()))[:, q].cpu()), q


@pytest.mark.gpu
def test_trainer_sliding_window_gpu_eager_and_cuda_graph():
    from prime_b200.config import load_config
    from prime_b200.trainer import Trainer

    base = ["--name_model", "debugmodel", "--sliding_window", "48", "--data.seq_length", "256", "--optim.batch_size", "4",
            "--train.micro_bs", "2", "--optim.warmup_steps", "2", "--optim.total_steps", "10", "--optim.optim.lr", "3e-3",
            "--train.attn_impl", "native"]  # fmt: skip
    runs = {}
    for graphs in ("false", "true"):
        t = Trainer(load_config(base + ["--train.cuda_graphs", graphs]), model_overrides={"n_heads": 4})  # head size 64
        assert t.model.args.sliding_window == 48 and t.accum == 2
        runs[graphs] = [float(t.inner_step().loss.item()) for _ in range(8)]
        t.close()
    eager, graph = runs["false"], runs["true"]
    assert all(np.isfinite(eager)) and eager[-1] < eager[0]
    # the first loss comes from the forward alone; later steps of eager and captured micro-steps differ in rounding only (the
    # document-mask test measures about 1e-3 relative after a few steps on this model)
    assert graph[0] == eager[0]
    np.testing.assert_allclose(graph, eager, rtol=2e-3)
