"""Document-masked attention over packed token rows: bounds, the fp32 oracle, the native sm_90a kernels, the model, the trainer.

A token at position q of row b attends key k iff doc_start[b, q] <= k <= q, where a document starts at s == 0 or after an EOS."""

import json
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from prime_b200 import ops
from prime_b200.ops import reference as R

ROOT = Path(__file__).resolve().parents[1]
EOS = 7


def _naive_bounds(row: list[int], eos: int) -> tuple[list[int], list[int]]:
    S = len(row)
    start, end = [0] * S, [0] * S
    cur = 0
    for s in range(S):
        if s > 0 and row[s - 1] == eos:
            cur = s
        start[s] = cur
    cur = S
    for s in reversed(range(S)):
        if row[s] == eos:
            cur = s + 1
        end[s] = cur
    return start, end


def _row(S: int, eos_at: list[int], seed: int = 0) -> list[int]:
    g = np.random.default_rng(seed)
    row = [int(x) for x in g.integers(8, 200, size=S)]  # never EOS
    for p in eos_at:
        row[p] = EOS
    return row


# position lists of EOS tokens per layout (S = 256)
LAYOUTS = {
    "no_eos": [],
    "eos_at_0": [0],
    "eos_at_last": [255],
    "consecutive": [10, 11, 12, 100, 101],
    "on_32_64_128": [31, 63, 127, 191],  # documents start exactly at 32, 64, 128, 192
    "between_tiles": [20, 45, 70, 150, 200, 230],
    "all_eos": list(range(256)),
}


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_document_bounds_cpu(layout):
    S = 256
    row = _row(S, LAYOUTS[layout])
    ds, de = ops.document_bounds(torch.tensor([row]), EOS)
    assert ds.dtype == torch.int32 and de.dtype == torch.int32 and ds.shape == (1, S)
    es, ee = _naive_bounds(row, EOS)
    assert ds[0].tolist() == es and de[0].tolist() == ee


def test_document_bounds_literal_rows():
    t = torch.tensor([[5, EOS, 9, EOS, EOS, 3, 4, EOS], [2] * 8, [EOS, 2, 3, 4, 5, 6, 7 + 1, 9]])
    ds, de = ops.document_bounds(t, EOS)
    assert ds.tolist() == [[0, 0, 2, 2, 4, 5, 5, 5], [0] * 8, [0, 1, 1, 1, 1, 1, 1, 1]]
    assert de.tolist() == [[2, 2, 4, 4, 5, 8, 8, 8], [8] * 8, [1, 8, 8, 8, 8, 8, 8, 8]]
    # several rows at once, each with its own boundaries
    rows = [_row(256, LAYOUTS[k], seed=i) for i, k in enumerate(sorted(LAYOUTS))]
    ds, de = ops.document_bounds(torch.tensor(rows), EOS)
    for i, r in enumerate(rows):
        assert (ds[i].tolist(), de[i].tolist()) == _naive_bounds(r, EOS)


def test_reference_attention_is_block_diagonal():
    """Masked attention on a packed row == plain causal attention of every document on its own (outputs and gradients)."""
    torch.manual_seed(0)
    H, Hkv, D = 4, 2, 16
    lens = [5, 1, 17, 9]
    S = sum(lens)
    eos_at = list(np.cumsum(lens) - 1)
    row = _row(S, eos_at)
    ds, _ = ops.document_bounds(torch.tensor([row]), EOS)
    q = torch.randn(1, S, H, D, dtype=torch.float64, requires_grad=True)
    k = torch.randn(1, S, Hkv, D, dtype=torch.float64, requires_grad=True)
    v = torch.randn(1, S, Hkv, D, dtype=torch.float64, requires_grad=True)
    out = R.attention(q, k, v, True, doc_start=ds).double()
    dout = torch.randn_like(out)
    gq, gk, gv = torch.autograd.grad(out, (q, k, v), dout)
    s0 = 0
    for n in lens:
        sl = slice(s0, s0 + n)
        qs, ks, vs = (t.detach()[:, sl].clone().requires_grad_(True) for t in (q, k, v))
        o = R.attention(qs, ks, vs, True).double()
        torch.testing.assert_close(out[:, sl], o, rtol=1e-6, atol=1e-6)
        rq, rk, rv = torch.autograd.grad(o, (qs, ks, vs), dout[:, sl])
        torch.testing.assert_close(gq[:, sl], rq, rtol=1e-6, atol=1e-6)
        torch.testing.assert_close(gk[:, sl], rk, rtol=1e-6, atol=1e-6)
        torch.testing.assert_close(gv[:, sl], rv, rtol=1e-6, atol=1e-6)
        s0 += n
    with pytest.raises(ValueError):
        R.attention(q, k, v, False, doc_start=ds)
    with pytest.raises(ValueError):
        ops.attention(q, k, v, causal=False, doc=ops.document_bounds(torch.tensor([row]), EOS))


def _packed_docs(lens: list[int], seed: int) -> list[list[int]]:
    g = np.random.default_rng(seed)
    return [[int(x) for x in g.integers(8, 2000, size=n - 1)] + [EOS] for n in lens]


def _translation_invariance(device, dtype, S_packed: int, S_alone: int, attn_impl: str = "auto") -> float:
    from prime_b200.models.llama import build_model

    # 4 heads of 64: a head size the native kernels take (the debug model's own 8 × 32 runs only on the CPU and sdpa paths)
    m = build_model("debugmodel", device=device, dtype=dtype, seed=3, n_heads=4)
    m.attn_impl = attn_impl
    m.doc_eos_id = EOS
    a, b = _packed_docs([37, 90], seed=1)
    c = _packed_docs([S_packed - 127], seed=2)[0]
    packed = torch.tensor([a + b + c], device=device)
    alone = torch.tensor([b + _packed_docs([S_alone - len(b)], seed=4)[0]], device=device)
    with torch.no_grad():
        lp = m(packed)[0, len(a) : len(a) + len(b)].float()
        la = m(alone)[0, : len(b)].float()
        m.doc_eos_id = None  # plain causal: docB then sees docA and its logits change
        lc = m(packed)[0, len(a) : len(a) + len(b)].float()
    assert float((lc - la).norm() / la.norm()) > 1e-3
    return float((lp - la).norm() / la.norm())


def test_model_logits_do_not_depend_on_position_in_window():
    """RoPE is relative and no query sees outside its document: docB's logits are the same wherever it sits in the row."""
    assert _translation_invariance("cpu", torch.float32, 256, 160) < 1e-5


def _tokenize(tmp_path: Path, docs: list[str]) -> Path:
    sys.path.insert(0, str(ROOT))
    from tools.tokenize_corpus import main as tokenize

    (tmp_path / "docs.jsonl").write_text("\n".join(json.dumps({"text": d}) for d in docs))
    tokenize([str(tmp_path / "docs.jsonl"), "--tokenizer", "bytes", "--out", str(tmp_path / "ds")])
    return tmp_path / "ds"


def _corpus_docs(n: int = 60) -> list[str]:
    words = ["alpha", "beta", "gamma", "delta", "epsilon", "zeta", "eta", "theta"]
    return [" ".join(words[(i + j) % len(words)] for j in range(3 + (i * 7) % 23)) + "." for i in range(n)]


def test_config_defaults_and_eos_resolution(tmp_path):
    from prime_b200.config import Config, load_config
    from prime_b200.data import document_eos_id

    assert Config().data.document_mask is False and Config().data.eos_id is None
    assert document_eos_id(Config().data) is None  # off: nothing is looked up
    ds = _tokenize(tmp_path, _corpus_docs(5))
    cfg = load_config(["--data.fake", "false", "--data.dataset_name_or_paths", str(ds), "--data.document_mask", "true"])
    assert document_eos_id(cfg.data) == 256  # from the bytes tokenizer's .meta.json
    cfg = load_config(["--data.fake", "false", "--data.dataset_name_or_paths", str(ds), "--data.document_mask", "true", "--data.eos_id", "3"])
    assert document_eos_id(cfg.data) == 3  # explicit id wins
    with pytest.raises(ValueError, match="eos_id"):
        document_eos_id(load_config(["--data.document_mask", "true"]).data)  # synthetic data, no id
    raw = tmp_path / "raw"
    raw.mkdir()
    np.arange(1000, dtype=np.uint16).tofile(raw / "x.bin")  # a raw shard without sidecar
    with pytest.raises(ValueError, match="eos_id"):
        document_eos_id(load_config(["--data.fake", "false", "--data.dataset_name_or_paths", str(raw), "--data.document_mask", "true"]).data)
    # synthetic data with an explicit id is accepted
    assert document_eos_id(load_config(["--data.document_mask", "true", "--data.eos_id", "5"]).data) == 5


def test_trainer_refuses_document_mask_without_eos():
    from prime_b200.config import load_config
    from prime_b200.trainer import Trainer

    with pytest.raises(ValueError, match="eos_id"):
        Trainer(load_config(["--name_model", "debugmodel", "--data.seq_length", "32", "--data.document_mask", "true",
                             "--optim.batch_size", "2", "--train.micro_bs", "2"]))  # fmt: skip


def _losses(p: Path) -> dict[int, float]:
    return {r["step"]: r["loss"] for r in map(json.loads, p.read_text().splitlines())}


def test_trainer_document_mask_cpu_run_and_exact_resume(tmp_path):
    from prime_b200 import checkpoint as ck
    from prime_b200.config import load_config
    from prime_b200.train import train

    ds = _tokenize(tmp_path, _corpus_docs())
    base = ["--name_model", "debugmodel", "--data.fake", "false", "--data.dataset_name_or_paths", str(ds), "--data.seq_length", "32",
            "--data.document_mask", "true", "--optim.batch_size", "4", "--train.micro_bs", "2", "--optim.warmup_steps", "2",
            "--optim.total_steps", "12", "--optim.optim.lr", "3e-3", "--diloco.inner_steps", "4"]  # fmt: skip
    a, b = tmp_path / "a", tmp_path / "b"
    out = train(load_config(base + ["--monitor.jsonl_path", str(a / "log.jsonl")]))
    straight = _losses(a / "log.jsonl")
    assert out["step"] == 12 and all(np.isfinite(list(straight.values())))
    assert straight[12] < straight[1] - 0.5
    train(load_config(base + ["--ckpt.path", str(b), "--ckpt.interval", "4", "--monitor.jsonl_path", str(b / "l1.jsonl")]), max_steps=4)
    assert ck.list_steps(b) == [4]
    train(load_config(base + ["--ckpt.path", str(b), "--ckpt.interval", "4", "--ckpt.resume", "latest", "--monitor.jsonl_path", str(b / "l2.jsonl")]))
    assert {**_losses(b / "l1.jsonl"), **_losses(b / "l2.jsonl")} == straight
    # the switch reaches the model: the same run without masking computes a different first loss
    train(load_config([x if x != "true" else "false" for x in base] + ["--monitor.jsonl_path", str(tmp_path / "plain.jsonl")]), max_steps=1)
    assert _losses(tmp_path / "plain.jsonl")[1] != straight[1]


def test_eval_ppl_document_mask_flags(tmp_path, monkeypatch):
    from prime_b200 import eval as ev
    from prime_b200.models.llama import build_model

    ds = _tokenize(tmp_path, _corpus_docs())
    monkeypatch.setattr(ev, "load_model", lambda a, device: build_model("debugmodel", dtype=torch.float32, seed=0))

    def ppl(*extra):
        argv = ["ppl", "--hf", str(tmp_path), "--data", str(ds), "--seq", "64", "--batches", "2", "--batch-size", "2", "--device", "cpu"]
        return ev.main(argv + list(extra))["loss"]

    plain, masked, explicit = ppl(), ppl("--document-mask"), ppl("--eos-id", "256")
    assert masked == explicit and masked != plain


# ====================================================================================================================== GPU
def _dev():
    return torch.device("cuda", 0)


def _rel_err(a: torch.Tensor, b: torch.Tensor) -> float:
    return float((a.detach().float() - b.detach().float()).norm() / (b.detach().float().norm() + 1e-12))


def _gpu_rows(layout: str, B: int, S: int) -> torch.Tensor:
    """int64 [B, S] token rows with EOS placed by ``layout``; every row has its own boundaries."""
    rows = []
    for b in range(B):
        g = np.random.default_rng(100 * b + S)
        if layout == "doc7":
            eos = list(range(6 + b, S, 7))
        elif layout == "mixed":  # lengths from 1 to 300, straddling the 32 / 64-token tiles
            eos, p = [], int(g.integers(0, 40))
            while p < S:
                eos.append(p)
                p += int(g.integers(1, 300))
        elif layout == "tile64":  # documents start exactly on 64-token tiles (and one on a 32-token dK/dV tile)
            eos = [63, 127 + 64 * b, 191 + 64 * b, S - 33]
        elif layout == "eos_last":
            eos = [int(g.integers(0, S // 2)), S - 1]
        else:
            raise KeyError(layout)
        rows.append(_row(S, [e for e in eos if e < S], seed=b))
    return torch.tensor(rows, device=_dev())


GPU_SHAPES = [(2, 256, 4, 4, 128), (2, 256, 8, 2, 64), (2, 1024, 4, 1, 128), (3, 1024, 4, 2, 64), (2, 4096, 2, 2, 128), (1, 4096, 4, 1, 64)]


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["doc7", "mixed", "tile64", "eos_last"])
@pytest.mark.parametrize("B,S,H,Hkv,D", GPU_SHAPES)
def test_native_document_masked_attention_matches_reference(B, S, H, Hkv, D, layout):
    from prime_b200.ops import attention_native as A

    torch.manual_seed(S + H + D)
    tok = _gpu_rows(layout, B, S)
    doc = ops.document_bounds(tok, EOS)  # native kernel on CUDA
    rs, re_ = R.document_bounds(tok.cpu(), EOS)
    assert torch.equal(doc[0].cpu(), rs) and torch.equal(doc[1].cpu(), re_)
    W = (H + 2 * Hkv) * D
    qkv = (torch.randn(B, S, W, device=_dev()) * 0.7).to(torch.bfloat16).requires_grad_(True)
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
    assert _rel_err(g[:, :, :H], gr[:, :, :H]) < 3e-2, f"dQ rel err {_rel_err(g[:, :, :H], gr[:, :, :H])}"
    assert _rel_err(g[:, :, H : H + Hkv], gr[:, :, H : H + Hkv]) < 3e-2, f"dK rel err {_rel_err(g[:, :, H : H + Hkv], gr[:, :, H : H + Hkv])}"
    assert _rel_err(g[:, :, H + Hkv :], gr[:, :, H + Hkv :]) < 3e-2, f"dV rel err {_rel_err(g[:, :, H + Hkv :], gr[:, :, H + Hkv :])}"


@pytest.mark.gpu
@pytest.mark.parametrize("B,S,H,Hkv,D", [(2, 512, 4, 2, 128), (1, 1024, 8, 8, 64), (1, 256, 4, 1, 128), (3, 384, 2, 2, 64)])
def test_single_document_is_bitwise_causal(B, S, H, Hkv, D):
    """A row without EOS is one document: output, lse2 and gradients of the masked kernels equal the causal kernels' bit for bit."""
    import math

    from prime_b200.ops import _lib
    from prime_b200.ops import attention_native as A
    from prime_b200.ops.functional import _ptr, _stream

    lib = _lib.load()
    torch.manual_seed(11)
    doc = ops.document_bounds(_gpu_rows("doc7", B, S).fill_(9), EOS)
    assert int(doc[0].max()) == 0 and int(doc[1].min()) == S
    W = (H + 2 * Hkv) * D
    qkv = (torch.randn(B, S, W, device=_dev()) * 0.7).to(torch.bfloat16)
    scale = 1.0 / math.sqrt(D)
    o1, o2 = (torch.empty(B, S, H * D, dtype=torch.bfloat16, device=_dev()) for _ in range(2))
    l1, l2 = (torch.empty(B, H, S, dtype=torch.float32, device=_dev()) for _ in range(2))
    _lib.check(lib.pb_flash_attn_fwd(_ptr(qkv), _ptr(o1), _ptr(l1), None, B, S, H, Hkv, D, scale, 1, _stream()), "fwd")
    _lib.check(lib.pb_flash_attn_fwd(_ptr(qkv), _ptr(o2), _ptr(l2), _ptr(doc[0]), B, S, H, Hkv, D, scale, 1, _stream()), "fwd doc")
    torch.cuda.synchronize()
    assert torch.equal(o1, o2) and torch.equal(l1, l2)
    dout = torch.randn(B, S, H * D, device=_dev()).to(torch.bfloat16)
    grads = []
    for d in (None, doc):
        x = qkv.clone().requires_grad_(True)
        A.flash_attention_qkv(x, H, Hkv, True, d).backward(dout)
        grads.append(x.grad)
    torch.cuda.synchronize()
    assert torch.equal(grads[0], grads[1])


@pytest.mark.gpu
@pytest.mark.parametrize("pre_rotated", [False, True])
@pytest.mark.parametrize("H,Hkv,D", [(4, 4, 128), (8, 2, 64)])
def test_rope_attention_with_document_mask(H, Hkv, D, pre_rotated):
    """RoPE ⊕ masked attention as one autograd node; ``pre_rotated`` = the rotation ran in the QKV GEMM epilogue."""
    torch.manual_seed(5)
    B, S, dim = 2, 512, 512
    W = (H + 2 * Hkv) * D
    doc = ops.document_bounds(_gpu_rows("mixed", B, S), EOS)
    x = (torch.randn(B, S, dim, device=_dev()) * 0.5).to(torch.bfloat16).requires_grad_(True)
    w = (torch.randn(W, dim, device=_dev()) * 0.05).to(torch.bfloat16).requires_grad_(True)
    cos, sin = R.rope_tables(S, D, device=_dev())
    if pre_rotated:
        qkv = ops.linear_qkv_rope(x, w, cos, sin, H, Hkv)
    else:
        qkv = ops.linear(x, w)
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
    # the sdpa fallback with its boolean mask agrees with the native kernels
    if not pre_rotated:
        with torch.no_grad():
            sd = ops.rope_attention_qkv(ops.linear(x, w), cos, sin, H, Hkv, causal=True, impl="sdpa", doc=doc)
        assert _rel_err(sd, ref) < 2e-2


@pytest.mark.gpu
def test_model_logits_do_not_depend_on_position_in_window_gpu():
    assert _translation_invariance(_dev(), torch.bfloat16, 256, 128, attn_impl="native") < 2e-2


@pytest.mark.gpu
def test_trainer_document_mask_gpu_eager_and_cuda_graph(tmp_path):
    from prime_b200.config import load_config
    from prime_b200.trainer import Trainer

    ds = _tokenize(tmp_path, _corpus_docs(200))
    base = ["--name_model", "debugmodel", "--data.fake", "false", "--data.dataset_name_or_paths", str(ds), "--data.seq_length", "128",
            "--data.document_mask", "true", "--optim.batch_size", "4", "--train.micro_bs", "2", "--optim.warmup_steps", "2",
            "--optim.total_steps", "10", "--optim.optim.lr", "3e-3", "--train.attn_impl", "native"]  # fmt: skip
    runs = {}
    for graphs in ("false", "true"):
        t = Trainer(load_config(base + ["--train.cuda_graphs", graphs]), model_overrides={"n_heads": 4})  # head size 64
        assert t.model.doc_eos_id == 256 and t.accum == 2
        runs[graphs] = [float(t.inner_step().loss.item()) for _ in range(8)]
        t.close()
    eager, graph = runs["false"], runs["true"]
    assert all(np.isfinite(eager)) and eager[-1] < eager[0]
    # the first loss comes from the forward alone: the replayed graph computed the document bounds of the batch it was given
    assert graph[0] == eager[0]
    # later steps: eager and captured micro-steps of this engine are not bitwise equal even without document masking (about 1e-3
    # relative after a few steps on this model, either way)
    np.testing.assert_allclose(graph, eager, rtol=2e-3)
