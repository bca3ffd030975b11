"""Speculative decoding on an H100: the verify-step kernels against fp64 and against the decode kernels, the accept kernel against
``reference.spec_accept``, the law of the emitted tokens, self-draft acceptance, greedy agreement and graph replay."""

import math

import numpy as np
import pytest
import torch

from prime_b200 import inference, ops
from prime_b200.models.llama import build_model
from prime_b200.ops import reference as Rf


def _dev():
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def native():
    from prime_b200.ops import _lib

    return _lib.load()  # a GPU box without the native library is a hard failure, never a silent fallback


def _verify64(q, kv, length, lo_q, window):
    """fp64 attention of q [B, T, H, D] by the verify rule."""
    B, T, H, D = q.shape
    cap = kv.shape[1]
    Hkv = kv.shape[2] // (2 * D)
    kf = kv[..., : Hkv * D].double().reshape(B, cap, Hkv, D).repeat_interleave(H // Hkv, dim=2)
    vf = kv[..., Hkv * D :].double().reshape(B, cap, Hkv, D).repeat_interleave(H // Hkv, dim=2)
    pos = length.long().view(B, 1) - T + torch.arange(T, device=q.device).view(1, T)  # [B, T]
    start = torch.zeros_like(pos) if lo_q is None else lo_q.long()
    if window:
        start = torch.maximum(start, pos + 1 - window)
    k = torch.arange(cap, device=q.device).view(1, 1, cap)
    vis = (k >= start.unsqueeze(-1)) & (k <= pos.unsqueeze(-1))  # [B, T, cap]
    s = torch.einsum("bthd,bkhd->bthk", q.double(), kf) / math.sqrt(D)
    p = s.masked_fill(~vis.unsqueeze(2), -math.inf).softmax(-1)
    return torch.einsum("bthk,bkhd->bthd", p, vf)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["plain", "window", "lo", "eos"])
@pytest.mark.parametrize("T", [1, 2, 5, 16])
@pytest.mark.parametrize("G", [1, 4, 8, 16])
@pytest.mark.parametrize("D", [64, 128])
def test_verify_attn_matches_fp64_and_decode_at_t1(native, D, G, T, mode):
    dev = _dev()
    g = torch.Generator(device=dev).manual_seed(D * 1000 + G * 10 + T)
    Hkv, cap = 2, 2048
    H = G * Hkv
    lens = [T, T + 1, 64 + T, 700, 2048]
    B = len(lens)
    kv = torch.randn(B, cap, 2 * Hkv * D, device=dev, generator=g).to(torch.bfloat16)
    qkv = torch.randn(B, T, (H + 2 * Hkv) * D, device=dev, generator=g).to(torch.bfloat16)
    length = torch.tensor(lens, dtype=torch.int32, device=dev)
    window = 100 if mode == "window" else 0
    lo_q = None
    if mode == "lo":
        lo_q = torch.tensor([0, 1, 30, 500, 1000], dtype=torch.int32, device=dev).view(B, 1).expand(B, T).contiguous()
    elif mode == "eos":  # an EOS at draft t0 - 1 opens a document at the query of t0
        t0 = T // 2
        lo_q = torch.zeros(B, T, dtype=torch.int32, device=dev)
        lo_q[:, t0:] = (length - T + t0).view(B, 1)
    out = ops.verify_attention(qkv, kv, length, lo_q, window, H, Hkv)
    q = qkv.view(B, T, H + 2 * Hkv, D)[:, :, :H]
    ref = _verify64(q, kv, length, lo_q, window)
    err = (out.view(B, T, H, D).double() - ref).abs()
    assert bool((err <= 2.0**-7 * ref.abs() + 4e-3).all()), float(err.max())
    if T == 1:
        dec = ops.decode_attention(qkv.view(B, -1), kv, length, None if lo_q is None else lo_q[:, 0].contiguous(), window, H, Hkv)
        assert torch.equal(out.view(B, -1), dec)


@pytest.mark.gpu
@pytest.mark.parametrize("T", [1, 3, 9])
def test_kv_append_tokens_and_verify_advance_match_their_references(native, T):
    dev = _dev()
    g = torch.Generator(device=dev).manual_seed(T)
    B, H, Hkv, D, cap = 3, 8, 2, 128, 256
    cos, sin = Rf.rope_tables(cap, D, device=dev)
    qkv = torch.randn(B, T, (H + 2 * Hkv) * D, device=dev, generator=g).to(torch.bfloat16)
    kv = torch.randn(B, cap, 2 * Hkv * D, device=dev, generator=g).to(torch.bfloat16)
    length = torch.tensor([T, 100, cap + 2], dtype=torch.int32, device=dev)  # row 2 partly past the capacity: left alone
    q1, kv1 = qkv.clone(), kv.clone()
    ops.kv_append_tokens(q1, kv1, length, cos, sin, H, Hkv)
    q2, kv2 = qkv.float().cpu(), kv.float().cpu()  # the fp32 reference path, rounded as the kernel rounds
    ops.kv_append_tokens(q2, kv2, length.cpu(), cos.cpu(), sin.cpu(), H, Hkv)
    assert torch.equal(q1.float().cpu(), q2.to(torch.bfloat16).float()) and torch.equal(kv1.float().cpu(), kv2.to(torch.bfloat16).float())

    eos = 7
    toks = torch.tensor([[7, 1, 7, 2, 3][:T] + [4] * max(0, T - 5) for _ in range(B)], dtype=torch.int64)[:, :T]
    state = [torch.tensor([5, 9, 0], dtype=torch.int32), torch.tensor([0, 3, 0], dtype=torch.int32), torch.tensor([7, 1, 2])]
    gpu = [s.to(dev) for s in state]
    lo_g = ops.verify_advance(toks.to(dev).contiguous(), *gpu, eos)
    lo_c = ops.verify_advance(toks, *state, eos)
    assert torch.equal(lo_g.cpu(), lo_c) and all(torch.equal(a.cpu(), b) for a, b in zip(gpu, state))


def _accept_case(V, B, k, knobs, seed):
    dev = _dev()
    g = torch.Generator().manual_seed(seed)
    tl = (torch.randn(B, k + 1, V, generator=g) * 2.5).to(torch.bfloat16)
    dl = (tl[:, :k].transpose(0, 1).float() + torch.randn(k, B, V, generator=g)).to(torch.bfloat16)
    L = 300
    cache = lambda: inference.KVCache(torch.empty(1, 1, 1, 8), torch.full((B,), L + k + 1, dtype=torch.int32),  # noqa: E731
                                      torch.zeros(B, dtype=torch.int32), torch.zeros(B, dtype=torch.int64), None, None, None)  # fmt: skip
    seeds = torch.arange(B, dtype=torch.int64) * 7919 + seed
    toks = torch.empty(B, k + 1, dtype=torch.int64)
    toks[:, 0] = 1
    for i in range(k):  # the drafts as the draft sampler draws them
        toks[:, i + 1] = ops.sample_tokens(dl[i].to(dev), **knobs, seeds=seeds.to(dev), positions=torch.full((B,), L + i + 1, dtype=torch.int32,
                                                                                                             device=dev)).cpu()  # fmt: skip
    lo_q = torch.arange(k + 1, dtype=torch.int32).repeat(B, 1)
    st = inference.SampleState.allocate([[1] * 10] * B, 64, 4096, None, "cpu")
    out = {}
    for where in ("cpu", "cuda"):
        dv = torch.device(where)
        t, d = cache(), cache()
        for c in (t, d):
            c.len, c.lo, c.last_tok = c.len.to(dv), c.lo.to(dv), c.last_tok.to(dv)
        s = inference.SampleState(*(x.to(dv) if isinstance(x, torch.Tensor) else x for x in (st.tokens.clone(), st.history.clone(),
                                  st.n_out.clone(), st.active.clone(), st.prompt_len.clone())), st.max_seq_len, st.eos_id)  # fmt: skip
        pend, dr, ac = (torch.zeros(B, dtype=torch.int64, device=dv) for _ in range(3))
        ops.spec_accept(tl.to(dv), dl.to(dv), **knobs, seeds=seeds.to(dv), tokens=toks.to(dv), lo_q=lo_q.to(dv), target=t, draft=d,
                        state=s, pending=pend, drafted=dr, accepted=ac)  # fmt: skip
        out[where] = [x.cpu() for x in (ac, pend, s.history, s.n_out, t.len, t.lo, t.last_tok, d.len, d.lo, d.last_tok, dr)]
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("knobs", [dict(temperature=0.0), dict(temperature=1.0), dict(temperature=0.8, top_p=0.9),
                                   dict(temperature=1.2, top_k=50, min_p=0.02)], ids=["greedy", "t1", "topp", "topk-minp"])  # fmt: skip
@pytest.mark.parametrize("V", [32000, 128256])
def test_spec_accept_kernel_matches_reference(native, V, knobs):
    B, k = 96, 4
    out = _accept_case(V, B, k, knobs, seed=V % 97)
    cpu, gpu = out["cpu"], out["cuda"]
    rows = torch.ones(B, dtype=torch.bool)
    for a, b in zip(cpu, gpu):
        rows &= (a == b).view(B, -1).all(-1)
    # rows may differ only where two fp64 exp results round to different fixed-point masses: allowed on under 1 % of the rows
    assert int((~rows).sum()) <= B // 100, f"{int((~rows).sum())} of {B} rows differ"
    assert int(cpu[0].sum()) > 0 or knobs.get("temperature") == 0.0


@pytest.mark.gpu
@pytest.mark.parametrize("knobs", [dict(temperature=1.0), dict(temperature=0.8, top_p=0.9)], ids=["t1", "t08-topp09"])
def test_first_emitted_token_has_the_target_law(native, knobs):
    """16 384 rows of one round, seeds s + b, k = 3, a draft whose logits are the target's plus noise: the first token the round
    emits (d_1 if accepted, else the residual draw) follows the target's filtered distribution P_1."""
    from scipy.stats import chisquare

    dev = _dev()
    V, B, k = 2048, 16384, 3
    g = torch.Generator().manual_seed(11)
    p1 = (torch.randn(V, generator=g) * 2.0).to(torch.bfloat16)
    tl = torch.stack([p1] + [(torch.randn(V, generator=g) * 2).to(torch.bfloat16) for _ in range(k)]).expand(B, k + 1, V).contiguous()
    dl = torch.stack([(p1.float() + torch.randn(V, generator=g)).to(torch.bfloat16) for _ in range(k)]).view(k, 1, V).expand(k, B, V).contiguous()
    L = 77
    seeds = torch.arange(B, dtype=torch.int64, device=dev) + 1000
    toks = torch.zeros(B, k + 1, dtype=torch.int64, device=dev)
    for i in range(k):
        toks[:, i + 1] = ops.sample_tokens(dl[i].to(dev), **knobs, seeds=seeds,
                                           positions=torch.full((B,), L + i + 1, dtype=torch.int32, device=dev))  # fmt: skip
    mk = lambda: inference.KVCache(torch.empty(1), torch.full((B,), L + k + 1, dtype=torch.int32, device=dev),  # noqa: E731
                                   torch.zeros(B, dtype=torch.int32, device=dev), torch.zeros(B, dtype=torch.int64, device=dev),
                                   None, None, None)  # fmt: skip
    st = inference.SampleState.allocate([[1] * 10] * B, 8, 4096, None, dev)
    st.n_out.zero_()
    z = [torch.zeros(B, dtype=torch.int64, device=dev) for _ in range(3)]
    ops.spec_accept(tl.to(dev), dl.to(dev), **knobs, seeds=seeds, tokens=toks, lo_q=torch.zeros(B, k + 1, dtype=torch.int32, device=dev),
                    target=mk(), draft=mk(), state=st, pending=z[0], drafted=z[1], accepted=z[2])  # fmt: skip
    first = st.history[:, 0].cpu()
    P = Rf.spec_masses(p1.view(1, V), **{"temperature": knobs["temperature"], "top_k": 0, "top_p": knobs.get("top_p", 1.0),
                                         "min_p": 0.0})[0].double()  # fmt: skip
    expected = (P / P.sum() * B).numpy()
    counts = np.bincount(first.numpy(), minlength=V).astype(float)
    assert counts[expected == 0].sum() == 0  # nothing outside the target's keep-set
    order = np.argsort(-expected)
    obs, exp = [], []
    o = e = 0.0
    for j in order:  # pool the tail so that every cell expects at least 5
        if expected[j] == 0:
            continue
        o, e = o + counts[j], e + expected[j]
        if e >= 5:
            obs.append(o)
            exp.append(e)
            o = e = 0.0
    if e > 0:
        obs[-1] += o
        exp[-1] += e
    pval = chisquare(obs, exp).pvalue
    assert 0.0 < float(z[2].sum()) < 3 * B  # some drafts accepted, some rejected
    assert pval > 1e-4, pval


@pytest.mark.gpu
@pytest.mark.parametrize("temperature,floor", [(0.0, 0.98), (1.0, 0.95)])
def test_self_draft_accepts_nearly_everything(native, temperature, floor):
    dev = _dev()
    t = build_model("debugmodel", device=dev, seed=1)
    prompts = [[1 + (7 * b + j) % 2000 for j in range(5 + 3 * b)] for b in range(8)]
    r = inference.generate_speculative(t, t, prompts, k=4, max_new=64, temperature=temperature, seed=3)
    assert r.accepted >= floor * r.drafted, (r.accepted, r.drafted)


def _margins(model, seq, P, dev):
    """Teacher-forced top-2 logit margins of model at positions P-1 .. len(seq)-2 (the logits that chose seq[P:])."""
    logits = model(torch.tensor([seq], device=dev)).float()[0]
    top = logits.topk(2, dim=-1).values
    return (top[:, 0] - top[:, 1])[P - 1 : len(seq) - 1].cpu()


@pytest.mark.gpu
def test_greedy_speculation_agrees_with_greedy_generation_on_1b_shape(native):
    dev = _dev()
    t = build_model("1B", device=dev, seed=0)
    d = build_model("150M", device=dev, seed=1)
    prompts = [[1 + (13 * b + 7 * j) % 31999 for j in range(40 + 17 * b)] for b in range(4)]
    ref = inference.generate_batch(t, prompts, max_new=48, sampler="device")
    for draft in (d, t):
        got = inference.generate_speculative(t, draft, prompts, k=4, max_new=48).ids
        for b, p in enumerate(prompts):
            m = _margins(t, ref[b], len(p), dev)
            near = (m < 0.05).nonzero()
            stop = len(p) + (int(near[0]) if len(near) else len(m))
            assert got[b][: stop + 1] == ref[b][: stop + 1], b


@pytest.mark.gpu
@pytest.mark.parametrize("knobs", [dict(temperature=0.0), dict(temperature=1.0, top_p=0.9)], ids=["greedy", "topp"])
def test_captured_round_equals_eager_round(native, knobs):
    dev = _dev()
    t = build_model("debugmodel", device=dev, seed=1)
    d = build_model("debugmodel", device=dev, seed=2, n_layers=1)
    t.doc_eos_id = d.doc_eos_id = 17
    prompts = [[5, 17, 9, 4], [3] * 20, [17, 17, 2]]
    a = inference.generate_speculative(t, d, prompts, k=3, max_new=40, graphs=True, seed=9, **knobs)
    b = inference.generate_speculative(t, d, prompts, k=3, max_new=40, graphs=False, seed=9, **knobs)
    assert a == b
