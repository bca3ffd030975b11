"""Speculative decoding on the CPU: the accept rule of ``ops.spec_accept`` (``reference.spec_accept_row``) keeps the target's
distribution exactly, greedy speculation reproduces greedy generation token for token, and bad input is refused before any device
work."""

import pytest
import torch

from prime_b200 import inference
from prime_b200.models.llama import build_model
from prime_b200.ops import reference as Rf

# (temperature, top_k, top_p, min_p)
KNOBS = [(1.0, 0, 1.0, 0.0), (0.7, 0, 1.0, 0.0), (1.3, 10, 1.0, 0.0), (1.0, 0, 0.8, 0.0), (0.8, 20, 0.9, 0.05), (1.0, 0, 1.0, 0.2)]


def _accept_share(P: int, Q: int) -> float:
    """P(accept) over the 2^24 values of r: #{r : (2r + 1)·Q < 2^25·P} / 2^24."""
    if P == 0:
        return 0.0
    if Q == 0:
        return 1.0
    odd = (((1 << 25) * P - 1) // Q + 1) // 2  # odd numbers 2r + 1 <= (2^25·P - 1) // Q
    return min(odd, 1 << 24) / 2.0**24


@pytest.mark.parametrize("knobs", KNOBS)
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_accept_rule_keeps_the_target_distribution(knobs, seed):
    g = torch.Generator().manual_seed(seed)
    V = 50
    p = torch.randn(1, V, generator=g) * 2
    q = p + torch.randn(1, V, generator=g) * 1.5  # a draft near the target; with filters it drafts tokens outside its keep-set
    P = [int(x) for x in Rf.spec_masses(p, *knobs)[0]]
    Q = [int(x) for x in Rf.spec_masses(q, *knobs)[0]]
    sq = sum(Q)
    R = [max(0, a - b) for a, b in zip(P, Q)]
    if sum(R) == 0:
        R = P
    law = [0.0] * V
    for d in range(V):
        if Q[d] == 0:
            continue
        acc = _accept_share(P[d], Q[d])
        law[d] += Q[d] / sq * acc
        for y in range(V):
            law[y] += Q[d] / sq * (1 - acc) * R[y] / sum(R)
    sp = sum(P)
    for y in range(V):
        assert abs(law[y] - P[y] / sp) <= 2.0**-20, (y, law[y], P[y] / sp)


@pytest.mark.parametrize("knobs", KNOBS[:3])
def test_accept_rule_implementation_matches_its_formula(knobs):
    """spec_accept_row's decision is the integer comparison with r from Philox counter (L + 1, 1, 0, 0)."""
    g = torch.Generator().manual_seed(7)
    V, L = 40, 33
    p, q = torch.randn(1, 2, V, generator=g), torch.randn(1, V, generator=g)
    P, Q = Rf.spec_masses(p[0], *knobs), Rf.spec_masses(q, *knobs)
    seen = set()
    for seed in range(200):
        d = int(torch.multinomial(Q[0].double(), 1, generator=g))
        n, y = Rf.spec_accept_row(P, Q, [d], seed, L, greedy=False)
        r = Rf._philox_r(seed, L + 1, 1)
        assert (n == 1) == ((2 * r + 1) * int(Q[0, d]) < (1 << 25) * int(P[0, d]))
        assert int(P[n, y]) > 0  # y is always a token the target keeps
        seen.add(n)
    assert seen == {0, 1}


def test_greedy_rule_is_argmax():
    g = torch.Generator().manual_seed(3)
    p = torch.randn(4, 30, generator=g)
    P = Rf.spec_masses(p, 0.0)
    am = p.argmax(-1).tolist()
    Q = torch.zeros(3, 30, dtype=torch.long)
    assert Rf.spec_accept_row(P, Q, am[:3], 0, 10, greedy=True) == (3, am[3])
    assert Rf.spec_accept_row(P, Q, [am[0], (am[1] + 1) % 30, am[2]], 0, 10, greedy=True) == (1, am[1])


# ------------------------------------------------------------------------------------------------------ end to end on the CPU
def _pair(**target_overrides):
    t = build_model("debugmodel", dtype=torch.float32, seed=1, **target_overrides)
    d = build_model("debugmodel", dtype=torch.float32, seed=2, n_layers=1)
    return t, d


PROMPTS = [[1, 2, 3, 4, 5], [7, 8, 9], [10] * 12, [300]]


@pytest.mark.parametrize("k", [1, 3, 8])
def test_greedy_speculation_equals_greedy_generation(k):
    t, d = _pair()
    ref = inference.generate_batch(t, PROMPTS, max_new=20, sampler="device")
    for draft in (d, t):
        r = inference.generate_speculative(t, draft, PROMPTS, k=k, max_new=20)
        assert r.ids == ref
        assert 0 < r.drafted <= k * 19 * len(PROMPTS) and 0 <= r.accepted <= r.drafted
    s = inference.generate_speculative(t, t, PROMPTS, k=k, max_new=20)
    assert s.accepted == s.drafted and s.rounds == -(-19 // (k + 1))  # self-draft: k + 1 tokens per round


def test_eos_in_the_middle_of_an_accepted_run_stops_the_row():
    t, _ = _pair()
    ref0 = inference.generate_batch(t, PROMPTS, max_new=20, sampler="device")
    eos = ref0[0][len(PROMPTS[0]) + 4]  # the fifth new token of row 0: inside the first run of 8 self-drafted tokens
    ref = inference.generate_batch(t, PROMPTS, max_new=20, sampler="device", eos_id=eos)
    assert ref[0][-1] == eos and len(ref[0]) == len(PROMPTS[0]) + 5
    for k in (1, 3, 8):
        assert inference.generate_speculative(t, t, PROMPTS, k=k, max_new=20, eos_id=eos).ids == ref


@pytest.mark.parametrize("max_new,max_seq_len", [(1, 2048), (2, 2048), (7, 2048), (30, 16)])
def test_max_new_and_max_seq_len_cut_offs(max_new, max_seq_len):
    t, d = _pair(max_seq_len=max_seq_len)
    ref = inference.generate_batch(t, PROMPTS, max_new=max_new, sampler="device")
    for k in (1, 3, 8):
        assert inference.generate_speculative(t, d, PROMPTS, k=k, max_new=max_new).ids == ref
        assert inference.generate_speculative(t, t, PROMPTS, k=k, max_new=max_new).ids == ref


def test_document_masking_and_window_on_the_target():
    t, d = _pair(sliding_window=6)
    t.doc_eos_id = d.doc_eos_id = 5
    prompts = [[1, 2, 5, 3, 4, 5, 9], [5, 5, 7], [11, 12, 13, 14, 15, 16, 17, 18, 19]]
    ref = inference.generate_batch(t, prompts, max_new=24, sampler="device")
    # a drafted EOS starts a new document for the later queries of the verify step: use the target's own EOS-bearing output
    for k in (1, 3, 8):
        assert inference.generate_speculative(t, d, prompts, k=k, max_new=24).ids == ref
        assert inference.generate_speculative(t, t, prompts, k=k, max_new=24).ids == ref


def test_eos_among_the_drafts_opens_a_document_in_the_verify_step():
    t, _ = _pair()
    ref0 = inference.generate_batch(t, PROMPTS, max_new=12, sampler="device")
    t.doc_eos_id = ref0[0][len(PROMPTS[0]) + 2]  # drafted (and accepted) in the middle of a self-drafted run
    ref = inference.generate_batch(t, PROMPTS, max_new=12, sampler="device")
    assert inference.generate_speculative(t, t, PROMPTS, k=8, max_new=12).ids == ref


def test_sampled_speculation_is_deterministic_and_self_draft_accepts_all():
    t, d = _pair()
    kw = dict(k=3, max_new=16, temperature=0.9, top_p=0.9, seed=5)
    a = inference.generate_speculative(t, d, PROMPTS, **kw)
    assert a == inference.generate_speculative(t, d, PROMPTS, **kw)
    s = inference.generate_speculative(t, t, PROMPTS, **kw)
    assert s.accepted == s.drafted  # P == Q exactly: every draft is accepted


# ------------------------------------------------------------------------------------------------------------- bad input
def test_bad_pairs_and_k_are_refused():
    t, d = _pair()
    other_v = build_model("debugmodel", dtype=torch.float32, seed=2, vocab_size=1024)
    with pytest.raises(ValueError, match="vocabulary"):
        inference.generate_speculative(t, other_v, PROMPTS, max_new=4)
    d.doc_eos_id = 3
    with pytest.raises(ValueError, match="doc_eos_id"):
        inference.generate_speculative(t, d, PROMPTS, max_new=4)
    d.doc_eos_id = None
    for k in (0, 16):
        with pytest.raises(ValueError, match="k must be"):
            inference.generate_speculative(t, d, PROMPTS, k=k, max_new=4)
    with pytest.raises(ValueError, match="top_p"):
        inference.generate_speculative(t, d, PROMPTS, max_new=4, temperature=1.0, top_p=0.0)


def test_speculative_launchers_reject_impossible_arguments_before_touching_the_device():
    from prime_b200.ops import _lib

    try:
        lib = _lib.load()
    except Exception as e:  # noqa: BLE001
        pytest.skip(f"native library not loadable here: {e}")
    a = 1 << 20  # 16-byte aligned, never dereferenced: every call below is rejected first
    odd = a + 2

    def adv(tokens=a, lo_q=a, last=a, B=4, T=3):
        return lib.pb_verify_advance(tokens, T, -1, a, a, lo_q, last, B, None)

    assert adv(tokens=None) == -1 and adv(lo_q=None) == -1 and adv(B=0) == -3 and adv(T=0) == -3 and adv(last=odd) == -6
    assert adv(lo_q=a + 1) == -6

    def app(qkv=a, kv=a, B=2, T=4, H=8, Hkv=2, D=128, cap=256):
        return lib.pb_kv_append_tokens(qkv, kv, a, a, a, B, T, H, Hkv, D, cap, None)

    assert app(kv=None) == -1 and app(D=96) == -2 and app(T=0) == -3 and app(H=6, Hkv=4) == -3 and app(qkv=odd) == -6

    def attn(qkv=a, lo=None, window=0, out=a, part=None, T=5, H=8, Hkv=2, D=64, cap=256, splits=1):
        return lib.pb_verify_attn(qkv, a, a, lo, window, out, part, 2, T, H, Hkv, D, cap, splits, 0.125, None)

    assert attn(out=None) == -1 and attn(splits=2) == -1 and attn(D=32) == -2 and attn(T=0) == -3 and attn(H=6, Hkv=4) == -3
    assert attn(window=-1) == -4 and attn(splits=0) == -5 and attn(qkv=odd) == -6 and attn(lo=a + 1) == -6

    def acc(target=a, draft=a, B=2, k=3, V=2048, ldt=2048, temperature=1.0, top_p=1.0, history=a, n_out=a, max_new=8, seeds=a):
        ptrs = [seeds, a, a, a, a, a, a, a, a, a, history, n_out, a, a]
        return lib.pb_spec_accept(target, ldt, draft, V, B, k, V, temperature, 0, top_p, 0.0, *ptrs, max_new, 64, -1, a, a, None)

    assert acc(target=None) == -1 and acc(history=None) == -1 and acc(seeds=None) == -1
    assert acc(k=0) == -7 and acc(k=16) == -7
    assert acc(B=0) == -3 and acc(V=0) == -3 and acc(ldt=100) == -3
    assert acc(temperature=-1.0) == -4 and acc(top_p=0.0) == -4 and acc(max_new=0) == -5
    assert acc(target=a + 1) == -6 and acc(history=a + 4) == -6 and acc(n_out=a + 2) == -6
