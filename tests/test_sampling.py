"""Token sampling on the CPU: the Philox stream against its known answers, the torch reference (``ops.reference.sample_tokens``)
against the fp64 oracle of ``test_sampling_gpu.py`` on random and heavily tied logits, the same comparison rejecting plausible
bugs, device-sampled generation against the recompute loop, and the launcher's argument checks."""

import math

import pytest
import torch

from prime_b200 import eval as ev
from prime_b200 import ops
from prime_b200.models.llama import build_model
from prime_b200.ops import reference as Rf
from test_sampling_gpu import GRID, compare_tokens, logit_rows, oracle, philox_py, uniforms

# key (lo, hi), counter words → output words (Random123's known-answer vectors for Philox4x32-10)
KAT = [((0x00000000, 0x00000000), (0, 0, 0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
       ((0xFFFFFFFF, 0xFFFFFFFF), (M := 0xFFFFFFFF, M, M, M), (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
       ((0xA4093822, 0x299F31D0), (0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]  # fmt: skip


@pytest.mark.parametrize("i", range(len(KAT)))
def test_philox_known_answers(i):
    (k0, k1), ctr, want = KAT[i]
    got = Rf.philox4x32_10(torch.tensor([k0, k1]), torch.tensor(ctr))
    assert [int(v) for v in got] == list(want)
    assert philox_py(k0 | k1 << 32, ctr) == want


def _positions(B, P, base=3):
    return [[base + 11 * b + q for q in range(P)] for b in range(B)]


def _reference_draws(logits, knobs, seeds, positions):
    """Tokens [B, P] of the reference, one call per position column."""
    B, P = len(positions), len(positions[0])
    s = torch.tensor(seeds, dtype=torch.int64)
    cols = [Rf.sample_tokens(logits, knobs[0], knobs[1], knobs[2], knobs[3], s, torch.tensor([p[q] for p in positions])) for q in range(P)]
    return torch.stack(cols, dim=1)


def _tied_logits(B, V, seed):
    """Heavily tied rows: a handful of distinct bf16 values."""
    g = torch.Generator().manual_seed(seed)
    return (torch.randint(-4, 5, (B, V), generator=g).float() * 0.5).to(torch.bfloat16)


CASES = {"randn": lambda: logit_rows(8, 3000, 2.0, seed=1), "tied": lambda: _tied_logits(8, 3000, seed=2),
         "wide": lambda: logit_rows(8, 500, 30.0, seed=3)}  # fmt: skip
EDGE = [(1.0, 1, 1.0, 0.0), (1.0, 3000, 1.0, 0.0), (1.0, 3010, 1.0, 0.0), (1.0, 0, 1e-7, 0.0), (0.9, 0, 1.0, 1.0),
        (1.0, 5, 0.3, 0.2)]  # fmt: skip


@pytest.mark.parametrize("case", sorted(CASES))
def test_reference_matches_oracle(case):
    logits = CASES[case]()
    B, V = logits.shape
    seeds = [17 + 5 * b for b in range(B)]
    pos = _positions(B, 64)
    u = uniforms(seeds, pos)
    draws = ambiguous = 0
    for knobs in GRID + EDGE:
        ref, amb = oracle(logits, *knobs, u)
        got = _reference_draws(logits, knobs, seeds, pos)
        ambiguous += compare_tokens(got, ref, amb, f"{case} {knobs}")
        draws += got.numel()
        if knobs[0] > 0:  # the keep-set itself, row by row, wherever the oracle's is unambiguous
            keep = Rf.sample_keep(logits, *knobs)
            for b in range(B):
                if not bool(amb[b].all()):
                    kept = set(int(i) for i in ref[b][~amb[b]])
                    assert all(bool(keep[b, i]) for i in kept), (case, knobs, b)
    assert ambiguous < 0.01 * draws


def test_keep_set_edges():
    x = torch.tensor([[3.0, 1.0, 3.0, 2.0, 2.0, -1.0]])
    assert Rf.sample_keep(x, 1.0, top_k=1).tolist() == [[True, False, True, False, False, False]]  # ties at the k-th stay
    assert Rf.sample_keep(x, 1.0, top_k=3).tolist() == [[True, False, True, True, True, False]]
    assert Rf.sample_keep(x, 1.0, top_k=6).all() and Rf.sample_keep(x, 1.0, top_k=16).all()
    assert Rf.sample_keep(x, 1.0, top_p=1e-6).tolist() == [[True, False, True, False, False, False]]  # the top tie group
    assert Rf.sample_keep(x, 1.0, min_p=1.0).tolist() == [[True, False, True, False, False, False]]
    assert Rf.sample_keep(torch.full((1, 7), 0.25), 0.5, top_k=2, top_p=0.1, min_p=1.0).all()  # all equal: one tie group
    # top-p crossing inside the second group keeps all of it: masses e^0, e^0, e^-1, e^-1 (, e^-2, e^-4)
    m = math.exp(-1)
    need = (2 + m) / (2 + 2 * m + math.exp(-2) + math.exp(-4))
    assert Rf.sample_keep(x, 1.0, top_p=need).tolist() == [[True, False, True, True, True, False]]


# ------------------------------------------------------------------------------------------- the comparison rejects bugs
def _draw_with(logits, keep, seeds, positions, shift=0):
    """The reference's draw over a given keep-set, with the result moved ``shift`` indices (a mutant of the inverse CDF)."""
    mass = Rf.sample_masses(logits, 1.0)
    cum = torch.where(keep, mass, 0).cumsum(-1)
    r = Rf.sample_uniform_bits(torch.tensor(seeds), torch.tensor(positions))
    a = 2 * r + 1
    M = cum[:, -1]
    target = a * (M >> 25) + ((a * (M & (2**25 - 1))) >> 25)
    return ((cum <= target.view(-1, 1)).sum(-1) + shift).clamp(max=logits.shape[1] - 1)


def _mutant_case():
    logits = _tied_logits(6, 400, seed=9)
    seeds = [3 + b for b in range(6)]
    pos = _positions(6, 64, base=20)
    knobs = (1.0, 0, 0.6, 0.0)
    ref, amb = oracle(logits, *knobs, uniforms(seeds, pos))
    keep = Rf.sample_keep(logits, *knobs)

    def draws(keep_=keep, seeds_=seeds, pos_=pos, shift=0):
        return torch.stack([_draw_with(logits, keep_, seeds_, [p[q] for p in pos_], shift) for q in range(len(pos[0]))], dim=1)

    return logits, keep, ref, amb, draws


def _rejects(got, ref, amb) -> bool:
    try:
        compare_tokens(got, ref, amb, "mutant")
    except AssertionError:
        return True
    return False


def test_checker_accepts_the_correct_draw():
    _, _, ref, amb, draws = _mutant_case()
    assert not _rejects(draws(), ref, amb)


def test_checker_rejects_top_p_dropping_the_boundary_tie_group():
    logits, keep, ref, amb, draws = _mutant_case()
    lf = logits.float()
    boundary = torch.where(keep, lf, math.inf).amin(-1, keepdim=True)  # the lowest kept value: the group that crossed p
    assert _rejects(draws(keep_=keep & (lf > boundary)), ref, amb)


def test_checker_rejects_inverse_cdf_off_by_one():
    _, _, ref, amb, draws = _mutant_case()
    assert _rejects(draws(shift=1), ref, amb)


def test_checker_rejects_counter_from_the_loop_step():
    _, _, ref, amb, draws = _mutant_case()
    steps = [list(range(64)) for _ in range(6)]  # the step index instead of the token's position in its row
    assert _rejects(draws(pos_=steps), ref, amb)


def test_checker_rejects_swapped_row_seeds():
    _, _, ref, amb, draws = _mutant_case()
    seeds = [3 + b for b in range(6)]
    seeds[0], seeds[1] = seeds[1], seeds[0]
    assert _rejects(draws(seeds_=seeds), ref, amb)


# ------------------------------------------------------------------------------------------------------ generation (CPU)
def test_device_sampled_generation_equals_recompute_row_by_row():
    model = build_model("debugmodel", device="cpu", dtype=torch.float32, max_seq_len=40)
    prompts = [[5, 9, 100, 3], [7] * 31, [1, 2]]
    kw = dict(temperature=0.9, top_k=200, top_p=0.9, min_p=0.02)
    batch = ev.generate_batch(model, prompts, max_new=16, seed=21, sampler="device", **kw)
    assert [len(r) for r in batch] == [20, 40, 18]  # max_new, max_seq_len, max_new
    assert batch == [ev._generate_recompute(model, p, max_new=16, seed=21 + b, sampler="device", **kw) for b, p in enumerate(prompts)]
    assert batch == ev.generate_batch(model, prompts, max_new=16, seed=21, sampler="device", **kw)
    assert batch != ev.generate_batch(model, prompts, max_new=16, seed=22, sampler="device", **kw)
    # EOS: the row stops right after it, the EOS kept; the other rows go on
    eos = batch[0][6]
    stopped = ev.generate_batch(model, prompts, max_new=16, seed=21, sampler="device", eos_id=eos, **kw)
    assert stopped[0][: len(stopped[0])] == batch[0][: len(stopped[0])] and stopped[0][-1] == eos and len(stopped[0]) <= 7
    for b, p in enumerate(prompts):
        assert stopped[b] == ev._generate_recompute(model, p, max_new=16, seed=21 + b, sampler="device", eos_id=eos, **kw)


def test_device_greedy_equals_host_greedy():
    model = build_model("debugmodel", device="cpu", dtype=torch.float32)
    prompts = [[5, 9, 100, 3], [7] * 11, [1, 2]]
    host = ev.generate_batch(model, prompts, max_new=24)
    assert ev.generate_batch(model, prompts, max_new=24, sampler="device", top_p=0.5, min_p=0.3) == host


def test_host_sampler_defaults_keep_their_stream():
    """top_p = 1 and min_p = 0 leave the host sampler's draws as they were; top-p restricts them to the reference keep-set."""
    g = torch.Generator().manual_seed(0)
    row = torch.randn(300, generator=g) * 3
    from prime_b200.inference import sample

    old = []
    gen = torch.Generator().manual_seed(4)
    for _ in range(50):  # the draw of earlier versions, written out
        x = row / 0.8
        kth = torch.topk(x, 40).values[-1]
        old.append(int(torch.multinomial(torch.softmax(x.masked_fill(x < kth, float("-inf")), -1), 1, generator=gen)))
    gen = torch.Generator().manual_seed(4)
    assert [sample(row, 0.8, 40, gen) for _ in range(50)] == old
    keep = Rf.sample_keep(row.view(1, -1), 0.8, 40, 0.5, 0.0)[0]
    gen = torch.Generator().manual_seed(4)
    assert all(bool(keep[sample(row, 0.8, 40, gen, top_p=0.5)]) for _ in range(50))


def test_sample_tokens_rejects_bad_arguments():
    x = torch.zeros(2, 10)
    s, p = torch.zeros(2, dtype=torch.int64), torch.zeros(2, dtype=torch.int32)
    for bad in (dict(temperature=-1.0), dict(temperature=math.inf), dict(temperature=1.0, top_k=-1), dict(temperature=1.0, top_p=0.0),
                dict(temperature=1.0, top_p=1.5), dict(temperature=1.0, min_p=-0.1), dict(temperature=1.0, min_p=1.1)):
        with pytest.raises(ValueError):
            ops.sample_tokens(x, **bad, seeds=s, positions=p)


def test_sample_launcher_rejects_impossible_arguments_before_touching_the_device():
    from prime_b200.ops import _lib

    try:
        lib = _lib.load()
    except Exception as e:  # noqa: BLE001
        pytest.skip(f"native library not loadable here: {e}")
    a = 1 << 20  # 16-byte aligned, never dereferenced: every call below is rejected first

    def call(logits=a, ld=64, B=2, V=64, T=1.0, k=0, p=1.0, m=0.0, seeds=a, pos=a, out=a, hist=None, n_out=None, act=None, plen=None,
             max_new=8, max_seq=64):  # fmt: skip
        return lib.pb_sample_tokens(logits, ld, B, V, T, k, p, m, seeds, pos, out, hist, n_out, act, plen, max_new, max_seq, -1, None)

    assert call(logits=None) == -1 and call(seeds=None) == -1 and call(pos=None) == -1 and call(out=None) == -1
    assert call(hist=a) == -1 and call(hist=a, n_out=a, act=a) == -1  # bookkeeping is all or nothing
    assert call(B=0) == -3 and call(V=0) == -3 and call(ld=63) == -3 and call(V=1 << 23, ld=1 << 23) == -3
    assert call(T=-0.5) == -4 and call(T=math.inf) == -4 and call(T=math.nan) == -4 and call(k=-1) == -4
    assert call(p=0.0) == -4 and call(p=1.01) == -4 and call(p=math.nan) == -4 and call(m=-0.01) == -4 and call(m=1.5) == -4
    book = dict(hist=a, n_out=a, act=a, plen=a)
    assert call(**book, max_new=0) == -5 and call(**book, max_seq=0) == -5
    assert call(logits=a + 1) == -6 and call(seeds=a + 4) == -6 and call(out=a + 4) == -6 and call(pos=a + 2) == -6
    assert call(**{**book, "hist": a + 4}) == -6 and call(**{**book, "n_out": a + 2}) == -6 and call(**{**book, "plen": a + 1}) == -6
