"""Device token sampling (``ops.sample_tokens``, csrc/sample_sm90.cu) against an fp64 oracle, token for token, and device-sampled
generation on CUDA.

The oracle below is written from the contract alone (``ops.sample_tokens``' docstring), in fp64 and with its own Philox in Python
integers. The kernel computes a token's mass p_i = exp((l_i - l_max)·(1/T)) in fp64 and rounds it to a 2^-40 fixed-point integer:

    x = (l - l_max)·(1/T)   three fp64 roundings (difference, reciprocal, product): |dx| <= 3·2^-53·|x|
    exp                     CUDA's and torch's fp64 exp: <= 1 ulp; taken as 2^-51 relative
    fixed point             <= 2^-41 absolute

so |p_kernel - p_i| <= err_i = p_i·(3·2^-53·|x_i| + 2^-51)·(1 + 2^-10) + 2^-41 (the last factor covers the second-order terms).
Every mass sum is exact in the kernel, so a prefix, the kept mass and the top-p mass are off by at most the sum of err_i over their
terms. A draw is ambiguous when the oracle's target u·mass(kept) lies within E = 2·sum(err over the kept set) + 2^-39 of an
inclusive prefix (both sides of the comparison move), or the row's keep-set is: the top-p mass of the chosen tie group or of the
one above it lies within E_p = 2·sum(err over the top-k set) + 2^-39 of top_p·mass(S), or a logit lies within the fp32 error of
the min-p bound l_max + T·ln(min_p). Only ambiguous draws may differ, and they must stay under 1 % of the draws.
"""

import math

import numpy as np
import pytest
import torch

from prime_b200 import eval as ev
from prime_b200 import inference, ops
from prime_b200.models.llama import build_model

M32 = 0xFFFFFFFF


# ---------------------------------------------------------------------------------------------------------------- the oracle
def philox_py(key: int, counter: tuple[int, int, int, int]) -> tuple[int, int, int, int]:
    """Philox4x32-10 on Python integers: key = 64-bit integer (lo, hi words), counter = four 32-bit words."""
    k0, k1 = key & M32, (key >> 32) & M32
    c = list(counter)
    for r in range(10):
        if r:
            k0, k1 = (k0 + 0x9E3779B9) & M32, (k1 + 0xBB67AE85) & M32
        p0, p1 = 0xD2511F53 * c[0], 0xCD9E8D57 * c[2]
        c = [((p1 >> 32) ^ c[1] ^ k0) & M32, p1 & M32, ((p0 >> 32) ^ c[3] ^ k1) & M32, p0 & M32]
    return tuple(c)


def uniforms(seeds: list[int], positions: list[list[int]]) -> torch.Tensor:
    """u [B, P] in fp64: ((x0 >> 8) + 0.5)·2^-24 for each row's seed at each position."""
    return torch.tensor([[((philox_py(s % 2**64, (q & M32, 0, 0, 0))[0] >> 8) + 0.5) * 2.0**-24 for q in pos]
                         for s, pos in zip(seeds, positions)], dtype=torch.float64)  # fmt: skip


def f32(x: float) -> float:
    return float(np.float32(x))


def oracle(logits: torch.Tensor, temperature: float, top_k: int, top_p: float, min_p: float, u: torch.Tensor):
    """Tokens [B, P] and an ambiguity mask [B, P] for logits [B, V] (any device) and uniforms u [B, P], all in fp64. The sampling
    parameters are taken as the fp32 values the kernel receives."""
    l = logits.double()
    B, V = l.shape
    u = u.to(l.device)
    if temperature == 0:
        return l.argmax(-1, keepdim=True).expand(B, u.shape[1]).cpu(), torch.zeros(u.shape, dtype=torch.bool)
    T, p, m = f32(temperature), f32(top_p), f32(min_p)
    lmax = l.amax(-1, keepdim=True)
    x = (l - lmax) / T
    prob = x.exp()
    err = prob * (3 * 2.0**-53 * x.abs() + 2.0**-51) * (1 + 2.0**-10) + 2.0**-41
    keep = torch.ones_like(l, dtype=torch.bool)
    amb_row = torch.zeros(B, dtype=torch.bool, device=l.device)
    if 0 < top_k < V:
        keep = l >= l.topk(top_k, dim=-1).values[:, -1:]
    if p < 1:
        # mass of {i in S : l_i >= v} for every value v, through the descending order of S
        vals = torch.where(keep, l, -math.inf)
        sv, order = vals.sort(-1, descending=True)
        cm = torch.where(keep.gather(1, order), prob.gather(1, order), 0.0).cumsum(-1)
        n_ge = torch.searchsorted(-sv.contiguous(), -sv.contiguous(), right=True)  # elements >= each sorted value
        mass_ge = cm.gather(1, n_ge - 1)
        total = torch.where(keep, prob, 0.0).sum(-1, keepdim=True)
        need = p * total
        ok = (mass_ge >= need) & torch.isfinite(sv)
        t = torch.where(ok, sv, -math.inf).amax(-1, keepdim=True)  # the largest value whose upper set reaches need
        at_t = (sv == t) & torch.isfinite(sv)
        g_t = torch.where(at_t, mass_ge, math.inf).amin(-1, keepdim=True)
        grp = torch.where(at_t, prob.gather(1, order), 0.0).sum(-1, keepdim=True)
        e_p = 2 * torch.where(keep, err, 0.0).sum(-1, keepdim=True) + 2.0**-39
        above = g_t - grp  # the mass of the groups above t; the top group has none above it to fall back to
        amb_row |= ((g_t - need <= e_p) | ((above > 0) & (need - above <= e_p))).view(B)
        keep &= l >= t
    if m > 0:
        off = T * math.log(m)
        thr = lmax + off
        e_m = 0.0 if off == 0 else 2.0**-22 * abs(off) + 2.0**-23 * thr.abs()
        keep &= l >= thr
        amb_row |= ((l - thr).abs() <= e_m).any(-1) if off != 0 else torch.zeros_like(amb_row)
    C = torch.where(keep, prob, 0.0).cumsum(-1)
    target = u * C[:, -1:]
    tok = torch.searchsorted(C, target, right=True)  # the first index whose inclusive prefix exceeds target
    last = torch.where(keep, torch.arange(V, device=l.device), -1).amax(-1, keepdim=True)
    tok = torch.where(tok < V, tok, last)
    E = 2 * torch.where(keep, err, 0.0).sum(-1, keepdim=True) + 2.0**-39
    amb = torch.searchsorted(C, target + E, right=True) > torch.searchsorted(C, target - E, right=False)
    return tok.cpu(), (amb | amb_row.view(B, 1)).cpu()


def compare_tokens(got: torch.Tensor, ref: torch.Tensor, amb: torch.Tensor, what: str) -> int:
    """Raise on any mismatch the oracle does not mark ambiguous; returns the number of ambiguous draws."""
    bad = (got.cpu() != ref) & ~amb
    if bool(bad.any()):
        b, q = (int(v) for v in bad.nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {got.numel()} draws differ; first at row {b} draw {q}: got {int(got[b, q])} "
                             f"oracle {int(ref[b, q])}")  # fmt: skip
    return int(amb.sum())


# (temperature, top_k, top_p, min_p)
GRID = [(0.0, 0, 1.0, 0.0), (0.7, 0, 1.0, 0.0), (1.0, 0, 1.0, 0.0), (1.5, 0, 1.0, 0.0),
        (1.0, 1, 1.0, 0.0), (1.0, 40, 1.0, 0.0), (0.7, 1000, 1.0, 0.0),
        (1.0, 0, 0.9, 0.0), (0.7, 0, 0.5, 0.0), (1.5, 0, 1e-6, 0.0),
        (1.0, 0, 1.0, 0.05), (1.5, 0, 1.0, 1.0),
        (0.8, 50, 0.9, 0.0), (0.7, 1000, 0.95, 0.02), (1.0, 0, 0.9, 0.1)]  # fmt: skip
POSITIONS = 256


def logit_rows(B: int, V: int, scale: float, seed: int, ld: int | None = None, device="cpu") -> torch.Tensor:
    """bf16 randn·scale [B, V] (a view of a [B, ld] buffer when ld > V); row 1 all equal, row 2 one spike over a flat floor."""
    g = torch.Generator().manual_seed(seed)
    buf = (torch.randn(B, ld or V, generator=g) * scale).to(torch.bfloat16)
    x = buf[:, :V]
    if B > 2:
        x[1] = 1.25
        x[2] = -3.0
        x[2, V // 3] = 7.5
    return x.to(device) if ld is None else buf.to(device)[:, :V]


# ------------------------------------------------------------------------------------------------------------------- GPU
def _dev():
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def native():
    from prime_b200.ops import _lib

    return _lib.load()  # a GPU box without the native library is a hard failure, never a silent fallback


def _draw(logits, knobs, seeds, pos0):
    """Tokens [B, POSITIONS]: one launch per position, every row at position pos0[b] + q."""
    out = []
    for q in range(POSITIONS):
        out.append(ops.sample_tokens(logits, **knobs, seeds=seeds, positions=pos0 + q).clone())
    return torch.stack(out, dim=1)


@pytest.mark.gpu
@pytest.mark.parametrize("scale", [1.0, 8.0, 30.0])
@pytest.mark.parametrize("V,ld", [(2048, None), (32000, None), (32001, 32008), (128256, None)], ids=["2048", "32000", "32001-padded", "128256"])
def test_sample_tokens_matches_fp64_oracle(native, V, ld, scale):
    dev = _dev()
    B = 64
    logits = logit_rows(B, V, scale, seed=V + int(scale), ld=ld, device=dev)
    seeds_l = [1000 * V + 7 * b for b in range(B)]
    pos0_l = [b * 37 for b in range(B)]
    seeds = torch.tensor(seeds_l, dtype=torch.int64, device=dev)
    pos0 = torch.tensor(pos0_l, dtype=torch.int32, device=dev)
    u = uniforms(seeds_l, [[p + q for q in range(POSITIONS)] for p in pos0_l])
    draws = ambiguous = 0
    for T, k, p, m in GRID:
        knobs = dict(temperature=T, top_k=k, top_p=p, min_p=m)
        ref, amb = oracle(logits, T, k, p, m, u)
        for nb in (1, 5, B):
            got = _draw(logits[:nb], knobs, seeds[:nb], pos0[:nb])
            ambiguous += compare_tokens(got, ref[:nb], amb[:nb], f"V={V} scale={scale} B={nb} {knobs}")
            draws += got.numel()
    print(f"[sample oracle] V={V} ld={ld} scale={scale}: {ambiguous} of {draws} draws ambiguous")
    assert ambiguous < 0.01 * draws


@pytest.mark.gpu
def test_sample_tokens_is_deterministic_and_capturable(native):
    dev = _dev()
    B, V = 64, 128256
    logits = logit_rows(B, V, 1.0, seed=5, device=dev)
    seeds = torch.arange(B, dtype=torch.int64, device=dev) * 3 + 11
    pos = torch.full((B,), 77, dtype=torch.int32, device=dev)
    for knobs in (dict(temperature=0.8, top_p=0.9), dict(temperature=1.0, top_k=40, top_p=0.95, min_p=0.01), dict(temperature=0.0)):
        a = ops.sample_tokens(logits, **knobs, seeds=seeds, positions=pos)
        b = ops.sample_tokens(logits, **knobs, seeds=seeds, positions=pos)
        assert torch.equal(a, b), knobs
        out = torch.empty(B, dtype=torch.int64, device=dev)
        ops.sample_tokens(logits, **knobs, seeds=seeds, positions=pos, out=out)  # warm-up outside the capture
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            ops.sample_tokens(logits, **knobs, seeds=seeds, positions=pos, out=out)
        out.fill_(-1)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, a), knobs


@pytest.mark.gpu
def test_sample_tokens_distribution_chi_square(native):
    """A fixed V = 16 distribution drawn at 2^16 positions of one seeded stream: Pearson's chi-square against the exact
    probabilities stays under the 0.999 quantile of chi-square with 15 degrees of freedom (37.70). The stream is seeded, so the
    statistic is the same on every run."""
    dev = _dev()
    V, n = 16, 1 << 16
    logits = (torch.linspace(-2.0, 1.5, V) * torch.tensor([1.0, -1.0] * 8)).to(torch.bfloat16).view(1, V)
    p = torch.softmax(logits.double(), -1)[0]
    counts = torch.zeros(V, dtype=torch.float64)
    row = logits.to(dev).expand(1024, V).contiguous()
    seeds = torch.full((1024,), 20240917, dtype=torch.int64, device=dev)
    for c in range(n // 1024):
        pos = torch.arange(c * 1024, (c + 1) * 1024, dtype=torch.int32, device=dev)
        tok = ops.sample_tokens(row, temperature=1.0, seeds=seeds, positions=pos)
        counts += torch.bincount(tok.cpu(), minlength=V).double()
    chi2 = float(((counts - n * p) ** 2 / (n * p)).sum())
    print(f"[sample chi-square] V=16, 2^16 draws: chi2 = {chi2:.2f} (15 dof)")
    assert chi2 < 37.70


def _kv_model(D, Hkv, window, seed=0):
    from prime_b200.models.llama import ModelArgs, Transformer

    args = ModelArgs(dim=512, n_layers=2, n_heads=512 // D, n_kv_heads=Hkv, vocab_size=2048, max_seq_len=1024, sliding_window=window)
    with torch.device(_dev()):
        m = Transformer(args)
    m.to(torch.bfloat16)
    m.init_weights(seed)
    return m.eval()


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["d64", "d128-window-docs", "d32-fallback"])
def test_device_greedy_equals_host_greedy_on_cuda(native, variant):
    if variant == "d32-fallback":
        model = build_model("debugmodel", device="cuda", dtype=torch.bfloat16).eval()
    else:
        model = _kv_model(64, 2, None) if variant == "d64" else _kv_model(128, 2, 48)
    if variant == "d128-window-docs":
        model.doc_eos_id = 7
    prompts = [list(range(3, 40)), [11, 12], list(range(5, 140))]
    host = ev.generate_batch(model, prompts, max_new=40)
    assert ev.generate_batch(model, prompts, max_new=40, sampler="device") == host
    assert ev.generate_batch(model, prompts, max_new=40, sampler="device", graphs=False) == host
    # an EOS stop: the first row's fifth new token ends it, the other rows run on
    eos = host[0][len(prompts[0]) + 4]
    host_eos = ev.generate_batch(model, prompts, max_new=40, eos_id=eos)
    assert ev.generate_batch(model, prompts, max_new=40, eos_id=eos, sampler="device") == host_eos
    assert len(host_eos[0]) <= len(prompts[0]) + 5


@pytest.mark.gpu
def test_device_sampling_graphs_equal_eager_and_reproduce(native):
    model = _kv_model(64, 2, None)
    prompts = [list(range(3, 40)), [11, 12], list(range(5, 300))]
    kw = dict(max_new=48, temperature=0.8, top_p=0.9, top_k=100, seed=5, sampler="device")
    a = ev.generate_batch(model, prompts, **kw)
    assert a == ev.generate_batch(model, prompts, **kw, graphs=False)
    assert a == ev.generate_batch(model, prompts, **kw)
    assert a != ev.generate_batch(model, prompts, **{**kw, "seed": 6})
    # row b of a batch is the single-prompt run with seed + b
    assert a[1] == ev.generate(model, prompts[1], **{**kw, "seed": 6})


@pytest.mark.gpu
def test_device_sampled_generation_reads_the_host_rarely(native):
    from torch.profiler import ProfilerActivity, profile

    model = _kv_model(64, 2, None)
    prompts = [list(range(3, 40)), [11, 12]]
    kw = dict(max_new=64, temperature=0.8, top_p=0.9, seed=1, sampler="device")
    ev.generate_batch(model, prompts, **kw)  # warm-up: library load, graph pools
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = ev.generate_batch(model, prompts, **kw)
        torch.cuda.synchronize()
    assert all(len(r) == len(p) + 64 for r, p in zip(out, prompts))
    d2h = sum(e.count for e in prof.key_averages() if "dtoh" in e.key.lower().replace(" ", "").replace("devicetohost", "dtoh"))
    print(f"[device sampling] 64 tokens: {d2h} device-to-host copies")
    assert d2h <= math.ceil(63 / inference.CHECK_EVERY) + 2
