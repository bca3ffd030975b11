"""Numerics of every native sm_90a kernel against a plain PyTorch fp32 reference of the same op."""

import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def _dev():
    return torch.device("cuda", 0)


def _rel_err(a: torch.Tensor, b: torch.Tensor) -> float:
    return float((a.float() - b.float()).norm() / (b.float().norm() + 1e-12))


@pytest.fixture(scope="module", autouse=True)
def _lib_loaded():
    from prime_b200.ops import _lib

    _lib.load()  # a GPU box without the native library is a hard failure, never a silent fallback
    yield


# ------------------------------------------------------------------ GEMM
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, True), (True, False)])
@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (256, 512, 256), (384, 1000 // 8 * 8, 136), (2048, 2048, 2048), (136, 264, 72)])
def test_gemm_layouts(M, N, K, a_mn, b_mn):
    from prime_b200 import ops

    torch.manual_seed(M + N + K)
    A = torch.randn(M, K, device=_dev(), dtype=torch.bfloat16)
    B = torch.randn(N, K, device=_dev(), dtype=torch.bfloat16)
    ref = A.float() @ B.float().t()
    a = A.t().contiguous() if a_mn else A
    b = B.t().contiguous() if b_mn else B
    out = ops.gemm(a, b, a_mn_major=a_mn, b_mn_major=b_mn)
    torch.cuda.synchronize()
    assert out.shape == (M, N) and out.dtype == torch.bfloat16
    assert _rel_err(out, ref) < 1e-2, f"rel err {_rel_err(out, ref)}"


def test_gemm_fp32_accumulate():
    from prime_b200 import ops

    torch.manual_seed(0)
    M, N, K = 512, 768, 1024
    A = torch.randn(K, M, device=_dev(), dtype=torch.bfloat16)  # stored [K, M]  (dW = dyᵀ x pattern)
    B = torch.randn(K, N, device=_dev(), dtype=torch.bfloat16)
    C = torch.randn(M, N, device=_dev(), dtype=torch.float32)
    ref = C + A.float().t() @ B.float()
    ops.gemm(A, B, a_mn_major=True, b_mn_major=True, out=C, accumulate=True)
    torch.cuda.synchronize()
    assert _rel_err(C, ref) < 2e-3


def test_gemm_many_tiles_persistent():
    """More tiles than SMs, K long enough to wrap the smem ring many times, both accumulator stages in use."""
    from prime_b200 import ops

    torch.manual_seed(1)
    M, N, K = 4096, 4096, 1024
    A = torch.randn(M, K, device=_dev(), dtype=torch.bfloat16) * 0.1
    B = torch.randn(N, K, device=_dev(), dtype=torch.bfloat16) * 0.1
    out = ops.gemm(A, B)
    ref = A.float() @ B.float().t()
    assert _rel_err(out, ref) < 1e-2


def test_linear_autograd_matches_torch():
    from prime_b200 import ops

    torch.manual_seed(2)
    x = torch.randn(4, 96, 512, device=_dev(), dtype=torch.bfloat16, requires_grad=True)
    w = (torch.randn(1536, 512, device=_dev(), dtype=torch.bfloat16) * 0.05).requires_grad_(True)
    y = ops.linear(x, w)
    dy = torch.randn_like(y)
    y.backward(dy)
    xr = x.detach().float().requires_grad_(True)
    wr = w.detach().float().requires_grad_(True)
    yr = torch.nn.functional.linear(xr, wr)
    yr.backward(dy.float())
    assert _rel_err(y, yr) < 1e-2
    assert _rel_err(x.grad, xr.grad) < 1e-2
    assert _rel_err(w.grad, wr.grad) < 1e-2


def test_linear_main_grad_fusion():
    from prime_b200 import ops

    torch.manual_seed(3)
    x = torch.randn(256, 256, device=_dev(), dtype=torch.bfloat16, requires_grad=True)
    w = (torch.randn(512, 256, device=_dev(), dtype=torch.bfloat16) * 0.05).requires_grad_(True)
    w.main_grad = torch.zeros(512, 256, device=_dev(), dtype=torch.float32)
    for _ in range(2):
        ops.linear(x, w).sum().backward()
    assert w.grad is None
    ref = 2 * torch.ones(256, 512, device=_dev()).t() @ x.detach().float()
    assert _rel_err(w.main_grad, ref) < 5e-3


# ------------------------------------------------------------------ norm / rope / swiglu / loss
@pytest.mark.parametrize("D", [1024, 2048, 4096, 5120])
def test_rmsnorm_fwd_bwd(D):
    from prime_b200 import ops
    from prime_b200.ops import reference as R

    torch.manual_seed(D)
    x = torch.randn(300, D, device=_dev(), dtype=torch.bfloat16, requires_grad=True)
    w = (1 + 0.1 * torch.randn(D, device=_dev())).to(torch.bfloat16).requires_grad_(True)
    y = ops.rmsnorm(x, w, 1e-5)
    dy = torch.randn_like(y)
    y.backward(dy)
    xr, wr = x.detach().float().requires_grad_(True), w.detach().float().requires_grad_(True)
    yr = R.rmsnorm(xr, wr, 1e-5)
    yr.backward(dy.float())
    assert _rel_err(y, yr) < 1e-2
    assert _rel_err(x.grad, xr.grad) < 1e-2
    assert _rel_err(w.grad, wr.grad) < 2e-2


def test_add_rmsnorm_fwd_bwd():
    from prime_b200 import ops
    from prime_b200.ops import reference as R

    torch.manual_seed(7)
    D = 2048
    x = torch.randn(4, 64, D, device=_dev(), dtype=torch.bfloat16, requires_grad=True)
    r = torch.randn(4, 64, D, device=_dev(), dtype=torch.bfloat16, requires_grad=True)
    w = torch.ones(D, device=_dev(), dtype=torch.bfloat16, requires_grad=True)
    y, h = ops.add_rmsnorm(x, r, w)
    dy, dh = torch.randn_like(y), torch.randn_like(h)
    torch.autograd.backward([y, h], [dy, dh])
    xr, rr, wr = (t.detach().float().requires_grad_(True) for t in (x, r, w))
    yr, hr = R.add_rmsnorm(xr, rr, wr)
    torch.autograd.backward([yr, hr], [dy.float(), dh.float()])
    assert _rel_err(h, hr) < 1e-2 and _rel_err(y, yr) < 1e-2
    assert _rel_err(x.grad, xr.grad) < 1e-2 and _rel_err(r.grad, rr.grad) < 1e-2
    assert _rel_err(w.grad, wr.grad) < 2e-2


@pytest.mark.parametrize("H,Hkv,D", [(16, 16, 128), (8, 2, 64)])
def test_rope_qkv(H, Hkv, D):
    from prime_b200 import ops
    from prime_b200.ops import reference as R

    torch.manual_seed(11)
    B, S = 2, 96
    W = (H + 2 * Hkv) * D
    qkv = torch.randn(B, S, W, device=_dev(), dtype=torch.bfloat16)
    cos, sin = R.rope_tables(S, D, device=_dev())
    base = qkv.clone().requires_grad_(True)
    out = ops.rope_qkv(base * 1.0, cos, sin, H, Hkv)  # *1.0: non-leaf so the in-place rotate is legal
    ref4 = qkv.float().view(B, S, H + 2 * Hkv, D)
    ref = torch.cat((R.rope(ref4[:, :, : H + Hkv], cos, sin), ref4[:, :, H + Hkv :]), dim=2).view(B, S, W)
    assert _rel_err(out, ref) < 1e-2
    g = torch.randn_like(out)
    out.backward(g.clone())
    g4 = g.float().view(B, S, H + 2 * Hkv, D)
    gref = torch.cat((R.rope(g4[:, :, : H + Hkv], cos, -sin), g4[:, :, H + Hkv :]), dim=2).view(B, S, W)
    assert _rel_err(base.grad, gref) < 1e-2


def test_swiglu_fwd_bwd():
    from prime_b200 import ops
    from prime_b200.ops import reference as R

    torch.manual_seed(13)
    gu = torch.randn(200, 2 * 5632, device=_dev(), dtype=torch.bfloat16, requires_grad=True)
    out = ops.swiglu(gu)
    d = torch.randn_like(out)
    out.backward(d)
    gr = gu.detach().float().requires_grad_(True)
    outr = R.swiglu(gr)
    outr.backward(d.float())
    assert _rel_err(out, outr) < 1e-2 and _rel_err(gu.grad, gr.grad) < 1e-2


@pytest.mark.parametrize("V", [32000, 2048])
def test_cross_entropy_fused(V):
    from prime_b200 import ops

    torch.manual_seed(17)
    R_ = 257
    logits = (torch.randn(R_, V, device=_dev()) * 2).to(torch.bfloat16)
    tgt = torch.randint(0, V, (R_,), device=_dev())
    tgt[5] = -100
    zr = logits.float().requires_grad_(True)
    lr = torch.nn.functional.cross_entropy(zr, tgt, ignore_index=-100)
    lr.backward()
    z = (logits.clone() * 1.0).requires_grad_(True)
    zz = z * 1.0
    loss = ops.cross_entropy(zz, tgt, grad_scale=0.5, unit_upstream=True)
    loss.backward()
    assert abs(float(loss) - float(lr)) < 2e-3 * max(1.0, abs(float(lr)))
    assert _rel_err(z.grad, 0.5 * zr.grad) < 2e-2


# ------------------------------------------------------------------ optimizer / outer kernels (single GPU, 1 "peer")
def test_fused_engine_matches_collective_single_gpu():
    """fused (P2P kernels with F=1) vs collective (torch ops) engines must produce the same parameters."""
    import copy

    from prime_b200.models.llama import build_model
    from prime_b200.parallel.fsdp import AdamHyper, ShardedEngine
    from prime_b200.parallel.mesh import WorldInfo, build_mesh
    from prime_b200.parallel.symm import SymmetricHeap

    dev = _dev()
    torch.manual_seed(0)
    m1 = build_model("debugmodel", device=dev, dtype=torch.bfloat16, seed=3)
    m2 = copy.deepcopy(m1)
    mesh = build_mesh(WorldInfo(), device=dev)
    heap = SymmetricHeap(256 << 20, 0, 1, lambda h: [h], dev)
    hyper = AdamHyper(lr=1e-3, max_norm=1.0)
    e1 = ShardedEngine(m1, mesh, hyper, backend="fused", heap=heap)
    e2 = ShardedEngine(m2, mesh, hyper, backend="collective")
    V = m1.args.vocab_size
    for _ in range(3):
        tok = torch.randint(0, V, (2, 64), device=dev)
        for m, e in ((m1, e1), (m2, e2)):
            e.zero_grad()
            e.set_micro_step(True)
            m.loss(tok, tok).backward()
            e.finish_backward()
            e.step()
    torch.cuda.synchronize()
    heap.check_errors()
    assert _rel_err(e1.master, e2.master) < 1e-4
    assert abs(float(e1.last_grad_norm) - float(e2.last_grad_norm)) < 1e-2 * float(e2.last_grad_norm)
    assert torch.equal(e1.param_flat.float() == 0, e2.param_flat.float() == 0)
    assert _rel_err(e1.param_flat, e2.param_flat) < 1e-3
    heap.close()


def test_outer_step_fused_matches_reference():
    from prime_b200.models.llama import build_model
    from prime_b200.ops import reference as R
    from prime_b200.parallel.diloco import DilocoOuter, OuterHyper
    from prime_b200.parallel.fsdp import AdamHyper, ShardedEngine
    from prime_b200.parallel.mesh import WorldInfo, build_mesh
    from prime_b200.parallel.symm import SymmetricHeap

    dev = _dev()
    m = build_model("debugmodel", device=dev, dtype=torch.bfloat16, seed=4)
    mesh = build_mesh(WorldInfo(), device=dev)
    heap = SymmetricHeap(256 << 20, 0, 1, lambda h: [h], dev)
    eng = ShardedEngine(m, mesh, AdamHyper(), backend="fused", heap=heap)
    outer = DilocoOuter(eng, OuterHyper(lr=0.7, momentum=0.9, nesterov=True, compression="int8"))
    theta0 = outer.theta0.clone()
    eng.master.add_(torch.randn_like(eng.master) * 1e-3)  # pretend H inner steps moved the weights
    pseudo = theta0 - eng.master
    q, s = R.quantize_int8_blockwise(pseudo, 1024)
    avg = R.dequantize_int8_blockwise(q, s, 1024)
    mom = torch.zeros_like(theta0)
    R.nesterov_outer_step(theta0, avg, mom, lr=0.7, momentum=0.9, nesterov=True)
    outer.step()
    torch.cuda.synchronize()
    heap.check_errors()
    # kernel and oracle evaluate the same formulas in the same precision; what is left is FMA contraction (one ulp of the product
    # in front of rint), which can still round a tie the other way: allow at most 3 elements per million to be off, and those by
    # no more than one quantisation step through the update (lr · (1 + momentum) · absmax / 127)
    step = 0.7 * 1.9 * float(pseudo.abs().max()) / 127.0

    def close(got, want):
        d = (got - want).abs()
        bad = d > (1e-7 + 1e-5 * want.abs())
        assert int(bad.sum()) <= max(1, 3 * want.numel() // 1_000_000), f"{int(bad.sum())} elements differ"
        assert float(d.max()) <= 1.05 * step, f"max |Δ| {float(d.max()):.3e} exceeds one quantisation step ({step:.3e})"

    close(outer.theta0, theta0)
    close(eng.master, theta0)
    close(outer.momentum, mom)
    # bf16 parameters were refreshed from the new θ
    b = eng.buckets[1]
    got = eng.param_flat[b.start : b.start + b.shard_size].float()
    want = outer.theta0[b.shard_start : b.shard_start + b.shard_size].to(torch.bfloat16).float()  # the kernel's own new θ, rounded
    assert torch.equal(got, want)
    heap.close()


def test_trainer_loss_decreases_on_gpu():
    from prime_b200.config import Config
    from prime_b200.trainer import Trainer

    cfg = Config.model_validate(
        {"name_model": "debugmodel", "data": {"seq_length": 128}, "optim": {"batch_size": 8, "warmup_steps": 2, "optim": {"lr": 3e-3}},
         "train": {"micro_bs": 4}, "diloco": {"inner_steps": 5}}
    )  # fmt: skip
    t = Trainer(cfg)
    losses = [float(t.inner_step().loss.item()) for _ in range(15)]
    assert all(math.isfinite(x) for x in losses)
    assert losses[-1] < losses[0] - 0.5, losses
    assert t.outer.outer_step_count == 3
    t.close()


# ------------------------------------------------------------------ native flash attention
@pytest.mark.parametrize("B,S,H,Hkv,D", [(2, 256, 4, 4, 128), (1, 512, 4, 2, 128), (2, 384, 8, 8, 64), (1, 128, 2, 1, 64), (1, 1024, 2, 2, 128),
                                         (3, 768, 2, 1, 128)])  # fmt: skip
@pytest.mark.parametrize("causal", [True, False])
def test_flash_attention_fwd_bwd(B, S, H, Hkv, D, causal):
    from prime_b200.ops import attention_native as A
    from prime_b200.ops import reference as R

    torch.manual_seed(S + H + D)
    W = (H + 2 * Hkv) * D
    qkv = (torch.randn(B, S, W, device=_dev()) * 0.7).to(torch.bfloat16).requires_grad_(True)
    assert A.supported(qkv, H, Hkv)
    out = A.flash_attention_qkv(qkv, H, Hkv, causal)
    dout = torch.randn_like(out)
    out.backward(dout)
    torch.cuda.synchronize()
    ref_in = qkv.detach().float().requires_grad_(True)
    x = ref_in.view(B, S, H + 2 * Hkv, D)
    ref = R.attention(x[:, :, :H], x[:, :, H : H + Hkv], x[:, :, H + Hkv :], causal).reshape(B, S, H * D)
    ref.backward(dout.float())
    assert _rel_err(out, ref) < 2e-2, f"fwd rel err {_rel_err(out, ref)}"
    g, gr = qkv.grad.view(B, S, H + 2 * Hkv, D), ref_in.grad.view(B, S, H + 2 * Hkv, D)
    assert _rel_err(g[:, :, :H], gr[:, :, :H]) < 3e-2, f"dQ rel err {_rel_err(g[:, :, :H], gr[:, :, :H])}"
    assert _rel_err(g[:, :, H : H + Hkv], gr[:, :, H : H + Hkv]) < 3e-2, "dK"
    assert _rel_err(g[:, :, H + Hkv :], gr[:, :, H + Hkv :]) < 3e-2, "dV"


@pytest.mark.parametrize("H,Hkv,D", [(4, 4, 128), (8, 2, 64)])
def test_rope_attention_fused_node_matches_reference(H, Hkv, D):
    """RoPE ⊕ flash attention as one autograd node (in-place rotation, in-place inverse rotation of its own dQKV)."""
    from prime_b200 import ops
    from prime_b200.ops import reference as R

    torch.manual_seed(5)
    B, S = 2, 256
    W = (H + 2 * Hkv) * D
    base = (torch.randn(B, S, W, device=_dev()) * 0.7).to(torch.bfloat16).requires_grad_(True)
    cos, sin = R.rope_tables(S, D, device=_dev())
    out = ops.rope_attention_qkv(base * 1.0, cos, sin, H, Hkv, causal=True, impl="native")
    dout = torch.randn_like(out)
    out.backward(dout)
    torch.cuda.synchronize()
    ref_in = base.detach().float().requires_grad_(True)
    x = ref_in.view(B, S, H + 2 * Hkv, D)
    rot = R.rope(x[:, :, : H + Hkv], cos, sin)
    ref = R.attention(rot[:, :, :H], rot[:, :, H:], x[:, :, H + Hkv :], True).reshape(B, S, H * D)
    ref.backward(dout.float())
    assert _rel_err(out, ref) < 2e-2
    assert _rel_err(base.grad, ref_in.grad) < 3e-2


def _out_buffer(M, N, dtype, padded):
    """(output view [M, N], full buffer): with ``padded`` the view is the first N columns of an [M, N + 8] buffer (row pitch
    N + 8), so a kernel that ignores the output's row stride, or stores past column N, fails the caller's checks."""
    full = torch.full((M, N + 8 if padded else N), 7.0, device=_dev(), dtype=dtype)
    return full[:, :N], full


@pytest.mark.parametrize("out_layout", ["dense_out", "padded_out"])
@pytest.mark.parametrize("M,N,K,a_mn,b_mn", [(256, 256, 64, False, False), (384, 1000, 136, False, True), (640, 264, 4096, True, True), (4096, 4096, 1024, True, False)])
def test_gemm_transposed_layouts_at_larger_shapes(M, N, K, a_mn, b_mn, out_layout):
    """Every K-major / MN-major operand combination against the fp32 reference, with ragged N and K and up to 4096² outputs, written
    into a dense output or into the first N columns of a wider buffer (whose padding must stay untouched)."""
    from prime_b200 import ops

    torch.manual_seed(M + N)
    A = torch.randn(M, K, device=_dev(), dtype=torch.bfloat16) * 0.1
    B = torch.randn(N, K, device=_dev(), dtype=torch.bfloat16) * 0.1
    a = A.t().contiguous() if a_mn else A
    b = B.t().contiguous() if b_mn else B
    out, full = _out_buffer(M, N, torch.bfloat16, out_layout == "padded_out")
    ops.gemm(a, b, a_mn_major=a_mn, b_mn_major=b_mn, out=out)
    torch.cuda.synchronize()
    assert _rel_err(out, A.float() @ B.float().t()) < 1e-2
    assert bool((full[:, N:] == 7.0).all()), "store past column N"


@pytest.mark.parametrize("out_layout", ["dense_out", "padded_out"])
@pytest.mark.parametrize("split", [-1, 2, 3, 8])
def test_gemm_split_k_reduce_add(split, out_layout):
    """Weight-gradient pattern: fp32 C += AᵀB with K sliced across work items, every slice adding its partial tile into C.
    K = 17·64 + 8 is not divisible by any split (ragged last slice, and with split 8 an empty one). C is dense or the first N
    columns of a wider buffer, whose padding must stay untouched."""
    from prime_b200 import ops

    old_s = ops.set_gemm_split_k(split)
    try:
        torch.manual_seed(3)
        M, N, K = 512, 768, 17 * 64 + 8
        A = torch.randn(K, M, device=_dev(), dtype=torch.bfloat16)
        B = torch.randn(K, N, device=_dev(), dtype=torch.bfloat16)
        C, full = _out_buffer(M, N, torch.float32, out_layout == "padded_out")
        C.copy_(torch.randn(M, N, device=_dev(), dtype=torch.float32))
        ref = C + A.float().t() @ B.float()
        ops.gemm(A, B, a_mn_major=True, b_mn_major=True, out=C, accumulate=True)
        torch.cuda.synchronize()
        assert _rel_err(C, ref) < 2e-3
        assert bool((full[:, N:] == 7.0).all()), "store past column N"
    finally:
        ops.set_gemm_split_k(old_s)


@pytest.mark.parametrize("H,Hkv,D", [(4, 4, 128), (8, 2, 64)])
def test_qkv_gemm_rope_epilogue_and_attention_unrotate(H, Hkv, D):
    """RoPE in the QKV GEMM epilogue (forward) + inverse RoPE in the dQ/dK epilogues of the attention backward: compare
    y = attention(rope(x Wᵀ)) and the gradients w.r.t. x and W with the fp32 reference (flash attention path end to end)."""
    from prime_b200 import ops
    from prime_b200.ops import reference as R

    torch.manual_seed(9)
    B, S, dim = 2, 256, 512
    W = (H + 2 * Hkv) * D
    x = (torch.randn(B, S, dim, device=_dev()) * 0.5).to(torch.bfloat16).requires_grad_(True)
    w = (torch.randn(W, dim, device=_dev()) * 0.05).to(torch.bfloat16).requires_grad_(True)
    cos, sin = R.rope_tables(S, D, device=_dev())
    assert ops.rope_fusable(x, H, Hkv, D)
    qkv = ops.linear_qkv_rope(x, w, cos, sin, H, Hkv)
    # the epilogue-rotated projection itself
    ref_qkv4 = (x.detach().float() @ w.detach().float().t()).view(B, S, H + 2 * Hkv, D)
    ref_rot = torch.cat((R.rope(ref_qkv4[:, :, : H + Hkv], cos, sin), ref_qkv4[:, :, H + Hkv :]), dim=2).view(B, S, W)
    assert _rel_err(qkv.detach(), ref_rot) < 1e-2
    out = ops.rope_attention_qkv(qkv, cos, sin, H, Hkv, causal=True, impl="native", pre_rotated=True)
    dout = torch.randn_like(out)
    out.backward(dout)
    torch.cuda.synchronize()
    xr = x.detach().float().requires_grad_(True)
    wr = w.detach().float().requires_grad_(True)
    q4 = (xr @ wr.t()).view(B, S, H + 2 * Hkv, D)
    rot = R.rope(q4[:, :, : H + Hkv], cos, sin)
    ref = R.attention(rot[:, :, :H], rot[:, :, H:], q4[:, :, H + Hkv :], True).reshape(B, S, H * D)
    ref.backward(dout.float())
    assert _rel_err(out, ref) < 2e-2
    assert _rel_err(x.grad, xr.grad) < 4e-2, _rel_err(x.grad, xr.grad)
    assert _rel_err(w.grad, wr.grad) < 4e-2, _rel_err(w.grad, wr.grad)


@pytest.mark.parametrize("M,FF,K", [(512, 1024, 256), (640, 5632, 2048), (384, 192, 136)])
def test_gemm_swiglu_epilogue(M, FF, K):
    """gate/up projection with SwiGLU in the epilogue vs the unfused linear → swiglu path, forward and gradients."""
    from prime_b200 import ops

    torch.manual_seed(M + FF)
    x = (torch.randn(M, K, device=_dev()) * 0.5).to(torch.bfloat16).requires_grad_(True)
    w = (torch.randn(2 * FF, K, device=_dev()) * 0.05).to(torch.bfloat16).requires_grad_(True)
    h = ops.linear_swiglu(x, w)
    dh = torch.randn_like(h)
    h.backward(dh)
    torch.cuda.synchronize()
    xr = x.detach().clone().requires_grad_(True)
    wr = w.detach().clone().requires_grad_(True)
    hr = ops.swiglu(ops.linear(xr, wr))
    hr.backward(dh)
    assert _rel_err(h, hr) < 1e-3, _rel_err(h, hr)  # same bf16-rounded gate/up → near bit-identical
    assert _rel_err(x.grad, xr.grad) < 1e-3 and _rel_err(w.grad, wr.grad) < 1e-3
    ref = torch.nn.functional.silu(x.detach().float() @ w.detach().float()[:FF].t()) * (x.detach().float() @ w.detach().float()[FF:].t())
    assert _rel_err(h, ref) < 2e-2


# ------------------------------------------------------------------ MXFP8 (block-scaled fp8)
@pytest.mark.parametrize("R,C,transpose", [(256, 384, False), (200, 1024, False), (4096, 2048, False), (256, 384, True), (1024, 200, True), (2048, 5632, True)])
def test_quantize_mxfp8_matches_reference(R, C, transpose):
    from prime_b200 import ops
    from prime_b200.ops import reference as Rf

    torch.manual_seed(R + C)
    x = (torch.randn(R, C, device=_dev()) * torch.rand(R, 1, device=_dev()) * 8).to(torch.bfloat16)
    q, sf = ops.quantize_mxfp8(x, transpose)
    q_ref, sf_ref = Rf.quantize_mxfp8(x, transpose)
    torch.cuda.synchronize()
    rows, k = q.shape
    idx = Rf._mxfp8_sf_index(rows, k, _dev()).reshape(-1)
    assert torch.equal(sf[idx], sf_ref[idx]), "UE8M0 scales differ"
    assert torch.equal(q, q_ref), f"{int((q != q_ref).sum())} e4m3 values differ"
    deq = Rf.dequantize_mxfp8(q, sf)
    tgt = (x.t() if transpose else x).float()
    assert _rel_err(deq, tgt) < 0.04


@pytest.mark.parametrize("out_layout", ["dense_out", "padded_out"])
@pytest.mark.parametrize("M,N,K", [(128, 192, 128), (256, 384, 512), (300, 520, 256), (1024, 2112, 1024), (4096, 3072, 2048), (136, 8, 128)])
def test_gemm_mxfp8_matches_dequantized_reference(M, N, K, out_layout):
    """``dense_out``: the op allocates C. ``padded_out``: C is the first N columns of a wider buffer, whose padding must stay
    untouched."""
    from prime_b200 import ops
    from prime_b200.ops import reference as Rf

    torch.manual_seed(M * 3 + N + K)
    # per-row magnitudes spread over a few octaves so wrong scale bytes (wrong row / wrong K block) cannot cancel out
    A = (torch.randn(M, K, device=_dev()) * torch.exp2(torch.randint(-3, 4, (M, 1), device=_dev()).float())).to(torch.bfloat16)
    B = (torch.randn(N, K, device=_dev()) * torch.exp2(torch.randint(-3, 4, (N, 1), device=_dev()).float())).to(torch.bfloat16)
    A[:, K // 2 :] *= 4  # and across K blocks
    aq, asf = ops.quantize_mxfp8(A)
    bq, bsf = ops.quantize_mxfp8(B)
    if out_layout == "padded_out":
        out, full = _out_buffer(M, N, torch.bfloat16, True)
        ops.gemm_mxfp8(aq, asf, bq, bsf, out=out)
    else:
        out = full = ops.gemm_mxfp8(aq, asf, bq, bsf)
    torch.cuda.synchronize()
    ref = Rf.dequantize_mxfp8(aq, asf) @ Rf.dequantize_mxfp8(bq, bsf).t()
    assert _rel_err(out, ref) < 6e-3, f"rel err {_rel_err(out, ref)}"
    assert _rel_err(out, A.float() @ B.float().t()) < 0.06  # and the quantisation itself is sane
    assert bool((full[:, N:] == 7.0).all()), "store past column N"


def test_linear_mxfp8_autograd():
    from prime_b200 import ops

    torch.manual_seed(5)
    x = torch.randn(4, 256, 1024, device=_dev(), dtype=torch.bfloat16, requires_grad=True)
    w = (torch.randn(1536, 1024, device=_dev()) * 0.03).to(torch.bfloat16).requires_grad_(True)
    y = ops.linear_mxfp8(x, w)
    dy = torch.randn_like(y)
    y.backward(dy)
    torch.cuda.synchronize()
    xr, wr = x.detach().float().requires_grad_(True), w.detach().float().requires_grad_(True)
    yr = xr @ wr.t()
    yr.backward(dy.float())
    assert _rel_err(y, yr) < 0.05
    assert _rel_err(x.grad, xr.grad) < 0.05
    assert _rel_err(w.grad, wr.grad) < 1e-2  # weight gradient stays bf16 x bf16 → fp32


def test_model_fp8_mode_tracks_bf16_loss():
    from prime_b200.models.llama import build_model

    torch.manual_seed(0)
    model = build_model("150M", "llama2", device=_dev(), dtype=torch.bfloat16, seed=0, n_layers=2)
    tokens = torch.randint(0, model.args.vocab_size, (2, 256), device=_dev())
    targets = torch.randint(0, model.args.vocab_size, (2, 256), device=_dev())
    losses = {}
    grads = {}
    for fp8 in (False, True):
        model.set_fp8(fp8)
        model.zero_grad(set_to_none=True)
        loss = model.loss(tokens, targets)
        loss.backward()
        losses[fp8] = float(loss)
        grads[fp8] = model.layers[0].feed_forward.w2.grad.float().clone()
    assert abs(losses[True] - losses[False]) < 0.02 * abs(losses[False]), losses
    assert _rel_err(grads[True], grads[False]) < 0.15


# ------------------------------------------------------------------ round 2: embedding, fp32 outer step, per-element bounds
def _max_rel(a: torch.Tensor, b: torch.Tensor) -> float:
    """max |a-b| / (|b| + 5 % of max|b|): a wrong row / tile shows up here even when the Frobenius ratio stays small."""
    a, b = a.float(), b.float()
    return float(((a - b).abs() / (b.abs() + 0.05 * b.abs().max())).max())


@pytest.mark.parametrize("T,V,D", [(4096, 32000, 2048), (20000, 2048, 256), (130, 1000, 1024)])
def test_embedding_fwd_bwd_deterministic(T, V, D):
    from prime_b200 import ops

    dev = _dev()
    torch.manual_seed(T)
    W = torch.randn(V, D, device=dev, dtype=torch.bfloat16)
    tok = torch.randint(0, V, (T,), device=dev)
    tok[: T // 4] = tok[0]  # a heavily repeated token: one long run after the sort
    W.main_grad = torch.zeros(V, D, device=dev, dtype=torch.float32)
    Wp = torch.nn.Parameter(W)
    Wp.main_grad = W.main_grad
    out = ops.embedding(tok.view(1, T), Wp)
    assert torch.equal(out[0], W[tok])
    dout = torch.randn(1, T, D, device=dev, dtype=torch.bfloat16)
    out.backward(dout)
    ref = torch.zeros(V, D, device=dev, dtype=torch.float32).index_add_(0, tok, dout[0].float())
    assert _rel_err(Wp.main_grad, ref) < 1e-5 and _max_rel(Wp.main_grad, ref) < 1e-3
    first = Wp.main_grad.clone()
    Wp.main_grad.zero_()
    ops.embedding(tok.view(1, T), Wp).backward(dout)
    assert torch.equal(first, Wp.main_grad)  # bitwise reproducible (sorted, one owner per row, no atomics)


def test_outer_step_fused_fp32_matches_reference():
    from prime_b200.models.llama import build_model
    from prime_b200.ops import reference as R
    from prime_b200.parallel.diloco import DilocoOuter, OuterHyper
    from prime_b200.parallel.fsdp import AdamHyper, ShardedEngine
    from prime_b200.parallel.mesh import WorldInfo, build_mesh
    from prime_b200.parallel.symm import SymmetricHeap

    dev = _dev()
    m = build_model("debugmodel", device=dev, dtype=torch.bfloat16, seed=4)
    mesh = build_mesh(WorldInfo(), device=dev)
    heap = SymmetricHeap(256 << 20, 0, 1, lambda h: [h], dev)
    eng = ShardedEngine(m, mesh, AdamHyper(), backend="fused", heap=heap, master_in_heap=True)
    outer = DilocoOuter(eng, OuterHyper(lr=0.7, momentum=0.9, nesterov=True, compression="no"))
    theta0 = outer.theta0.clone()
    eng.master.add_(torch.randn_like(eng.master) * 1e-3)
    pseudo = theta0 - eng.master
    mom = torch.zeros_like(theta0)
    R.nesterov_outer_step(theta0, pseudo, mom, lr=0.7, momentum=0.9, nesterov=True)
    outer.step()
    torch.cuda.synchronize()
    heap.check_errors()
    torch.testing.assert_close(outer.theta0, theta0, rtol=1e-5, atol=1e-7)
    torch.testing.assert_close(eng.master, theta0, rtol=1e-5, atol=1e-7)
    b = eng.buckets[1]
    got = eng.param_flat[b.pstart : b.pstart + b.shard_size].float()
    torch.testing.assert_close(got, theta0[b.shard_start : b.shard_start + b.shard_size].to(torch.bfloat16).float())
    assert outer.device_seconds() > 0
    heap.close()


@pytest.mark.parametrize("M,N,K,a_mn,b_mn", [(512, 768, 1024, False, False), (384, 1000, 136, False, True), (640, 264, 2048, True, True)])
def test_gemm_per_element_bound(M, N, K, a_mn, b_mn):
    """Per-element check next to the norm checks above (VERDICT r1: a wrong row or tile passes a Frobenius-ratio test)."""
    from prime_b200 import ops

    torch.manual_seed(M * 3 + N)
    A = torch.randn(M, K, device=_dev(), dtype=torch.bfloat16)
    B = torch.randn(N, K, device=_dev(), dtype=torch.bfloat16)
    ref = A.float() @ B.float().t()
    out = ops.gemm(A.t().contiguous() if a_mn else A, B.t().contiguous() if b_mn else B, a_mn_major=a_mn, b_mn_major=b_mn)
    # bf16 output rounding is 2^-9 relative; the bound is per element, relative to |ref| + 5 % of the largest magnitude
    assert _max_rel(out, ref) < 1.5e-2
    out32 = torch.zeros(M, N, device=_dev(), dtype=torch.float32)
    ops.gemm(A.t().contiguous() if a_mn else A, B.t().contiguous() if b_mn else B, a_mn_major=a_mn, b_mn_major=b_mn, out=out32)
    assert _max_rel(out32, ref) < 1e-4


@pytest.mark.parametrize("causal", [True, False])
def test_flash_attention_per_element_bound(causal):
    from prime_b200 import ops
    from prime_b200.ops import reference as R

    dev = _dev()
    B, S, H, D = 2, 512, 4, 128
    torch.manual_seed(11)
    qkv = (torch.randn(B, S, 3 * H * D, device=dev) * 0.7).to(torch.bfloat16).requires_grad_(True)
    out = ops.attention_qkv(qkv, H, H, causal=causal, impl="native")
    dout = torch.randn_like(out)
    out.backward(dout)
    x = qkv.detach().float().view(B, S, 3 * H, D).requires_grad_(True)
    ref = R.attention(x[:, :, :H], x[:, :, H : 2 * H], x[:, :, 2 * H :], causal).reshape(B, S, H * D)
    ref.backward(dout.float())
    assert _max_rel(out, ref) < 3e-2
    assert _max_rel(qkv.grad, x.grad.view(B, S, -1)) < 4e-2


def test_fresh_grad_mode_matches_memset_mode():
    """zero_grad without the 4·N-byte memset (first wgrad of a step overwrites) must give the same gradients."""
    import copy

    from prime_b200.models.llama import build_model
    from prime_b200.parallel.fsdp import AdamHyper, ShardedEngine
    from prime_b200.parallel.mesh import WorldInfo, build_mesh

    dev = _dev()
    m1 = build_model("debugmodel", device=dev, dtype=torch.bfloat16, seed=9)
    m2 = copy.deepcopy(m1)
    mesh = build_mesh(WorldInfo(), device=dev)
    e1 = ShardedEngine(m1, mesh, AdamHyper(), backend="collective", fresh_grads=True)
    e2 = ShardedEngine(m2, mesh, AdamHyper(), backend="collective", fresh_grads=False)
    V = m1.args.vocab_size
    for step in range(2):
        for m, e in ((m1, e1), (m2, e2)):
            torch.manual_seed(100 + step)
            e.zero_grad()
            for micro in range(2):
                tok = torch.randint(0, V, (2, 64), device=dev)
                e.set_micro_step(micro == 1)
                m.loss(tok, tok, grad_scale=0.5).backward()
            e.finish_backward()
        assert torch.equal(e1.grad_flat, e2.grad_flat)
        e1.step()
        e2.step()


@pytest.mark.parametrize("M,D,FF", [(512, 256, 1024), (1024, 2048, 5632), (384, 136, 192)])
def test_mlp_swiglu_fused_backward(M, D, FF):
    """One autograd node for the SwiGLU MLP: the SwiGLU derivative rides in the down-projection's dgrad epilogue (EPI = 3)."""
    from prime_b200 import ops

    dev = _dev()
    torch.manual_seed(M + FF)
    x = (torch.randn(2, M // 2, D, device=dev) * 0.5).to(torch.bfloat16).requires_grad_(True)
    w13 = (torch.randn(2 * FF, D, device=dev) * D**-0.5).to(torch.bfloat16).requires_grad_(True)
    w2 = (torch.randn(D, FF, device=dev) * FF**-0.5).to(torch.bfloat16).requires_grad_(True)
    y = ops.mlp_swiglu(x, w13, w2)
    dy = torch.randn_like(y)
    y.backward(dy)
    xr, w13r, w2r = (t.detach().float().requires_grad_(True) for t in (x, w13, w2))
    gu = xr @ w13r.t()
    gub = gu + (gu.to(torch.bfloat16).float() - gu).detach()  # the kernel rounds gate/up to bf16 before the activation (straight-through)
    h = torch.nn.functional.silu(gub[..., :FF]) * gub[..., FF:]
    yr = h @ w2r.t()
    yr.backward(dy.float())
    assert _rel_err(y, yr) < 1e-2 and _max_rel(y, yr) < 4e-2
    assert _rel_err(x.grad, xr.grad) < 1.5e-2 and _max_rel(x.grad, xr.grad) < 6e-2
    assert _rel_err(w13.grad, w13r.grad) < 1.5e-2 and _rel_err(w2.grad, w2r.grad) < 1.5e-2
    # and it agrees with the composition of the separate ops (same kernels except the fused epilogue)
    x2, w13b, w2b = (t.detach().clone().requires_grad_(True) for t in (x, w13, w2))
    y2 = ops.linear(ops.linear_swiglu(x2, w13b), w2b)
    y2.backward(dy)
    assert torch.equal(y, y2)
    assert _rel_err(x.grad, x2.grad) < 4e-3 and _rel_err(w13.grad, w13b.grad) < 4e-3


@pytest.mark.parametrize("mode", ["fwd", "dgrad", "swiglu", "swiglu_bwd", "rope", "ahead"])
def test_weight_gather_gemm_single_rank(mode):
    """IO = 3 (parameter all-gather ⊕ GEMM) with a 1-rank group: the copier, the readiness counters, the gated TMA producer, the
    rotated tile / K order and the gather-ahead list all run (the "peer" is this GPU), so the ZeRO-3 kernel is covered on a
    single-GPU box and under compute-sanitizer; the multi-GPU variants live in tests/test_multigpu.py."""
    import ctypes

    from prime_b200 import ops
    from prime_b200.ops import reference
    from prime_b200.parallel.fsdp import RowShard
    from prime_b200.parallel.symm import SymmetricHeap

    dev = _dev()
    heap = SymmetricHeap(256 << 20, 0, 1, lambda h: [h], dev)
    torch.manual_seed(17)
    M, K = 768, 512

    def shard(W):
        rows, cols = W.shape
        sh = heap.alloc(rows * cols, torch.bfloat16).view(rows, cols)
        sh.copy_(W)
        full = torch.zeros(rows, cols, dtype=torch.bfloat16, device=dev)
        flags = torch.zeros(64, dtype=torch.int32, device=dev)
        peers = (ctypes.c_void_p * 1)(heap.peer_ptr(0, sh))
        return RowShard(rows, cols, 1, 0, rows, peers, full.data_ptr(), flags, sh, full=full), full

    x = (torch.randn(M, K, device=dev) * 0.5).to(torch.bfloat16)
    try:
        if mode in ("fwd", "dgrad", "ahead"):
            W = (torch.randn(1088, K, device=dev) * 0.05).to(torch.bfloat16)  # 1088 rows: the last 128-row box is clipped
            z, full = shard(W)
            if mode == "fwd":
                y = ops.gemm_wgather(x, z)
                ref = x.float() @ W.float().t()
            elif mode == "dgrad":
                dy = (torch.randn(M, 1088, device=dev) * 0.5).to(torch.bfloat16)
                y = ops.gemm_wgather(dy, z, b_mn_major=True)
                ref = dy.float() @ W.float()
            else:
                W2 = (torch.randn(640, 1088, device=dev) * 0.05).to(torch.bfloat16)
                z2, full2 = shard(W2)
                z.next_fwd = z2
                y1 = ops.gemm_wgather(x, z)
                torch.cuda.synchronize()
                assert torch.equal(full2, W2) and ops.functional._resident(z2)  # gathered ahead by the first kernel
                y = ops.gemm_wgather(y1, z2)  # resident: plain kernel
                ref = y1.float() @ W2.float().t()
            assert torch.equal(full, W)
        elif mode in ("swiglu", "swiglu_bwd"):
            FF = 576
            W13 = (torch.randn(2 * FF, K, device=dev) * 0.05).to(torch.bfloat16)
            z13, _ = shard(W13)
            gu = torch.empty(M, 2 * FF, dtype=torch.bfloat16, device=dev)
            h = torch.empty(M, FF, dtype=torch.bfloat16, device=dev)
            ops.gemm_wgather(x, z13, out=gu, swiglu_h=h)
            gur = (x.float() @ W13.float().t()).to(torch.bfloat16).float()
            if mode == "swiglu":
                y, ref = h, torch.nn.functional.silu(gur[:, :FF]) * gur[:, FF:]
                assert _rel_err(gu, gur) < 1e-2
            else:
                W2 = (torch.randn(K, FF, device=dev) * 0.05).to(torch.bfloat16)
                z2, _ = shard(W2)
                dy = (torch.randn(M, K, device=dev) * 0.5).to(torch.bfloat16)
                y = ops.gemm_wgather(dy, z2, b_mn_major=True, swiglu_bwd_gu=gu)
                dh = dy.float() @ W2.float()
                g, u = gu[:, :FF].float(), gu[:, FF:].float()
                sg = torch.sigmoid(g)
                ref = torch.cat((dh * u * sg * (1 + g * (1 - sg)), dh * g * sg), dim=1)
        else:
            H, D, S = 2, 128, 256
            Wq = (torch.randn(3 * H * D, K, device=dev) * 0.05).to(torch.bfloat16)
            zq, _ = shard(Wq)
            cos, sin = reference.rope_tables(S, D, 10000.0, device=dev)
            y = ops.gemm_wgather(x, zq, rope=(cos, sin, S, 2 * H * D, D))
            r = (x.float() @ Wq.float().t()).view(-1, S, 3 * H, D)
            ref = torch.cat((reference.rope(r[:, :, : 2 * H], cos, sin), r[:, :, 2 * H :]), dim=2).reshape(M, -1)
        torch.cuda.synchronize()
        heap.check_errors()
        assert _rel_err(y, ref) < 1e-2 and _max_rel(y, ref) < 5e-2
    finally:
        ops.reset_gather_cache()
        heap.close()
