"""2-GPU checks of the fused NVLink paths (run on the box with `gpurun --gpus 2`): the P2P reduce-scatter⊕AdamW⊕
all-gather and the int8 outer all-gather⊕Nesterov must agree with the NCCL-collective implementation of the
same algorithm, and replicas must stay bitwise consistent."""

import json
import os
import socket
import subprocess
import sys
import textwrap
from pathlib import Path

import pytest

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]
ROOT = Path(__file__).resolve().parent.parent

WORKER = textwrap.dedent(
    """
    import json, sys, torch
    import torch.distributed as dist
    sys.path.insert(0, {root!r})
    from prime_b200.config import Config
    from prime_b200.trainer import Trainer

    def run(fused):
        cfg = Config.model_validate({cfg!r})
        cfg.train.fused_comm = fused
        t = Trainer(cfg)
        losses = [float(t.inner_step().loss.item()) for _ in range({steps})]
        torch.cuda.synchronize()
        if t.heap is not None:
            t.heap.check_errors()
        out = dict(losses=losses, master=t.engine.master.clone(), params=t.engine.param_flat.clone().float(),
                   gnorm=float(t.engine.last_grad_norm), outer=t.outer.outer_step_count if t.outer else 0)
        t.close()
        return out

    a = run(True)
    b = run(False)
    rel = float((a["master"] - b["master"]).norm() / b["master"].norm())
    prel = float((a["params"] - b["params"]).norm() / b["params"].norm())
    # replica consistency of the fused path: every rank of an FSDP group / every worker after an outer step
    h = a["params"].double().sum().reshape(1)
    hs = [torch.zeros_like(h) for _ in range(dist.get_world_size())]
    dist.all_gather(hs, h)
    if dist.get_rank() == 0:
        print("RESULT " + json.dumps(dict(rel=rel, prel=prel, la=a["losses"], lb=b["losses"], ga=a["gnorm"], gb=b["gnorm"],
              hashes=[float(x) for x in hs], outer=a["outer"])))
    dist.barrier()
    dist.destroy_process_group()
    """
)


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _run(nproc, cfg, steps, tmp_path, env=None):
    script = tmp_path / "w.py"
    script.write_text(WORKER.format(root=str(ROOT), cfg=cfg, steps=steps))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}", "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), str(script)]  # fmt: skip
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env={**os.environ, **(env or {})})
    assert p.returncode == 0, p.stdout[-4000:] + p.stderr[-4000:]
    return json.loads([l for l in p.stdout.splitlines() if l.startswith("RESULT ")][-1][7:])


BASE = {"name_model": "debugmodel", "data": {"seq_length": 128}, "optim": {"batch_size": 8, "warmup_steps": 2, "optim": {"lr": 3e-3}},
        "train": {"micro_bs": 2}}  # fmt: skip


def test_fsdp2_fused_matches_collective(tmp_path):
    cfg = {**BASE, "mesh": {"fsdp_size": 2}}
    r = _run(2, cfg, 5, tmp_path)
    assert r["rel"] < 2e-3 and r["prel"] < 5e-3, r
    assert abs(r["ga"] - r["gb"]) < 2e-2 * r["gb"], r
    assert r["hashes"][0] == r["hashes"][1], r  # both ranks hold identical bf16 parameters
    assert r["la"][-1] < r["la"][0]


# NVLS (multimem.ld_reduce / multimem.st over a VMM heap bound to an NVSwitch multicast object); the tests skip themselves only where
# the driver reports no multicast support.
def test_fsdp2_nvls_reduce_scatter_matches_collective(tmp_path):
    """PB_NVLS=1: the heap is VMM-backed with a multicast mapping and the gradient reduce-scatter is summed by the switch."""
    from prime_b200.parallel.multicast import nvls_available

    if not nvls_available(0):
        pytest.skip("multicast unsupported on this box")
    r = _run(2, {**BASE, "mesh": {"fsdp_size": 2}}, 5, tmp_path, env={"PB_NVLS": "1"})
    assert r["rel"] < 2e-3 and r["prel"] < 5e-3, r
    assert abs(r["ga"] - r["gb"]) < 2e-2 * r["gb"], r
    assert r["hashes"][0] == r["hashes"][1], r
    assert r["la"][-1] < r["la"][0]


def test_diloco2_fused_outer_matches_collective(tmp_path):
    cfg = {**BASE, "mesh": {"num_workers": 2}, "diloco": {"inner_steps": 3}}
    r = _run(2, cfg, 6, tmp_path)
    assert r["outer"] == 2
    assert r["rel"] < 2e-3, r
    assert r["hashes"][0] == r["hashes"][1], r  # workers identical right after an outer step


CG_WORKER = textwrap.dedent(
    """
    import json, sys, torch
    import torch.distributed as dist
    sys.path.insert(0, {root!r})
    from prime_b200 import ops
    from prime_b200.parallel.mesh import init_distributed
    from prime_b200.parallel.symm import SymmetricHeap, dist_exchange
    from prime_b200.parallel.collective_gemm import CollectiveGemm

    w = init_distributed("nccl")
    dev = torch.device("cuda", w.local_rank)
    n, r = w.world_size, w.rank
    heap = SymmetricHeap(512 << 20, r, n, dist_exchange(), dev)
    cg = CollectiveGemm(heap, list(range(n)))
    torch.manual_seed(1234)  # same tensors on every rank, then shard
    M_local, N, K = 512, 1024, 768
    A_full = (torch.randn(n * M_local, K, device=dev) * 0.1).to(torch.bfloat16)
    B = (torch.randn(N, K, device=dev) * 0.1).to(torch.bfloat16)
    # ---- all-gather + GEMM
    a_sym = heap.alloc(M_local * K, torch.bfloat16).view(M_local, K)
    a_sym.copy_(A_full[r * M_local:(r + 1) * M_local])
    for _ in range(2):  # twice: flags and the gathered scratch are reusable
        C = cg.all_gather_gemm(a_sym, B)
    ref = A_full.float() @ B.float().t()
    e_ag = float((C.float() - ref).norm() / ref.norm())
    for o in range(n):  # by-product: the remote row blocks, copied exactly once over NVLink
        if o != r:
            assert torch.equal(cg.gathered[o * M_local:(o + 1) * M_local], A_full[o * M_local:(o + 1) * M_local]), "gathered copy differs"
    # ---- GEMM + reduce-scatter (K sharded)
    Kl = K // n
    M = n * M_local
    a_k = A_full[:, r * Kl:(r + 1) * Kl].contiguous()
    b_k = B[:, r * Kl:(r + 1) * Kl].contiguous()
    out_sym = heap.alloc((M // n) * N, torch.float32).view(M // n, N)
    for _ in range(2):  # twice: the buffers and flags are reusable
        cg.gemm_reduce_scatter(a_k, b_k, out_sym)
    torch.cuda.synchronize()
    partial = [A_full[:, i * Kl:(i + 1) * Kl].float() @ B[:, i * Kl:(i + 1) * Kl].float().t() for i in range(n)]
    ref_rs = sum(partial)[r * (M // n):(r + 1) * (M // n)]
    e_rs = float((out_sym - ref_rs).norm() / ref_rs.norm())
    heap.check_errors()
    errs = [None] * n
    dist.all_gather_object(errs, (e_ag, e_rs))
    if r == 0:
        print("RESULT " + json.dumps(dict(errs=errs)))
    dist.barrier()
    heap.close()
    dist.destroy_process_group()
    """
)


def test_fused_allgather_gemm_and_gemm_reduce_scatter(tmp_path):
    """ONE kernel each: A tiles pulled from the owning rank's memory by TMA inside the GEMM; fp32 tiles reduce-added into the
    owning rank's buffer by TMA from the GEMM epilogue. Compared with the dense single-device result."""
    script = tmp_path / "cg_worker.py"
    script.write_text(CG_WORKER.format(root=str(ROOT)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), str(script)]  # fmt: skip
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")][-1]
    errs = json.loads(line[len("RESULT "):])["errs"]
    for e_ag, e_rs in errs:
        assert e_ag < 1e-2, errs
        assert e_rs < 2e-3, errs


SP_WORKER = textwrap.dedent(
    """
    import json, sys, torch
    import torch.distributed as dist
    sys.path.insert(0, {root!r})
    from prime_b200.parallel.mesh import init_distributed
    from prime_b200.parallel.symm import SymmetricHeap, dist_exchange
    from prime_b200.parallel.tensor_parallel import SequenceParallelMLP

    w = init_distributed("nccl")
    dev = torch.device("cuda", w.local_rank)
    n, r = w.world_size, w.rank
    heap = SymmetricHeap(256 << 20, r, n, dist_exchange(), dev)
    torch.manual_seed(7)  # identical full tensors on every rank, then shard
    T, D, FF = 1024, 512, 1024
    x = (torch.randn(T, D, device=dev) * 0.5).to(torch.bfloat16)
    w13 = (torch.randn(2 * FF, D, device=dev) * 0.04).to(torch.bfloat16)
    w2 = (torch.randn(D, FF, device=dev) * 0.04).to(torch.bfloat16)
    dy = (torch.randn(T, D, device=dev) * 0.5).to(torch.bfloat16)
    mlp = SequenceParallelMLP(heap, list(range(n)), D, FF, T // n)
    mlp.load_full_weights(w13, w2)
    tl = T // n
    for _ in range(2):  # twice: symmetric buffers and flags are reusable, gradients accumulate like any nn.Module
        mlp.zero_grad(set_to_none=True)
        x_local = x[r * tl:(r + 1) * tl].clone().requires_grad_(True)
        y_local = mlp(x_local)
        y_local.backward(dy[r * tl:(r + 1) * tl])
    torch.cuda.synchronize()
    # dense fp32 reference on the full tensors
    xr, w13r, w2r = x.float().requires_grad_(True), w13.float().requires_grad_(True), w2.float().requires_grad_(True)
    gu = xr @ w13r.t()
    h = torch.nn.functional.silu(gu[:, :FF]) * gu[:, FF:]
    yr = h @ w2r.t()
    yr.backward(dy.float())
    rel = lambda a, b: float((a.float() - b.float()).norm() / (b.float().norm() + 1e-12))
    f = FF // n
    errs = dict(
        y=rel(y_local, yr[r * tl:(r + 1) * tl]),
        dx=rel(x_local.grad, xr.grad[r * tl:(r + 1) * tl]),
        dw13=rel(mlp.w13.grad, torch.cat([w13r.grad[r * f:(r + 1) * f], w13r.grad[FF + r * f:FF + (r + 1) * f]])),
        dw2=rel(mlp.w2.grad, w2r.grad[:, r * f:(r + 1) * f]),
    )
    heap.check_errors()
    allerrs = [None] * n
    dist.all_gather_object(allerrs, errs)
    if r == 0:
        print("RESULT " + json.dumps(allerrs))
    dist.barrier()
    heap.close()
    dist.destroy_process_group()
    """
)


def test_sequence_parallel_mlp_forward_backward(tmp_path):
    """SwiGLU MLP, sequence-sharded activations × hidden-sharded weights: all cross-GPU traffic inside the four fused collective
    GEMMs (all-gather ⊕ GEMM with K-major and MN-major B, GEMM ⊕ reduce-scatter likewise); output and all gradients vs dense fp32."""
    script = tmp_path / "sp_worker.py"
    script.write_text(SP_WORKER.format(root=str(ROOT)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), str(script)]  # fmt: skip
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")][-1]
    for errs in json.loads(line[len("RESULT "):]):
        assert errs["y"] < 1.5e-2 and errs["dx"] < 1.5e-2 and errs["dw13"] < 1.5e-2 and errs["dw2"] < 1.5e-2, errs


NVLS_WORKER = textwrap.dedent(
    """
    import ctypes, json, os, sys, torch
    import torch.distributed as dist
    sys.path.insert(0, {root!r})
    from prime_b200.ops import _lib
    from prime_b200.parallel.multicast import MulticastHeap, nvls_available
    from prime_b200.parallel.symm import dist_exchange

    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
    dev = torch.device("cuda", rank)
    if not nvls_available(rank):
        if rank == 0:
            print("RESULT " + json.dumps(dict(skipped="multicast unsupported on this box")))
        dist.destroy_process_group()
        sys.exit(0)
    heap = MulticastHeap(64 << 20, rank, world, dist_exchange(), dev)
    lib = _lib.load()
    out = dict()
    g = torch.Generator(device="cpu").manual_seed(1234)
    n = 1 << 20
    parts = [torch.randn(n, generator=g) for _ in range(world)]  # every rank knows every rank's input
    want = torch.stack(parts).sum(0)
    # in-place all-reduce through the switch, f32 then bf16, twice each (the barrier counters must carry across launches)
    x32 = heap.alloc(n, torch.float32)
    xb = heap.alloc(n, torch.bfloat16)
    for rep in range(2):
        x32.copy_(parts[rank]); xb.copy_(parts[rank].bfloat16())
        heap.all_reduce_(x32); heap.all_reduce_(xb)
        torch.cuda.synchronize()
        out[f"f32_{{rep}}"] = float((x32.cpu() - want).abs().max() / want.abs().max())
        wb = torch.stack([p.bfloat16().float() for p in parts]).sum(0)
        out[f"bf16_{{rep}}"] = float((xb.float().cpu() - wb).abs().max() / wb.abs().max())
    # NVLS gradient reduce-scatter against the peer-load kernel: same shard, same scale, same sum of squares
    grads = heap.alloc(n, torch.float32)
    grads.copy_(parts[rank])
    torch.cuda.synchronize(); dist.barrier()
    shard = n // world
    off = rank * shard
    grid = lib.pb_grad_reduce_grid()
    o_mc, o_p2p = torch.zeros(shard, device=dev), torch.zeros(shard, device=dev)
    ss_mc, ss_p2p = torch.zeros(grid, device=dev), torch.zeros(grid, device=dev)
    s = torch.cuda.current_stream().cuda_stream
    pp = heap.peers(range(world), grads)
    table = _lib.SegTable.of([(off, 0, shard)])
    for mc, o, ss in ((heap.mc_ptr(grads), o_mc, ss_mc), (None, o_p2p, ss_p2p)):  # the one launcher, with and without mc_grads
        _lib.check(lib.pb_grad_reduce(ctypes.byref(pp), mc, ctypes.byref(table), 0.5, o.data_ptr(), ss.data_ptr(), None, 0, 0,
                                      heap.err.data_ptr(), 0, s), "pb_grad_reduce")
    torch.cuda.synchronize()
    out["rs"] = float((o_mc - o_p2p).abs().max() / o_p2p.abs().max())
    out["rs_sumsq"] = abs(float(ss_mc.sum()) / float(ss_p2p.sum()) - 1.0)
    heap.check_errors()
    dist.barrier()
    heap.close()
    if rank == 0:
        print("RESULT " + json.dumps(out))
    dist.destroy_process_group()
    """
)


def test_nvls_multicast_all_reduce_and_grad_reduce(tmp_path):
    """multimem.ld_reduce / multimem.st over a VMM heap bound to an NVSwitch multicast object: the in-place all-reduce matches
    the dense sum, and the NVLS gradient reduce-scatter matches the peer-load kernel it can replace (PB_NVLS=1)."""
    script = tmp_path / "nvls_worker.py"
    script.write_text(NVLS_WORKER.format(root=str(ROOT)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), str(script)]  # fmt: skip
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    res = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")][-1][len("RESULT "):])
    if "skipped" in res:
        pytest.skip(res["skipped"])
    assert max(res["f32_0"], res["f32_1"]) < 1e-6, res
    assert max(res["bf16_0"], res["bf16_1"]) < 1e-2, res
    assert res["rs"] < 1e-6 and res["rs_sumsq"] < 1e-5, res


WG_WORKER = textwrap.dedent(
    """
    import ctypes, json, sys, torch
    import torch.distributed as dist
    sys.path.insert(0, {root!r})
    from prime_b200 import ops
    from prime_b200.ops import reference
    from prime_b200.parallel.fsdp import RowShard
    from prime_b200.parallel.mesh import init_distributed
    from prime_b200.parallel.symm import SymmetricHeap, dist_exchange

    w = init_distributed("nccl")
    dev = torch.device("cuda", w.local_rank)
    n, r = w.world_size, w.rank
    heap = SymmetricHeap(512 << 20, r, n, dist_exchange(), dev)
    torch.manual_seed(4321)  # identical full tensors on every rank, then shard by rows

    def shard(Wfull):
        rows, cols = Wfull.shape
        rpr = rows // n
        sh = heap.alloc(rpr * cols, torch.bfloat16).view(rpr, cols)
        sh.copy_(Wfull[r * rpr:(r + 1) * rpr])
        full = torch.zeros(rows, cols, dtype=torch.bfloat16, device=dev)
        flags = torch.zeros(64, dtype=torch.int32, device=dev)
        peers = (ctypes.c_void_p * n)(*[heap.peer_ptr(q, sh) for q in range(n)])
        return RowShard(rows, cols, n, r, rpr, peers, full.data_ptr(), flags, sh), full

    def errs(got, ref):
        got, ref = got.float(), ref.float()
        return [float((got - ref).norm() / ref.norm()), float(((got - ref).abs() / (ref.abs() + 0.05 * ref.abs().max())).max())]

    out = dict()
    M, K = {M}, {K}
    x = (torch.randn(M, K, device=dev) * 0.5).to(torch.bfloat16)
    # rows not a multiple of 128·n: the copier's last box of every rank block is clipped
    for name, N in (("fwd", {N}), ("fwd_ragged", {N} + 64 * n)):
        Wf = (torch.randn(N, K, device=dev) * 0.05).to(torch.bfloat16)
        z, full = shard(Wf)
        torch.cuda.synchronize(); dist.barrier()
        for _ in range(2):  # twice: flags and scratch are reusable
            y = ops.gemm_wgather(x, z)
        out[name] = errs(y, x.float() @ Wf.float().t())
        out[name + "_gathered_exact"] = bool(torch.equal(full, Wf))
        # input gradient: dx = dy · W, contraction over the sharded rows
        dy = (torch.randn(M, N, device=dev) * 0.5).to(torch.bfloat16)
        full.zero_()
        z.ver[0] += 1  # the scratch no longer holds W: force the in-kernel gather again
        dx = ops.gemm_wgather(dy, z, b_mn_major=True)
        out[name + "_dgrad"] = errs(dx, dy.float() @ Wf.float())
    # gather-ahead: the kernel that computes with W_a also pulls W_b (the next GEMM's weight) into ITS scratch; the next call then
    # finds W_b resident and runs the plain kernel on it
    Wa = (torch.randn({N}, K, device=dev) * 0.05).to(torch.bfloat16)
    Wb = (torch.randn(K + 64 * n, {N}, device=dev) * 0.05).to(torch.bfloat16)
    za, fa = shard(Wa)
    zb, fb = shard(Wb)
    za.next_fwd = zb
    torch.cuda.synchronize(); dist.barrier()
    ya = ops.gemm_wgather(x, za)
    torch.cuda.synchronize()
    out["ahead_a"] = errs(ya, x.float() @ Wa.float().t())
    out["ahead_b_gathered_exact"] = bool(torch.equal(fb, Wb))
    yb = ops.gemm_wgather(ya, zb)  # resident: no gather
    out["ahead_b"] = errs(yb, ya.float() @ Wb.float().t())
    out["ahead_b_was_resident_exact"] = bool(ops.functional._resident(zb))
    # SwiGLU epilogue: W13 = [gate rows | up rows]
    FF = {FF}
    W13 = (torch.randn(2 * FF, K, device=dev) * 0.05).to(torch.bfloat16)
    z13, _ = shard(W13)
    gu = torch.empty(M, 2 * FF, dtype=torch.bfloat16, device=dev)
    h = torch.empty(M, FF, dtype=torch.bfloat16, device=dev)
    torch.cuda.synchronize(); dist.barrier()
    ops.gemm_wgather(x, z13, out=gu, swiglu_h=h)
    gur = x.float() @ W13.float().t()
    out["swiglu_gu"] = errs(gu, gur)
    gb = gur.to(torch.bfloat16).float()
    out["swiglu_h"] = errs(h, torch.nn.functional.silu(gb[:, :FF]) * gb[:, FF:])
    # SwiGLU-backward epilogue on the down-projection's input gradient: W2 [K, FF] sharded by rows, d_gate_up = swiglu'(gu) ⊙ (dy·W2)
    W2 = (torch.randn(K, FF, device=dev) * 0.05).to(torch.bfloat16)
    z2, _ = shard(W2)
    dy2 = (torch.randn(M, K, device=dev) * 0.5).to(torch.bfloat16)
    torch.cuda.synchronize(); dist.barrier()
    dgu = ops.gemm_wgather(dy2, z2, b_mn_major=True, swiglu_bwd_gu=gu)
    dh = dy2.float() @ W2.float()
    gf, uf = gu[:, :FF].float(), gu[:, FF:].float()
    sg = torch.sigmoid(gf)
    out["swiglu_bwd"] = errs(dgu, torch.cat((dh * uf * sg * (1 + gf * (1 - sg)), dh * gf * sg), dim=1))
    # RoPE epilogue on the leading (Q, K) head columns of a fused QKV projection
    H, D, S = 4, 128, 256
    Wq = (torch.randn(3 * H * D, K, device=dev) * 0.05).to(torch.bfloat16)
    zq, _ = shard(Wq)
    cos, sin = reference.rope_tables(S, D, 10000.0, device=dev)
    torch.cuda.synchronize(); dist.barrier()
    yq = ops.gemm_wgather(x[: (M // S) * S], zq, rope=(cos, sin, S, 2 * H * D, D))
    ref = (x[: (M // S) * S].float() @ Wq.float().t()).view(-1, S, 3 * H, D)
    rot = reference.rope(ref[:, :, : 2 * H], cos, sin)
    ref = torch.cat((rot, ref[:, :, 2 * H:]), dim=2).reshape(-1, 3 * H * D)
    out["rope"] = errs(yq, ref)
    torch.cuda.synchronize()
    heap.check_errors()
    allo = [None] * n
    dist.all_gather_object(allo, out)
    if r == 0:
        print("RESULT " + json.dumps(allo))
    dist.barrier()
    heap.close()
    dist.destroy_process_group()
    """
)


def _ngpu():
    import torch

    return torch.cuda.device_count()


@pytest.mark.parametrize("nproc", [2, 4, 8])
def test_weight_gather_gemm(tmp_path, nproc):
    """ZeRO-3 hot path: parameter all-gather fused into the consuming GEMM (IO = 3) — forward, ragged row blocks, input gradient
    (contraction over the sharded dimension), SwiGLU and RoPE epilogues — against dense fp32, with per-element bounds."""
    if _ngpu() < nproc:
        pytest.skip(f"needs {nproc} GPUs")
    script = tmp_path / "wg_worker.py"
    script.write_text(WG_WORKER.format(root=str(ROOT), M=1024, K=512, N=1024 * nproc // 2, FF=512 * nproc // 2))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc), "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), str(script)]  # fmt: skip
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    for res in json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")][-1][len("RESULT "):]):
        for k, v in res.items():
            if k.endswith("_exact"):
                assert v, res
            else:
                assert v[0] < 1e-2 and v[1] < 5e-2, (k, res)


Z3_WORKER = textwrap.dedent(
    """
    import json, sys, torch
    import torch.distributed as dist
    sys.path.insert(0, {root!r})
    from prime_b200.config import Config
    from prime_b200.trainer import Trainer

    def run(reshard, fused=True):
        cfg = Config.model_validate({cfg!r})
        cfg.train.reshard_after_forward = reshard
        cfg.train.fused_comm = fused
        t = Trainer(cfg)
        assert t.engine.shard_params == bool(reshard)
        losses = [float(t.inner_step().loss.item()) for _ in range({steps})]
        torch.cuda.synchronize()
        t.check_health()
        eng = t.engine
        # full bf16 value of one big weight and of the embedding, gathered through the public helper
        wq = eng.full_param(t.model.layers[0].attention.wqkv).float().clone()
        emb = eng.full_param(t.model.tok_embeddings.weight).float().clone()
        out = dict(losses=losses, wq=wq, emb=emb, gnorm=float(eng.last_grad_norm), outer=t.outer.outer_step_count if t.outer else 0,
                   pbytes=(eng.pshard.numel() if eng.shard_params else 0) * 2 + eng.param_flat.numel() * 2)
        t.close()
        return out

    a = run(True)
    b = run(False)
    rel = lambda x, y: float((x - y).norm() / y.norm())
    res = dict(la=a["losses"], lb=b["losses"], wq=rel(a["wq"], b["wq"]), emb=rel(a["emb"], b["emb"]), ga=a["gnorm"], gb=b["gnorm"],
               outer=a["outer"], pbytes_z3=a["pbytes"], pbytes_rep=b["pbytes"])
    h = a["wq"].double().sum().reshape(1)
    hs = [torch.zeros_like(h) for _ in range(dist.get_world_size())]
    dist.all_gather(hs, h)
    res["hashes"] = [float(x) for x in hs]
    if dist.get_rank() == 0:
        print("RESULT " + json.dumps(res))
    dist.barrier()
    dist.destroy_process_group()
    """
)


@pytest.mark.parametrize("mesh", [{"fsdp_size": 2}, {"fsdp_size": 2, "num_workers": 2}, {"fsdp_size": 4}])
def test_zero3_training_matches_replicated(tmp_path, mesh):
    """train.reshard_after_forward: parameters sharded 1/F and gathered inside the GEMMs must train like the replicated engine
    (same data, same init): losses, one large weight, the embedding and the gradient norm; with DiLoCo on top in the 2x2 case."""
    n = mesh["fsdp_size"] * mesh.get("num_workers", 1)
    if _ngpu() < n:
        pytest.skip(f"needs {n} GPUs")
    cfg = {"name_model": "150M", "data": {"seq_length": 256}, "optim": {"batch_size": 4 * mesh["fsdp_size"], "warmup_steps": 2, "optim": {"lr": 1e-3}},
           "train": {"micro_bs": 2}, "mesh": mesh}  # fmt: skip
    if mesh.get("num_workers", 1) > 1:
        cfg["diloco"] = {"inner_steps": 2}
    script = tmp_path / "z3.py"
    script.write_text(Z3_WORKER.format(root=str(ROOT), cfg=cfg, steps=4))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), str(script)]  # fmt: skip
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-4000:] + p.stderr[-4000:]
    r = json.loads([l for l in p.stdout.splitlines() if l.startswith("RESULT ")][-1][7:])
    assert all(abs(x - y) < 2e-2 for x, y in zip(r["la"], r["lb"])), r
    assert r["wq"] < 5e-3 and r["emb"] < 5e-3 and abs(r["ga"] - r["gb"]) < 3e-2 * r["gb"], r
    assert len(set(r["hashes"])) == 1, r  # every rank gathers the same full weight
    assert r["pbytes_z3"] < 0.7 * r["pbytes_rep"], r  # parameter memory really shrank


def test_diloco2_fused_fp32_outer_matches_collective(tmp_path):
    """diloco.compression = "no": the fused outer step reads the peers' fp32 inner masters straight out of the symmetric heap."""
    cfg = {**BASE, "mesh": {"num_workers": 2}, "diloco": {"inner_steps": 3, "compression": "no"}}
    r = _run(2, cfg, 6, tmp_path)
    assert r["outer"] == 2
    assert r["rel"] < 1e-4, r
    assert r["hashes"][0] == r["hashes"][1], r
