"""Full-model parity at the Llama-1B shape: logits and every parameter gradient of the native bf16 model (wgmma GEMMs, flash
attention, fused epilogues, native embedding / loss) against an independent fp32 PyTorch model with the same weights
(``baseline/torch_b0.Llama`` — nn.Linear, SDPA, complex-multiply RoPE). VERDICT r1 #7."""

import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def _load_into_b0(ours, ref):
    """Copy the native model's (fused-layout) weights into the stock model (same fused layout: [q;k;v] rows, [gate;up] rows)."""
    with torch.no_grad():
        ref.tok_embeddings.weight.copy_(ours.tok_embeddings.weight.float())
        for a, b in zip(ours.layers, ref.layers):
            b.wqkv.weight.copy_(a.attention.wqkv.float())
            b.wo.weight.copy_(a.attention.wo.float())
            b.w13.weight.copy_(a.feed_forward.w13.float())
            b.w2.weight.copy_(a.feed_forward.w2.float())
            b.attention_norm.weight.copy_(a.attention_norm.weight.float())
            b.ffn_norm.weight.copy_(a.ffn_norm.weight.float())
        ref.norm.weight.copy_(ours.norm.weight.float())
        ref.output.weight.copy_(ours.output.float())


def _rel(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / (b.norm() + 1e-12))


def _max_rel(a, b):
    a, b = a.float(), b.float()
    return float(((a - b).abs() / (b.abs() + 0.05 * b.abs().max())).max())


@pytest.mark.parametrize("n_layers,S", [(1, 1024), (18, 512)])
def test_llama_1b_shape_logits_and_grads_match_fp32_torch(n_layers, S):
    from baseline.torch_b0 import Llama as RefLlama
    from prime_b200.models.llama import build_model

    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    ours = build_model("1B", device=dev, dtype=torch.bfloat16, seed=11, n_layers=n_layers, max_seq_len=S)
    ref = RefLlama(2048, n_layers, 16, 32000, max_seq=S).to(dev).float()
    _load_into_b0(ours, ref)
    B = 2
    tok = torch.randint(0, 32000, (B, S), device=dev)
    tgt = torch.randint(0, 32000, (B, S), device=dev)
    logits = ours(tok)
    keep = logits.detach().clone()  # the loss kernel overwrites the logits with their gradient
    loss = torch.nn.functional.cross_entropy(logits.float().view(-1, 32000), tgt.view(-1))
    loss.backward()
    rl = ref(tok)
    rloss = torch.nn.functional.cross_entropy(rl.view(-1, 32000), tgt.view(-1))
    rloss.backward()
    tol = 1.5e-2 if n_layers == 1 else 4e-2
    assert _rel(keep, rl) < tol, (_rel(keep, rl),)
    assert _max_rel(keep, rl) < 6 * tol
    assert abs(float(loss) - float(rloss)) < 2e-2 * float(rloss)
    pairs = [("embed", ours.tok_embeddings.weight.grad, ref.tok_embeddings.weight.grad), ("output", ours.output.grad, ref.output.weight.grad),
             ("norm", ours.norm.weight.grad, ref.norm.weight.grad)]  # fmt: skip
    for i, (a, b) in enumerate(zip(ours.layers, ref.layers)):
        pairs += [(f"l{i}.wqkv", a.attention.wqkv.grad, b.wqkv.weight.grad), (f"l{i}.wo", a.attention.wo.grad, b.wo.weight.grad),
                  (f"l{i}.w13", a.feed_forward.w13.grad, b.w13.weight.grad), (f"l{i}.w2", a.feed_forward.w2.grad, b.w2.weight.grad),
                  (f"l{i}.anorm", a.attention_norm.weight.grad, b.attention_norm.weight.grad)]  # fmt: skip
    gtol = 3e-2 if n_layers == 1 else 8e-2
    worst = max((_rel(a, b), name) for name, a, b in pairs)
    assert worst[0] < gtol, worst


def test_native_loss_path_matches_torch_cross_entropy():
    """model.loss(): native count → fused CE (register-resident rows) → fixed-order mean, with ignore_index and grad scaling."""
    from prime_b200 import ops

    dev = torch.device("cuda", 0)
    torch.manual_seed(3)
    for V, R in ((32000, 512), (2048, 300), (128256, 64)):
        z = (torch.randn(R, V, device=dev) * 2).to(torch.bfloat16)
        t = torch.randint(0, V, (R,), device=dev)
        t[::7] = -100
        zr = z.float().requires_grad_(True)
        ref = torch.nn.functional.cross_entropy(zr, t, ignore_index=-100)
        ref.backward()
        zz = z.clone().requires_grad_(True)
        acc = torch.zeros((), device=dev)
        loss = ops.cross_entropy(zz.view(1, R, V), t.view(1, R), grad_scale=0.25, unit_upstream=True, loss_acc=acc)
        loss.backward()
        assert abs(float(loss) - float(ref)) < 2e-3 * abs(float(ref)) and abs(float(acc) - float(loss)) < 1e-6
        assert _rel(zz.grad.view(R, V), 0.25 * zr.grad) < 1e-2
        assert float(zz.grad.view(R, V)[::7].abs().max()) == 0.0  # ignored rows get no gradient
