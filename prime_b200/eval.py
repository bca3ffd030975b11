"""Offline evaluation of a trained model: perplexity over a tokenised corpus and (small-scale) sampling.

    python -m prime_b200.eval ppl --ckpt runs/x/ckpt/step_001000 --model 1B --data data/c4_val --seq 1024 --batches 50
    python -m prime_b200.eval ppl --hf path/to/llama --data data/c4_val
    python -m prime_b200.eval ppl --ckpt … --model 1B --data data/c4_val --document-mask   # attention within documents only
    python -m prime_b200.eval generate --ckpt … --model 1B --prompt-ids 1,306,626 --max-new 32
    python -m prime_b200.eval generate --ckpt … --model 1B --prompt-ids 1,306,626 --temperature 0.8 --top-p 0.9 --sampler device
    python -m prime_b200.eval generate --ckpt … --model 1B --draft-ckpt … --draft-model 150M --spec-k 4 --prompt-ids 1,306,626
    python -m prime_b200.eval generate --ckpt … --model 1B --prompt-ids 1,306,626 --kv-dtype fp8   # e4m3 KV cache: half the bytes
    python -m prime_b200.eval generate --ckpt … --model 1B --prompt-ids 1,306,626 --weight-dtype fp8   # e4m3 projection weights

The model is rebuilt on one device from the per-rank optimizer shards (``checkpoint.assemble_full_model``) or from a Hugging
Face directory (``models.hf.load_hf_dir``); the forward runs through the same ops as training (native kernels on an H100, the
reference ops on the CPU).  Generation runs on a KV cache (``inference.py``): one prefill of the prompt, padded to a multiple of 128
on CUDA, then one decode step per token (the split-KV decode-attention kernel, the step replayed from a CUDA graph on the GPU), so
T new tokens cost one prompt forward and T single-token steps instead of T full forwards. ``generate_batch`` samples ragged
prompt lists together. Sliding windows and document masking (``Transformer.doc_eos_id``) behave as in the full forward.

``--weight-dtype fp8`` (both commands; with a draft model it converts the draft as well) runs ``inference.quantize_weights`` after
loading: the four projections of every block and the LM head are held as e4m3 with a power-of-two scale per 32 values (about 1.03
bytes per weight instead of 2). Decode and verify steps read those bytes in place (``ops.linear`` on an ``ops.MXWeight``); prefill and
perplexity run the bf16 kernels on the exactly dequantised weights. The embedding and the norms stay as loaded.
"""

from __future__ import annotations

import argparse
import json
import math

import torch
import torch.nn.functional as F

from . import ops
from .data import MemmapTokenDataset
from .inference import generate_batch, generate_speculative, quantize_weights, sample
from .models.llama import Transformer


@torch.no_grad()
def perplexity(model: Transformer, dataset, *, batches: int, batch_size: int, device: torch.device | str) -> dict:
    """Mean next-token loss (nats) and perplexity over ``batches`` × ``batch_size`` windows of ``dataset``."""
    model.eval()
    tot, n = 0.0, 0
    for _ in range(batches):
        x, y = dataset.next_batch(batch_size)
        tok = torch.from_numpy(x).to(device)
        tgt = torch.from_numpy(y).to(device)
        logits = model(tok)
        tot += float(F.cross_entropy(logits.float().reshape(-1, logits.shape[-1]), tgt.reshape(-1), reduction="sum"))
        n += tgt.numel()
    loss = tot / max(n, 1)
    return {"loss": loss, "perplexity": math.exp(min(loss, 50.0)), "tokens": n}


def generate(model: Transformer, prompt: list[int], *, max_new: int, temperature: float = 0.0, top_k: int = 0, top_p: float = 1.0,
             min_p: float = 0.0, seed: int = 0, eos_id: int | None = None, sampler: str = "host", kv_dtype: str = "bf16") -> list[int]:  # fmt: skip
    """Greedy (temperature 0) or temperature / top-k / top-p / min-p sampling; returns prompt + continuation. ``sampler``: "host"
    (the random stream of earlier versions) or "device" (``ops.sample_tokens``'s Philox stream), see ``generate_batch``; ``kv_dtype``:
    "bf16" or "fp8" (an e4m3 KV cache)."""
    return generate_batch(model, [prompt], max_new=max_new, temperature=temperature, top_k=top_k, top_p=top_p, min_p=min_p, seed=seed,
                          eos_id=eos_id, sampler=sampler, kv_dtype=kv_dtype)[0]  # fmt: skip


@torch.no_grad()
def _generate_recompute(model: Transformer, prompt: list[int], *, max_new: int, temperature: float = 0.0, top_k: int = 0,
                        top_p: float = 1.0, min_p: float = 0.0, seed: int = 0, eos_id: int | None = None,
                        sampler: str = "host") -> list[int]:  # fmt: skip
    """:func:`generate` without a cache: the whole prefix is run again for every token (padded to a multiple of 128 on CUDA). The
    oracle of the cached path and the baseline of its speed-up. ``sampler="device"`` draws each token with ``ops.sample_tokens`` on
    the model's device, keyed by ``seed`` at the token's position: row b of ``generate_batch(seed=s)`` is this with seed s + b."""
    model.eval()
    dev = next(model.parameters()).device
    ids = list(prompt)
    gen = torch.Generator(device="cpu").manual_seed(seed)
    seeds = torch.tensor([seed], dtype=torch.int64, device=dev)
    pad_to = 128 if dev.type == "cuda" else 1
    for _ in range(max_new):
        n = len(ids)
        if n >= model.args.max_seq_len:
            break
        padded = ids + [0] * ((-n) % pad_to)
        logits = model(torch.tensor([padded], dtype=torch.int64, device=dev))[0, n - 1]
        if sampler == "device":
            pos = torch.tensor([n], dtype=torch.int32, device=dev)
            nxt = int(ops.sample_tokens(logits.view(1, -1), temperature=temperature, top_k=top_k, top_p=top_p, min_p=min_p, seeds=seeds,
                                        positions=pos)[0])  # fmt: skip
        else:
            nxt = sample(logits.float().cpu(), temperature, top_k, gen, top_p, min_p)
        ids.append(nxt)
        if eos_id is not None and nxt == eos_id:
            break
    return ids


def load_model(a, device: str, prefix: str = "") -> Transformer:
    """The model named by ``--ckpt`` / ``--hf`` / ``--model`` / ``--type-model`` (``prefix="draft_"``: the ``--draft-*`` ones)."""
    dtype = torch.bfloat16 if device.startswith("cuda") else torch.float32
    hf = getattr(a, prefix + "hf")
    if hf:
        from .models.hf import load_hf_dir

        return load_hf_dir(hf, device=device, dtype=dtype)
    from .checkpoint import assemble_full_model

    return assemble_full_model(getattr(a, prefix + "ckpt"), getattr(a, prefix + "model"), getattr(a, prefix + "type_model")).to(
        device=device, dtype=dtype)  # fmt: skip


def main(argv: list[str] | None = None) -> dict:
    ap = argparse.ArgumentParser(prog="python -m prime_b200.eval", description=__doc__.split("\n\n")[0])
    sub = ap.add_subparsers(dest="cmd", required=True)
    for name in ("ppl", "generate"):
        p = sub.add_parser(name)
        src = p.add_mutually_exclusive_group(required=True)
        src.add_argument("--ckpt", help="checkpoint step directory written by the trainer")
        src.add_argument("--hf", help="Hugging Face Llama checkpoint directory")
        p.add_argument("--model", default="1B")
        p.add_argument("--type-model", default="llama2", choices=["llama2", "llama3"])
        p.add_argument("--device", default="cuda" if torch.cuda.is_available() else "cpu")
        p.add_argument("--weight-dtype", default="bf16", choices=["bf16", "fp8"],
                       help="projection weights: as loaded, or fp8 = e4m3 with a power-of-two scale per 32 values (inference only)")
    p = sub.choices["ppl"]
    p.add_argument("--data", required=True, help="token files / directory / glob (see tools/tokenize_corpus.py)")
    p.add_argument("--seq", type=int, default=1024)
    p.add_argument("--batches", type=int, default=20)
    p.add_argument("--batch-size", type=int, default=8)
    p.add_argument("--document-mask", action="store_true",
                   help="document-masked attention: a token attends only to earlier tokens of its own document (EOS id from the "
                        "first shard's .meta.json unless --eos-id is given)")  # fmt: skip
    p.add_argument("--eos-id", type=int, default=None, help="EOS id that ends a document; implies --document-mask")
    g = sub.choices["generate"]
    g.add_argument("--prompt-ids", required=True, help="comma-separated token ids")
    g.add_argument("--max-new", type=int, default=32)
    g.add_argument("--temperature", type=float, default=0.0)
    g.add_argument("--top-k", type=int, default=0)
    g.add_argument("--top-p", type=float, default=1.0, help="nucleus sampling: keep the smallest top set holding this share of the mass")
    g.add_argument("--min-p", type=float, default=0.0, help="keep tokens with at least this share of the top token's probability")
    g.add_argument("--sampler", default="host", choices=["host", "device"],
                   help="host: CPU generator, as earlier versions; device: sample inside the captured decode step (Philox stream)")
    g.add_argument("--seed", type=int, default=0)
    dsrc = g.add_mutually_exclusive_group()
    dsrc.add_argument("--draft-ckpt", help="speculative decoding: the draft model's checkpoint step directory")
    dsrc.add_argument("--draft-hf", help="speculative decoding: the draft model's Hugging Face directory")
    g.add_argument("--draft-model", default="150M")
    g.add_argument("--draft-type-model", default="llama2", choices=["llama2", "llama3"])
    g.add_argument("--spec-k", type=int, default=4, help="draft tokens per speculative round")
    g.add_argument("--kv-dtype", default="bf16", choices=["bf16", "fp8"],
                   help="KV-cache storage: bf16, or fp8 = e4m3 with a power-of-two scale per 32 values (about half the bytes)")
    a = ap.parse_args(argv)
    spec = a.cmd == "generate" and (a.draft_ckpt or a.draft_hf)
    if spec and a.sampler == "host":
        raise SystemExit("speculative decoding samples on the device: --sampler host cannot be combined with a draft model")
    model = load_model(a, a.device)
    if a.weight_dtype == "fp8":
        quantize_weights(model)
    if a.cmd == "ppl":
        if a.document_mask or a.eos_id is not None:
            from .data import eos_id_from_meta

            eos = a.eos_id if a.eos_id is not None else eos_id_from_meta(a.data)
            if eos is None:
                raise SystemExit(f"--document-mask: no eos_id in the .meta.json of the first shard of {a.data!r}; pass --eos-id")
            model.doc_eos_id = eos
        ds = MemmapTokenDataset(a.data, a.seq, vocab_size=model.args.vocab_size, shuffle=False)
        out = perplexity(model, ds, batches=min(a.batches, max(1, ds.windows // a.batch_size)), batch_size=a.batch_size, device=a.device)
    elif spec:
        draft = load_model(a, a.device, "draft_")
        if a.weight_dtype == "fp8":
            quantize_weights(draft)
        r = generate_speculative(model, draft, [[int(x) for x in a.prompt_ids.split(",")]], k=a.spec_k,
                                 max_new=a.max_new, temperature=a.temperature, top_k=a.top_k, top_p=a.top_p, min_p=a.min_p,
                                 seed=a.seed, kv_dtype=a.kv_dtype)  # fmt: skip
        out = {"ids": r.ids[0], "spec": {"rounds": r.rounds, "drafted": r.drafted, "accepted": r.accepted,
                                         "acceptance": r.accepted / max(r.drafted, 1)}}  # fmt: skip
    else:
        ids = generate(model, [int(x) for x in a.prompt_ids.split(",")], max_new=a.max_new, temperature=a.temperature, top_k=a.top_k,
                       top_p=a.top_p, min_p=a.min_p, seed=a.seed, sampler=a.sampler, kv_dtype=a.kv_dtype)  # fmt: skip
        out = {"ids": ids}
    print(json.dumps(out))
    return out


if __name__ == "__main__":
    main()
