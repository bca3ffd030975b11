"""Hugging Face ``LlamaForCausalLM`` interchange: import pretrained weights into the fused-QKV / fused-gate-up layout this
engine trains, export a trained model as a directory ``transformers`` loads (``config.json`` + safetensors shards).

    python -m prime_b200.models.hf export --ckpt runs/<run>/ckpt/step_1000 --model 1B --out hf_out/   # engine checkpoint → HF
    python -m prime_b200.models.hf import --hf path/to/llama --out weights.pt                          # HF → reference naming

Layout differences handled here (checked against ``transformers`` on CPU in ``tests/test_model_cpu.py``):

* **RoPE convention.** This engine rotates interleaved pairs (x[2i], x[2i+1]) — the Meta reference, and what the RoPE GEMM
  epilogue and the attention-backward epilogues implement. HF rotates (x[i], x[i + D/2]) and stores ``q_proj`` / ``k_proj``
  with the rows of every head permuted accordingly. Import undoes that permutation per head, export applies it.
* **Fused projections.** ``wqkv`` = [q; k; v] rows, ``w13`` = [gate; up] rows.
* **Untied head only.** ``tie_word_embeddings`` checkpoints are imported by copying the embedding into the head; exporting always
  writes an untied head. RoPE scaling variants (``rope_scaling`` ≠ null) are refused rather than silently ignored.
* **Sliding window.** A model with ``ModelArgs.sliding_window`` is exported as a ``MistralForCausalLM`` (same tensors and names,
  ``sliding_window`` in the config). Import stays Llama-only.
"""

from __future__ import annotations

import argparse
import json
from pathlib import Path

import torch

from .llama import ModelArgs, Transformer

_MAX_SHARD_BYTES = 4 << 30


def _to_interleaved(w: torch.Tensor, n_heads: int) -> torch.Tensor:
    """HF row order (per head: first half = even pair members, second half = odd) → interleaved pairs."""
    out, inp = w.shape
    d = out // n_heads
    return w.view(n_heads, 2, d // 2, inp).transpose(1, 2).reshape(out, inp)


def _to_half_split(w: torch.Tensor, n_heads: int) -> torch.Tensor:
    """Interleaved pairs → HF row order (inverse of :func:`_to_interleaved`)."""
    out, inp = w.shape
    d = out // n_heads
    return w.view(n_heads, d // 2, 2, inp).transpose(1, 2).reshape(out, inp)


def args_from_hf_config(cfg: dict) -> ModelArgs:
    """``config.json`` of a Llama-architecture checkpoint → :class:`ModelArgs`."""
    arch = cfg.get("architectures") or ["LlamaForCausalLM"]
    if cfg.get("model_type", "llama") != "llama" or not any("Llama" in a for a in arch):
        raise ValueError(f"not a Llama-architecture checkpoint: model_type={cfg.get('model_type')!r}, architectures={arch}")
    if cfg.get("rope_scaling"):
        raise ValueError(f"rope_scaling={cfg['rope_scaling']!r} is not supported (plain RoPE with rope_theta only)")
    if cfg.get("attention_bias") or cfg.get("mlp_bias"):
        raise ValueError("projection biases are not supported")
    dim, heads = int(cfg["hidden_size"]), int(cfg["num_attention_heads"])
    if cfg.get("head_dim") not in (None, dim // heads):
        raise ValueError(f"head_dim={cfg['head_dim']} differs from hidden_size / num_attention_heads = {dim // heads}")
    theta = cfg.get("rope_theta")
    if theta is None:  # transformers ≥ 5 nests it
        theta = (cfg.get("rope_parameters") or {}).get("rope_theta", 10000.0)
    return ModelArgs(
        dim=dim,
        n_layers=int(cfg["num_hidden_layers"]),
        n_heads=heads,
        n_kv_heads=int(cfg.get("num_key_value_heads") or heads),
        vocab_size=int(cfg["vocab_size"]),
        norm_eps=float(cfg.get("rms_norm_eps", 1e-5)),
        rope_theta=float(theta),
        max_seq_len=int(cfg.get("max_position_embeddings", 2048)),
        intermediate_size=int(cfg["intermediate_size"]),
    )


def hf_config_from_args(a: ModelArgs, dtype: torch.dtype = torch.bfloat16) -> dict:
    """``config.json`` of :func:`save_hf_dir`. A model with a sliding window is a ``MistralForCausalLM``: the same tensors, names and
    RoPE layout as Llama, with the window in every layer."""
    cfg = {
        "architectures": ["LlamaForCausalLM"],
        "model_type": "llama",
        "hidden_size": a.dim,
        "intermediate_size": a.ffn_hidden,
        "num_hidden_layers": a.n_layers,
        "num_attention_heads": a.n_heads,
        "num_key_value_heads": a.kv_heads,
        "head_dim": a.head_dim,
        "vocab_size": a.vocab_size,
        "rms_norm_eps": a.norm_eps,
        "rope_theta": a.rope_theta,
        "rope_scaling": None,
        "max_position_embeddings": a.max_seq_len,
        "hidden_act": "silu",
        "attention_bias": False,
        "mlp_bias": False,
        "tie_word_embeddings": False,
        "torch_dtype": str(dtype).replace("torch.", ""),
    }
    if a.sliding_window is not None:
        cfg.update(architectures=["MistralForCausalLM"], model_type="mistral", sliding_window=a.sliding_window)
    return cfg


@torch.no_grad()
def load_hf_state_dict(model: Transformer, sd: dict[str, torch.Tensor]) -> None:
    """Copy an HF ``LlamaForCausalLM`` state dict into ``model`` (shapes must match ``model.args``)."""
    a = model.args
    H, Hkv = a.n_heads, a.kv_heads
    get = lambda k: sd[k]  # noqa: E731
    model.tok_embeddings.weight.copy_(get("model.embed_tokens.weight"))
    for i, layer in enumerate(model.layers):
        p = f"model.layers.{i}."
        q = _to_interleaved(get(p + "self_attn.q_proj.weight"), H)
        k = _to_interleaved(get(p + "self_attn.k_proj.weight"), Hkv)
        layer.attention.wqkv.copy_(torch.cat([q, k, get(p + "self_attn.v_proj.weight")]))
        layer.attention.wo.copy_(get(p + "self_attn.o_proj.weight"))
        layer.feed_forward.w13.copy_(torch.cat([get(p + "mlp.gate_proj.weight"), get(p + "mlp.up_proj.weight")]))
        layer.feed_forward.w2.copy_(get(p + "mlp.down_proj.weight"))
        layer.attention_norm.weight.copy_(get(p + "input_layernorm.weight"))
        layer.ffn_norm.weight.copy_(get(p + "post_attention_layernorm.weight"))
    model.norm.weight.copy_(get("model.norm.weight"))
    model.output.copy_(sd["lm_head.weight"] if "lm_head.weight" in sd else get("model.embed_tokens.weight"))


def to_hf_state_dict(model: Transformer) -> dict[str, torch.Tensor]:
    a = model.args
    H, Hkv, D, hid = a.n_heads, a.kv_heads, a.head_dim, a.ffn_hidden
    out: dict[str, torch.Tensor] = {"model.embed_tokens.weight": model.tok_embeddings.weight.detach()}
    for i, layer in enumerate(model.layers):
        p = f"model.layers.{i}."
        wqkv = layer.attention.wqkv.detach()
        out[p + "self_attn.q_proj.weight"] = _to_half_split(wqkv[: H * D], H)
        out[p + "self_attn.k_proj.weight"] = _to_half_split(wqkv[H * D : (H + Hkv) * D], Hkv)
        out[p + "self_attn.v_proj.weight"] = wqkv[(H + Hkv) * D :]
        out[p + "self_attn.o_proj.weight"] = layer.attention.wo.detach()
        w13 = layer.feed_forward.w13.detach()
        out[p + "mlp.gate_proj.weight"] = w13[:hid]
        out[p + "mlp.up_proj.weight"] = w13[hid:]
        out[p + "mlp.down_proj.weight"] = layer.feed_forward.w2.detach()
        out[p + "input_layernorm.weight"] = layer.attention_norm.weight.detach()
        out[p + "post_attention_layernorm.weight"] = layer.ffn_norm.weight.detach()
    out["model.norm.weight"] = model.norm.weight.detach()
    out["lm_head.weight"] = model.output.detach()
    return out


# ---------------------------------------------------------------------------------------------------------- directories
def read_hf_dir(path: str | Path) -> tuple[dict, dict[str, torch.Tensor]]:
    """(config, state dict) of an HF checkpoint directory: safetensors (single file or sharded with an index) or ``pytorch_model.bin``."""
    d = Path(path)
    cfg = json.loads((d / "config.json").read_text())
    sd: dict[str, torch.Tensor] = {}
    idx = d / "model.safetensors.index.json"
    files = sorted(set(json.loads(idx.read_text())["weight_map"].values())) if idx.exists() else [f.name for f in sorted(d.glob("*.safetensors"))]
    if files:
        from safetensors.torch import load_file

        for f in files:
            sd.update(load_file(str(d / f)))
    elif (d / "pytorch_model.bin").exists():
        sd = torch.load(d / "pytorch_model.bin", map_location="cpu", weights_only=True)
    else:
        raise FileNotFoundError(f"no *.safetensors or pytorch_model.bin in {d}")
    return cfg, sd


def load_hf_dir(path: str | Path, *, device="cpu", dtype=torch.bfloat16) -> Transformer:
    """Build a :class:`Transformer` with the architecture and weights of an HF Llama checkpoint directory."""
    cfg, sd = read_hf_dir(path)
    args = args_from_hf_config(cfg)
    with torch.device(device):
        model = Transformer(args)
    model.to(dtype)
    load_hf_state_dict(model, sd)
    return model


def save_hf_dir(model: Transformer, path: str | Path, *, dtype: torch.dtype | None = None, max_shard_bytes: int = _MAX_SHARD_BYTES) -> list[str]:
    """Write ``config.json`` + safetensors shard(s) (+ index when sharded) that ``AutoModelForCausalLM.from_pretrained`` loads."""
    from safetensors.torch import save_file

    d = Path(path)
    d.mkdir(parents=True, exist_ok=True)
    dtype = dtype or next(model.parameters()).dtype
    sd = {k: v.to(device="cpu", dtype=dtype).contiguous() for k, v in to_hf_state_dict(model).items()}
    shards: list[dict[str, torch.Tensor]] = [{}]
    size = 0
    for k, v in sd.items():
        nbytes = v.numel() * v.element_size()
        if shards[-1] and size + nbytes > max_shard_bytes:
            shards.append({})
            size = 0
        shards[-1][k] = v
        size += nbytes
    names = []
    if len(shards) == 1:
        names = ["model.safetensors"]
        save_file(shards[0], str(d / names[0]), metadata={"format": "pt"})
    else:
        weight_map = {}
        for i, sh in enumerate(shards):
            name = f"model-{i + 1:05d}-of-{len(shards):05d}.safetensors"
            save_file(sh, str(d / name), metadata={"format": "pt"})
            names.append(name)
            weight_map.update({k: name for k in sh})
        total = sum(v.numel() * v.element_size() for v in sd.values())
        (d / "model.safetensors.index.json").write_text(json.dumps({"metadata": {"total_size": total}, "weight_map": weight_map}, indent=1))
    (d / "config.json").write_text(json.dumps(hf_config_from_args(model.args, dtype), indent=1))
    return names


# ---------------------------------------------------------------------------------------------------------------- CLI
def _model_from_engine_ckpt(ckpt: str, name: str, type_model: str) -> Transformer:
    """Rebuild the full bf16 model from a sharded engine checkpoint (every ``shard_*.pt`` holds its slice of the fp32 masters)."""
    from ..checkpoint import assemble_full_model

    return assemble_full_model(ckpt, name, type_model)


def main(argv: list[str] | None = None) -> None:
    ap = argparse.ArgumentParser(prog="python -m prime_b200.models.hf", description=__doc__.split("\n\n")[0])
    sub = ap.add_subparsers(dest="cmd", required=True)
    e = sub.add_parser("export", help="engine checkpoint (or reference-named .pt state dict) → HF directory")
    e.add_argument("--ckpt", required=True, help="checkpoint step directory written by the trainer, or a .pt state dict in reference naming")
    e.add_argument("--model", default="1B", help="model size name (configs of prime_b200.models.llama)")
    e.add_argument("--type-model", default="llama2", choices=["llama2", "llama3"])
    e.add_argument("--out", required=True)
    e.add_argument("--dtype", default="bfloat16", choices=["bfloat16", "float16", "float32"])
    i = sub.add_parser("import", help="HF directory → .pt state dict in reference naming (tok_embeddings / layers.N.attention.wq …)")
    i.add_argument("--hf", required=True)
    i.add_argument("--out", required=True)
    a = ap.parse_args(argv)
    if a.cmd == "export":
        if Path(a.ckpt).is_file():
            from .llama import build_model, from_reference_state_dict

            model = build_model(a.model, a.type_model, dtype=torch.float32, seed=None)
            from_reference_state_dict(model, torch.load(a.ckpt, map_location="cpu", weights_only=True))
        else:
            model = _model_from_engine_ckpt(a.ckpt, a.model, a.type_model)
        names = save_hf_dir(model, a.out, dtype=getattr(torch, a.dtype))
        print(json.dumps({"out": a.out, "files": ["config.json", *names], "params": model.num_params()}))
    else:
        from .llama import to_reference_state_dict

        model = load_hf_dir(a.hf, dtype=torch.float32)
        torch.save({k: v.clone() for k, v in to_reference_state_dict(model).items()}, a.out)
        print(json.dumps({"out": a.out, "params": model.num_params(), "args": model.args.__dict__}))


if __name__ == "__main__":
    main()
