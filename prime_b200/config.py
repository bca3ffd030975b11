"""Training configuration: pydantic schema, TOML loading and CLI overrides.

Surface follows the DiLoCo engine's public contract named in BASELINE.json
(``diloco.train @configs/1B/h100.toml --optim.lr 3e-4``): nested sections
``data / optim / train / ckpt / diloco / mesh``; unknown keys are rejected.

The merge order (CLI > TOML > defaults) and the ``extra="forbid"`` +
friendly-error pattern mirror the reference's job-config tier
(reference: packages/prime/src/prime_cli/utils/config.py:62-111 and
packages/prime/src/prime_cli/commands/rl.py:478-552) — re-implemented here,
not copied.
"""

from __future__ import annotations

import sys
import tomllib
from pathlib import Path
from typing import Any, Literal, Sequence

from pydantic import BaseModel, ConfigDict, Field, ValidationError, model_validator


class _Section(BaseModel):
    model_config = ConfigDict(extra="forbid", validate_assignment=True)


class DataConfig(_Section):
    seq_length: int = 1024
    fake: bool = True  # synthetic tokens (no network in the sandbox)
    dataset_name_or_paths: str = ""  # comma-separated token files (.bin / .npy), directories or globs (tools/tokenize_corpus.py writes them)
    token_dtype: Literal["auto", "uint16", "uint32"] = "auto"  # raw .bin files: auto = uint16 up to 65 536 vocabulary entries, else uint32
    shuffle: bool = True  # per-epoch permutation of the sequence windows (seeded by data.seed)
    # held-out corpus for the periodic validation loss (same formats as dataset_name_or_paths); with data.fake a second synthetic stream
    eval_dataset_name_or_paths: str = ""
    # document masking of packed windows: a token attends only to earlier tokens of its own document (documents end with EOS).
    # The EOS id is data.eos_id, or else the "eos_id" of the first shard's .meta.json (tools/tokenize_corpus.py writes it)
    document_mask: bool = False
    eos_id: int | None = None
    num_workers: int = 2
    seed: int = 1337
    pin_memory: bool = True


class AdamConfig(_Section):
    lr: float = 4e-4
    weight_decay: float = 0.1
    betas1: float = 0.9
    betas2: float = 0.95
    eps: float = 1e-8


class OptimConfig(_Section):
    optim: AdamConfig = Field(default_factory=AdamConfig)
    sched_type: Literal["cosine", "linear", "wsd-sqrt", "constant"] = "cosine"
    warmup_steps: int = 1000
    stable_steps: int = 80_000
    total_steps: int = 88_000
    batch_size: int = 512  # global sequences per optimizer step, per DiLoCo worker
    max_norm: float = 1.0
    # "delayed" (clip with the previous step's norm) is not offered: the fused norm exchange is already off the critical path
    clip_mode: Literal["exact", "none"] = "exact"


class TrainConfig(_Section):
    micro_bs: int = 16
    ac_ckpt: bool | int = False
    # ZeRO-3: bf16 parameters sharded 1/F, gathered from the peers INSIDE the consuming GEMMs (parallel/fsdp.py). None = automatic:
    # on for models of 5 B parameters and more when fsdp_size > 1, off below that (small models stay resident)
    reshard_after_forward: bool | None = None
    cuda_graphs: bool = False
    log_model_hash: bool = False
    attn_impl: Literal["auto", "native", "sdpa"] = "auto"
    fp8: bool = False
    fused_comm: bool = True  # P2P fused reduce-scatter/AdamW/all-gather kernels
    memory_profile: bool = False
    # start from existing weights instead of the random init: a Hugging Face Llama directory (config.json + safetensors) or a .pt
    # state dict in reference naming (models/hf.py, models/llama.py); every rank loads the same file, then training proceeds as usual
    init_weights: str | None = None
    eval_interval: int = 0  # validation loss every N optimizer steps (0 = never): forward only, mean over all ranks of the world
    eval_batches: int = 8  # micro-batches per rank and evaluation


class CkptConfig(_Section):
    path: str | None = None
    interval: int | None = None
    topk: int | None = None
    resume: str | None = None
    async_write: bool = True
    live_recovery: bool = True
    live_recovery_port: int = 0
    skip_dataloader: bool = False


class DilocoConfig(_Section):
    outer_lr: float = 0.7
    outer_momentum: float = 0.9
    nesterov: bool = True
    inner_steps: int = 100
    compression: Literal["no", "int8", "uint8"] = "int8"
    quant_block: int = 1024
    retry_all_reduce: int = 3
    # fall back to plain averaging of parameters when only one worker is alive
    skip_outer_when_alone: bool = False


class MeshConfig(_Section):
    """Two-level mesh on one NVSwitch box: ``workers × fsdp`` ranks."""

    fsdp_size: int = 0  # 0 → derive (world // num_workers)
    num_workers: int = 0  # 0 → derive (world // fsdp_size), default 1 worker
    elastic: bool = False  # worker groups launched separately, joined via global store
    heartbeat_interval_s: float = 2.0
    heartbeat_timeout_s: float = 20.0
    backend: Literal["auto", "nccl", "gloo"] = "auto"


class MonitorConfig(_Section):
    log_interval: int = 1
    jsonl_path: str | None = None
    prometheus_port: int | None = None
    wandb: bool = False
    clocks: bool = False


ModelName = Literal["debugmodel", "10M", "150M", "271M", "1B", "7B", "10B", "13B", "26B", "70B"]


class Config(_Section):
    name_model: ModelName = "150M"
    type_model: Literal["llama2", "llama3"] = "llama2"
    # sliding-window attention in every layer (as in Mistral): a query attends only its W most recent keys, itself included; it
    # composes with data.document_mask. Part of the model's definition, so checkpoints record it. None = full causal attention
    sliding_window: int | None = Field(default=None, ge=1)
    project: str = "prime_b200"
    run_id: str | None = None
    seed: int = 42
    data: DataConfig = Field(default_factory=DataConfig)
    optim: OptimConfig = Field(default_factory=OptimConfig)
    train: TrainConfig = Field(default_factory=TrainConfig)
    ckpt: CkptConfig = Field(default_factory=CkptConfig)
    diloco: DilocoConfig | None = None
    mesh: MeshConfig = Field(default_factory=MeshConfig)
    monitor: MonitorConfig = Field(default_factory=MonitorConfig)

    @model_validator(mode="after")
    def _check(self) -> "Config":
        if self.optim.batch_size % self.train.micro_bs != 0 and self.optim.batch_size > self.train.micro_bs:
            raise ValueError(
                f"optim.batch_size ({self.optim.batch_size}) must be a multiple of train.micro_bs ({self.train.micro_bs})"
            )
        if self.ckpt.interval is not None and self.diloco is not None:
            if self.ckpt.interval % self.diloco.inner_steps != 0:
                raise ValueError("ckpt.interval must be a multiple of diloco.inner_steps")
        return self


# --------------------------------------------------------------------------- #
# loading
# --------------------------------------------------------------------------- #


def _set_dotted(tree: dict[str, Any], dotted: str, value: Any) -> None:
    parts = dotted.split(".")
    node = tree
    for p in parts[:-1]:
        nxt = node.get(p)
        if not isinstance(nxt, dict):
            nxt = {}
            node[p] = nxt
        node = nxt
    node[parts[-1]] = value


def _coerce(raw: str) -> Any:
    low = raw.lower()
    if low in ("true", "false"):
        return low == "true"
    if low in ("none", "null"):
        return None
    for cast in (int, float):
        try:
            return cast(raw)
        except ValueError:
            pass
    return raw


def parse_cli(argv: Sequence[str]) -> tuple[list[Path], dict[str, Any]]:
    """Split ``@file.toml`` arguments from ``--a.b value`` / ``--a.b=value`` / ``--flag`` overrides."""
    files: list[Path] = []
    overrides: dict[str, Any] = {}
    i = 0
    argv = list(argv)
    while i < len(argv):
        tok = argv[i]
        if tok.startswith("@"):
            files.append(Path(tok[1:].strip() or argv[i + 1]))
            if tok == "@":
                i += 1
        elif tok.startswith("--"):
            key = tok[2:]
            if "=" in key:
                key, val = key.split("=", 1)
                _set_dotted(overrides, key.replace("-", "_"), _coerce(val))
            elif key.startswith("no-") or key.startswith("no_"):
                _set_dotted(overrides, key[3:].replace("-", "_"), False)
            elif i + 1 < len(argv) and not argv[i + 1].startswith("--") and not argv[i + 1].startswith("@"):
                _set_dotted(overrides, key.replace("-", "_"), _coerce(argv[i + 1]))
                i += 1
            else:
                _set_dotted(overrides, key.replace("-", "_"), True)
        else:
            raise SystemExit(f"unrecognised argument {tok!r} (use @file.toml or --section.key value)")
        i += 1
    return files, overrides


def deep_merge(base: dict[str, Any], over: dict[str, Any]) -> dict[str, Any]:
    out = dict(base)
    for k, v in over.items():
        if isinstance(v, dict) and isinstance(out.get(k), dict):
            out[k] = deep_merge(out[k], v)
        else:
            out[k] = v
    return out


def load_toml(path: Path) -> dict[str, Any]:
    try:
        with open(path, "rb") as f:
            return tomllib.load(f)
    except FileNotFoundError:
        raise SystemExit(f"config file not found: {path}")
    except tomllib.TOMLDecodeError as e:
        raise SystemExit(f"invalid TOML in {path}: {e}")


def format_validation_error(err: ValidationError) -> str:
    lines = ["invalid configuration:"]
    for e in err.errors():
        loc = ".".join(str(x) for x in e["loc"])
        lines.append(f"  {loc or '<root>'}: {e['msg']}")
    return "\n".join(lines)


def load_config(argv: Sequence[str] | None = None, *, base: dict[str, Any] | None = None) -> Config:
    files, overrides = parse_cli(sys.argv[1:] if argv is None else argv)
    tree: dict[str, Any] = dict(base or {})
    for f in files:
        tree = deep_merge(tree, load_toml(f))
    tree = deep_merge(tree, overrides)
    try:
        return Config.model_validate(tree)
    except ValidationError as e:
        raise SystemExit(format_validation_error(e))
