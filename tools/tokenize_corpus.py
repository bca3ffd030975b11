#!/usr/bin/env python
"""Text corpus → token shards the trainer memory-maps (``data.dataset_name_or_paths``).

    python tools/tokenize_corpus.py --tokenizer /models/llama-2-7b --out data/c4 corpus/*.jsonl corpus/notes.txt
    python tools/tokenize_corpus.py --tokenizer bytes --out data/tiny README.md        # no tokenizer files needed
    python -m diloco.train @configs/1B/h100.toml --data.fake false --data.dataset_name_or_paths data/c4

Inputs: ``.txt`` (one document per file), ``.jsonl`` / ``.json`` lines with a ``--field`` (default ``text``) per document.
Tokenizers: a local Hugging Face tokenizer directory (``transformers.AutoTokenizer``), a SentencePiece ``.model`` file, or
``bytes`` (UTF-8 bytes + EOS = 256; vocabulary 257 — for smoke runs with ``--vocab_size``-overridden debug models).
Every document is followed by EOS; documents are concatenated and cut into shards of ``--shard-tokens`` tokens:
``shard_00000.bin`` (uint16 when the vocabulary fits, else uint32) + ``shard_00000.meta.json`` (dtype, vocab_size, n_tokens,
tokenizer) — the sidecar is what ``MemmapTokenDataset`` reads the dtype from.  There is no network in the build sandbox, so
nothing is downloaded: the tokenizer must be on disk.
"""

from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path
from typing import Callable, Iterator

import numpy as np


def load_tokenizer(spec: str) -> tuple[Callable[[str], list[int]], int, int, str]:
    """→ (encode, vocab_size, eos_id, description)."""
    if spec == "bytes":
        return (lambda t: list(t.encode("utf-8"))), 257, 256, "bytes"
    p = Path(spec)
    if p.is_file() and p.suffix == ".model":
        import sentencepiece as spm

        sp = spm.SentencePieceProcessor(model_file=str(p))
        eos = sp.eos_id() if sp.eos_id() >= 0 else sp.piece_to_id("</s>")
        return (lambda t: sp.encode(t)), sp.get_piece_size(), eos, f"sentencepiece:{p.name}"
    from transformers import AutoTokenizer

    tok = AutoTokenizer.from_pretrained(spec, local_files_only=True)
    eos = tok.eos_token_id if tok.eos_token_id is not None else tok.sep_token_id
    if eos is None:
        raise SystemExit(f"tokenizer {spec} defines no EOS token")
    return (lambda t: tok.encode(t, add_special_tokens=False)), len(tok), int(eos), f"hf:{spec}"


def documents(files: list[str], field: str) -> Iterator[str]:
    for f in files:
        p = Path(f)
        if p.suffix in (".jsonl", ".json"):
            with open(p, encoding="utf-8") as fh:
                for n, line in enumerate(fh, 1):
                    line = line.strip()
                    if not line:
                        continue
                    rec = json.loads(line)
                    if field not in rec:
                        raise SystemExit(f"{p}:{n}: no field {field!r}")
                    yield str(rec[field])
        else:
            yield p.read_text(encoding="utf-8", errors="replace")


def main(argv: list[str] | None = None) -> dict:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("inputs", nargs="+")
    ap.add_argument("--tokenizer", required=True, help="HF tokenizer directory, SentencePiece .model file, or 'bytes'")
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--field", default="text")
    ap.add_argument("--shard-tokens", type=int, default=1 << 27, help="tokens per shard (default 128 Mi)")
    a = ap.parse_args(argv)
    encode, vocab, eos, desc = load_tokenizer(a.tokenizer)
    dtype = np.uint16 if vocab <= 65536 else np.uint32
    out = Path(a.out)
    out.mkdir(parents=True, exist_ok=True)
    buf = np.empty(a.shard_tokens, dtype=dtype)
    fill = n_docs = n_tokens = 0
    shards: list[str] = []

    def flush() -> None:
        nonlocal fill
        if fill == 0:
            return
        name = f"shard_{len(shards):05d}"
        buf[:fill].tofile(out / f"{name}.bin")
        (out / f"{name}.meta.json").write_text(json.dumps({"dtype": np.dtype(dtype).name, "vocab_size": vocab, "n_tokens": fill,
                                                           "tokenizer": desc, "eos_id": eos}))  # fmt: skip
        shards.append(f"{name}.bin")
        fill = 0

    for doc in documents(a.inputs, a.field):
        ids = np.asarray(encode(doc) + [eos], dtype=np.int64)
        if ids.size and int(ids.max()) >= vocab:
            raise SystemExit(f"tokenizer produced id {int(ids.max())} ≥ vocabulary size {vocab}")
        n_docs += 1
        n_tokens += ids.size
        while ids.size:
            k = min(ids.size, a.shard_tokens - fill)
            buf[fill : fill + k] = ids[:k]
            fill += k
            ids = ids[k:]
            if fill == a.shard_tokens:
                flush()
    flush()
    summary = {"out": str(out), "shards": shards, "documents": n_docs, "tokens": n_tokens, "vocab_size": vocab, "dtype": np.dtype(dtype).name,
               "tokenizer": desc}  # fmt: skip
    (out / "dataset.json").write_text(json.dumps(summary, indent=1))
    print(json.dumps(summary))
    return summary


if __name__ == "__main__":
    sys.exit(0 if main() else 1)
