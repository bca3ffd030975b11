"""Data pipeline: synthetic token streams (the sandbox has no network) and memory-mapped token files.

Batches are produced on the host in *pinned* memory and copied host→device asynchronously on a side
stream, double-buffered, so the H2D copy of step i+1 overlaps the compute of step i.  The loader is
checkpointable (``state_dict``: RNG state / file cursor).
"""

from __future__ import annotations

from dataclasses import dataclass
from pathlib import Path

import numpy as np
import torch


@dataclass
class Batch:
    input_ids: torch.Tensor  # [B, S] int64
    labels: torch.Tensor  # [B, S] int64


class FakeTokenDataset:
    """Deterministic pseudo-random tokens with a learnable structure (next token depends on the previous
    one), so the loss measurably decreases in smoke tests."""

    def __init__(self, vocab_size: int, seq_len: int, seed: int = 0, rank: int = 0, world: int = 1):
        self.vocab_size, self.seq_len = vocab_size, seq_len
        self.rng = np.random.default_rng(seed * 10007 + rank)
        self.rank, self.world = rank, world
        self.n_served = 0

    def next_batch(self, batch_size: int) -> tuple[np.ndarray, np.ndarray]:
        V, S = self.vocab_size, self.seq_len
        start = self.rng.integers(0, V, size=(batch_size, 1), dtype=np.int64)
        steps = self.rng.integers(1, 4, size=(batch_size, S), dtype=np.int64)
        toks = (start + np.cumsum(steps, axis=1)) % V
        full = np.concatenate([start % V, toks], axis=1)
        self.n_served += batch_size
        return full[:, :-1], full[:, 1:]

    def state_dict(self) -> dict:
        return {"rng": self.rng.bit_generator.state, "n_served": self.n_served}

    def load_state_dict(self, sd: dict) -> None:
        self.rng.bit_generator.state = sd["rng"]
        self.n_served = sd["n_served"]


def _expand_paths(spec: str) -> list[Path]:
    """Comma-separated files, directories (every ``*.bin`` / ``*.npy`` inside, sorted) or glob patterns."""
    import glob

    out: list[Path] = []
    for part in (x.strip() for x in spec.split(",")):
        if not part:
            continue
        p = Path(part)
        if p.is_dir():
            found = sorted(f for f in p.iterdir() if f.suffix in (".bin", ".npy"))
        elif any(c in part for c in "*?["):
            found = sorted(Path(f) for f in glob.glob(part, recursive=True))
        else:
            found = [p]
        if not found:
            raise FileNotFoundError(f"dataset path {part!r} matches no token file")
        out += found
    if not out:
        raise ValueError("no dataset paths given")
    return out


def _open_tokens(f: Path, dtype) -> np.ndarray:
    if f.suffix == ".npy":
        a = np.load(f, mmap_mode="r")
        if a.ndim != 1 or a.dtype.kind not in "ui":
            raise ValueError(f"{f}: expected a 1-D integer token array, got {a.dtype} {a.shape}")
        return a
    meta = f.with_suffix(".meta.json")  # written by tools/tokenize_corpus.py next to every shard
    if meta.exists():
        import json

        dtype = np.dtype(json.loads(meta.read_text())["dtype"])
    if f.stat().st_size % np.dtype(dtype).itemsize:
        raise ValueError(f"{f}: {f.stat().st_size} bytes is not a whole number of {np.dtype(dtype).name} tokens — set data.token_dtype "
                         "(or keep the .meta.json that tools/tokenize_corpus.py wrote next to the shard)")  # fmt: skip
    return np.memmap(f, dtype=dtype, mode="r")


class MemmapTokenDataset:
    """Pre-tokenised corpus: flat token files (raw ``.bin`` of uint16 / uint32, or 1-D ``.npy``), cut into windows of
    ``seq_len + 1`` tokens (inputs and next-token labels).

    * every data rank reads a disjoint strided subset of the windows (sample k of rank r is window ``k·world + r`` of the epoch);
    * ``shuffle``: the window order of every epoch is an affine permutation ``(a·i + b) mod N`` with ``gcd(a, N) = 1`` derived
      from (seed, epoch) — a bijection evaluated in O(1), so a 100-billion-token corpus needs no index array and the position
      is one integer (``cursor``) in the checkpoint;
    * token ids are range-checked against the model's vocabulary on the way out (a uint16 file read as uint32, or a tokenizer
      that does not belong to the model, otherwise shows up as a device-side index fault in the embedding much later).
    """

    def __init__(self, paths: str, seq_len: int, rank: int = 0, world: int = 1, dtype=None, *, vocab_size: int | None = None,
                 shuffle: bool = True, seed: int = 0):  # fmt: skip
        if dtype is None:
            dtype = np.uint16 if (vocab_size or 0) <= 65536 else np.uint32
        self.files = _expand_paths(paths)
        self.arrays = [_open_tokens(f, dtype) for f in self.files]
        self.seq_len, self.rank, self.world = seq_len, rank, world
        self.vocab_size, self.shuffle, self.seed = vocab_size, shuffle, seed
        per_file = np.array([(len(a) - 1) // seq_len for a in self.arrays], dtype=np.int64)
        self.first_window = np.concatenate([[0], np.cumsum(per_file)])  # window index → file by searchsorted
        self.windows = int(self.first_window[-1])
        if self.windows < world:
            raise ValueError(f"dataset has {self.windows} windows of {seq_len} tokens — fewer than the {world} data ranks")
        self.cursor = 0  # samples drawn by THIS rank
        self._perm_epoch, self._perm = -1, (1, 0)

    # -------------------------------------------------------------- order
    def _affine(self, epoch: int) -> tuple[int, int]:
        if epoch != self._perm_epoch:
            import math

            rng = np.random.default_rng([self.seed, epoch])
            n = self.windows
            a = int(rng.integers(1, max(n, 2)))
            while math.gcd(a, n) != 1:
                a = a + 1 if a + 1 < n else 1
            self._perm_epoch, self._perm = epoch, (a, int(rng.integers(0, n)))
        return self._perm

    def _index(self, k: int) -> int:
        """Window of this rank's k-th sample."""
        g = k * self.world + self.rank
        epoch, i = divmod(g, self.windows)
        if not self.shuffle:
            return i
        a, b = self._affine(epoch)
        return (a * i + b) % self.windows

    def _window(self, idx: int) -> np.ndarray:
        f = int(np.searchsorted(self.first_window, idx, side="right")) - 1
        s = (idx - int(self.first_window[f])) * self.seq_len
        return np.asarray(self.arrays[f][s : s + self.seq_len + 1], dtype=np.int64)

    def next_batch(self, batch_size: int) -> tuple[np.ndarray, np.ndarray]:
        full = np.stack([self._window(self._index(self.cursor + j)) for j in range(batch_size)])
        self.cursor += batch_size
        if self.vocab_size is not None and int(full.max()) >= self.vocab_size:
            raise ValueError(f"token id {int(full.max())} ≥ vocab_size {self.vocab_size}: wrong tokenizer for this model, or the file's "
                             "dtype is not what data.token_dtype says")  # fmt: skip
        return full[:, :-1], full[:, 1:]

    @property
    def epoch(self) -> int:
        return (self.cursor * self.world) // self.windows

    def state_dict(self) -> dict:
        return {"cursor": self.cursor}

    def load_state_dict(self, sd: dict) -> None:
        self.cursor = int(sd["cursor"])


class PinnedPrefetcher:
    """Ring of ``depth`` pinned-host → device slots; the H2D copy of batch i+k overlaps the compute of batch i.

    Contract: a batch returned by :meth:`next` stays valid until the following ``next()`` call *returns* (the trainer
    enqueues every kernel that reads batch i before it asks for batch i+1).  Two hazards are fenced per slot:

    * host side — the pinned buffer of a slot is rewritten on the CPU only after the previous H2D copy out of it has
      finished (``copied[i].synchronize()``); otherwise a host that runs ahead of the GPU (CUDA graphs, log_interval > 1,
      ``read_loss=False`` benches) would let the pending DMA read a newer or torn batch;
    * device side — the copy into a device slot waits for the event recorded after the last consumer of that slot
      (``consumed[i]``), not for everything enqueued on the compute stream, so prefetch really runs ahead.
    """

    def __init__(self, dataset, batch_size: int, device: torch.device, depth: int = 4):
        self.ds, self.bs, self.device = dataset, batch_size, device
        self.cuda = device.type == "cuda"
        S = dataset.seq_len
        self.depth = max(2, depth)
        self.host = [torch.empty((2, batch_size, S), dtype=torch.int64, pin_memory=self.cuda) for _ in range(self.depth)]
        if self.cuda:
            self.dev = [torch.empty((2, batch_size, S), dtype=torch.int64, device=device) for _ in range(self.depth)]
            self.stream = torch.cuda.Stream(device=device)
            self.copied = [torch.cuda.Event() for _ in range(self.depth)]  # H2D out of host[i] / into dev[i] finished
            self.consumed = [torch.cuda.Event() for _ in range(self.depth)]  # every kernel reading dev[i] was enqueued before this
            self._copied_armed = [False] * self.depth
            self._consumed_armed = [False] * self.depth
        self.slot = 0
        self._handed: int | None = None  # slot currently owned by the consumer
        self.h2d_bytes_per_batch = 2 * batch_size * S * 8
        self.host_waits = 0  # times the CPU had to wait for an in-flight DMA before reusing a pinned slot (diagnostic)
        self._inflight: list[int] = []
        self._states: list[dict] = []  # dataset state BEFORE each in-flight batch was drawn (checkpoint = oldest one)
        for _ in range(self.depth - 1):
            self._issue()

    def state_dict(self) -> dict:
        """Position of the next batch the *consumer* will see (prefetched-but-unconsumed batches are replayed on resume)."""
        import copy

        return copy.deepcopy(self._states[0]) if self._states else self.ds.state_dict()

    def load_state_dict(self, sd: dict) -> None:
        self.ds.load_state_dict(sd)
        self.reset()

    def _issue(self) -> None:
        i = self.slot
        import copy

        self._states.append(copy.deepcopy(self.ds.state_dict()))
        x, y = self.ds.next_batch(self.bs)
        if self.cuda and self._copied_armed[i]:
            if not self.copied[i].query():
                self.host_waits += 1
            self.copied[i].synchronize()  # the DMA that last read host[i] is done: safe to rewrite it on the CPU
        self.host[i][0].copy_(torch.from_numpy(np.ascontiguousarray(x)))
        self.host[i][1].copy_(torch.from_numpy(np.ascontiguousarray(y)))
        if self.cuda:
            if self._consumed_armed[i]:
                self.stream.wait_event(self.consumed[i])  # the last consumer of dev[i] is done before we overwrite it
            with torch.cuda.stream(self.stream):
                self.dev[i].copy_(self.host[i], non_blocking=True)
                self.copied[i].record(self.stream)
            self._copied_armed[i] = True
        self._inflight.append(i)
        self.slot = (self.slot + 1) % self.depth

    def _release_handed(self) -> None:
        if self.cuda and self._handed is not None:
            self.consumed[self._handed].record(torch.cuda.current_stream())
            self._consumed_armed[self._handed] = True
        self._handed = None

    def reset(self) -> None:
        """Drop prefetched batches (they were drawn before a dataset ``load_state_dict``) and refill the pipeline."""
        if self.cuda:
            torch.cuda.current_stream().synchronize()
            self.stream.synchronize()
            self._copied_armed = [False] * self.depth
            self._consumed_armed = [False] * self.depth
        self._handed = None
        self._inflight.clear()
        self._states.clear()
        self.slot = 0
        for _ in range(self.depth - 1):
            self._issue()

    def next(self) -> Batch:
        self._release_handed()  # the batch handed out last time has been fully enqueued by now
        self._issue()
        i = self._inflight.pop(0)
        self._states.pop(0)
        if self.cuda:
            torch.cuda.current_stream().wait_event(self.copied[i])
            t = self.dev[i]
            self._handed = i
        else:
            t = self.host[i].clone()
        return Batch(t[0], t[1])


def eos_id_from_meta(paths: str) -> int | None:
    """EOS id recorded in the ``.meta.json`` sidecar of the first token file of ``paths`` (None without a sidecar or an id)."""
    import json

    meta = _expand_paths(paths)[0].with_suffix(".meta.json")
    if not meta.exists():
        return None
    eos = json.loads(meta.read_text()).get("eos_id")
    return None if eos is None else int(eos)


def document_eos_id(cfg_data) -> int | None:
    """EOS id for document masking (``data.document_mask``): ``data.eos_id``, else the first shard's sidecar; None when masking is
    off. Raises ``ValueError`` when masking is on and no EOS id can be found."""
    if not cfg_data.document_mask:
        return None
    if cfg_data.eos_id is not None:
        return int(cfg_data.eos_id)
    if cfg_data.fake or not cfg_data.dataset_name_or_paths:
        raise ValueError("data.document_mask=true with synthetic data needs an explicit data.eos_id")
    eos = eos_id_from_meta(cfg_data.dataset_name_or_paths)
    if eos is None:
        raise ValueError(f"data.document_mask=true: no eos_id in the .meta.json of the first shard of {cfg_data.dataset_name_or_paths!r} "
                         "(tools/tokenize_corpus.py writes it); set data.eos_id")  # fmt: skip
    return eos


def build_dataset(cfg_data, vocab_size: int, rank: int, world: int):
    if cfg_data.fake or not cfg_data.dataset_name_or_paths:
        return FakeTokenDataset(vocab_size, cfg_data.seq_length, cfg_data.seed, rank, world)
    dt = {"auto": None, "uint16": np.uint16, "uint32": np.uint32}[getattr(cfg_data, "token_dtype", "auto")]
    return MemmapTokenDataset(cfg_data.dataset_name_or_paths, cfg_data.seq_length, rank, world, dt, vocab_size=vocab_size,
                              shuffle=getattr(cfg_data, "shuffle", True), seed=cfg_data.seed)  # fmt: skip
