"""Sharded checkpointing: every rank writes ONLY its 1/F optimizer shard, asynchronously, with an atomic publish.

Layout::

    <ckpt.path>/step_000200/            ← appears atomically (rename of ``.tmp-step_000200``)
        meta.json                       ← written last by rank 0: config, mesh, step counters, shard table
        rank_00003.pbck                 ← JSON header + raw little-endian tensor bytes (no pickle → safe to load)
    <ckpt.path>/latest                  ← text file naming the newest complete step (written after the rename)

Write path (``save``): the shard (master + m + v + θ₀ + momentum = 20 B/param/F) is first cloned on the device at HBM
speed (≈7 ms for a whole 1B model; the device has the room), so training resumes immediately; the clone drains to
reusable pinned host buffers on a side stream (PCIe 5, ≈0.4 s for 22 GB, overlapped with the next steps), a writer thread
streams the pinned buffers to disk and fsyncs, then ranks meet on a barrier and rank 0 publishes by rename.

Resume (``load``): ``ckpt.resume = <dir> | "latest"``; the shard table is validated against the live engine
(bucket layout, fsdp size) before any tensor is copied; the data loader position and RNG state come back too.

This is the training-side analogue of the reference's only "checkpoint-like" pipelines — the resumable chunked upload of
``prime env push`` (reference: packages/prime/src/prime_cli/commands/env.py:1150-1340) and hosted-RL checkpoint listing
(reference: packages/prime/src/prime_cli/api/rl.py:316-340); BASELINE.json's DiLoCo contract requires the real thing.
"""

from __future__ import annotations

import json
import os
import shutil
import struct
import threading
import time
from dataclasses import dataclass
from pathlib import Path
from typing import Any

import numpy as np
import torch
import torch.distributed as dist

from .parallel.layout import plan_layout, use_zero3

MAGIC = b"PBCK0001"
_NP = {torch.float32: np.float32, torch.int8: np.int8, torch.int64: np.int64, torch.uint8: np.uint8, torch.float16: np.float16,
       torch.int32: np.int32, torch.bfloat16: np.uint16}  # fmt: skip
_DT = {str(k).replace("torch.", ""): k for k in _NP}


def step_dir(root: Path, step: int) -> Path:
    return Path(root) / f"step_{step:06d}"


def list_steps(root: Path) -> list[int]:
    out = []
    for p in Path(root).glob("step_*"):
        if p.is_dir() and (p / "meta.json").exists():
            try:
                out.append(int(p.name.split("_", 1)[1]))
            except ValueError:
                pass
    return sorted(out)


def resolve_resume(spec: str, root: str | None) -> Path | None:
    """``"latest"`` → newest complete step under ``root``; otherwise a path to a step directory (or a root holding steps)."""
    if spec == "latest":
        if root is None:
            return None
        steps = list_steps(Path(root))
        return step_dir(Path(root), steps[-1]) if steps else None
    p = Path(spec)
    if (p / "meta.json").exists():
        return p
    steps = list_steps(p)
    if steps:
        return step_dir(p, steps[-1])
    raise FileNotFoundError(f"no complete checkpoint at {spec}")


# ------------------------------------------------------------------------------------------------- shard file format
def write_shard(path: Path, tensors: dict[str, torch.Tensor], extra: dict[str, Any]) -> int:
    """Header (JSON: name → dtype/shape/offset/nbytes, plus ``extra``) then 64-byte-aligned raw tensor bytes. Returns bytes written."""
    table, off = {}, 0
    for name, t in tensors.items():
        nbytes = t.numel() * t.element_size()
        table[name] = {"dtype": str(t.dtype).replace("torch.", ""), "shape": list(t.shape), "offset": off, "nbytes": nbytes}
        off += (nbytes + 63) & ~63
    header = json.dumps({"tensors": table, "extra": extra}).encode()
    pad = (-(len(MAGIC) + 8 + len(header))) % 64
    with open(path, "wb") as f:
        f.write(MAGIC)
        f.write(struct.pack("<Q", len(header) + pad))
        f.write(header + b" " * pad)
        base = f.tell()
        for name, t in tensors.items():
            f.seek(base + table[name]["offset"])
            if t.numel():
                f.write(memoryview(t.contiguous().view(-1).view(torch.uint8).numpy()))
        f.truncate(base + off)
        f.flush()
        os.fsync(f.fileno())
        return base + off


def read_shard(path: Path, device: torch.device | str = "cpu") -> tuple[dict[str, torch.Tensor], dict[str, Any]]:
    with open(path, "rb") as f:
        if f.read(8) != MAGIC:
            raise ValueError(f"{path} is not a prime_b200 checkpoint shard")
        (hlen,) = struct.unpack("<Q", f.read(8))
        header = json.loads(f.read(hlen))
        base = f.tell()
    mm = np.memmap(path, dtype=np.uint8, mode="r", offset=base) if any(d["nbytes"] for d in header["tensors"].values()) else None
    out = {}
    for name, d in header["tensors"].items():
        dt = _DT[d["dtype"]]
        if d["nbytes"] == 0:
            out[name] = torch.empty(d["shape"], dtype=dt, device=device)
            continue
        raw = torch.from_numpy(np.array(mm[d["offset"] : d["offset"] + d["nbytes"]]))  # copy out of the mapping
        out[name] = raw.view(dt).reshape(d["shape"]).to(device)
    return out, header["extra"]


# ------------------------------------------------------------------------------------------------- manager
@dataclass
class SaveHandle:
    step: int
    thread: threading.Thread | None
    error: list[BaseException]

    def wait(self) -> None:
        if self.thread is not None:
            self.thread.join()
        if self.error:
            raise RuntimeError(f"checkpoint step {self.step} failed") from self.error[0]


class CheckpointManager:
    def __init__(self, root: str | Path, *, rank: int, world_size: int, topk: int | None = None, async_write: bool = True,
                 device: torch.device | None = None):  # fmt: skip
        self.root = Path(root)
        self.rank, self.world = rank, world_size
        self.topk, self.async_write = topk, async_write
        self.device = device or torch.device("cpu")
        self.cuda = self.device.type == "cuda"
        self._pending: SaveHandle | None = None
        self._pinned: dict[str, torch.Tensor] = {}
        self._stream = torch.cuda.Stream(device=self.device) if self.cuda else None
        self._snap_done = torch.cuda.Event() if self.cuda else None
        self.last_snapshot_s = 0.0
        self.last_write_s = 0.0
        self.last_bytes = 0
        self._pending_meta: dict[str, Any] = {}
        # host-side (gloo) group for the status exchange of asynchronous checkpoints: polling must not touch the device
        self._side = None
        if world_size > 1 and dist.is_initialized():
            try:
                self._side = dist.new_group(backend="gloo")
            except Exception:  # noqa: BLE001
                self._side = None
        if rank == 0:
            self.root.mkdir(parents=True, exist_ok=True)

    # -- snapshot: device clone at HBM speed on the training stream, then clone → pinned host on a side stream
    def _snapshot(self, tensors: dict[str, torch.Tensor]) -> dict[str, torch.Tensor]:
        t0 = time.perf_counter()
        host: dict[str, torch.Tensor] = {}
        if not self.cuda:
            host = {k: v.detach().clone() for k, v in tensors.items()}
        else:
            staged = {k: v.detach().clone() for k, v in tensors.items()}  # training may now overwrite the originals
            self._stream.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(self._stream):
                for k, v in staged.items():
                    if not v.is_cuda:  # host-side state (RNG): already a private copy
                        host[k] = v
                        continue
                    buf = self._pinned.get(k)
                    if buf is None or buf.shape != v.shape or buf.dtype != v.dtype:
                        buf = torch.empty(v.shape, dtype=v.dtype, pin_memory=True)
                        self._pinned[k] = buf
                    buf.copy_(v, non_blocking=True)
                    v.record_stream(self._stream)  # the caching allocator may reuse the clone only after the D2H
                    host[k] = buf
                self._snap_done.record(self._stream)
        self.last_snapshot_s = time.perf_counter() - t0
        return host

    def _barrier(self) -> None:
        if dist.is_initialized() and self.world > 1:
            dist.barrier()

    def _publish(self, step: int, meta: dict[str, Any]) -> None:
        tmp, final = self.root / f".tmp-step_{step:06d}", step_dir(self.root, step)
        (tmp / "meta.json").write_text(json.dumps(meta, indent=1))
        if final.exists():
            shutil.rmtree(final)
        os.replace(tmp, final)
        latest = self.root / ".latest.tmp"
        latest.write_text(final.name)
        os.replace(latest, self.root / "latest")
        if self.topk:
            for old in list_steps(self.root)[: -self.topk]:
                shutil.rmtree(step_dir(self.root, old), ignore_errors=True)

    def save(self, step: int, tensors: dict[str, torch.Tensor], extra: dict[str, Any], meta: dict[str, Any]) -> SaveHandle:
        """Snapshot now, write in the background. ``tensors`` = this rank's shard; ``meta`` = job-level description (rank 0)."""
        self.wait()  # one checkpoint in flight: the pinned buffers are reused
        tmp = self.root / f".tmp-step_{step:06d}"
        if self.rank == 0:
            if tmp.exists():
                shutil.rmtree(tmp)
            tmp.mkdir(parents=True)
        self._barrier()
        host = self._snapshot(tensors)
        handle = SaveHandle(step, None, [])

        def work() -> None:
            try:
                t0 = time.perf_counter()
                if self.cuda:
                    self._snap_done.synchronize()
                self.last_bytes = write_shard(tmp / f"rank_{self.rank:05d}.pbck", host, extra)
                self.last_write_s = time.perf_counter() - t0
            except BaseException as e:  # surfaced by wait()
                handle.error.append(e)

        if self.async_write and self.world == 1:
            # single-rank jobs can publish from the writer thread; multi-rank publish needs a collective → done in wait()
            def work_and_publish() -> None:
                work()
                if not handle.error:
                    try:
                        self._publish(step, {**meta, "step": step, "world_size": self.world})
                    except BaseException as e:
                        handle.error.append(e)

            handle.thread = threading.Thread(target=work_and_publish, name=f"ckpt-{step}", daemon=True)
            handle.thread.start()
            self._pending = handle
            return handle
        if self.async_write:
            handle.thread = threading.Thread(target=work, name=f"ckpt-{step}", daemon=True)
            handle.thread.start()
            self._pending = handle
            self._pending_meta = {**meta, "step": step, "world_size": self.world}
            return handle
        work()
        handle.wait()
        self._barrier()
        if self.rank == 0:
            self._publish(step, {**meta, "step": step, "world_size": self.world})
        self._barrier()
        return handle

    def _status(self, done: bool, failed: bool) -> tuple[bool, bool]:
        """(every rank done, any rank failed) — one tiny all-reduce; on the gloo side group when there is one."""
        if self.world == 1 or not dist.is_initialized():
            return done, failed
        dev = "cpu" if self._side is not None else self.device
        t = torch.tensor([0 if done else 1, 1 if failed else 0], dtype=torch.int32, device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX, group=self._side)
        return int(t[0]) == 0, int(t[1]) == 1

    def _finish(self, h: SaveHandle, failed: bool) -> None:
        self._pending = None
        if failed:  # every rank raises together: nobody is left waiting in a barrier
            cause = h.error[0] if h.error else None
            raise RuntimeError(f"checkpoint step {h.step} failed on {'this rank' if h.error else 'another rank'}") from cause
        publish_error: BaseException | None = None
        if self.rank == 0:
            try:
                self._publish(h.step, self._pending_meta)
            except BaseException as e:  # disk full, directory removed under us, …: tell the others instead of leaving them in a barrier
                publish_error = e
        # doubles as the barrier that used to follow the publish: nobody returns before rank 0 has renamed the directory (or failed to)
        _, failed = self._status(True, publish_error is not None)
        if failed:
            raise RuntimeError(f"checkpoint step {h.step}: every shard was written but rank 0 could not publish the directory") from publish_error

    def poll(self) -> bool:
        """Call once per training step on every rank: publishes the asynchronously written checkpoint as soon as ALL shards are on
        disk (instead of at the next ``save``/exit, which left the newest checkpoint invisible to resume for a whole interval).
        Never blocks on the writer thread. Returns True when a checkpoint was published by this call."""
        h = self._pending
        if h is None or self.world == 1:
            return False
        mine_done = h.thread is None or not h.thread.is_alive()
        done, failed = self._status(mine_done, bool(h.error) and mine_done)
        if failed or done:
            if h.thread is not None:
                h.thread.join()
            self._finish(h, failed)
            return not failed
        return False

    def wait(self) -> None:
        """Finish the in-flight checkpoint (called before the next save, before exit, and by tests)."""
        h = self._pending
        if h is None:
            return
        if h.thread is not None:
            h.thread.join()
        if self.world == 1:
            self._pending = None
            h.wait()
            return
        _, failed = self._status(True, bool(h.error))  # exchange error status BEFORE anybody raises or enters the barrier
        self._finish(h, failed)

    def load(self, path: Path) -> tuple[dict[str, torch.Tensor], dict[str, Any], dict[str, Any]]:
        meta = json.loads((Path(path) / "meta.json").read_text())
        if meta.get("world_size") != self.world:
            raise ValueError(f"checkpoint {path} was written by {meta.get('world_size')} ranks; this job has {self.world} "
                             "— restart with the same mesh, or rewrite it offline: python -m prime_b200.checkpoint reshard --src <step dir> --out <new step dir> "
                             "--model <size> --fsdp-size <F>")  # fmt: skip
        tensors, extra = read_shard(Path(path) / f"rank_{self.rank:05d}.pbck", self.device)
        return tensors, extra, meta


# ------------------------------------------------------------------------------------------------- trainer glue
def trainer_state(trainer) -> tuple[dict[str, torch.Tensor], dict[str, Any]]:
    eng, outer = trainer.engine, trainer.outer
    tensors = {"master": eng.master, "exp_avg": eng.exp_avg, "exp_avg_sq": eng.exp_avg_sq}
    extra: dict[str, Any] = {
        "trainer_step": trainer.step_count, "engine_step": eng.step_count, "fsdp_size": eng.F, "fsdp_rank": eng.mesh.fsdp_rank,
        "layout": eng.layout.signature,
        "data": trainer.loader.state_dict(),
        "shard_params": bool(getattr(eng, "shard_params", False)),
    }  # fmt: skip
    tensors["rng_cpu"] = torch.get_rng_state()
    if eng.device.type == "cuda":
        tensors["rng_cuda"] = torch.cuda.get_rng_state(eng.device)
    if outer is not None:
        tensors.update(theta0=outer.theta0, momentum=outer.momentum)
        extra["outer_step"] = outer.outer_step_count
    return tensors, extra


def restore_trainer(trainer, tensors: dict[str, torch.Tensor], extra: dict[str, Any], *, skip_dataloader: bool = False) -> None:
    eng, outer = trainer.engine, trainer.outer
    eng.layout.check_saved(extra["layout"], extra["fsdp_size"], extra.get("shard_params", False))
    with torch.no_grad():
        eng.master.copy_(tensors["master"])
        eng.exp_avg.copy_(tensors["exp_avg"])
        eng.exp_avg_sq.copy_(tensors["exp_avg_sq"])
        eng.step_count = int(extra["engine_step"])
        if outer is not None and "theta0" in tensors:
            outer.theta0.copy_(tensors["theta0"])
            outer.momentum.copy_(tensors["momentum"])
            outer.outer_step_count = int(extra.get("outer_step", 0))
        elif outer is not None:
            # the run was saved without [diloco] and is resumed with it: the outer parameters start at the LOADED weights (not at
            # the constructor's random init, whose pseudo-gradient would wipe out the checkpoint at the first outer step)
            outer.theta0.copy_(eng.master)
            outer.momentum.zero_()
            outer.outer_step_count = 0
        eng.publish_params()
        if "rng_cpu" in tensors:
            torch.set_rng_state(tensors["rng_cpu"].cpu())
        if "rng_cuda" in tensors and eng.device.type == "cuda":
            torch.cuda.set_rng_state(tensors["rng_cuda"].cpu(), eng.device)
    trainer.step_count = int(extra["trainer_step"])
    if not skip_dataloader and extra.get("data") is not None:  # None: a rank added by an offline reshard starts its own stream
        trainer.loader.load_state_dict(extra["data"])


# ------------------------------------------------------------------------------------------------- offline assembly / resharding
SHARDED_KINDS = ("master", "exp_avg", "exp_avg_sq", "theta0", "momentum")  # per-rank 1/F slices of parameter-shaped state


def _read_all_ranks(d: Path) -> tuple[dict, list[tuple[dict[str, torch.Tensor], dict[str, Any]]]]:
    meta = json.loads((d / "meta.json").read_text())
    return meta, [read_shard(d / f"rank_{r:05d}.pbck", "cpu") for r in range(int(meta["world_size"]))]


def assemble_full_model(path: str | Path, name_model: str, type_model: str = "llama2", *, dtype: torch.dtype = torch.float32, **overrides):
    """Rebuild the complete model on the CPU from a published checkpoint step directory: every ``rank_*.pbck`` holds its rank's
    1/F slice of the fp32 master weights, cut either as contiguous bucket slices (replicated-parameter mode) or as one row block
    per weight (ZeRO-3). The layout is recomputed with the engine's own planner (``parallel/layout.py``).
    Used by ``python -m prime_b200.models.hf export`` and ``examples/inspect_checkpoint.py``; DiLoCo workers are identical after
    an outer step, the first worker's shards are taken. The sliding window is taken from the run's recorded config (the bucket
    layout does not depend on it), so a windowed model is never rebuilt with full attention."""
    from .models.llama import build_model

    d = Path(path)
    meta = json.loads((d / "meta.json").read_text())
    overrides.setdefault("sliding_window", (meta.get("config") or {}).get("sliding_window"))
    shards: dict[int, torch.Tensor] = {}
    extra0: dict[str, Any] | None = None
    for r in range(int(meta["world_size"])):
        tensors, extra = read_shard(d / f"rank_{r:05d}.pbck", "cpu")
        fr = int(extra["fsdp_rank"])
        if fr not in shards:
            shards[fr] = tensors["master"].float()
            extra0 = extra0 or extra
        if len(shards) == int(extra["fsdp_size"]):
            break
    assert extra0 is not None
    F = int(extra0["fsdp_size"])
    if sorted(shards) != list(range(F)):
        raise ValueError(f"checkpoint {d} is incomplete: have fsdp ranks {sorted(shards)} of {F}")
    model = build_model(name_model, type_model, dtype=dtype, seed=None, **overrides)
    layout = plan_layout(model, F, bool(extra0.get("shard_params", False)))
    if not layout.matches(extra0["layout"]):
        raise ValueError(f"checkpoint {d} was written for a different model than {type_model}/{name_model} (bucket layout differs)")
    full = layout.gather(shards)
    with torch.no_grad():
        for qn, p in model.named_parameters():
            p.copy_(full[qn])
    return model


def reshard_checkpoint(src: str | Path, dst: str | Path, name_model: str, type_model: str = "llama2", *, fsdp_size: int,
                       shard_params: bool | None = None, **overrides) -> dict[str, Any]:  # fmt: skip
    """Rewrite a published checkpoint for a different FSDP group size and / or parameter mode, offline on the CPU.

    Every worker's optimizer state (fp32 masters, AdamW moments, and the outer θ₀ / momentum) is gathered into whole parameters with
    the source layout and cut again with the target layout — replicated ↔ ZeRO-3 and any F that divides the weights' row counts.
    The number of DiLoCo workers is kept (each worker keeps ITS moments). Counters, LR position and RNG state are carried over from
    the worker's first rank; the data position of every new rank is the furthest any old rank of that worker had read (no sample is
    repeated; with a different rank count the streams are re-striped, so bit-exact continuation of the loss curve is not expected
    — the optimizer state is).  → {"world_size", "fsdp_size", "workers", "bytes"}; resume with ``--mesh.fsdp_size <new F>``."""
    from .models.llama import build_model

    src, dst = Path(src), Path(dst)
    meta, ranks = _read_all_ranks(src)
    F0 = int(ranks[0][1]["fsdp_size"])
    world0 = len(ranks)
    if world0 % F0:
        raise ValueError(f"{src}: {world0} rank files do not divide into groups of fsdp_size={F0}")
    workers = world0 // F0
    sp0 = bool(ranks[0][1].get("shard_params", False))
    sp1 = use_zero3(sp0 if shard_params is None else shard_params, fused=True, fsdp_size=int(fsdp_size))
    model = build_model(name_model, type_model, device="meta", dtype=torch.float32, seed=None, **overrides)  # shapes only
    plan0, plan1 = plan_layout(model, F0, sp0), plan_layout(model, fsdp_size, sp1)
    if not plan0.matches(ranks[0][1]["layout"]):
        raise ValueError(f"checkpoint {src} was written for a different model than {type_model}/{name_model} (bucket layout differs)")
    tmp = dst.parent / f".tmp-{dst.name}"
    if tmp.exists():
        shutil.rmtree(tmp)
    tmp.mkdir(parents=True)
    written = 0
    for w in range(workers):
        group = ranks[w * F0 : (w + 1) * F0]
        if sorted(int(e["fsdp_rank"]) for _, e in group) != list(range(F0)):
            raise ValueError(f"{src}: ranks {w * F0}..{(w + 1) * F0 - 1} are not one FSDP group (rank = worker·F + fsdp_rank expected)")
        by_rank = {int(e["fsdp_rank"]): t for t, e in group}
        first_t, first_e = group[0]
        kinds = [k for k in SHARDED_KINDS if k in first_t]
        whole = {k: plan0.gather({r: by_rank[r][k].float() for r in range(F0)}) for k in kinds}
        data_states = [e.get("data") for _, e in group]
        furthest = max((d.get("cursor", d.get("n_served", 0)) for d in data_states if isinstance(d, dict)), default=None)
        for r in range(fsdp_size):
            tensors = {k: plan1.scatter(whole[k], r) for k in kinds}
            for k, v in first_t.items():  # RNG state and anything else that is not parameter-shaped: the worker's first rank's
                if k not in tensors:
                    tensors[k] = v
            # data position: an old rank keeps its own stream state; a rank that did not exist before starts a fresh stream (synthetic
            # data: seeded by its rank) or, for a corpus, at the furthest position any old rank of the worker had reached
            data = data_states[r] if r < F0 else None
            if isinstance(data_states[0], dict) and "cursor" in data_states[0]:
                data = {**data_states[0], "cursor": furthest}
            extra = {**first_e, "fsdp_size": int(fsdp_size), "fsdp_rank": r, "layout": plan1.signature, "shard_params": sp1, "data": data,
                     "resharded_from": {"fsdp_size": F0, "shard_params": sp0, "path": str(src)}}  # fmt: skip
            written += write_shard(tmp / f"rank_{w * fsdp_size + r:05d}.pbck", tensors, extra)
    new_meta = {**meta, "world_size": workers * fsdp_size, "mesh": f"dl{workers}xfsdp{fsdp_size}",
                "resharded_from": {"world_size": world0, "mesh": meta.get("mesh")}}  # fmt: skip
    (tmp / "meta.json").write_text(json.dumps(new_meta, indent=1))
    if dst.exists():
        shutil.rmtree(dst)
    os.replace(tmp, dst)
    (dst.parent / "latest").write_text(dst.name)
    return {"world_size": workers * fsdp_size, "fsdp_size": int(fsdp_size), "workers": workers, "bytes": written, "shard_params": sp1}


def main(argv: list[str] | None = None) -> None:
    import argparse

    ap = argparse.ArgumentParser(prog="python -m prime_b200.checkpoint", description="Offline checkpoint tools")
    sub = ap.add_subparsers(dest="cmd", required=True)
    r = sub.add_parser("reshard", help="rewrite a checkpoint for another fsdp_size / parameter mode")
    r.add_argument("--src", required=True, help="published step directory (…/step_000500)")
    r.add_argument("--out", required=True, help="new step directory (its parent becomes a ckpt.path to resume from)")
    r.add_argument("--model", required=True)
    r.add_argument("--type-model", default="llama2", choices=["llama2", "llama3"])
    r.add_argument("--fsdp-size", type=int, required=True)
    r.add_argument("--shard-params", choices=["keep", "true", "false"], default="keep", help="ZeRO-3 row shards (train.reshard_after_forward) in the output")
    a = ap.parse_args(argv)
    sp = None if a.shard_params == "keep" else a.shard_params == "true"
    print(json.dumps(reshard_checkpoint(a.src, a.out, a.model, a.type_model, fsdp_size=a.fsdp_size, shard_params=sp)))


if __name__ == "__main__":
    main()
