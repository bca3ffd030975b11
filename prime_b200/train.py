"""Training entrypoint: ``python -m prime_b200.train @configs/1B/h100.toml --optim.lr 3e-4`` (alias: ``python -m diloco.train``).

    torchrun --nproc-per-node 8 -m prime_b200.train @configs/1B/diloco_4x2.toml          # static mesh, one world
    GLOBAL_PORT=29400 GLOBAL_UNIQUE_ID=w0 torchrun --nproc-per-node 2 --master-port 29510 \
        -m prime_b200.train @configs/1B/elastic.toml                                       # one elastic worker (of many)

The loop: resume → [inner step]* with an outer DiLoCo step every H → periodic async sharded checkpoints → final
checkpoint on SIGTERM/SIGINT. In elastic mode the outer boundary first runs the membership rendezvous
(``parallel/elastic.py``): dead workers are dropped, joiners receive the live checkpoint from a survivor, and a failed
exchange is retried on the re-formed group (``diloco.retry_all_reduce`` times) before the worker falls back to a local
outer step.

The reference's nearest analogue of a train driver is the hosted-RL submit path — config merge, validation, submit, follow
logs (reference: packages/prime/src/prime_cli/commands/rl.py:608-900); BASELINE.json names this entrypoint's contract.
"""

from __future__ import annotations

import json
import signal
import sys
import time
from typing import Any, Sequence

import torch
import torch.distributed as dist

from .checkpoint import CheckpointManager, resolve_resume, restore_trainer, trainer_state
from .config import Config, load_config
from .trainer import Trainer
from .utils import JsonlSink, PrometheusSink, StepTimer, Throughput, get_logger


class _StopFlag:
    def __init__(self) -> None:
        self.set_by: str | None = None

    def install(self) -> None:
        for sig in (signal.SIGTERM, signal.SIGINT):
            try:
                signal.signal(sig, lambda s, _f: setattr(self, "set_by", signal.Signals(s).name))
            except ValueError:  # not the main thread (tests)
                pass


class _StopConsensus:
    """All ranks of a process world leave the loop at the SAME step: a signal sent to the whole process group reaches the ranks
    on different sides of a step boundary, and a rank that entered ``ckpt.save()`` (a barrier) while a peer started another
    ``inner_step`` (flag waits / collectives) would hang. One MAX all-reduce of a single int over a gloo side group — host
    memory only, no device sync — per step; single-rank worlds skip it."""

    def __init__(self, stop: _StopFlag):
        self.stop = stop
        self.group = None
        if dist.is_initialized() and dist.get_world_size() > 1:
            try:
                self.group = dist.new_group(backend="gloo")
            except Exception:  # noqa: BLE001 — no gloo in this build: fall back to the default group
                self.group = dist.group.WORLD

    def __call__(self) -> bool:
        mine = 1 if self.stop.set_by is not None else 0
        if self.group is None:
            return bool(mine)
        dev = "cpu" if dist.get_backend(self.group) == "gloo" else torch.device("cuda", torch.cuda.current_device())
        t = torch.tensor([mine], dtype=torch.int32, device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX, group=self.group)
        agreed = bool(int(t.item()))
        if agreed and self.stop.set_by is None:
            self.stop.set_by = "peer"
        return agreed


def _elastic_setup(cfg: Config, trainer: Trainer, log) -> Any:
    from .parallel.elastic import ElasticConfig, ElasticContext, display_name

    mesh = trainer.mesh
    backend = __import__("os").environ.get("PRIME_B200_ELASTIC_BACKEND") or ("nccl" if mesh.device.type == "cuda" else "gloo")
    ecfg = ElasticConfig(heartbeat_interval_s=cfg.mesh.heartbeat_interval_s, heartbeat_timeout_s=cfg.mesh.heartbeat_timeout_s,
                         min_workers=max(1, cfg.mesh.num_workers))  # fmt: skip
    ctx = ElasticContext.from_env(fsdp_rank=mesh.fsdp_rank, backend=backend, cfg=ecfg)
    eng, outer = trainer.engine, trainer.outer
    state = [eng.master, eng.exp_avg, eng.exp_avg_sq, outer.theta0, outer.momentum]
    retries = max(1, cfg.diloco.retry_all_reduce)
    xchg = None
    if eng.backend == "fused" and cfg.diloco.compression in ("int8", "uint8") and __import__("os").environ.get("PRIME_B200_ELASTIC_FUSED", "1") != "0":
        # fused outer step across the separately launched workers: cudaIpc exchange regions published through the global store
        from .parallel.elastic_exchange import ElasticExchange

        xchg = ElasticExchange(ctx.store, ctx.wid, mesh.fsdp_rank, eng.shard_total, mesh.device)
        outer.attach_exchange(xchg)
        trainer.heap.set_spin_timeout(max(2.0, min(20.0, cfg.mesh.heartbeat_timeout_s / 2)))  # a dead peer costs seconds, not 20
        ctx.exchange = xchg
        log.info("elastic: fused NVLink outer exchange (cudaIpc region of %.1f MiB per rank)", xchg.nbytes / 2**20)

    def meet() -> None:
        m = ctx.rendezvous()
        counters = {"trainer_step": trainer.step_count, "engine_step": eng.step_count, "outer_step": outer.outer_step_count}
        got = ctx.sync_state(state, counters)
        if got is not counters and got != counters:  # we were the joiner: adopt the survivor's clock
            trainer.step_count, eng.step_count, outer.outer_step_count = got["trainer_step"], got["engine_step"], got["outer_step"]
            eng.publish_params()
        outer.set_membership(list(range(m.size)), m.pg)
        if xchg is not None:
            xchg.connect(m.workers, m.epoch)
        trainer.global_workers = m.size
        for _, msg in ctx.events:
            log.info("elastic: %s", msg)
        ctx.events.clear()
        if m.changed:
            log.info("elastic: epoch %d members=%s", m.epoch, [display_name(w) for w in m.workers])

    def boundary() -> None:
        meet()

    # the exchange itself can still fail if a peer dies between the rendezvous and the collective: re-form and retry
    plain_step = outer.step

    def guarded_step() -> None:
        for attempt in range(retries):
            try:
                plain_step()
                return
            except Exception as e:  # noqa: BLE001  (gloo/NCCL raise RuntimeError / DistBackendError on a dead peer)
                log.warning("elastic: outer exchange failed (%s: %s); re-forming the group (attempt %d/%d)", type(e).__name__, str(e)[:120], attempt + 1, retries)
                meet()
        log.warning("elastic: giving up on the exchange; taking a local outer step")
        outer.set_membership([0], None)
        if xchg is not None:
            xchg.connect([ctx.wid], ctx.epoch)
        plain_step()

    outer.step = guarded_step  # type: ignore[method-assign]
    trainer.on_outer_boundary = boundary
    meet()  # cold start / late join: become a member (and receive the live checkpoint) before the first inner step
    m = ctx.membership
    if m is not None and m.source is not None and ctx.wid in m.joiners:
        # admitted at the survivors' outer boundary: they are about to exchange pseudo-gradients with us in the group, so take
        # part in that outer step now (our pseudo-gradient is the source's, cloned with the live checkpoint)
        guarded_step()
    return ctx


def train(cfg: Config, *, max_steps: int | None = None) -> dict[str, Any]:
    stop = _StopFlag()
    stop.install()
    trainer = Trainer(cfg)
    mesh = trainer.mesh
    worker = mesh.worker_id if not cfg.mesh.elastic else (__import__("os").environ.get("GLOBAL_UNIQUE_ID") or "w?")
    log = get_logger(worker, mesh.world.rank)
    leader = mesh.fsdp_rank == 0 and (cfg.mesh.elastic or mesh.worker_id == 0)
    n_params = sum(p.numel() for p in trainer.model.parameters())
    log.info("model %s/%s: %.1fM params | mesh %s%s | micro_bs %d × accum %d × seq %d | backend %s | attn %s",
             cfg.type_model, cfg.name_model, n_params / 1e6, mesh.describe(), " (elastic)" if cfg.mesh.elastic else "",
             trainer.micro_bs, trainer.accum, cfg.data.seq_length, trainer.engine.backend, cfg.train.attn_impl)  # fmt: skip

    ckpt: CheckpointManager | None = None
    if cfg.ckpt.path:
        root = cfg.ckpt.path if not cfg.mesh.elastic else f"{cfg.ckpt.path}/{worker}"
        ckpt = CheckpointManager(root, rank=mesh.world.rank, world_size=mesh.world.world_size, topk=cfg.ckpt.topk,
                                 async_write=cfg.ckpt.async_write, device=mesh.device)  # fmt: skip
    if cfg.ckpt.resume:
        src = resolve_resume(cfg.ckpt.resume, cfg.ckpt.path if not cfg.mesh.elastic else f"{cfg.ckpt.path}/{worker}")
        if src is None:
            log.info("resume=%s: no checkpoint found, starting fresh", cfg.ckpt.resume)
        else:
            mgr = ckpt or CheckpointManager(src.parent, rank=mesh.world.rank, world_size=mesh.world.world_size, device=mesh.device)
            tensors, extra, meta = mgr.load(src)
            restore_trainer(trainer, tensors, extra, skip_dataloader=cfg.ckpt.skip_dataloader)
            log.info("resumed from %s at step %d", src, trainer.step_count)

    elastic = _elastic_setup(cfg, trainer, log) if cfg.mesh.elastic and trainer.outer is not None else None

    n_gpus = mesh.world.world_size
    meter = Throughput(trainer.model.flops_per_token(cfg.data.seq_length), n_gpus)
    jsonl = JsonlSink(cfg.monitor.jsonl_path if leader else None)
    prom = PrometheusSink(cfg.monitor.prometheus_port if leader else None)
    clocks = None
    if cfg.monitor.clocks and mesh.device.type == "cuda":
        from .utils.clocks import ClockSampler

        clocks = ClockSampler(mesh.world.local_rank)
        clocks.start()

    total = cfg.optim.total_steps if max_steps is None else min(cfg.optim.total_steps, trainer.step_count + max_steps)
    meta = {"config": cfg.model_dump(), "mesh": mesh.describe(), "n_params": n_params}
    timer = StepTimer()
    step_delay = float(__import__("os").environ.get("PRIME_B200_STEP_DELAY_S", "0"))  # fault-injection aid for the elastic tests
    last: dict[str, Any] = {}
    cuda = mesh.device.type == "cuda"
    should_stop = _StopConsensus(stop)
    logged_at = trainer.step_count  # step of the previous log line: a line can come off the log_interval grid (outer step, last step)
    try:
        while trainer.step_count < total and not should_stop():
            r = trainer.inner_step()
            step = trainer.step_count
            if step_delay:
                time.sleep(step_delay)
            if step % cfg.monitor.log_interval == 0 or r.did_outer or step == total:
                loss = float(r.loss)  # the only device→host sync of the step
                trainer.check_health()  # a device-side peer wait timed out → raise here instead of training on a void step
                dt = timer.lap()
                n_steps, logged_at = max(1, step - logged_at), step
                # tokens of this worker-world only: MFU is per-GPU of THIS process world; global tok/s is scaled by membership
                meter.update(trainer.tokens_per_step * n_steps, dt)
                scale = trainer.global_workers if cfg.mesh.elastic else 1
                last = {"step": step, "loss": round(loss, 5), "lr": r.lr, "grad_norm": float(r.grad_norm) if r.grad_norm is not None else None,
                        "tokens_per_s": round(meter.tokens_per_s * scale, 1), "mfu": round(meter.mfu, 4), "step_s": round(dt / n_steps, 4),
                        "workers": trainer.global_workers, "outer": r.did_outer, "total_tokens": meter.total_tokens * scale}  # fmt: skip
                if r.did_outer and trainer.outer is not None:
                    last["outer_s"] = round(trainer.outer.last_seconds, 4)
                    last["outer_bytes"] = trainer.outer.last_bytes_on_wire
                if cfg.train.log_model_hash and r.did_outer:
                    last["param_hash"] = trainer.engine.param_hash()
                if cuda and cfg.train.memory_profile:
                    last["hbm_gb"] = round(torch.cuda.max_memory_allocated() / 2**30, 2)
                if leader:
                    log.info("step %d loss %.4f lr %.2e gnorm %s %.0f tok/s mfu %.3f%s", step, loss, r.lr,
                             f"{last['grad_norm']:.3f}" if last["grad_norm"] is not None else "-", last["tokens_per_s"], last["mfu"],
                             f" | outer {last['outer_s'] * 1e3:.1f} ms, {last['outer_bytes'] / 2**20:.1f} MiB on the wire" if r.did_outer else "")  # fmt: skip
                    jsonl.write({"time": time.time(), **last})
                    prom.write(last)
            if cfg.train.eval_interval and step % cfg.train.eval_interval == 0:
                t_eval = time.perf_counter()
                val = trainer.evaluate()  # ends in a device→host read, so the wall time below covers the whole pass
                timer.exclude(time.perf_counter() - t_eval)  # tokens/s and MFU of the next log line are training only
                last["val_loss"] = round(val, 5)
                if leader:
                    log.info("step %d validation loss %.4f (%d batches per rank)", step, val, cfg.train.eval_batches)
                    jsonl.write({"time": time.time(), "step": step, "val_loss": round(val, 5)})
            if ckpt is not None:
                ckpt.poll()  # publish an asynchronously written checkpoint as soon as every rank's shard is on disk
            if ckpt is not None and cfg.ckpt.interval and step % cfg.ckpt.interval == 0:
                trainer.check_health()
                tensors, extra = trainer_state(trainer)
                ckpt.save(step, tensors, extra, meta)
                if leader:
                    log.info("checkpoint step %d: snapshot %.1f ms (write continues in the background)", step, ckpt.last_snapshot_s * 1e3)
        if stop.set_by is not None:
            log.info("%s received: stopping at step %d", stop.set_by, trainer.step_count)
        if ckpt is not None and (stop.set_by is not None or (cfg.ckpt.interval and trainer.step_count % cfg.ckpt.interval != 0)):
            # synchronised final checkpoint so a restart resumes exactly here (only at an outer boundary is it DiLoCo-consistent;
            # mid-H checkpoints still restore this worker's own inner state exactly)
            trainer.check_health()
            tensors, extra = trainer_state(trainer)
            ckpt.save(trainer.step_count, tensors, extra, meta)
    finally:
        if ckpt is not None:
            ckpt.wait()
        if elastic is not None:
            elastic.close()
            if getattr(elastic, "exchange", None) is not None:
                torch.cuda.synchronize()
                elastic.exchange.close()
        if clocks is not None:
            last["clocks"] = clocks.finish()
        jsonl.close()
        trainer.close()
    return last


def main(argv: Sequence[str] | None = None) -> None:
    cfg = load_config(argv)
    summary = train(cfg)
    if int(__import__("os").environ.get("RANK", "0")) == 0:
        print(json.dumps({"final": summary}))
    if dist.is_initialized():
        dist.destroy_process_group()


if __name__ == "__main__":
    main(sys.argv[1:])
