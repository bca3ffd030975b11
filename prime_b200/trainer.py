"""Trainer: the public training API (``Trainer(cfg).step()``) behind ``diloco.train`` and ``bench.py``.

One *inner step* = ``accum`` micro-batches of forward/backward (gradients accumulate in fp32 in the
GEMM epilogues) → bucketed gradient reduce-scatter → clip → partitioned AdamW → parameter all-gather.
Every ``diloco.inner_steps`` inner steps the outer optimizer runs (int8 pseudo-gradient all-reduce
across workers ⊕ Nesterov).
"""

from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import torch
import torch.distributed as dist

from .config import Config
from .data import Batch, PinnedPrefetcher, build_dataset, document_eos_id
from .models.llama import Transformer, build_model
from .optim.schedule import lr_at
from .parallel.diloco import DilocoOuter, OuterHyper
from .parallel.fsdp import AdamHyper, ShardedEngine
from .parallel.layout import plan_layout, use_zero3
from .parallel.mesh import Mesh, WorldInfo, build_mesh, init_distributed


@dataclass
class StepResult:
    loss: torch.Tensor  # device scalar, mean over micro-batches of this rank
    lr: float
    grad_norm: torch.Tensor | None
    tokens: int  # tokens consumed by the WHOLE job in this step
    did_outer: bool


class Trainer:
    def __init__(self, cfg: Config, *, mesh: Mesh | None = None, model_overrides: dict | None = None):
        self.cfg = cfg
        if mesh is None:
            world = init_distributed(cfg.mesh.backend) if (_env_world() > 1 or dist.is_initialized()) else WorldInfo.from_env()
            if torch.cuda.is_available():
                torch.cuda.set_device(world.device_index)
            if cfg.mesh.elastic:  # this process world IS one worker; other workers are reached through the elastic coordinator
                mesh = build_mesh(world, 1, world.world_size)
            else:
                mesh = build_mesh(world, cfg.mesh.num_workers, cfg.mesh.fsdp_size)
        self.mesh = mesh
        self.device = mesh.device
        cuda = self.device.type == "cuda"
        torch.manual_seed(cfg.seed)
        dtype = torch.bfloat16 if cuda else torch.float32
        doc_eos_id = document_eos_id(cfg.data)  # before any allocation: a missing EOS id is a configuration error
        overrides = dict(model_overrides or {})
        overrides.setdefault("max_seq_len", max(cfg.data.seq_length, 128))
        overrides.setdefault("sliding_window", cfg.sliding_window)
        self.memory_plan = self._plan_memory(cfg, mesh, overrides) if cuda else None  # refuse what cannot fit BEFORE allocating
        # identical init on every rank (same seed) — workers start from the same θ₀
        self.model: Transformer = build_model(cfg.name_model, cfg.type_model, device=self.device, dtype=dtype, seed=cfg.seed, **overrides)
        if cfg.train.init_weights:
            load_initial_weights(self.model, cfg.train.init_weights)  # before the engine takes the parameters into its buffers
        self.model.attn_impl = cfg.train.attn_impl
        # document masking: the bounds kernel reads the token buffer inside the forward, so a captured micro-step stays valid
        self.model.doc_eos_id = doc_eos_id
        self.model.ac_ckpt = cfg.train.ac_ckpt
        self.model.set_fp8(cfg.train.fp8)  # MXFP8 forward / dgrad GEMMs (opt-in; the headline benchmark is bf16)
        self.heap = None
        use_fused = cuda and cfg.train.fused_comm
        shard_params = use_zero3(cfg.train.reshard_after_forward, fused=use_fused, fsdp_size=mesh.fsdp_size,
                                 n_params=sum(p.numel() for p in self.model.parameters()))
        if cfg.train.reshard_after_forward and not shard_params:
            raise ValueError("train.reshard_after_forward=true needs CUDA, train.fused_comm=true and mesh.fsdp_size > 1 "
                             "(the parameter gather runs inside the GEMM kernels over the symmetric NVLink heap)")  # fmt: skip
        if shard_params and cfg.train.fp8:
            raise ValueError("train.fp8 and train.reshard_after_forward cannot be combined yet (the MXFP8 GEMM has no gather variant)")
        fp32_outer = cfg.diloco is not None and cfg.diloco.compression == "no" and use_fused and not cfg.mesh.elastic
        if use_fused:
            from .parallel.symm import SymmetricHeap, dist_exchange

            nbytes = plan_layout(self.model, mesh.fsdp_size, shard_params).heap_bytes(fp32_master=fp32_outer)
            heap_cls = SymmetricHeap
            if _want_nvls() and mesh.world.world_size > 1:
                from .parallel.multicast import MulticastHeap, nvls_available

                if not nvls_available(self.device.index or 0):
                    raise RuntimeError("PB_NVLS=1 but this device cannot join an NVSwitch multicast object")
                heap_cls = MulticastHeap  # VMM + multicast mapping: the gradient reduce-scatter is summed inside the switch
            self.heap = heap_cls(nbytes, mesh.world.rank, mesh.world.world_size, dist_exchange(), self.device)

        o = cfg.optim
        hyper = AdamHyper(o.optim.lr, o.optim.betas1, o.optim.betas2, o.optim.eps, o.optim.weight_decay,
                          o.max_norm if o.clip_mode != "none" else 0.0)  # fmt: skip
        self.engine = ShardedEngine(self.model, mesh, hyper, backend="fused" if use_fused else "collective", heap=self.heap,
                                    shard_params=shard_params, master_in_heap=fp32_outer, fresh_grads=not cfg.train.cuda_graphs)  # fmt: skip
        self.outer: DilocoOuter | None = None
        if cfg.diloco is not None:
            d = cfg.diloco
            comp = "int8" if d.compression in ("int8", "uint8") else "no"
            self.outer = DilocoOuter(self.engine, OuterHyper(d.outer_lr, d.outer_momentum, d.nesterov, comp), collective=cfg.mesh.elastic)
        self.on_outer_boundary = None  # callable run right before every outer step (elastic rendezvous lives here)
        self.global_workers = mesh.num_workers  # elastic: updated by the coordinator at every boundary
        self.data_rank, self.data_world = mesh.world.rank, mesh.world.world_size

        # batch plan: optim.batch_size sequences per worker per step
        per_rank = max(1, o.batch_size // mesh.fsdp_size)
        self.micro_bs = min(cfg.train.micro_bs, per_rank)
        self.accum = max(1, per_rank // self.micro_bs)
        self.tokens_per_step = self.micro_bs * self.accum * cfg.data.seq_length * mesh.world.world_size
        effective = self.micro_bs * self.accum * mesh.fsdp_size
        if effective != o.batch_size:
            import warnings

            warnings.warn(f"optim.batch_size={o.batch_size} is not a multiple of fsdp_size × micro_bs = {mesh.fsdp_size} × {self.micro_bs}: "
                          f"every worker steps on {effective} sequences", stacklevel=2)  # fmt: skip
        if cfg.mesh.elastic:  # no global rank exists: derive a stable, distinct data stream from the worker's name
            import os
            import zlib

            name = os.environ.get("GLOBAL_UNIQUE_ID") or os.environ.get("GLOBAL_RANK") or "w0"
            self.data_rank = (zlib.crc32(name.encode()) % 65536) * mesh.fsdp_size + mesh.fsdp_rank
            self.data_world = 65536 * mesh.fsdp_size
        self.dataset = build_dataset(cfg.data, self.model.args.vocab_size, self.data_rank, self.data_world)
        self.loader = PinnedPrefetcher(self.dataset, self.micro_bs, self.device)
        self.step_count = 0
        self._loss_acc = torch.zeros((), dtype=torch.float32, device=self.device)
        self._graph = None
        self._graph_launches = 0
        if cfg.train.cuda_graphs and cuda:
            self._capture_micro_step()

    # ------------------------------------------------------------------ CUDA graph of one micro-step
    def _capture_micro_step(self) -> None:
        """Capture fwd + bwd (+ stray-grad fold) of one micro-batch into a CUDA graph.

        ~2.3k kernel launches per optimizer step become `accum` graph launches; gradients accumulate into the
        static fp32 main_grad buffers from inside the graph; bucket reduction then runs after the replay.
        """
        from . import ops

        eng, S = self.engine, self.cfg.data.seq_length
        self._g_tokens = torch.zeros((self.micro_bs, S), dtype=torch.int64, device=self.device)
        self._g_labels = torch.zeros((self.micro_bs, S), dtype=torch.int64, device=self.device)
        eng.capture_mode = True
        scale = 1.0 / self.accum

        def micro() -> torch.Tensor:
            ops.reset_gather_cache()  # ZeRO-3: a captured micro-step gathers every weight itself, whatever ran before it
            loss = self.model.loss(self._g_tokens, self._g_labels, grad_scale=scale, loss_acc=self._loss_acc)
            loss.backward()
            eng.fold_micro_grads()
            return loss.detach()

        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):  # warm-up outside capture: binds contexts, fills the tensor-map cache, sizes pools
            for _ in range(2):
                micro()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        eng.zero_grad()
        self._graph = torch.cuda.CUDAGraph()
        n0 = ops.launch_count()
        with torch.cuda.graph(self._graph):
            self._g_loss = micro()
        self._graph_launches = ops.launch_count() - n0
        eng.zero_grad()

    # ------------------------------------------------------------------ one optimizer step
    def current_lr(self) -> float:
        o = self.cfg.optim
        return lr_at(self.step_count, base_lr=o.optim.lr, sched_type=o.sched_type, warmup_steps=o.warmup_steps,
                     total_steps=o.total_steps, stable_steps=o.stable_steps)  # fmt: skip

    def inner_step(self, batches: list[Batch] | None = None) -> StepResult:
        eng = self.engine
        if eng.trace is not None:
            eng.trace.begin_step()
        eng.zero_grad()
        self._loss_acc.zero_()
        for i in range(self.accum):
            batch = batches[i] if batches is not None else self.loader.next()
            last = i == self.accum - 1
            eng.set_micro_step(last)
            if self._graph is not None:
                self._g_tokens.copy_(batch.input_ids, non_blocking=True)
                self._g_labels.copy_(batch.labels, non_blocking=True)
                self._graph.replay()
                _count_launches(self._graph_launches)
                if eng.shard_params:
                    from . import ops as _ops

                    _ops.reset_gather_cache()
                loss = self._g_loss
                if last:
                    eng.finish_backward()
            else:
                loss = self.model.loss(batch.input_ids, batch.labels, grad_scale=1.0 / self.accum, loss_acc=self._loss_acc)
                loss.backward()
                if last:
                    eng.finish_backward()
                else:
                    eng.fold_micro_grads()
        lr = self.current_lr()
        eng.step(lr)
        self.step_count += 1
        did_outer = False
        if self.outer is not None and self.step_count % self.cfg.diloco.inner_steps == 0:
            if self.on_outer_boundary is not None:
                self.on_outer_boundary()
            self.outer.step()
            did_outer = True
        tokens = self.tokens_per_step * (self.global_workers if self.cfg.mesh.elastic else 1)
        return StepResult(self._loss_acc / self.accum, lr, eng.last_grad_norm, tokens, did_outer)

    # ------------------------------------------------------------------ memory budget
    @staticmethod
    def _plan_memory(cfg: Config, mesh: Mesh, overrides: dict, capacity: int | None = None):
        """Per-GPU HBM budget of this configuration (``utils/memory_plan.py``). Raises ``MemoryPlanError`` when model + optimizer state
        alone exceed the device — every rank computes the same numbers, so all of them refuse together instead of one dying in
        ``cudaMalloc`` while its peers wait in the heap handle exchange. Anything else that goes wrong in here is logged, not fatal."""
        from .utils import memory_plan as mp
        from .utils.logging import get_logger

        log = get_logger(mesh.worker_id, mesh.world.rank)
        try:
            if capacity is None:
                capacity = int(torch.cuda.get_device_properties(mesh.device).total_memory)
            plan = mp.plan_from_config(cfg, mesh.world.world_size, capacity=capacity, fsdp_size=mesh.fsdp_size,
                                       model_overrides={k: v for k, v in overrides.items() if k != "max_seq_len"})  # fmt: skip
        except Exception as e:  # noqa: BLE001 — the plan is advice; never let a bug in it stop a run that would have fitted
            log.warning("memory plan skipped: %s", e)
            return None
        mp.check(plan, log)
        return plan

    # ------------------------------------------------------------------ validation
    @torch.no_grad()
    def evaluate(self, batches: int | None = None) -> float:
        """Mean next-token loss over ``batches`` micro-batches per rank of the held-out stream (``data.eval_dataset_name_or_paths``; with
        synthetic data a second stream with its own seed), averaged over the ranks of this process world. Forward only, through the
        same model and kernels as training; the evaluation stream restarts at the same position every time, so values are comparable."""
        import torch.distributed as dist

        from .data import FakeTokenDataset, MemmapTokenDataset

        cfg, V = self.cfg, self.model.args.vocab_size
        if cfg.data.eval_dataset_name_or_paths and not cfg.data.fake:
            ds = MemmapTokenDataset(cfg.data.eval_dataset_name_or_paths, cfg.data.seq_length, self.data_rank % max(1, self.mesh.world.world_size),
                                    self.mesh.world.world_size, vocab_size=V, shuffle=False)  # fmt: skip
        else:
            ds = FakeTokenDataset(V, cfg.data.seq_length, cfg.data.seed + 7919, self.data_rank, self.data_world)
        was_training = self.model.training
        self.model.eval()
        total = torch.zeros(2, dtype=torch.float64, device=self.device)
        for _ in range(batches or cfg.train.eval_batches):
            x, y = ds.next_batch(self.micro_bs)
            tok, tgt = torch.from_numpy(np.ascontiguousarray(x)).to(self.device), torch.from_numpy(np.ascontiguousarray(y)).to(self.device)
            logits = self.model(tok)
            total[0] += torch.nn.functional.cross_entropy(logits.float().reshape(-1, logits.shape[-1]), tgt.reshape(-1), reduction="sum").double()
            total[1] += tgt.numel()
        if dist.is_initialized() and self.mesh.world.world_size > 1:
            dist.all_reduce(total)
        self.model.train(was_training)
        return float(total[0] / total[1].clamp(min=1))

    # ------------------------------------------------------------------ helpers
    def check_health(self) -> None:
        """Raise if a device-side peer wait timed out (a rank stalled or died): the kernels then skipped their stores, so the
        step is void and nothing may be checkpointed. Synchronises; call it where the loop already does (log / outer / ckpt)."""
        if self.heap is not None:
            self.heap.check_errors()

    def flops_per_step(self) -> float:
        return self.model.flops_per_token(self.cfg.data.seq_length) * self.tokens_per_step

    def close(self) -> None:
        if self.heap is not None:
            torch.cuda.synchronize()
            self.heap.close()
            self.heap = None


def load_initial_weights(model: Transformer, source: str) -> None:
    """``train.init_weights``: copy pretrained weights into ``model`` (any device / dtype). A directory is read as a Hugging Face
    Llama checkpoint (RoPE row permutation and fused QKV / gate-up handled by ``models/hf.py``), a file as a state dict in reference
    naming. The architecture must be the one the config names — a mismatch is an error, not a partial load."""
    from pathlib import Path

    src = Path(source)
    if src.is_dir():
        from .models import hf

        cfg, sd = hf.read_hf_dir(src)
        want, have = hf.args_from_hf_config(cfg), model.args
        for f in ("dim", "n_layers", "n_heads", "vocab_size"):
            if getattr(want, f) != getattr(have, f):
                raise ValueError(f"train.init_weights: {src} has {f}={getattr(want, f)}, the configured model has {getattr(have, f)}")
        if want.kv_heads != have.kv_heads or want.ffn_hidden != have.ffn_hidden:
            raise ValueError(f"train.init_weights: {src} has kv_heads={want.kv_heads}, ffn={want.ffn_hidden}; the configured model has "
                             f"kv_heads={have.kv_heads}, ffn={have.ffn_hidden}")  # fmt: skip
        hf.load_hf_state_dict(model, sd)
    elif src.is_file():
        from .models.llama import from_reference_state_dict

        from_reference_state_dict(model, torch.load(src, map_location="cpu", weights_only=True))
    else:
        raise FileNotFoundError(f"train.init_weights: {source} is neither a Hugging Face checkpoint directory nor a state-dict file")


def _count_launches(n: int) -> None:
    from .ops.functional import _count

    _count(n)


def _want_nvls() -> bool:
    import os

    return os.environ.get("PB_NVLS", "0") == "1"


def _env_world() -> int:
    import os

    return int(os.environ.get("WORLD_SIZE", "1"))
