"""parallel/layout.py: the shard layout of the sharded engine, pinned by a golden file, and the symmetric-heap size derived from it."""

import gzip
import json
from pathlib import Path

import pytest
import torch

from prime_b200.models.llama import Transformer, get_model_args
from prime_b200.parallel.fsdp import reduce_segments
from prime_b200.parallel.layout import SHARD_ALIGN, plan_layout

GOLDEN = json.loads(gzip.decompress((Path(__file__).parent / "golden" / "shard_layouts.json.gz").read_bytes()))
MODELS = sorted({(g["type_model"], g["name_model"]) for g in GOLDEN.values()})


def _meta_model(type_model, name):
    with torch.device("meta"):
        return Transformer(get_model_args(name, type_model))


def _configs(type_model, name):
    return [g for g in GOLDEN.values() if (g["type_model"], g["name_model"]) == (type_model, name)]


@pytest.mark.parametrize("type_model,name", MODELS)
def test_layout_reproduces_the_golden_file(type_model, name):
    """Buckets, parameter offsets, row pieces and totals, for F in {1, 2, 4, 8} replicated and {2, 4, 8} under ZeRO-3. A checkpoint
    records this layout, so any change here stops existing checkpoints from loading."""
    model = _meta_model(type_model, name)
    for g in _configs(type_model, name):
        lay = plan_layout(model, g["fsdp_size"], g["shard_params"])
        got = {
            "buckets": [
                {"name": b.name, "kind": b.kind, "start": b.start, "size": b.size, "shard_start": b.shard_start, "shard_size": b.shard_size,
                 "pstart": b.pstart, "params": [[qn, off] for qn, _, off in b.params], "pieces": [list(x) for x in b.pieces]}
                for b in lay.buckets
            ],
            "total": lay.total, "shard_total": lay.shard_total, "pflat_total": lay.pflat_total,
        }  # fmt: skip
        want = {k: g[k] for k in got}
        assert got == want, (type_model, name, g["fsdp_size"], g["shard_params"])


def _heap_used(g, fp32_master: bool) -> int:
    """Bytes taken from the symmetric heap by its control block, the engine and the outer step, replayed with the heap's
    1024-byte alignment from the golden totals (``SymmetricHeap.__init__``, ``ShardedEngine._allocate``, ``DilocoOuter``)."""
    sizes = [4096 * 4, 64 * 4, 64 * 4]  # flags, error words, norm slots
    sizes += [max(g["pflat_total"], 8) * 2, g["total"] * 4]  # bf16 param_flat, fp32 main_grad
    if g["shard_params"]:
        sizes.append(g["shard_total"] * 2)  # bf16 row shards
    if fp32_master:
        sizes.append(g["shard_total"] * 4)  # fp32 masters (the fused fp32 outer step allocates nothing else in the heap)
    else:
        sizes += [g["shard_total"], g["shard_total"] // SHARD_ALIGN * 4]  # int8 outer payload + fp32 block scales
    cursor = 0
    for n in sizes:
        cursor = (cursor + 1023) // 1024 * 1024 + n
    return cursor


@pytest.mark.parametrize("type_model,name", MODELS)
def test_heap_bytes_cover_every_allocation(type_model, name):
    model = _meta_model(type_model, name)
    for g in _configs(type_model, name):
        lay = plan_layout(model, g["fsdp_size"], g["shard_params"])
        for fp32_master in (False, True):
            spare = lay.heap_bytes(fp32_master=fp32_master) - _heap_used(g, fp32_master)
            assert spare >= 64e6, (type_model, name, g["fsdp_size"], g["shard_params"], fp32_master, spare)


@pytest.mark.parametrize("type_model,name", MODELS)
def test_reduce_segments_follow_the_layout(type_model, name):
    """The engine's gradient reduce-scatter tables, (offset in main_grad, offset in the shard, elements) per bucket: a flat bucket is
    rank r's contiguous 1/F slice (at F = 1 the whole bucket, reduced in place: its shard starts where it does), a row-sharded
    bucket is rank r's row block of every weight, in parameter order."""
    model = _meta_model(type_model, name)
    for g in _configs(type_model, name):
        F = g["fsdp_size"]
        lay = plan_layout(model, F, g["shard_params"])
        for r in sorted({0, F // 2, F - 1}):
            tables = reduce_segments(lay, r)
            assert len(tables) == len(lay.buckets)
            for b, t in zip(lay.buckets, tables):
                got = [(t.src_off[i], t.dst_off[i], t.n[i]) for i in range(t.nseg)]
                if b.kind == "flat":
                    want = [(b.start + r * b.shard_size, b.shard_start, b.shard_size)]
                    assert F > 1 or b.shard_start == b.start
                else:
                    want = [(b.start + off + r * (p.numel() // F), b.shard_start + soff, p.numel() // F)
                            for (_, p, off), (soff, _) in zip(b.params, b.pieces)]  # fmt: skip
                assert got == want, (type_model, name, F, g["shard_params"], r, b.name)
