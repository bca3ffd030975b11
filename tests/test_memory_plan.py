"""utils/memory_plan.py: the per-GPU HBM budget computed before anything is allocated (CPU-only arithmetic, so it is tested here)."""

import json
import logging
from types import SimpleNamespace

import pytest
import torch

from prime_b200.models.llama import Transformer, get_model_args
from prime_b200.parallel.layout import plan_layout
from prime_b200.utils import memory_plan as mp


@pytest.mark.parametrize("type_model,name", [("llama2", "debugmodel"), ("llama2", "150M"), ("llama2", "7B"), ("llama3", "7B"), ("llama2", "70B")])
def test_parameter_count_equals_the_models(type_model, name):
    a = get_model_args(name, type_model)
    with torch.device("meta"):
        model = Transformer(a)
    assert mp.count_params(a)["total"] == sum(p.numel() for p in model.parameters())


def test_headline_config_fits_and_70b_is_refused_with_the_reason():
    ok = mp.plan_memory(get_model_args("1B"), fsdp_size=2, micro_bs=16, seq_len=1024, diloco=True, name="llama2/1B")
    assert ok.verdict == "fits" and ok.total_bytes < 80e9
    mp.check(ok)  # no exception
    big = mp.plan_memory(get_model_args("70B"), fsdp_size=8, micro_bs=1, seq_len=4096, name="llama2/70B")
    assert big.verdict == "does_not_fit" and big.largest().name.startswith("fp32 main_grad")
    with pytest.raises(mp.MemoryPlanError) as e:
        mp.check(big)
    msg = str(e.value)
    assert "fp32 main_grad" in msg and "80 GB" in msg and "fsdp 8" in msg


def test_skip_switch_turns_the_refusal_into_a_warning(monkeypatch, caplog):
    monkeypatch.setenv("PB_SKIP_MEMORY_CHECK", "1")
    big = mp.plan_memory(get_model_args("70B"), fsdp_size=8)
    with caplog.at_level(logging.WARNING):
        mp.check(big, logging.getLogger("t"))
    assert "cannot fit" in caplog.text


def test_estimate_alone_only_warns(caplog):
    p = mp.plan_memory(get_model_args("7B"), fsdp_size=8, micro_bs=16, seq_len=4096)
    assert p.state_bytes < p.capacity < p.total_bytes and p.verdict == "tight"
    with caplog.at_level(logging.WARNING):
        mp.check(p, logging.getLogger("t"))
    assert "lower train.micro_bs" in caplog.text
    q = mp.plan_memory(get_model_args("7B"), fsdp_size=8, micro_bs=16, seq_len=4096, ac_ckpt=True)
    assert q.total_bytes < 0.5 * p.total_bytes  # checkpointing every block keeps one residual per layer


def test_zero3_rule_is_the_trainers():
    a = get_model_args("7B")
    assert "ZeRO-3" in mp.plan_memory(a, fsdp_size=8).describe
    assert "replicated" in mp.plan_memory(a, fsdp_size=1).describe  # nothing to shard over
    assert "replicated" in mp.plan_memory(a, fsdp_size=8, fused=False).describe  # the gather lives in the fused GEMMs
    assert "replicated" in mp.plan_memory(get_model_args("1B"), fsdp_size=8).describe  # below 5 B parameters
    z3, z1 = mp.plan_memory(a, fsdp_size=8, shard_params=True), mp.plan_memory(a, fsdp_size=8, shard_params=False)
    saved = z1.state_bytes - z3.state_bytes
    n = mp.count_params(a)["total"]
    assert 0.95 < saved / (2 * n * 7 / 8 - 2 * (mp.count_params(a)["layer_2d"] + mp.count_params(a)["head"])) < 1.05


def test_torch_side_rows_match_the_measured_1b_run():
    """`bench.py --gpus 1` on an H100 80GB HBM3 (llama2/1B, fsdp 1, replicated parameters, DiLoCo, micro_bs 16 × seq 1024): torch's
    max_memory_allocated was 42.02 GB (the symmetric heap is not in it). The plan must be at or a little above that, never below."""
    p = mp.plan_memory(get_model_args("1B"), fsdp_size=1, micro_bs=16, seq_len=1024, shard_params=False, diloco=True)
    torch_gb = sum(r.nbytes for r in p.rows if r.where == "torch") / 1e9
    assert 42.02 <= torch_gb <= 42.02 * 1.06


def test_heap_rows_equal_the_trainers_heap_sizing():
    """trainer.py sizes the symmetric heap with the shard layout's ``heap_bytes``: the plan's heap rows must add up to it."""
    for name, F, z3 in (("1B", 2, False), ("7B", 8, True)):
        a = get_model_args(name)
        with torch.device("meta"):
            model = Transformer(a)
        nbytes = plan_layout(model, F, z3).heap_bytes()
        plan = mp.plan_memory(a, fsdp_size=F, shard_params=z3)
        assert abs(plan.heap_bytes - nbytes) / nbytes < 0.005, (name, plan.heap_bytes, nbytes)


def test_trainer_hook_refuses_before_building_the_model():
    from prime_b200.config import Config
    from prime_b200.trainer import Trainer

    cfg = Config(name_model="debugmodel")
    mesh = SimpleNamespace(worker_id=0, fsdp_size=1, device=torch.device("cpu"), world=SimpleNamespace(rank=0, world_size=1))
    plan = Trainer._plan_memory(cfg, mesh, {"max_seq_len": 128}, capacity=int(80e9))
    assert plan is not None and plan.verdict == "fits"
    with pytest.raises(mp.MemoryPlanError):
        Trainer._plan_memory(cfg, mesh, {"max_seq_len": 128}, capacity=1 << 20)
    # a bug inside the planner must not stop a run: unknown override → logged, None
    assert Trainer._plan_memory(cfg, mesh, {"no_such_field": 1}, capacity=int(80e9)) is None


def test_cli(capsys):
    assert mp.main(["--model", "70B", "--fsdp", "8", "--json"]) == 1
    out = json.loads(capsys.readouterr().out)
    assert out["verdict"] == "does_not_fit" and out["largest_micro_bs"] == 0
    assert mp.main(["@configs/7B/fsdp_8.toml", "--world", "8"]) == 0
    text = capsys.readouterr().out
    assert "ZeRO-3" in text and "→ fits" in text
    assert mp.main(["--model", "7B", "--fsdp", "8", "--seq", "4096", "--json"]) == 0  # 13B state alone exceeds an 80 GB part at F = 8
    assert json.loads(capsys.readouterr().out)["largest_micro_bs"] >= 1
