"""Training entrypoint on CPU: checkpoint shard format, atomic publish + top-k, bit-exact resume, and a real elastic run
(three independently launched workers over gloo; one is SIGKILLed, a fourth joins and receives the live checkpoint)."""

import json
import os
import signal
import subprocess
import sys
import time
from pathlib import Path

import pytest
import torch

from prime_b200 import checkpoint as ck
from prime_b200.config import load_config
from prime_b200.train import train

ROOT = Path(__file__).resolve().parents[1]
BASE = ["--name_model", "debugmodel", "--data.seq_length", "32", "--optim.batch_size", "4", "--train.micro_bs", "2",
        "--optim.warmup_steps", "2", "--optim.total_steps", "8", "--diloco.inner_steps", "4"]  # fmt: skip


def test_shard_roundtrip_all_dtypes(tmp_path):
    t = {"f32": torch.randn(1000), "bf16": torch.randn(7, 9).bfloat16(), "i8": torch.randint(-128, 127, (333,), dtype=torch.int8),
         "i64": torch.arange(5), "empty": torch.zeros(0)}  # fmt: skip
    n = ck.write_shard(tmp_path / "s.pbck", t, {"k": [1, 2], "nested": {"a": "b"}})
    assert n == (tmp_path / "s.pbck").stat().st_size
    back, extra = ck.read_shard(tmp_path / "s.pbck")
    assert extra == {"k": [1, 2], "nested": {"a": "b"}} and set(back) == set(t)
    for k in t:
        assert back[k].dtype == t[k].dtype and back[k].shape == t[k].shape and torch.equal(back[k], t[k])
    (tmp_path / "junk").write_bytes(b"not a checkpoint")
    with pytest.raises(ValueError):
        ck.read_shard(tmp_path / "junk")


def test_publish_is_atomic_and_topk_prunes(tmp_path):
    m = ck.CheckpointManager(tmp_path, rank=0, world_size=1, topk=2, async_write=True)
    for step in (4, 8, 12):
        h = m.save(step, {"x": torch.full((10,), float(step))}, {"s": step}, {"note": "t"})
        h.wait()
    assert ck.list_steps(tmp_path) == [8, 12] and (tmp_path / "latest").read_text() == "step_000012"
    assert not list(tmp_path.glob(".tmp-*"))
    # a crashed writer leaves only a .tmp dir, which is never mistaken for a checkpoint
    (tmp_path / ".tmp-step_000016").mkdir()
    (tmp_path / "step_000020").mkdir()  # no meta.json → incomplete
    assert ck.resolve_resume("latest", str(tmp_path)) == tmp_path / "step_000012"
    t, extra, meta = m.load(tmp_path / "step_000012")
    assert t["x"][0] == 12 and extra == {"s": 12} and meta["step"] == 12 and meta["note"] == "t"
    with pytest.raises(ValueError):
        ck.CheckpointManager(tmp_path, rank=0, world_size=2).load(tmp_path / "step_000012")
    assert ck.resolve_resume("latest", str(tmp_path / "nothing")) is None
    with pytest.raises(FileNotFoundError):
        ck.resolve_resume(str(tmp_path / "nothing"), None)


def _losses(jsonl: Path) -> dict[int, float]:
    return {r["step"]: r["loss"] for r in map(json.loads, jsonl.read_text().splitlines())}


def test_resume_is_bit_exact(tmp_path):
    a, b = tmp_path / "a", tmp_path / "b"
    train(load_config(BASE + ["--monitor.jsonl_path", str(a / "log.jsonl")]))
    straight = _losses(a / "log.jsonl")
    train(load_config(BASE + ["--ckpt.path", str(b), "--ckpt.interval", "4", "--monitor.jsonl_path", str(b / "log1.jsonl")]), max_steps=4)
    assert ck.list_steps(b) == [4]
    out = train(load_config(BASE + ["--ckpt.path", str(b), "--ckpt.interval", "4", "--ckpt.resume", "latest", "--monitor.jsonl_path", str(b / "log2.jsonl")]))
    resumed = {**_losses(b / "log1.jsonl"), **_losses(b / "log2.jsonl")}
    assert out["step"] == 8 and sorted(resumed) == list(range(1, 9))
    assert resumed == straight  # optimizer shards, outer state, LR schedule position and data stream all came back
    assert ck.list_steps(b) == [4, 8]


def test_sigterm_writes_a_final_checkpoint(tmp_path):
    cmd = [sys.executable, "-m", "prime_b200.train", *BASE, "--optim.total_steps", "100000", "--ckpt.path", str(tmp_path / "c"), "--ckpt.interval", "1000"]
    logf = tmp_path / "train.log"
    with open(logf, "w") as lf:
        p = subprocess.Popen(cmd, cwd=ROOT, env={**os.environ, "PYTHONPATH": str(ROOT)}, stdout=lf, stderr=subprocess.STDOUT)
        try:
            deadline = time.time() + 120
            while time.time() < deadline and "step 3 " not in logf.read_text():
                time.sleep(0.1)
            p.send_signal(signal.SIGTERM)
            assert p.wait(timeout=60) == 0, logf.read_text()
        finally:
            if p.poll() is None:  # never leave a 100000-step job behind
                p.kill()
    log, err = logf.read_text(), ""
    steps = ck.list_steps(tmp_path / "c")
    assert len(steps) == 1 and steps[0] >= 3 and "SIGTERM received" in log + err


WORKER = """
import os, sys
sys.path.insert(0, {root!r})
from prime_b200.config import load_config
from prime_b200.train import train
cfg = load_config({argv!r})
print("FINAL", train(cfg), flush=True)
"""


@pytest.mark.slow
def test_elastic_drop_and_join_end_to_end(tmp_path):
    from prime_b200.parallel import elastic as el

    served = el.serve(0)
    argv = ["--name_model", "debugmodel", "--data.seq_length", "32", "--optim.batch_size", "2", "--train.micro_bs", "2", "--optim.warmup_steps", "2",
            "--optim.total_steps", "60", "--diloco.inner_steps", "4", "--mesh.elastic", "true", "--mesh.num_workers", "3",
            "--mesh.heartbeat_interval_s", "0.1", "--mesh.heartbeat_timeout_s", "1.5", "--train.log_model_hash", "true"]  # fmt: skip

    def launch(name, extra=()):
        env = {**os.environ, "PYTHONPATH": str(ROOT), "GLOBAL_ADDR": "127.0.0.1", "GLOBAL_PORT": str(served.port), "GLOBAL_UNIQUE_ID": name,
               "PRIME_B200_STEP_DELAY_S": "0.3"}  # fmt: skip
        log = open(tmp_path / f"{name}.log", "w")
        return subprocess.Popen([sys.executable, "-c", WORKER.format(root=str(ROOT), argv=argv + ["--monitor.jsonl_path", str(tmp_path / f"{name}.jsonl"), *extra])],
                                cwd=ROOT, env=env, stdout=log, stderr=subprocess.STDOUT)  # fmt: skip

    def wait_for(path, needle, timeout=120):
        t0 = time.time()
        while time.time() - t0 < timeout:
            if path.exists() and needle in path.read_text():
                return
            time.sleep(0.1)
        raise AssertionError(f"{needle!r} never appeared in {path.name}:\n{path.read_text() if path.exists() else ''}")

    procs = {n: launch(n) for n in ("w0", "w1", "w2")}
    try:
        wait_for(tmp_path / "w0.log", "members=['w0', 'w1', 'w2']")
        wait_for(tmp_path / "w0.log", "step 5 ")  # past the first outer step with 3 workers
        procs["w2"].kill()  # no goodbye: must be detected by heartbeat timeout
        wait_for(tmp_path / "w0.log", "members=['w0', 'w1']")
        procs["w3"] = launch("w3")
        wait_for(tmp_path / "w3.log", "received live checkpoint from w0")
        wait_for(tmp_path / "w0.log", "members=['w0', 'w1', 'w3']")
        for n in ("w0", "w1", "w3"):
            assert procs[n].wait(timeout=180) == 0, (tmp_path / f"{n}.log").read_text()
    finally:
        for p in procs.values():
            if p.poll() is None:
                p.kill()
    rows = {n: [json.loads(x) for x in (tmp_path / f"{n}.jsonl").read_text().splitlines()] for n in ("w0", "w1", "w3")}
    assert {r["workers"] for r in rows["w0"]} >= {3, 2}
    # after every outer step the replicas hold the same parameters, including the worker that joined mid-run
    final = {n: [r for r in rows[n] if r.get("outer")][-1] for n in rows}
    assert final["w0"]["step"] == final["w1"]["step"] == final["w3"]["step"] == 60
    assert final["w0"]["param_hash"] == final["w1"]["param_hash"] == final["w3"]["param_hash"]
    del served.store


def test_every_shipped_config_validates():
    seen = {}
    for f in sorted((ROOT / "configs").glob("*/*.toml")):
        cfg = load_config([f"@{f}"])
        seen[f"{f.parent.name}/{f.name}"] = cfg
    # the five BASELINE.json configurations
    assert seen["150M/gloo_2x1.toml"].diloco.inner_steps == 10 and seen["150M/gloo_2x1.toml"].mesh.backend == "gloo"
    c = seen["1B/diloco_4x2.toml"]
    assert (c.name_model, c.diloco.inner_steps, c.mesh.num_workers, c.mesh.fsdp_size, c.diloco.compression) == ("1B", 100, 4, 2, "int8")
    # config 3 (7B DiLoCo H=500, 2 workers × 4-GPU FSDP) is not shipped: on an 80 GB part its state alone leaves no room for activations
    from prime_b200.models.llama import get_model_args
    from prime_b200.utils import memory_plan as mp

    plan = mp.plan_memory(get_model_args("7B"), fsdp_size=4, micro_bs=1, seq_len=4096, shard_params=True, diloco=True)
    assert plan.verdict != "fits" and plan.state_bytes > 0.95 * plan.capacity and not any(k.startswith("7B/diloco") for k in seen)
    assert seen["7B/fsdp_8.toml"].diloco is None and seen["7B/fsdp_8.toml"].mesh.fsdp_size == 8
    assert seen["1B/elastic.toml"].mesh.elastic and seen["1B/elastic.toml"].mesh.num_workers == 4


@pytest.mark.slow
def test_entrypoint_under_torchrun_gloo_2_workers(tmp_path):
    """BASELINE config 1 shape (2 workers × 1 rank, gloo, int8 outer exchange) through ``python -m diloco.train`` — shrunk to the debug model."""
    port = 29650 + os.getpid() % 200
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port", str(port),
           "-m", "diloco.train", f"@{ROOT / 'configs/150M/gloo_2x1.toml'}", "--name_model", "debugmodel", "--data.seq_length", "32",
           "--optim.total_steps", "6", "--diloco.inner_steps", "3", "--optim.warmup_steps", "1", "--train.log_model_hash", "true",
           "--ckpt.path", str(tmp_path / "ck"), "--ckpt.interval", "3", "--monitor.jsonl_path", str(tmp_path / "log.jsonl")]  # fmt: skip
    r = subprocess.run(cmd, cwd=ROOT, env={**os.environ, "PYTHONPATH": str(ROOT)}, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    rows = [json.loads(x) for x in (tmp_path / "log.jsonl").read_text().splitlines()]
    outers = [x for x in rows if x["outer"]]
    assert [x["step"] for x in outers] == [3, 6] and all(x["outer_bytes"] > 0 for x in outers)
    assert ck.list_steps(tmp_path / "ck") == [3, 6]
    assert sorted(p.name for p in (tmp_path / "ck" / "step_000006").iterdir()) == ["meta.json", "rank_00000.pbck", "rank_00001.pbck"]


def test_assemble_full_model_and_hf_export(tmp_path):
    """Offline: published checkpoint → complete model (the engine's own layout planner) → HF directory that transformers loads."""
    transformers = pytest.importorskip("transformers")
    from prime_b200.models import hf

    out = train(load_config(BASE + ["--ckpt.path", str(tmp_path / "ck"), "--ckpt.interval", "8", "--train.log_model_hash", "true"]))
    step = tmp_path / "ck" / "step_000008"
    m = ck.assemble_full_model(step, "debugmodel")
    with torch.no_grad():
        assert abs(float(sum(p.sum() for p in m.parameters())) - out["param_hash"]) < 1e-3 * abs(out["param_hash"])
    with pytest.raises(ValueError, match="different model"):
        ck.assemble_full_model(step, "10M")
    hf.main(["export", "--ckpt", str(step), "--model", "debugmodel", "--out", str(tmp_path / "hf"), "--dtype", "float32"])
    loaded = transformers.AutoModelForCausalLM.from_pretrained(tmp_path / "hf", torch_dtype=torch.float32, attn_implementation="eager").eval()
    tok = torch.randint(0, m.args.vocab_size, (1, 24))
    with torch.no_grad():
        torch.testing.assert_close(loaded(tok).logits, m(tok), rtol=1e-4, atol=1e-4)
    hf.main(["import", "--hf", str(tmp_path / "hf"), "--out", str(tmp_path / "ref.pt")])
    sd = torch.load(tmp_path / "ref.pt", weights_only=True)
    torch.testing.assert_close(sd["layers.1.attention.wq.weight"], m.layers[1].attention.wqkv[: m.args.dim], rtol=0, atol=0)


@pytest.mark.slow
def test_assemble_full_model_from_fsdp2_shards(tmp_path):
    """Two FSDP ranks (gloo): each rank file holds half of every bucket; the assembled model sums to the logged parameter hash."""
    port = 29450 + os.getpid() % 200
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port", str(port),
           "-m", "diloco.train", *BASE, "--mesh.num_workers", "1", "--mesh.backend", "gloo", "--train.log_model_hash", "true",
           "--ckpt.path", str(tmp_path / "ck"), "--ckpt.interval", "8", "--monitor.jsonl_path", str(tmp_path / "log.jsonl")]  # fmt: skip
    r = subprocess.run(cmd, cwd=ROOT, env={**os.environ, "PYTHONPATH": str(ROOT)}, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    rows = [json.loads(x) for x in (tmp_path / "log.jsonl").read_text().splitlines()]
    m = ck.assemble_full_model(tmp_path / "ck" / "step_000008", "debugmodel")
    with torch.no_grad():
        total = float(sum(p.sum() for p in m.parameters()))
    assert abs(total - rows[-1]["param_hash"]) < 1e-3 * abs(total), (total, rows[-1]["param_hash"])


def test_assemble_full_model_from_zero3_row_shards_planned_by_the_layout(tmp_path):
    """ZeRO-3 checkpoints cut every 2-D weight into one row block per rank (and keep the 1-D gains in a small flat bucket).
    The engine only runs that mode on GPUs, so the rank files are synthesised here with the engine's own planner and an
    independent statement of the row cut."""
    from prime_b200.models.llama import build_model
    from prime_b200.parallel.layout import plan_layout

    F = 2
    src = build_model("debugmodel", dtype=torch.float32, seed=21)
    plan = plan_layout(src, F, True)
    assert {b.kind for b in plan.buckets} == {"rows", "flat"}
    layout = plan.signature
    step = tmp_path / "step_000001"
    step.mkdir()
    for r in range(F):
        master = torch.zeros(plan.shard_total)
        for b in plan.buckets:
            if b.kind == "rows":
                for (_, p, _), (soff, piece) in zip(b.params, b.pieces):
                    rpr = p.shape[0] // F
                    master[b.shard_start + soff : b.shard_start + soff + piece] = p.data[r * rpr : (r + 1) * rpr].reshape(-1)
            else:
                flat = torch.zeros(b.size)
                for _, p, off in b.params:
                    flat[off : off + p.numel()] = p.data.reshape(-1)
                master[b.shard_start : b.shard_start + b.shard_size] = flat[r * b.shard_size : (r + 1) * b.shard_size]
        ck.write_shard(step / f"rank_{r:05d}.pbck", {"master": master}, {"fsdp_rank": r, "fsdp_size": F, "layout": layout, "shard_params": True})
    (step / "meta.json").write_text(json.dumps({"world_size": F, "step": 1}))
    got = ck.assemble_full_model(step, "debugmodel")
    for (k, a), (_, b) in zip(src.named_parameters(), got.named_parameters()):
        torch.testing.assert_close(a, b, rtol=0, atol=0, msg=k)


def _state(step_dir):
    meta = json.loads((step_dir / "meta.json").read_text())
    return [ck.read_shard(step_dir / f"rank_{r:05d}.pbck") for r in range(meta["world_size"])]


def test_reshard_checkpoint_round_trips_every_kind_of_state(tmp_path):
    """F=1 → F=2 → F=1 and replicated → ZeRO-3 row shards → replicated: masters, AdamW moments, θ₀ and the outer momentum come back
    bit-identical, the assembled model is the same at every stage, counters and the RNG state travel along."""
    train(load_config(BASE + ["--ckpt.path", str(tmp_path / "a"), "--ckpt.interval", "8"]))
    s1 = tmp_path / "a" / "step_000008"
    (t1, e1), = _state(s1)
    info = ck.reshard_checkpoint(s1, tmp_path / "b" / "step_000008", "debugmodel", fsdp_size=2)
    assert info == {"world_size": 2, "fsdp_size": 2, "workers": 1, "bytes": info["bytes"], "shard_params": False}
    two = _state(tmp_path / "b" / "step_000008")
    assert [e["fsdp_rank"] for _, e in two] == [0, 1] and all(e["fsdp_size"] == 2 and e["trainer_step"] == 8 and e["outer_step"] == e1["outer_step"] for _, e in two)
    assert all(t["master"].numel() < t1["master"].numel() for t, _ in two) and torch.equal(two[1][0]["rng_cpu"], t1["rng_cpu"])
    assert two[1][1]["data"] is None and two[0][1]["data"] == e1["data"]  # the new rank starts its own synthetic stream
    ck.reshard_checkpoint(tmp_path / "b" / "step_000008", tmp_path / "c" / "step_000008", "debugmodel", fsdp_size=2, shard_params=True)  # → ZeRO-3 cut
    z3 = _state(tmp_path / "c" / "step_000008")
    assert all(e["shard_params"] for _, e in z3) and z3[0][1]["layout"] != two[0][1]["layout"]
    ck.reshard_checkpoint(tmp_path / "c" / "step_000008", tmp_path / "d" / "step_000008", "debugmodel", fsdp_size=1)
    (t4, e4), = _state(tmp_path / "d" / "step_000008")
    assert e4["layout"] == e1["layout"] and e4["shard_params"] is False
    for k in ("master", "exp_avg", "exp_avg_sq", "theta0", "momentum"):
        assert torch.equal(t4[k], t1[k]), k
    want = ck.assemble_full_model(s1, "debugmodel")
    for stage in ("b", "c", "d"):
        got = ck.assemble_full_model(tmp_path / stage / "step_000008", "debugmodel")
        for (n, a), (_, b) in zip(want.named_parameters(), got.named_parameters()):
            assert torch.equal(a, b), (stage, n)
    with pytest.raises(ValueError, match="different model"):
        ck.reshard_checkpoint(s1, tmp_path / "x" / "step_000008", "10M", fsdp_size=2)


@pytest.mark.slow
def test_resume_from_a_resharded_checkpoint_with_twice_the_ranks(tmp_path):
    """Train on one rank, reshard the checkpoint offline to fsdp_size=2, resume under torchrun (gloo, 2 ranks): the run continues at
    the saved step with the saved optimizer state (first resumed loss close to the last loss before the checkpoint)."""
    train(load_config(BASE + ["--ckpt.path", str(tmp_path / "a"), "--ckpt.interval", "4", "--monitor.jsonl_path", str(tmp_path / "log1.jsonl")]), max_steps=4)
    ck.main(["reshard", "--src", str(tmp_path / "a" / "step_000004"), "--out", str(tmp_path / "b" / "step_000004"), "--model", "debugmodel", "--fsdp-size", "2"])
    port = 29350 + os.getpid() % 200
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port", str(port),
           "-m", "diloco.train", *BASE, "--mesh.num_workers", "1", "--mesh.backend", "gloo", "--ckpt.path", str(tmp_path / "b"), "--ckpt.resume", "latest",
           "--ckpt.interval", "8", "--monitor.jsonl_path", str(tmp_path / "log2.jsonl")]  # fmt: skip
    r = subprocess.run(cmd, cwd=ROOT, env={**os.environ, "PYTHONPATH": str(ROOT)}, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    before, after = _losses(tmp_path / "log1.jsonl"), _losses(tmp_path / "log2.jsonl")
    assert sorted(after) == [5, 6, 7, 8] and abs(after[5] - before[4]) < 0.5  # continues where it stopped (not from a fresh init: ≈ 8.3 → would jump)
    assert ck.list_steps(tmp_path / "b") == [4, 8]
    assert len(list((tmp_path / "b" / "step_000008").glob("rank_*.pbck"))) == 2


def test_training_starts_from_hugging_face_weights(tmp_path):
    """train.init_weights: the run starts at the imported weights (first loss = the imported model's loss, not a random init's),
    a different architecture is refused."""
    pytest.importorskip("safetensors")
    from prime_b200.models import hf
    from prime_b200.models.llama import build_model
    from prime_b200.trainer import Trainer

    donor = build_model("debugmodel", dtype=torch.float32, seed=123)
    hf.save_hf_dir(donor, tmp_path / "hf")
    cfg = load_config(BASE + ["--train.init_weights", str(tmp_path / "hf")])
    t = Trainer(cfg)
    for (n, a), (_, b) in zip(donor.named_parameters(), t.model.named_parameters()):
        torch.testing.assert_close(a, b.detach().float(), rtol=0, atol=0, msg=n)
    assert torch.equal(t.outer.theta0[: 16], t.engine.master[: 16])  # θ₀ is the imported model too
    t.close()
    torch.save({k: v.clone() for k, v in __import__("prime_b200.models.llama", fromlist=["x"]).to_reference_state_dict(donor).items()}, tmp_path / "ref.pt")
    t2 = Trainer(load_config(BASE + ["--train.init_weights", str(tmp_path / "ref.pt")]))
    torch.testing.assert_close(t2.model.output.detach(), donor.output, rtol=0, atol=0)
    t2.close()
    with pytest.raises(ValueError, match="init_weights"):
        Trainer(load_config(["--name_model", "10M", "--data.seq_length", "32", "--optim.batch_size", "4", "--train.micro_bs", "2", "--train.init_weights", str(tmp_path / "hf")]))
    with pytest.raises(FileNotFoundError):
        Trainer(load_config(BASE + ["--train.init_weights", str(tmp_path / "nope")]))


def test_periodic_validation_loss(tmp_path):
    """train.eval_interval: a forward-only loss on the held-out stream, logged next to the training metrics, comparable across calls."""
    from prime_b200.trainer import Trainer

    out = train(load_config(BASE + ["--train.eval_interval", "4", "--train.eval_batches", "2", "--monitor.jsonl_path", str(tmp_path / "log.jsonl"), "--optim.optim.lr", "3e-3"]))
    rows = [json.loads(x) for x in (tmp_path / "log.jsonl").read_text().splitlines()]
    vals = [r["val_loss"] for r in rows if "val_loss" in r and "loss" not in r]
    assert [r["step"] for r in rows if "val_loss" in r and "loss" not in r] == [4, 8] and all(v == v for v in vals) and out["val_loss"] == vals[-1]
    assert vals[1] < vals[0]  # same held-out batches both times: the model got better on them
    t = Trainer(load_config(BASE))
    a, b = t.evaluate(2), t.evaluate(2)
    assert a == b and abs(a - 7.7) < 1.5  # ln(2048) ≈ 7.6 at init; the stream restarts for every evaluation
    t.close()
