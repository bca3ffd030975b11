"""Local run manager (prime_b200/launch.py): run → list/get/metrics/logs, stop (final checkpoint) → restart (resume),
and supervised elastic workers: SIGKILL one, the supervisor respawns it, it rejoins through the live checkpoint.
The verb set mirrors the hosted one (reference: packages/prime/src/prime_cli/commands/rl.py:608-1510; its tests:
packages/prime/tests/test_rl_*.py) — here the "server" is a supervisor process on this box."""

import json
import os
import signal
import time
from pathlib import Path

import pytest

from prime_b200 import launch

ROOT = Path(__file__).resolve().parents[1]
CFG = f"@{ROOT / 'configs' / 'debug' / 'cpu.toml'}"


@pytest.fixture()
def runs(tmp_path, monkeypatch):
    monkeypatch.setenv("PRIME_B200_RUNS_DIR", str(tmp_path / "runs"))
    monkeypatch.setenv("CUDA_VISIBLE_DEVICES", "")  # the manager itself is device-agnostic; keep these runs on the CPU path
    yield tmp_path / "runs"
    for r in launch.iter_runs():  # never leave a supervisor behind, whatever the test did
        if r.status()["state"] in launch.ACTIVE:
            launch.stop_run(r, force=True, wait_s=30)


def wait_for(pred, timeout=120.0, what="condition"):
    t0 = time.monotonic()
    while time.monotonic() - t0 < timeout:
        v = pred()
        if v:
            return v
        time.sleep(0.2)
    raise AssertionError(f"timed out waiting for {what}")


def test_helpers_are_pure():
    assert launch._arg_value(["--a", "1", "--ckpt.path=/x", "--a", "2"], "--a") == "2"
    assert launch._arg_value(["--a", "1", "--ckpt.path=/x"], "--ckpt.path") == "/x" and launch._arg_value(["--a"], "--a") is None
    assert launch.gpu_slices(2, 2, None) == ["0,1", "2,3"] and launch.gpu_slices(2, 2, "4,5,6,7") == ["4,5", "6,7"]
    assert launch.gpu_slices(1, 8, None) == [None] and launch.gpu_slices(3, 0, None) == [None] * 3
    with pytest.raises(SystemExit):
        launch.gpu_slices(2, 2, "0,1,2")
    with pytest.raises(SystemExit):  # several independent worlds only make sense with the elastic rendezvous
        launch.create_run([CFG], name=None, gpus=0, workers=2, elastic=False, respawn=0, grace_s=1)


def test_worker_command_injects_paths_once(runs):
    run = launch.create_run([CFG, "--ckpt.path", "/data/ck"], name="n", gpus=4, workers=1, elastic=False, respawn=0, grace_s=5)
    cmd = launch.worker_command(run.spec, run, "w0", 29511, resume=True)
    assert cmd[1:4] == ["-m", "torch.distributed.run", "--nnodes=1"] and "--nproc-per-node=4" in cmd and cmd[cmd.index("--master-port") + 1] == "29511"
    assert cmd.count("--ckpt.path") == 1 and cmd[cmd.index("--ckpt.path") + 1] == "/data/ck"  # the user's choice stands
    assert cmd[cmd.index("--monitor.jsonl_path") + 1] == str(run.path / "metrics.jsonl") and cmd[-2:] == ["--ckpt.resume", "latest"]
    assert run.ckpt_root == Path("/data/ck") and launch.find_run("n").spec.id == run.spec.id and launch.find_run(run.spec.id[:9]).spec.id == run.spec.id
    solo = launch.create_run([CFG], name="solo", gpus=0, workers=1, elastic=False, respawn=0, grace_s=5)
    assert launch.worker_command(solo.spec, solo, "w0", 1, resume=False)[1:3] == ["-m", "prime_b200.train"]


def test_run_refuses_a_configuration_that_cannot_fit_before_starting_anything(runs, monkeypatch):
    """`run --gpus 8` with llama2/70B: model + optimizer state alone exceed an 80 GB part → the command ends with the memory table and
    no run directory, no supervisor, no ranks. A configuration the planner cannot read is not this check's business."""
    with pytest.raises(SystemExit) as e:
        launch.main(["run", "--gpus", "8", "--detach", "--", "--name_model", "70B", "--data.seq_length", "4096", "--train.micro_bs", "1"])
    assert "cannot fit a 80 GB GPU" in str(e.value) and "fp32 main_grad" in str(e.value)
    assert list(launch.iter_runs()) == []
    launch.preflight_memory(["--name_model", "7B", "--data.seq_length", "4096", "--train.micro_bs", "1"], 8)  # fits: no exception
    launch.preflight_memory(["--no_such_key", "1"], 8)  # unreadable: left to the workers
    monkeypatch.setenv("PB_SKIP_MEMORY_CHECK", "1")
    launch.preflight_memory(["--name_model", "70B"], 8)  # explicit override: no refusal


def test_run_then_inspect(runs, capsys):
    assert launch.main(["run", "--detach", "--name", "quick", CFG, "--optim.total_steps", "6"]) == 0
    rid = json.loads(capsys.readouterr().out)["run"]
    run = launch.find_run("quick")
    assert run.spec.id == rid
    wait_for(lambda: run.status()["state"] in launch.FINAL, what="run to finish")
    assert run.status()["state"] == "COMPLETED", run.log_path("w0").read_text()[-2000:]
    assert [w["exit_code"] for w in run.status()["workers"]] == [0]
    launch.main(["list", "-o", "json"])
    listed = json.loads(capsys.readouterr().out)["runs"]
    assert [(r["name"], r["state"], r["step"]) for r in listed] == [("quick", "COMPLETED", 6)]
    launch.main(["metrics", "quick", "-n", "2", "-o", "json"])
    assert [m["step"] for m in json.loads(capsys.readouterr().out)["metrics"]] == [5, 6]
    launch.main(["logs", "quick", "-n", "1"])
    assert '"final"' in capsys.readouterr().out
    launch.main(["list"])
    assert "COMPLETED" in capsys.readouterr().out
    launch.main(["delete", "quick"])
    assert not run.path.exists()


def test_stop_writes_a_checkpoint_and_restart_resumes(runs, capsys):
    launch.main(["run", "-d", "--name", "long", "-e", "PRIME_B200_STEP_DELAY_S=0.2", CFG, "--optim.total_steps", "500"])
    capsys.readouterr()
    run = launch.find_run("long")
    wait_for(lambda: (launch._last_jsonl(run.metrics_path) or {}).get("step", 0) >= 3, what="a few steps")
    assert launch.main(["stop", "long"]) == 0 and run.status()["state"] == "STOPPED"
    ck = run.checkpoints()
    assert len(ck) == 1 and ck[0]["step"] >= 3 and ck[0]["size_bytes"] > 0
    stopped_at = ck[0]["step"]
    with pytest.raises(SystemExit):
        launch.main(["restart", "nope"])
    launch.main(["restart", "long", "-d"])
    assert json.loads(capsys.readouterr().out.strip().splitlines()[-1])["resumed_from"] == stopped_at
    wait_for(lambda: (launch._last_jsonl(run.metrics_path) or {}).get("step", 0) > stopped_at + 1, what="progress after the resume")
    assert f"resumed from {ck[0]['path']} at step {stopped_at}" in run.log_path("w0").read_text()
    assert run.status()["restarts"] == 1
    with pytest.raises(SystemExit):  # refuses to delete a live run without --force
        launch.main(["delete", "long"])
    launch.main(["stop", "long", "--force"])
    assert run.status()["state"] == "STOPPED"


def test_killed_elastic_worker_is_respawned_and_rejoins(runs, capsys):
    launch.main(["run", "-d", "--name", "el", "--workers", "2", "--elastic", "--respawn", "1", "-e", "PRIME_B200_STEP_DELAY_S=0.12", CFG,
                 "--optim.total_steps", "72", "--mesh.num_workers", "2", "--mesh.heartbeat_interval_s", "0.2", "--mesh.heartbeat_timeout_s", "3",
                 "--train.log_model_hash", "true"])  # fmt: skip
    capsys.readouterr()
    run = launch.find_run("el")
    wait_for(lambda: (launch._last_jsonl(run.worker_metrics_path("w1")) or {}).get("step", 0) >= 5, what="both workers training")
    victim = next(w for w in run.status()["workers"] if w["name"] == "w1")
    os.killpg(victim["pid"], signal.SIGKILL)  # the exact process group the supervisor created for w1
    wait_for(lambda: next(w for w in run.status()["workers"] if w["name"] == "w1")["starts"] == 2, what="the respawn")
    wait_for(lambda: run.status()["state"] in launch.FINAL, timeout=240, what="the elastic run to finish")
    st = run.status()
    assert st["state"] == "COMPLETED" and {w["name"]: w["exit_code"] for w in st["workers"]} == {"w0": 0, "w1": 0}, run.log_path("w1").read_text()[-3000:]
    w1 = run.log_path("w1").read_text()
    assert "--- respawn #1" in w1 and "received live checkpoint from w0" in w1
    finals = [launch._last_jsonl(run.worker_metrics_path(w)) for w in ("w0", "w1")]
    assert finals[0]["step"] == finals[1]["step"] == 72 and finals[0]["workers"] == 2
    assert finals[0]["param_hash"] == finals[1]["param_hash"]  # the rejoined worker ends bit-identical with the survivor
