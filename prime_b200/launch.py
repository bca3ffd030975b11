"""Local run manager: start, watch, stop and resume training jobs on THIS box.

    python -m prime_b200.launch run @configs/1B/h100.toml --gpus 8 --detach           # one world of 8 ranks
    python -m prime_b200.launch run @configs/1B/elastic.toml --workers 4 --gpus 2 \\
           --elastic --respawn 3                                                      # 4 elastic DiLoCo workers × 2 GPUs
    python -m prime_b200.launch list | get <id> | logs <id> -f | metrics <id> | checkpoints <id>
    python -m prime_b200.launch stop <id>        # SIGTERM → final checkpoint → exit
    python -m prime_b200.launch restart <id>     # same arguments, resumes from the newest complete checkpoint

The verb set is the hosted-RL one (``prime rl run/list/get/stop/restart/logs/metrics/checkpoints``, reference:
packages/prime/src/prime_cli/commands/rl.py:608-1510) applied to local processes; ``--workers N --elastic`` is the
"several nodes on one box" launch the DiLoCo framework shipped as a shell script, plus supervision.

Every run owns a directory ``<runs>/<id>/``:

    spec.json       what was asked (immutable)               status.json    what is happening (supervisor-written, atomic)
    logs/<w>.log    stdout+stderr of each worker             metrics.jsonl  the leader's step records (``monitor.jsonl_path``)
    ckpt/           checkpoints (``ckpt.path``) unless the arguments name another place

A detached **supervisor** process (``_supervise``) owns the workers: it starts each one as the leader of its own process
group, forwards a stop request to exactly those groups, escalates to SIGKILL after the grace period, optionally respawns
crashed elastic workers (they re-enter through the live-checkpoint join), and records exit codes. ``stop`` therefore
signals one known PID and never matches processes by name.
"""

from __future__ import annotations

import argparse
import json
import os
import signal
import socket
import subprocess
import sys
import time
import uuid
from dataclasses import asdict, dataclass, field
from pathlib import Path
from typing import Any, Iterator, Sequence

ACTIVE = ("PENDING", "RUNNING", "STOPPING")
FINAL = ("COMPLETED", "FAILED", "STOPPED")
POLL_S = 0.25


# ------------------------------------------------------------------------------------------------------------ storage
def runs_root() -> Path:
    return Path(os.environ.get("PRIME_B200_RUNS_DIR") or Path.home() / ".prime_b200" / "runs")


def write_json_atomic(path: Path, doc: Any) -> None:
    tmp = path.with_name(f".{path.name}.{os.getpid()}.tmp")
    tmp.write_text(json.dumps(doc, indent=2))
    os.replace(tmp, path)


def read_json(path: Path) -> dict[str, Any] | None:
    try:
        return json.loads(path.read_text())
    except (FileNotFoundError, json.JSONDecodeError):
        return None


@dataclass
class RunSpec:
    id: str
    name: str
    train_args: list[str]  # argv of prime_b200.train as the user gave it
    gpus: int = 0  # ranks per worker (0/1: a single process without torchrun)
    workers: int = 1
    elastic: bool = False
    respawn: int = 0  # how many times a crashed elastic worker may be started again
    grace_s: float = 60.0
    cwd: str = field(default_factory=os.getcwd)
    env: dict[str, str] = field(default_factory=dict)
    created_at: float = field(default_factory=time.time)

    @property
    def worker_names(self) -> list[str]:
        return [f"w{k}" for k in range(self.workers)]


class Run:
    """A run directory and the questions one asks of it."""

    def __init__(self, path: Path):
        self.path = path
        doc = read_json(path / "spec.json")
        if doc is None:
            raise FileNotFoundError(f"{path} is not a run directory")
        self.spec = RunSpec(**doc)

    # where things are --------------------------------------------------------------------------------------------
    @property
    def metrics_path(self) -> Path:
        """The step records to show: the file the arguments name, else ours. Elastic workers each keep their own
        (``metrics-<w>.jsonl`` — any of them may die), and the freshest one speaks for the run."""
        named = _arg_value(self.spec.train_args, "--monitor.jsonl_path")
        if named:
            return Path(named)
        if self.spec.elastic:
            live = sorted(self.path.glob("metrics-*.jsonl"), key=lambda p: p.stat().st_mtime)
            return live[-1] if live else self.worker_metrics_path(self.spec.worker_names[0])
        return self.path / "metrics.jsonl"

    def worker_metrics_path(self, worker: str) -> Path:
        return self.path / (f"metrics-{worker}.jsonl" if self.spec.elastic else "metrics.jsonl")

    @property
    def ckpt_root(self) -> Path:
        return Path(_arg_value(self.spec.train_args, "--ckpt.path") or self.path / "ckpt")

    def log_path(self, worker: str) -> Path:
        return self.path / "logs" / f"{worker}.log"

    # state -------------------------------------------------------------------------------------------------------
    def status(self) -> dict[str, Any]:
        st = read_json(self.path / "status.json") or {"state": "PENDING", "workers": []}
        if st["state"] in ACTIVE and not _alive(st.get("supervisor_pid"), marker=self.spec.id):
            # the supervisor vanished without a verdict (machine reboot, SIGKILL): say so instead of "RUNNING" forever
            st = {**st, "state": "FAILED", "note": "supervisor is gone; no exit status was recorded"}
        return st

    def describe(self) -> dict[str, Any]:
        st = self.status()
        last = _last_jsonl(self.metrics_path)
        return {"id": self.spec.id, "name": self.spec.name, "state": st["state"], "workers": self.spec.workers, "gpus_per_worker": self.spec.gpus,
                "elastic": self.spec.elastic, "created_at": self.spec.created_at, "started_at": st.get("started_at"),
                "finished_at": st.get("finished_at"), "restarts": st.get("restarts", 0), "step": (last or {}).get("step"),
                "loss": (last or {}).get("loss"), "tokens_per_s": (last or {}).get("tokens_per_s"), "dir": str(self.path)}  # fmt: skip

    def checkpoints(self) -> list[dict[str, Any]]:
        """Complete step directories (per elastic worker when the run has several), newest last."""
        roots = [self.ckpt_root / w for w in self.spec.worker_names] if self.spec.elastic else [self.ckpt_root]
        out = []
        for root in roots:
            for d in sorted(root.glob("step_*")):
                if not (d / "meta.json").exists():
                    continue
                files = [f for f in d.iterdir() if f.is_file()]
                out.append({"step": int(d.name.split("_")[1]), "path": str(d), "worker": root.name if self.spec.elastic else None,
                            "files": len(files), "size_bytes": sum(f.stat().st_size for f in files), "written_at": (d / "meta.json").stat().st_mtime})  # fmt: skip
        return sorted(out, key=lambda c: (c["step"], c["worker"] or ""))


def _arg_value(argv: Sequence[str], flag: str) -> str | None:
    """Value of ``--flag v`` / ``--flag=v`` in a train argv (last one wins, like the config loader)."""
    found = None
    for i, a in enumerate(argv):
        if a == flag and i + 1 < len(argv):
            found = argv[i + 1]
        elif a.startswith(flag + "="):
            found = a.split("=", 1)[1]
    return found


def _last_jsonl(path: Path) -> dict[str, Any] | None:
    try:
        with open(path, "rb") as f:
            f.seek(0, os.SEEK_END)
            size = f.tell()
            f.seek(max(0, size - 8192))
            lines = [ln for ln in f.read().decode(errors="replace").splitlines() if ln.strip()]
    except FileNotFoundError:
        return None
    for ln in reversed(lines):
        try:
            return json.loads(ln)
        except json.JSONDecodeError:
            continue  # a line the writer has not finished yet
    return None


def _alive(pid: int | None, marker: str | None = None) -> bool:
    """Is ``pid`` running — and, when ``marker`` is given, is it still OUR process (guards against PID reuse)?"""
    if not pid:
        return False
    try:
        os.kill(pid, 0)
    except ProcessLookupError:
        return False
    except PermissionError:
        return marker is None
    if marker is None:
        return True
    try:
        return marker.encode() in Path(f"/proc/{pid}/cmdline").read_bytes()
    except OSError:
        return True  # no procfs: trust the PID


def find_run(ref: str) -> Run:
    """By id, unique id prefix, or name (newest of that name)."""
    root = runs_root()
    if (root / ref / "spec.json").exists():
        return Run(root / ref)
    runs = list(iter_runs())
    by_prefix = [r for r in runs if r.spec.id.startswith(ref)]
    if len(by_prefix) == 1:
        return by_prefix[0]
    if len(by_prefix) > 1:
        raise SystemExit(f"'{ref}' is ambiguous: {', '.join(r.spec.id for r in by_prefix)}")
    by_name = [r for r in runs if r.spec.name == ref]
    if by_name:
        return by_name[-1]
    raise SystemExit(f"no run '{ref}' under {root}")


def iter_runs() -> Iterator[Run]:
    root = runs_root()
    if not root.is_dir():
        return
    found = []
    for d in root.iterdir():
        try:
            found.append(Run(d))
        except (FileNotFoundError, TypeError, NotADirectoryError):
            continue
    yield from sorted(found, key=lambda r: r.spec.created_at)


# --------------------------------------------------------------------------------------------------------- supervisor
def free_port() -> int:
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def descendants(pid: int) -> list[int]:
    """Every live descendant of ``pid`` (children first). torchrun starts its ranks in their OWN sessions, so a signal to the
    launcher's process group does not reach them: a SIGKILL of "the worker" has to walk the tree (seen on the 8-GPU box: killpg
    took torchrun down, the ranks trained on as orphans next to their respawned successors)."""
    try:
        import psutil

        return [c.pid for c in psutil.Process(pid).children(recursive=True)]
    except Exception:  # noqa: BLE001 — psutil missing or the process is already gone: fall back to /proc
        kids: dict[int, list[int]] = {}
        for d in os.listdir("/proc"):
            if d.isdigit():
                try:
                    with open(f"/proc/{d}/stat") as f:
                        ppid = int(f.read().rsplit(")", 1)[1].split()[1])
                    kids.setdefault(ppid, []).append(int(d))
                except (OSError, ValueError, IndexError):
                    pass
        out, todo = [], [pid]
        while todo:
            for c in kids.get(todo.pop(), []):
                out.append(c)
                todo.append(c)
        return out


def signal_tree(pid: int, sig: int) -> None:
    """Deliver ``sig`` to the process group of ``pid`` AND to every descendant (collected first: they re-parent once the root dies).
    SIGTERM is forwarded by torchrun itself, so only the hard kill really needs the walk — doing it for both keeps one code path."""
    tree = descendants(pid) if sig == signal.SIGKILL else []
    try:
        os.killpg(pid, sig)
    except (ProcessLookupError, PermissionError):
        pass
    for c in tree:
        try:
            os.kill(c, sig)
        except (ProcessLookupError, PermissionError):
            pass


def gpu_slices(workers: int, per_worker: int, pool: str | None) -> list[str | None]:
    """``CUDA_VISIBLE_DEVICES`` for each worker: consecutive slices of the visible pool (or of 0..N-1)."""
    if per_worker <= 0 or workers <= 1:
        return [None] * workers
    ids = [x for x in pool.split(",") if x] if pool else [str(i) for i in range(workers * per_worker)]
    if len(ids) < workers * per_worker:
        raise SystemExit(f"{workers} workers × {per_worker} GPUs need {workers * per_worker} devices, {len(ids)} visible")
    return [",".join(ids[k * per_worker : (k + 1) * per_worker]) for k in range(workers)]


def worker_command(spec: RunSpec, run: Run, worker: str, master_port: int, resume: bool) -> list[str]:
    args = list(spec.train_args)
    if _arg_value(args, "--monitor.jsonl_path") is None:
        args += ["--monitor.jsonl_path", str(run.worker_metrics_path(worker))]
    if _arg_value(args, "--ckpt.path") is None:
        args += ["--ckpt.path", str(run.ckpt_root)]
    if resume and _arg_value(args, "--ckpt.resume") is None:
        args += ["--ckpt.resume", "latest"]
    if spec.elastic and _arg_value(args, "--mesh.elastic") is None:
        args += ["--mesh.elastic", "true"]
    if spec.gpus > 1:
        return [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={spec.gpus}", "--master-addr", "127.0.0.1",
                "--master-port", str(master_port), "-m", "prime_b200.train", *args]  # fmt: skip
    return [sys.executable, "-m", "prime_b200.train", *args]


@dataclass
class _Worker:
    name: str
    cmd: list[str]
    env: dict[str, str]
    proc: subprocess.Popen | None = None
    starts: int = 0
    exit_code: int | None = None

    def start(self, log_path: Path, cwd: str) -> None:
        log_path.parent.mkdir(parents=True, exist_ok=True)
        with open(log_path, "ab") as log:
            if self.starts:
                log.write(f"\n--- respawn #{self.starts} at {time.strftime('%Y-%m-%d %H:%M:%S')} ---\n".encode())
            # own session ⇒ own process group: a stop reaches torchrun AND its ranks, and nothing else
            self.proc = subprocess.Popen(self.cmd, cwd=cwd, env=self.env, stdout=log, stderr=subprocess.STDOUT, stdin=subprocess.DEVNULL,
                                         start_new_session=True)  # fmt: skip
        self.starts += 1
        self.exit_code = None

    def signal(self, sig: int) -> None:
        if self.proc is not None and self.proc.poll() is None:
            signal_tree(self.proc.pid, sig)

    def snapshot(self) -> dict[str, Any]:
        return {"name": self.name, "pid": self.proc.pid if self.proc else None, "starts": self.starts, "exit_code": self.exit_code}


def supervise(run_dir: Path, resume: bool = False) -> int:
    """Body of the detached supervisor. Returns the process exit code (0 unless the run FAILED)."""
    run = Run(run_dir)
    spec = run.spec
    prev = read_json(run.path / "status.json") or {}
    stop_requested: list[str] = []
    for sig in (signal.SIGTERM, signal.SIGINT):
        signal.signal(sig, lambda s, _f: stop_requested.append(signal.Signals(s).name))

    base_env = {**os.environ, **spec.env, "PYTHONUNBUFFERED": "1"}
    repo = str(Path(__file__).resolve().parents[1])
    base_env["PYTHONPATH"] = repo + (os.pathsep + base_env["PYTHONPATH"] if base_env.get("PYTHONPATH") else "")
    store = None
    if spec.elastic:
        port = free_port()
        with open(run.path / "logs" / "store.log", "ab") as store_log:
            store = subprocess.Popen([sys.executable, "-m", "prime_b200.parallel.elastic", "serve", "--port", str(port)], env=base_env,
                                     stdout=store_log, stderr=subprocess.STDOUT, start_new_session=True)  # fmt: skip
        base_env.update(GLOBAL_ADDR="127.0.0.1", GLOBAL_PORT=str(port))
    slices = gpu_slices(spec.workers, spec.gpus, base_env.get("CUDA_VISIBLE_DEVICES"))
    workers: list[_Worker] = []
    for k, name in enumerate(spec.worker_names):
        port = free_port()
        env = {**base_env, "MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port)}
        if spec.elastic:
            env["GLOBAL_UNIQUE_ID"] = name
        if slices[k] is not None:
            if spec.elastic:
                # elastic workers keep every GPU VISIBLE and are told which ones are theirs: the fused outer step maps the other
                # workers' exchange buffers by cudaIpc, which cannot reach a device hidden by CUDA_VISIBLE_DEVICES
                env["PRIME_B200_DEVICES"] = ",".join(str(k * spec.gpus + j) for j in range(spec.gpus))  # indices into the visible pool
            else:
                env["CUDA_VISIBLE_DEVICES"] = slices[k]
        workers.append(_Worker(name, worker_command(spec, run, name, port, resume), env))

    status: dict[str, Any] = {"state": "RUNNING", "supervisor_pid": os.getpid(), "started_at": time.time(), "finished_at": None,
                              "restarts": prev.get("restarts", 0) + (1 if resume else 0), "workers": []}  # fmt: skip

    def publish(state: str | None = None) -> None:
        if state:
            status["state"] = state
        status["workers"] = [w.snapshot() for w in workers]
        write_json_atomic(run.path / "status.json", status)

    for w in workers:
        w.start(run.log_path(w.name), spec.cwd)
    publish()

    deadline = None
    while True:
        running = 0
        for w in workers:
            if w.proc is None or w.exit_code is not None:
                continue
            rc = w.proc.poll()
            if rc is None:
                running += 1
                continue
            w.exit_code = rc
            if rc != 0 and not stop_requested and spec.elastic and w.starts <= spec.respawn:
                w.cmd = worker_command(spec, run, w.name, int(w.env["MASTER_PORT"]), resume=False)  # a rejoiner gets the LIVE checkpoint from a peer
                w.start(run.log_path(w.name), spec.cwd)
                running += 1
            publish()
        if running == 0:
            break
        if stop_requested and deadline is None:
            deadline = time.monotonic() + spec.grace_s
            publish("STOPPING")
            for w in workers:
                w.signal(signal.SIGTERM)
        if deadline is not None and time.monotonic() > deadline:
            for w in workers:
                w.signal(signal.SIGKILL)
            deadline = float("inf")
        time.sleep(POLL_S)

    if store is not None:
        store.terminate()
        try:
            store.wait(5)
        except subprocess.TimeoutExpired:
            store.kill()
    codes = [w.exit_code for w in workers]
    status["finished_at"] = time.time()
    if stop_requested:
        publish("STOPPED")
        return 0
    # an elastic run is a success if the job finished on at least one worker (the others dropping out is the feature)
    ok = any(c == 0 for c in codes) if spec.elastic else all(c == 0 for c in codes)
    publish("COMPLETED" if ok else "FAILED")
    return 0 if ok else 1


def spawn_supervisor(run: Run, resume: bool) -> int:
    """Start the supervisor detached from this terminal; returns its PID once it has published a status."""
    (run.path / "logs").mkdir(parents=True, exist_ok=True)
    before = (read_json(run.path / "status.json") or {}).get("started_at")
    cmd = [sys.executable, "-m", "prime_b200.launch", "_supervise", str(run.path), run.spec.id] + (["--resume"] if resume else [])
    repo = str(Path(__file__).resolve().parents[1])
    env = {**os.environ, "PYTHONPATH": repo + (os.pathsep + os.environ["PYTHONPATH"] if os.environ.get("PYTHONPATH") else "")}
    with open(run.path / "logs" / "supervisor.log", "ab") as log:
        p = subprocess.Popen(cmd, env=env, stdout=log, stderr=subprocess.STDOUT, stdin=subprocess.DEVNULL, start_new_session=True)
    t0 = time.monotonic()
    while time.monotonic() - t0 < 30:
        st = read_json(run.path / "status.json") or {}
        if st.get("supervisor_pid") == p.pid and st.get("started_at") != before:
            return p.pid
        if p.poll() is not None:
            raise SystemExit(f"supervisor exited with {p.returncode}; see {run.path / 'logs' / 'supervisor.log'}")
        time.sleep(0.05)
    raise SystemExit("supervisor did not come up within 30 s")


# ------------------------------------------------------------------------------------------------------------- verbs
def create_run(train_args: list[str], *, name: str | None, gpus: int, workers: int, elastic: bool, respawn: int, grace_s: float,
               env: dict[str, str] | None = None) -> Run:  # fmt: skip
    if workers > 1 and not elastic:
        raise SystemExit("--workers > 1 starts independent process worlds: that needs --elastic (a static DiLoCo mesh is ONE world: use --gpus)")
    rid = time.strftime("%y%m%d-%H%M%S-") + uuid.uuid4().hex[:6]
    path = runs_root() / rid
    (path / "logs").mkdir(parents=True)
    spec = RunSpec(id=rid, name=name or rid, train_args=train_args, gpus=gpus, workers=workers, elastic=elastic, respawn=respawn, grace_s=grace_s,
                   env=env or {})  # fmt: skip
    write_json_atomic(path / "spec.json", asdict(spec))
    return Run(path)


def preflight_memory(train_args: list[str], ranks_per_worker: int) -> None:
    """``run --gpus N``: the per-GPU memory plan of the configuration (``utils/memory_plan.py``) before the supervisor and N ranks are
    started. A plan whose exact part exceeds the device ends the command with the table; a configuration the planner cannot read is
    left to the workers (they print the real validation error); ``PB_SKIP_MEMORY_CHECK=1`` skips the refusal."""
    from .utils import memory_plan as mp

    try:
        from .config import load_config

        plan = mp.plan_from_config(load_config(train_args), ranks_per_worker)
    except BaseException:  # noqa: BLE001 — SystemExit from the config loader included: not this function's error to report
        return
    try:
        mp.check(plan)
    except mp.MemoryPlanError as e:
        raise SystemExit(str(e)) from None


def stop_run(run: Run, *, force: bool = False, wait_s: float = 120.0) -> dict[str, Any]:
    st = run.status()
    if st["state"] not in ACTIVE:
        return st
    pid = st.get("supervisor_pid")
    if _alive(pid, marker=run.spec.id):
        os.kill(pid, signal.SIGTERM)
        if force:  # do not wait for final checkpoints: take the workers' groups down now, the supervisor records the outcome
            for w in st.get("workers", []):
                if w.get("pid") and w.get("exit_code") is None:
                    try:
                        signal_tree(w["pid"], signal.SIGKILL)
                    except (ProcessLookupError, PermissionError):
                        pass
    t0 = time.monotonic()
    while time.monotonic() - t0 < wait_s:
        st = run.status()
        if st["state"] in FINAL:
            break
        time.sleep(POLL_S)
    return st


def follow(path: Path, *, tail: int | None, until) -> Iterator[str]:
    """Lines of a growing file; ends when ``until()`` is true and nothing is left to read."""
    pos = 0
    first = True
    while True:
        done = until()
        try:
            with open(path, "rb") as f:
                f.seek(pos)
                chunk = f.read()
        except FileNotFoundError:
            chunk = b""
        if chunk:
            end = chunk.rfind(b"\n") + 1  # hold back a partial last line
            if done:
                end = len(chunk)
            lines = chunk[:end].decode(errors="replace").splitlines()
            pos += end
            if first and tail is not None:
                lines = lines[-tail:] if tail else []
            first = False
            yield from lines
        if done:
            return
        time.sleep(POLL_S)


def _print_table(rows: list[dict[str, Any]], cols: Sequence[str]) -> None:
    def cell(v: Any) -> str:
        if v is None:
            return "-"
        if isinstance(v, float):
            return f"{v:.4g}"
        return str(v)

    table = [[c.upper() for c in cols]] + [[cell(r.get(c)) for c in cols] for r in rows]
    widths = [max(len(r[i]) for r in table) for i in range(len(cols))]
    for r in table:
        print("  ".join(v.ljust(w) for v, w in zip(r, widths)).rstrip())


def _age(ts: float | None) -> str | None:
    if ts is None:
        return None
    s = max(0, int(time.time() - ts))
    for unit, n in (("d", 86400), ("h", 3600), ("m", 60)):
        if s >= n:
            return f"{s // n}{unit}"
    return f"{s}s"


def main(argv: Sequence[str] | None = None) -> int:
    ap = argparse.ArgumentParser(prog="python -m prime_b200.launch", description="Run and manage local training jobs")
    sub = ap.add_subparsers(dest="verb", required=True)
    r = sub.add_parser("run", help="start a run (arguments after the options go to prime_b200.train)")
    r.add_argument("--name")
    r.add_argument("--gpus", type=int, default=0, help="ranks per worker (torchrun --nproc-per-node); 0 = one CPU/GPU process")
    r.add_argument("--workers", type=int, default=1, help="independent DiLoCo workers (needs --elastic when > 1)")
    r.add_argument("--elastic", action="store_true", help="workers meet through the global store; they may die and rejoin")
    r.add_argument("--respawn", type=int, default=0, help="restart a crashed elastic worker up to N times")
    r.add_argument("--grace", type=float, default=60.0, help="seconds between SIGTERM and SIGKILL on stop")
    r.add_argument("--env", "-e", action="append", default=[], metavar="KEY=VALUE", help="extra environment for the workers (repeatable)")
    r.add_argument("--detach", "-d", action="store_true", help="return once the run is up instead of following its log")
    r.add_argument("train_args", nargs=argparse.REMAINDER)
    for verb, text in (("get", "one run as JSON"), ("stop", "SIGTERM the run: final checkpoint, then exit"), ("restart", "start a finished run again from its newest checkpoint"),
                       ("delete", "remove a finished run's directory"), ("checkpoints", "complete checkpoints of a run"), ("metrics", "step records of a run"),
                       ("logs", "worker output")):  # fmt: skip
        p = sub.add_parser(verb, help=text)
        p.add_argument("run")
        p.add_argument("--output", "-o", choices=("table", "json"), default="table")
        if verb in ("stop", "delete"):
            p.add_argument("--force", "-f", action="store_true")
        if verb == "metrics":
            p.add_argument("--last", "-n", type=int, default=10)
        if verb == "logs":
            p.add_argument("--follow", "-f", action="store_true")
            p.add_argument("--tail", "-n", type=int, default=None)
            p.add_argument("--worker", "-w", default="w0")
        if verb == "restart":
            p.add_argument("--detach", "-d", action="store_true")
    ls = sub.add_parser("list", aliases=["ls"], help="all runs, oldest first")
    ls.add_argument("--output", "-o", choices=("table", "json"), default="table")
    ls.add_argument("--active", action="store_true", help="only runs that are still going")
    sv = sub.add_parser("_supervise")
    sv.add_argument("dir")
    sv.add_argument("marker", nargs="?")
    sv.add_argument("--resume", action="store_true")
    a = ap.parse_args(argv)

    if a.verb == "_supervise":
        return supervise(Path(a.dir), resume=a.resume)

    if a.verb == "run":
        targs = [t for t in a.train_args if t != "--"] if a.train_args[:1] == ["--"] else list(a.train_args)
        bad = [e for e in a.env if "=" not in e]
        if bad:
            raise SystemExit(f"--env wants KEY=VALUE, got {bad[0]!r}")
        if a.gpus > 0:
            preflight_memory(targs, a.gpus)  # refuse what cannot fit a GPU before any process is started
        run = create_run(targs, name=a.name, gpus=a.gpus, workers=a.workers, elastic=a.elastic, respawn=a.respawn, grace_s=a.grace,
                         env=dict(e.split("=", 1) for e in a.env))  # fmt: skip
        spawn_supervisor(run, resume=False)
        print(json.dumps({"run": run.spec.id, "dir": str(run.path)}), flush=True)
        return 0 if a.detach else _attach(run)

    if a.verb in ("list", "ls"):
        rows = [r_.describe() for r_ in iter_runs()]
        if a.active:
            rows = [x for x in rows if x["state"] in ACTIVE]
        if a.output == "json":
            print(json.dumps({"runs": rows}, indent=2))
        else:
            for x in rows:
                x["age"] = _age(x["created_at"])
            _print_table(rows, ("id", "name", "state", "workers", "gpus_per_worker", "step", "loss", "tokens_per_s", "age"))
        return 0

    run = find_run(a.run)
    if a.verb == "get":
        print(json.dumps({**run.describe(), "status": run.status(), "spec": asdict(run.spec)}, indent=2))
    elif a.verb == "stop":
        st = stop_run(run, force=a.force)
        print(json.dumps({"run": run.spec.id, "state": st["state"]}))
        return 0 if st["state"] in FINAL else 1
    elif a.verb == "restart":
        if run.status()["state"] in ACTIVE:
            raise SystemExit(f"run {run.spec.id} is still {run.status()['state']}; stop it first")
        spawn_supervisor(run, resume=bool(run.checkpoints()))
        print(json.dumps({"run": run.spec.id, "resumed_from": (run.checkpoints() or [{}])[-1].get("step")}), flush=True)
        return 0 if a.detach else _attach(run)
    elif a.verb == "delete":
        if run.status()["state"] in ACTIVE and not a.force:
            raise SystemExit(f"run {run.spec.id} is still going; stop it first (or --force)")
        if run.status()["state"] in ACTIVE:
            stop_run(run, force=True)
        import shutil

        shutil.rmtree(run.path)
        print(json.dumps({"deleted": run.spec.id}))
    elif a.verb == "checkpoints":
        rows = run.checkpoints()
        if a.output == "json":
            print(json.dumps({"checkpoints": rows}, indent=2))
        else:
            for x in rows:
                x["size"] = f"{x['size_bytes'] / 2**20:.1f} MiB"
                x["age"] = _age(x["written_at"])
            _print_table(rows, ("step", "worker", "files", "size", "age", "path"))
    elif a.verb == "metrics":
        try:
            recs = [json.loads(ln) for ln in run.metrics_path.read_text().splitlines() if ln.strip()]
        except FileNotFoundError:
            recs = []
        recs = recs[-a.last :] if a.last else recs
        if a.output == "json":
            print(json.dumps({"metrics": recs}, indent=2))
        else:
            _print_table(recs, ("step", "loss", "lr", "grad_norm", "tokens_per_s", "mfu", "step_s", "workers", "outer"))
    elif a.verb == "logs":
        path = run.log_path(a.worker)
        if not path.exists() and not a.follow:
            raise SystemExit(f"no log for worker {a.worker} (have: {', '.join(p.stem for p in (run.path / 'logs').glob('*.log'))})")
        until = (lambda: run.status()["state"] in FINAL) if a.follow else (lambda: True)
        try:
            for line in follow(path, tail=a.tail, until=until):
                print(line, flush=True)
        except KeyboardInterrupt:
            pass
    return 0


def _attach(run: Run) -> int:
    """Foreground mode: stream worker 0's log until the run ends. Ctrl-C stops the run (with its final checkpoint), as it
    would a foreground job; use ``--detach`` to leave it running."""
    try:
        for line in follow(run.log_path("w0"), tail=None, until=lambda: run.status()["state"] in FINAL):
            print(line, flush=True)
    except KeyboardInterrupt:
        print("\ninterrupt: stopping the run (final checkpoint) …", file=sys.stderr)
        stop_run(run)
    st = run.status()
    print(json.dumps({"run": run.spec.id, "state": st["state"]}))
    return 0 if st["state"] in ("COMPLETED", "STOPPED") else 1


if __name__ == "__main__":
    sys.exit(main())
