#!/usr/bin/env python
"""Differential CLI test: the same ``prime …`` command lines through the unmodified reference CLI and through this repo's CLI,
against the recording fake server of ``tools/wire_diff.py``. Compared per command: exit code, the HTTP requests sent (method,
path, query, JSON body) and — where the command prints JSON (``--output json``) — the parsed JSON: every key and value of the
reference's JSON must be present in this CLI's (which may add keys).

    python tools/cli_diff.py > cli_diff.json                   # exit code 1 on any difference
    python tools/cli_diff.py [6] --record tests/golden/reference_cli_diff.json.gz  # store the reference CLI's side for that stride (needs the reference)
    python tools/cli_diff.py --reference tests/golden/reference_cli_diff.json.gz  # compare against the stored side
"""

from __future__ import annotations

import json
import os
import shutil
import subprocess
import sys
import tempfile
import threading
import urllib.request
from http.server import ThreadingHTTPServer
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from tools.wire_diff import REF_PATHS, Recorder, covers, read_json, write_json  # noqa: E402

COMMANDS: list[list[str]] = [
    ["pods", "list", "--output", "json"], ["pods", "list", "--limit", "10", "--offset", "5", "-o", "json"], ["pods", "status", "p1", "-o", "json"],
    ["pods", "history", "-o", "json"], ["pods", "terminate", "p1", "--yes"],
    ["disks", "list", "-o", "json"], ["disks", "get", "d1", "-o", "json"], ["disks", "update", "d1", "--name", "newname"], ["disks", "terminate", "d1", "--yes"],
    ["availability", "list", "--gpu-type", "B200_180GB", "--gpu-count", "8", "-o", "json"], ["availability", "gpu-types"], ["availability", "disks", "-o", "json"],
    ["sandbox", "list", "-o", "json"], ["sandbox", "list", "--status", "RUNNING", "--label", "a", "--page", "2", "--num", "10", "-o", "json"],
    ["sandbox", "get", "s1", "-o", "json"], ["sandbox", "run", "s1", "echo ok"], ["sandbox", "logs", "s1"], ["sandbox", "delete", "s1", "--yes"],
    ["sandbox", "create", "--name", "bench", "--cpu-cores", "2", "--memory-gb", "4", "--yes", "python:3.11-slim"],
    ["sandbox", "expose", "s1", "8000", "--name", "web"], ["sandbox", "list-ports", "s1", "-o", "json"], ["sandbox", "unexpose", "s1", "e1", "--yes"],
    ["sandbox", "get", "missing"], ["sandbox", "get", "unauth"],
    ["eval", "list", "-o", "json"], ["eval", "get", "ev1", "-o", "json"], ["eval", "samples", "ev1", "-o", "json"],
    ["teams", "list", "-o", "json"], ["whoami"], ["secret", "list", "-o", "json"], ["env", "list", "-o", "json"], ["registry", "list", "-o", "json"],
    ["images", "list", "-o", "json"], ["rl", "list", "-o", "json"], ["rl", "models", "-o", "json"], ["rl", "get", "r1", "-o", "json"], ["deployments", "list", "-o", "json"],
    ["inference", "models", "-o", "json"], ["config", "view"], ["config", "set-team-id", "team-1"], ["config", "view"], ["--version"],
    # second batch: mutating commands and the remaining groups
    ["secret", "get", "sec1", "-o", "json"], ["secret", "create", "--name", "TOKEN", "--value", "v"], ["secret", "update", "sec1", "--name", "NEW"],
    ["secret", "delete", "sec1", "--yes"],
    ["env", "status", "owner/env"], ["env", "info", "owner/env"], ["env", "version", "list", "owner/env"], ["env", "action", "list", "owner/env"],
    ["env", "secret", "list", "owner/env"], ["env", "var", "list", "owner/env"], ["env", "delete", "owner/env", "--force"],
    ["rl", "stop", "r1", "--force"], ["rl", "delete", "r1", "--force"], ["rl", "restart", "r1", "--force"], ["rl", "logs", "r1", "--tail", "10"],
    ["rl", "metrics", "r1"], ["rl", "rollouts", "r1", "--step", "1"], ["rl", "progress", "r1"], ["rl", "distributions", "r1"],
    ["tunnel", "list"], ["tunnel", "status", "t1"], ["teams", "members", "--team-id", "t1", "-o", "json"],
    ["registry", "check-image", "python:3.11-slim"], ["images", "delete", "img:tag", "--yes"],
    ["config", "set-base-url", "http://example.invalid"], ["config", "set-frontend-url", "http://front.invalid"], ["config", "set-ssh-key-path", "/tmp/key"],
    ["config", "remove-team-id"], ["config", "set-share-resources-with-team", "true"], ["config", "view"],
    ["sandbox", "reset-cache", "--yes"], ["eval", "stop", "ev1"], ["eval", "logs", "ev1"], ["switch"], ["pods", "connect", "--help"],
    ["sandbox", "create", "--help"], ["env", "push", "--help"], ["rl", "run", "--help"],
    ["availability", "list", "--gpu-type", "B200_180GB", "-o", "json"], ["availability", "list", "--gpu-type", "B200_180GB", "--no-group-similar", "-o", "json"],
    # creation flows (flags only, no prompts): offer lookup by short id, explicit disk location, VM / GPU sandbox, bulk deletes
    ["pods", "create", "--id", "32fb75", "--name", "diffpod", "--disk-size", "2000", "--vcpus", "128", "--memory", "1024", "--image", "ubuntu_22_cuda_12", "--yes"],
    ["pods", "create", "--id", "nope00", "--yes"],
    ["disks", "create", "--size", "100", "--name", "d", "--country", "US", "--cloud-id", "c", "--data-center-id", "dc", "--provider-type", "x", "--yes"],
    ["sandbox", "create", "--name", "x", "--gpu-count", "1", "--gpu-type", "H100_80GB", "--vm", "--yes", "img:tag"],
    ["sandbox", "create", "--env", "A=1", "--env", "B=2", "--label", "l1", "--timeout-minutes", "30", "--yes", "python:3.11-slim"],
    ["sandbox", "delete", "--all", "--yes"], ["sandbox", "delete", "--label", "a", "--yes"], ["secret", "create", "--name", "N", "--value", "v", "--description", "d"],
    # the packaging pipeline (SURVEY §3.4): build the wheel, resolve, wheel upload + finalize, source archive upload + finalize
    ["env", "push", "--path", "myenv", "--visibility", "PRIVATE"], ["env", "push", "--path", "myenv", "--auto-bump"],
    # hosted evaluations (SURVEY §3.2): one environment from flags, sandbox access + secrets, a TOML file with two [[eval]] tables
    ["eval", "run", "owner/env", "--hosted", "-m", "org/m", "-n", "5", "-r", "2", "--eval-name", "diff-eval", "--timeout-minutes", "30"],
    ["eval", "run", "owner/env", "--hosted", "-m", "org/m", "--allow-sandbox-access", "--custom-secrets", '{"A": "1"}'],
    ["eval", "run", "evals.toml", "--hosted"],
    ["env", "init", "my-new-env"], ["env", "pull", "owner/env"], ["env", "uninstall", "myenv"], ["lab", "--help"], ["gepa", "--help"], ["upgrade", "--help"],
    # read commands against realistic payloads, JSON mode
    ["env", "list", "--output", "json"], ["env", "list", "--output", "json", "--search", "ma", "--page", "2", "-n", "20"], ["env", "status", "owner/env", "--output", "json"],
    ["env", "version", "list", "owner/env", "--output", "json"], ["env", "action", "list", "owner/env", "--output", "json"], ["env", "action", "logs", "owner/env", "A1"],
    ["secret", "list", "-o", "json"], ["secret", "get", "sec1", "-o", "json"], ["teams", "members", "--team-id", "t1", "-o", "json"], ["teams", "list", "-o", "json"],
    ["registry", "list", "-o", "json"], ["registry", "check-image", "ghcr.io/ok/img:1"], ["inference", "models", "-o", "json"], ["whoami"],
    ["images", "push", "app:v1", "--context", "ctx"], ["images", "push", "app:v1", "--context", "ctx", "--dockerfile", "ctx/Dockerfile", "--platform", "linux/amd64"],
    ["sandbox", "run", "s1", "--working-dir", "/w", "--env", "A=1", "--timeout", "7", "echo hi"], ["sandbox", "run", "s1", "sleep 1"],
    ["tunnel", "stop", "t1", "--yes"], ["tunnel", "stop", "t1,t2", "--yes"], ["tunnel", "stop", "--all", "--yes"],
    # the local evaluation path (model validation + billing preflight, then verifiers in a child process) and a hub install
    ["eval", "run", "owner/env", "-m", "org/m", "-n", "2", "-r", "1", "--skip-upload"], ["env", "install", "owner/env"],
    # the browser challenge login, headless: ephemeral RSA key, encrypted API key back, whoami, team choice (EOF → personal)
    ["login", "--headless"], ["config", "view"],
    # named contexts and account switching: save / use / --context / switch / reset, compared through the files they leave behind
    ["config", "set-api-key", "k-123"], ["config", "save", "staging"], ["config", "set-base-url", "http://other.invalid"], ["config", "save", "other"], ["config", "envs"],
    ["config", "use", "staging"], ["config", "view"], ["--context", "other", "config", "view"], ["--context", "nope", "config", "view"], ["switch", "team"],
    ["switch", "personal"], ["switch", "t1"], ["config", "reset", "--yes"], ["config", "use", "production"], ["config", "envs"],
    # environment secrets / variables, deployments, checkpoints, pushes into an existing evaluation or a training run
    ["env", "secret", "create", "owner/env", "--name", "TOKEN", "--value", "v", "--description", "d", "-o", "json"], ["env", "secret", "update", "owner/env", "--id", "es1", "--value", "v2"],
    ["env", "secret", "delete", "owner/env", "--id", "es1", "--yes"], ["env", "secret", "link", "sec1", "owner/env"], ["env", "secret", "unlink", "sec1", "owner/env", "--yes"],
    ["env", "var", "create", "owner/env", "--name", "VAR", "--value", "1"], ["deployments", "create", "a1", "--yes"], ["deployments", "delete", "a1"],
    ["rl", "checkpoints", "r1", "-o", "json"], ["rl", "models", "-o", "json"], ["eval", "push", "outputs/evals/gsm8k--org--m/run1", "--run-id", "r1"],
    ["eval", "push", "outputs/evals/gsm8k--org--m/run1", "--eval", "ev1", "-o", "json"], ["env", "action", "retry", "owner/env", "A1"],
    ["env", "version", "delete", "owner/env", "aaaaaaaa", "--force"], ["images", "list", "-o", "json"],
    ["config", "set-inference-url", "http://inf.invalid/api/v1"], ["rl", "ls", "-o", "json"], ["sandbox", "ls", "-o", "json"], ["env", "var", "update", "ev1", "owner/env", "--value", "2"],
    ["env", "var", "delete", "ev1", "owner/env", "--yes"], ["env", "build", "--help"], ["gepa", "run", "--help"], ["lab", "setup", "--help"], ["eval", "tui", "--help"],
    # invalid input: bad option values, missing arguments, failed validation, unknown names — same exit codes, and no request before the check
    ["pods", "list", "-o", "yaml"], ["sandbox", "list", "--page", "0"], ["sandbox", "create"], ["sandbox", "create", "--env", "BAD", "--yes", "img"], ["disks", "create", "--size", "0", "--yes"],
    ["rl", "list", "--num", "0"], ["env", "list", "--sort", "bogus"], ["env", "version", "delete", "owner/env", "abc"], ["sandbox", "delete"], ["sandbox", "delete", "s1", "--all", "--yes"],
    ["tunnel", "stop"], ["eval", "push", "/nonexistent"], ["eval", "samples"], ["secret", "create"], ["config", "use", "nope"], ["config", "save", "production"], ["rl", "run", "missing.toml"],
    ["nosuchcommand"], ["sandbox", "expose", "s1", "8000", "--protocol", "udp"], ["availability", "list", "--regions", "mars"], ["pods", "terminate"], ["deployments", "create"], ["rl", "get"],
    # third batch: flows that read or write local files
    ["rl", "run", "rl.toml"], ["rl", "run", "rl.toml", "-e", "WANDB_MODE=offline", "-o", "json"], ["rl", "init", "template.toml"],
    ["sandbox", "upload", "s1", "a.txt", "/tmp/a.txt"], ["sandbox", "download", "s1", "/tmp/a.txt", "got.txt"],
    ["eval", "push", "outputs/evals/gsm8k--org--m/run1", "--env", "owner/env"], ["eval", "push", "--env", "owner/env", "-o", "json"],
    ["eval", "push", "verifiers_example", "--env", "owner/env"], ["eval", "push", "verifiers_example", "-o", "json"],
]  # fmt: skip


RL_TOML = """model = "Qwen/Qwen3-4B-Instruct-2507"
name = "diff-run"
max_steps = 20
batch_size = 64
rollouts_per_example = 4
learning_rate = 1e-5

[[env]]
id = "owner/env"
args = { difficulty = "hard" }

[sampling]
max_tokens = 512
temperature = 0.8

[checkpoints]
interval = 10
"""


def prepare_files(home: Path) -> None:
    """Inputs of the file-based command lines, identical in both arms' working directories."""
    (home / "rl.toml").write_text(RL_TOML)
    (home / "a.txt").write_text("hello")
    (home / "ctx").mkdir()
    (home / "ctx" / "Dockerfile").write_text("FROM python:3.11-slim\nCOPY app.py /app.py\n")
    (home / "ctx" / "app.py").write_text("print(1)\n")
    (home / "evals.toml").write_text('model = "org/m"\nnum_examples = 5\nrollouts_per_example = 2\n\n[[eval]]\nenv_id = "owner/env"\n\n[[eval]]\nenv_id = "owner/env2"\nnum_examples = 7\n')
    make_env_project(home / "myenv")
    sample = Path(os.environ.get("PRIME_REFERENCE_ROOT", "/root/reference")) / "examples" / "verifiers_example"
    if sample.is_dir():  # the reference's own verifiers-format sample (SURVEY §2 row 75), pushed as it ships
        shutil.copytree(sample, home / "verifiers_example")
    run = home / "outputs" / "evals" / "gsm8k--org--m" / "run1"
    run.mkdir(parents=True)
    (run / "metadata.json").write_text(json.dumps({"env_id": "gsm8k", "env": "gsm8k", "model": "org/m", "num_examples": 2, "rollouts_per_example": 1,
                                                    "avg_reward": 0.5, "date": "2025-01-01", "time": "00:00:00", "sampling_args": {"max_tokens": 16}}))  # fmt: skip
    (run / "results.jsonl").write_text("\n".join(json.dumps({"example_id": i, "reward": 0.5, "task": "t", "prompt": [{"role": "user", "content": "q"}],
                                                              "completion": [{"role": "assistant", "content": "a"}]}) for i in range(2)))  # fmt: skip


ENV_BACKEND = '''
import base64, hashlib, io, os, tarfile, zipfile
NAME, VER = "myenv", "0.1.0"
META = f"Metadata-Version: 2.1\\\\nName: {NAME}\\\\nVersion: {VER}\\\\nSummary: diff env\\\\nRequires-Python: >=3.10\\\\nRequires-Dist: verifiers>=0.1.0\\\\n"
def _zi(name):
    z = zipfile.ZipInfo(name, date_time=(2020, 1, 1, 0, 0, 0)); z.external_attr = 0o644 << 16; return z
def build_wheel(wheel_directory, config_settings=None, metadata_directory=None):
    fn = f"{NAME}-{VER}-py3-none-any.whl"
    files = {"myenv.py": open("myenv.py", "rb").read(), f"{NAME}-{VER}.dist-info/METADATA": META.encode(),
             f"{NAME}-{VER}.dist-info/WHEEL": b"Wheel-Version: 1.0\\\\nGenerator: diff\\\\nRoot-Is-Purelib: true\\\\nTag: py3-none-any\\\\n"}
    rec = "".join(f"{k},sha256={base64.urlsafe_b64encode(hashlib.sha256(v).digest()).rstrip(b'=').decode()},{len(v)}\\\\n" for k, v in files.items())
    files[f"{NAME}-{VER}.dist-info/RECORD"] = (rec + f"{NAME}-{VER}.dist-info/RECORD,,\\\\n").encode()
    with zipfile.ZipFile(os.path.join(wheel_directory, fn), "w") as z:
        for k, v in files.items(): z.writestr(_zi(k), v)
    return fn
def build_sdist(sdist_directory, config_settings=None):
    fn = f"{NAME}-{VER}.tar.gz"
    with tarfile.open(os.path.join(sdist_directory, fn), "w:gz") as t:
        for f in ("pyproject.toml", "myenv.py", "README.md", "backend.py"):
            t.add(f, arcname=f"{NAME}-{VER}/{f}")
    return fn
def get_requires_for_build_wheel(config_settings=None): return []
def get_requires_for_build_sdist(config_settings=None): return []
'''


def make_env_project(d: Path) -> None:
    """A minimal verifiers environment whose wheel builds OFFLINE: an in-tree PEP 517 backend (no build requirements to download)
    that writes a deterministic wheel — both CLIs build byte-identical archives, so content hashes and uploads are comparable."""
    d.mkdir(parents=True, exist_ok=True)
    (d / "pyproject.toml").write_text('[project]\nname = "myenv"\nversion = "0.1.0"\ndescription = "diff env"\ntags = ["test"]\nrequires-python = ">=3.10"\n'
                                      'dependencies = ["verifiers>=0.1.0"]\n\n[build-system]\nrequires = []\nbuild-backend = "backend"\nbackend-path = ["."]\n')
    (d / "myenv.py").write_text("def load_environment(**kw):\n    return None\n")
    (d / "README.md").write_text("# myenv\n")
    (d / "backend.py").write_text(ENV_BACKEND)


def toml_of(path: Path):
    try:
        import tomllib

        return tomllib.loads(path.read_text())
    except Exception:  # noqa: BLE001
        return None


def run_cli(arm: str, base: str, home: str, args: list[str]) -> tuple[int, str, str]:
    code = "from prime_cli.main import run; run()" if arm == "reference" else "from prime_b200.platform.main import run; run()"
    env = {**os.environ, "HOME": home, "PRIME_API_BASE_URL": base, "PRIME_BASE_URL": base, "PRIME_INFERENCE_URL": base + "/api/v1", "PRIME_API_KEY": "k",
           "PRIME_DISABLE_VERSION_CHECK": "1", "NO_COLOR": "1", "COLUMNS": "200", "TERM": "dumb", "UV_OFFLINE": "1",
           "PYTHONPATH": os.pathsep.join(REF_PATHS if arm == "reference" else [str(ROOT)])}  # fmt: skip
    env.pop("PRIME_TEAM_ID", None)
    r = subprocess.run([sys.executable, "-c", f"import sys; sys.argv = ['prime', *{args!r}]; {code}"], env=env, capture_output=True, text=True,
                       cwd=home, timeout=120, stdin=subprocess.DEVNULL)  # fmt: skip
    return r.returncode, r.stdout, r.stderr


def parsed_json(stdout: str):
    s = stdout.strip()
    for opener in ("{", "["):
        i = s.find(opener)
        if i >= 0:
            try:
                return json.loads(s[i:])
            except json.JSONDecodeError:
                continue
    return None


def mask(req: dict) -> dict:
    """Auto-generated names carry a random 4-character suffix (``python-x7k2``): compare everything but the suffix."""
    import re

    body = req.get("body")
    if isinstance(body, dict) and isinstance(body.get("name"), str):
        req = {**req, "body": {**body, "name": re.sub(r"-[a-z0-9]{4}$", "-XXXX", body["name"])}}
    if isinstance(body, dict) and "encryptionPublicKey" in body:  # `prime login`: a fresh RSA key pair per run
        req = {**req, "body": {**body, "encryptionPublicKey": "<ephemeral public key>" if "BEGIN PUBLIC KEY" in str(body["encryptionPublicKey"]) else body["encryptionPublicKey"]}}
    if req.get("path", "").endswith("/versions") and isinstance(body, dict) and "sha256" in body:
        # the source tarball embeds file and gzip timestamps: its digest differs between two runs of the SAME CLI; the content hash
        # (over the source files) and the wheel digest are the comparable identifiers
        req = {**req, "body": {**req["body"], "sha256": "<tarball digest>"}}
    return req


def same_or_fewer_reads(ours: list, ref: list) -> tuple[bool, int]:
    """Identical, or this CLI sends the same requests minus some read-only GETs (it skips a lookup whose result the reference does
    not use, or fails a local precondition before listing) → (acceptable, number of GETs saved)."""
    ours, ref = [mask(r) for r in ours], [mask(r) for r in ref]
    if ours == ref:
        return True, 0
    i = 0
    dropped = []
    for r in ref:
        if i < len(ours) and ours[i] == r:
            i += 1
        else:
            dropped.append(r)
    ok = i == len(ours) and all(r["method"] == "GET" for r in dropped)
    return ok, len(dropped) if ok else 0


def main(stride: int = 1, reference: str | Path | None = None, record: str | Path | None = None) -> int:
    """``stride`` > 1 runs every stride-th command line (the test suite's quick pass). ``reference``: a JSON file with the reference
    CLI's exit codes, requests, JSON output and ~/.prime files per command line, written earlier by ``record`` (a full run); the
    reference packages are then not needed. Recordings are kept per stride: a command's requests depend on what the commands before
    it left in ~/.prime (a cached sandbox gateway token, say)."""
    recorded = read_json(reference)[str(stride)] if reference is not None else None
    to_record: dict = {"commands": {}}
    srv = ThreadingHTTPServer(("127.0.0.1", 0), Recorder)
    srv.daemon_threads = True
    threading.Thread(target=srv.serve_forever, daemon=True).start()
    base = f"http://127.0.0.1:{srv.server_address[1]}"
    rows, diffs = [], []
    with tempfile.TemporaryDirectory() as h1, tempfile.TemporaryDirectory() as h2:
        for h in (h1, h2):
            prepare_files(Path(h))
        for args in COMMANDS[::stride]:
            got = {}
            key = " ".join(args)
            for arm, home in (("reference", h1), ("ours", h2)):
                if arm == "reference" and recorded is not None:
                    got[arm] = {**recorded["commands"][key], "stdout_tail": "", "stderr_tail": ""}
                    continue
                rc, out, err = run_cli(arm, base, home, args)
                log = json.loads(urllib.request.urlopen(base + "/__log").read())
                got[arm] = {"exit_code": rc, "requests": [{k: e[k] for k in ("method", "path", "query", "body")} for e in log], "json": parsed_json(out),
                            "stdout_tail": out.strip()[-300:], "stderr_tail": err.strip()[-300:]}  # fmt: skip
            arms = (("ours", h2),) if recorded is not None else (("reference", h1), ("ours", h2))
            if args[:2] == ["env", "init"]:  # the scaffold each CLI wrote: same files, same contents
                for arm, home in arms:
                    root = Path(home) / "environments"
                    got[arm]["json"] = {str(p.relative_to(home)): (p.read_text() if p.is_file() else None) for p in sorted(root.rglob("*"))} if root.exists() else None
            if args[:2] == ["rl", "init"]:  # the template each CLI wrote: compare what it configures, not its comments
                for arm, home in arms:
                    got[arm]["json"] = toml_of(Path(home) / args[2])
            a, b = got["reference"], got["ours"]
            to_record["commands"][key] = {k: a[k] for k in ("exit_code", "requests", "json")}
            row = {"command": "prime " + " ".join(args), "exit_code": b["exit_code"], "requests": len(b["requests"]),
                   "same_exit_code": a["exit_code"] == b["exit_code"], "same_requests": same_or_fewer_reads(b["requests"], a["requests"])[0],
                   "reads_saved": same_or_fewer_reads(b["requests"], a["requests"])[1],
                   # JSON contract: every key / value the reference prints is printed here (this CLI may add keys); nothing to compare when
                   # the reference printed no JSON (e.g. its "No images found" text in JSON mode)
                   "same_json": covers(b["json"], a["json"]) if a["json"] is not None else None}  # fmt: skip
            rows.append(row)
            if not (row["same_exit_code"] and row["same_requests"] and row["same_json"] in (True, None)):
                diffs.append({"command": row["command"], "reference": a, "ours": b})
        # what the commands left on disk: users who switch keep their ~/.prime
        state = {}
        for arm, home in (("reference", h1), ("ours", h2)):
            if arm == "reference" and recorded is not None:
                state[arm] = recorded["dot_prime"]
                continue
            d = Path(home) / ".prime"
            files = {}
            for f in sorted(d.rglob("*.json")) if d.exists() else []:
                try:
                    files[str(f.relative_to(d))] = json.loads(f.read_text())
                except (OSError, ValueError):
                    files[str(f.relative_to(d))] = "<unreadable>"
            state[arm] = files

        def stable(v, home):  # expiry stamps of cached gateway tokens differ run to run; paths under the arm's private $HOME → "~";
            # the recording server's address (a free port per run) → "<server>"
            if isinstance(v, dict):
                return {k: stable(x, home) for k, x in v.items() if k not in ("cached_at", "expires_at", "last_check", "timestamp")}
            if isinstance(v, list):
                return [stable(x, home) for x in v]
            return v.replace(home, "~").replace(base, "<server>") if isinstance(v, str) else v

        ref_state = state["reference"] if recorded is not None else stable(state["reference"], h1)
        on_disk_same = stride > 1 or covers(stable(state["ours"], h2), ref_state)
        if record is not None and recorded is None:
            to_record["dot_prime"] = stable(state["reference"], h1)
            everything = read_json(record) if Path(record).exists() else {}
            everything[str(stride)] = to_record
            write_json(record, everything)
        if not on_disk_same:
            diffs.append({"command": "<files under ~/.prime after the run>", "reference": {"exit_code": 0, "requests": [], "json": state["reference"], "stdout_tail": "", "stderr_tail": ""},
                          "ours": {"exit_code": 0, "requests": [], "json": state["ours"], "stdout_tail": "", "stderr_tail": ""}})  # fmt: skip
    print(json.dumps({"commands": len(rows), "files_under_dot_prime": sorted(state["ours"]), "files_under_dot_prime_identical": on_disk_same, "read_only_requests_saved": sum(r["reads_saved"] for r in rows), "identical": sum(1 for r in rows if r["same_exit_code"] and r["same_requests"] and r["same_json"] in (True, None)),
                      "rows": rows, "differences": diffs}, indent=1))  # fmt: skip
    srv.shutdown()
    return 1 if diffs else 0


if __name__ == "__main__":
    import argparse

    ap = argparse.ArgumentParser()
    ap.add_argument("stride", nargs="?", type=int, default=1)
    ap.add_argument("--reference", default=None, help="recorded reference CLI (JSON) instead of running the reference packages")
    ap.add_argument("--record", default=None, help="add the reference CLI's results for this stride to this JSON file")
    a = ap.parse_args()
    sys.exit(main(a.stride, a.reference, a.record))
