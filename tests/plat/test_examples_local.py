"""This repo's own sandbox examples, run end to end against tools/local_sandbox_service.py (commands really execute, files really move,
exposed ports are really reachable) — nothing mocked on the client side."""

import os
import stat
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))


def run_example(name: str, tmp_path: Path, *argv: str, extra_env: dict | None = None, path_prefix: Path | None = None, timeout: int = 240):
    from tools import local_sandbox_service as svc_mod

    old_path = os.environ["PATH"]
    if path_prefix is not None:  # the service runs sandbox commands with ITS environment: stub binaries go in front of its PATH
        os.environ["PATH"] = f"{path_prefix}:{old_path}"
    httpd, svc = svc_mod.serve(0)
    try:
        env = {k: v for k, v in os.environ.items() if not k.startswith("PRIME_")}
        env.update(HOME=str(tmp_path), PRIME_API_BASE_URL=f"http://127.0.0.1:{httpd.server_address[1]}", PRIME_API_KEY="local-key",
                   PRIME_DISABLE_VERSION_CHECK="1", PYTHONPATH=str(ROOT), **(extra_env or {}))  # fmt: skip
        p = subprocess.run([sys.executable, str(ROOT / "examples" / name), *argv], env=env, cwd=tmp_path, capture_output=True, text=True, timeout=timeout,
                           stdin=subprocess.DEVNULL)  # fmt: skip
        created = len(svc.sandboxes)
        running = sum(1 for s in svc.sandboxes.values() if s.status != "TERMINATED")
        records = [s.record() for s in svc.sandboxes.values()]
        return p, created, running, records
    finally:
        os.environ["PATH"] = old_path
        httpd.shutdown()
        svc.close()


@pytest.mark.slow
@pytest.mark.parametrize("name", ["sandbox_quickstart.py", "sandbox_files.py", "sandbox_background_job.py", "sandbox_expose_port.py", "sandbox_async_fanout.py"])
def test_own_examples_run_and_clean_up(name, tmp_path):
    p, created, running, _ = run_example(name, tmp_path)
    assert p.returncode == 0, p.stdout[-1500:] + p.stderr[-1500:]
    assert created >= 1 and running == 0  # every example deletes what it made


@pytest.mark.slow
def test_tailnet_example_with_stub_tailscale(tmp_path):
    """examples/sandbox_tailnet_ssh.py against stand-in `tailscaled` / `tailscale` binaries: the daemon runs as a background job and is
    waited for through its socket, the auth key reaches `tailscale up` as a sandbox secret (environment) and is in no record or output."""
    bin_dir = tmp_path / "bin"
    bin_dir.mkdir()
    # the service maps the sandbox's /tmp under its scratch root, so the socket's host path can exceed the 108-byte AF_UNIX limit
    # when the temporary directory is deep: bind by basename from inside the socket's directory (the limit applies to that string)
    (bin_dir / "tailscaled").write_text(
        f"#!{sys.executable}\nimport os, socket, sys, time\n"
        "path = [a.split('=', 1)[1] for a in sys.argv if a.startswith('--socket=')][0]\n"
        "os.chdir(os.path.dirname(path) or '.')\n"
        "s = socket.socket(socket.AF_UNIX); s.bind(os.path.basename(path)); s.listen(1); time.sleep(120)\n")  # fmt: skip
    (bin_dir / "tailscale").write_text(
        "#!/bin/bash\nshift  # --socket=…\ncase \"$1\" in\n"
        "  up) [[ \"$*\" == *\"--authkey=tskey-test-123\"* ]] || { echo 'bad key' >&2; exit 1; } ;;\n"
        "  ip) echo 100.64.0.7 ;;\nesac\n")  # fmt: skip
    for f in bin_dir.iterdir():
        f.chmod(f.stat().st_mode | stat.S_IEXEC)
    p, created, running, records = run_example("sandbox_tailnet_ssh.py", tmp_path, extra_env={"TS_AUTHKEY": "tskey-test-123"}, path_prefix=bin_dir)
    assert p.returncode == 0, p.stdout[-1500:] + p.stderr[-1500:]
    assert "on the tailnet as 100.64.0.7" in p.stdout and "@100.64.0.7" in p.stdout and "sandbox deleted" in p.stdout
    assert created == 1 and running == 0
    assert "tskey-test-123" not in p.stdout + p.stderr and "tskey-test-123" not in str(records)
    # without the key the example refuses before it creates anything
    q, created, _, _ = run_example("sandbox_tailnet_ssh.py", tmp_path)
    assert q.returncode != 0 and "TS_AUTHKEY is not set" in q.stderr and created == 0
