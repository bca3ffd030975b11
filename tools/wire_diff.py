#!/usr/bin/env python
"""Differential wire test: ONE script, written against the reference's import names, runs against the unmodified reference
packages and against this repo (through ``prime_b200.compat``); a recording fake server logs every HTTP request each arm
sends. The request sequences (method, path, query, JSON body) and the outcome of every call must be identical.

    python tools/wire_diff.py > wire_diff.json                 # exit code 1 on any difference
    python tools/wire_diff.py --record tests/golden/reference_wire_diff.json.gz   # store the reference arm (needs the reference)
    python tools/wire_diff.py --reference tests/golden/reference_wire_diff.json.gz   # compare against the stored arm

What it covers: 108 SDK / API-client / MCP-tool calls — sync and async sandbox and evaluation clients, RL, deployments and tunnel clients, the
nine MCP tools; sandbox lifecycle, command execution, file transfer, ports, SSH sessions, bulk delete,
evaluation create / push / finalize / list, pods, disks, availability — and injected failures: 404 / 401 / 402 / 422, a flaky idempotent
GET (retried), a 503 on a non-idempotent POST (not retried), gateway 502 ``sandbox_not_found``, 408, 409. A failure counts as the same
when this repo raises the reference's exception class or a subclass of it. What it cannot cover: responses of the real service.
"""

from __future__ import annotations

import json
import os
import re
import subprocess
import sys
import tempfile
import threading
from http.server import BaseHTTPRequestHandler, ThreadingHTTPServer
from pathlib import Path
from urllib.parse import parse_qsl, urlsplit

ROOT = Path(__file__).resolve().parent.parent
REF = Path(os.environ.get("PRIME_REFERENCE_PACKAGES", "/root/reference/packages"))
REF_PATHS = [str(REF / p / "src") for p in ("prime", "prime-evals", "prime-sandboxes", "prime-tunnel", "prime-mcp-server")]
T = "2025-01-01T00:00:00Z"
SB = {"id": "s1", "name": "bench", "dockerImage": "python:3.11-slim", "startCommand": None, "cpuCores": 2, "memoryGB": 4, "diskSizeGB": 10,
      "diskMountPath": "/workspace", "gpuCount": 0, "gpuType": None, "vm": False, "status": "RUNNING", "timeoutMinutes": 60, "createdAt": T,
      "updatedAt": T, "userId": "u1", "teamId": None}  # fmt: skip
PORT = {"exposure_id": "e1", "sandbox_id": "s1", "port": 8000, "name": "web", "url": "https://x", "tls_socket": "x:443", "protocol": "HTTP"}
POD = {"id": "p1", "name": "pod", "gpuName": "H100_80GB", "gpuCount": 1, "status": "ACTIVE", "createdAt": T, "updatedAt": T, "providerType": "x",
       "installationStatus": "FINISHED", "teamId": None, "socket": "ON_DEMAND", "priceHr": 1.0, "userId": "u1", "type": "HOSTED", "resources": None,
       "ip": "1.2.3.4", "sshConnection": [None]}  # fmt: skip
DISK = {"id": "d1", "name": "disk", "size": 100, "status": "ACTIVE", "createdAt": T, "updatedAt": T, "providerType": "x", "userId": "u1", "teamId": None,
        "priceHr": 0.1, "info": {"country": "US", "dataCenterId": "dc", "cloudId": "c", "isMultinode": False}, "pods": [], "clusters": []}  # fmt: skip


def _spec(default, lo=None, hi=None):
    return {"minCount": lo, "defaultCount": default, "maxCount": hi, "pricePerUnit": 0.01, "step": 1, "defaultIncludedInPrice": True, "additionalInfo": None}


OFFER = {"cloudId": "c1", "gpuType": "B200_180GB", "socket": "SXM6", "provider": "hyperstack", "dataCenter": "dc1", "country": "US", "gpuCount": 8,
         "gpuMemory": 180, "security": "secure_cloud", "prices": {"onDemand": 31.2, "communityPrice": None, "isVariable": False, "currency": "USD"},
         "stockStatus": "Available", "vcpu": _spec(128), "memory": _spec(1024), "disk": _spec(2000, 100, 4000), "isSpot": False,
         "images": ["ubuntu_22_cuda_12"], "region": "united_states", "interconnect": None, "interconnectType": None, "internetSpeed": None,
         "provisioningTime": None, "prepaidTime": None}  # fmt: skip


def respond(method: str, path: str, host: str):
    r = [
        ("POST", r"/api/v1/sandbox/s1/auth$", {"gateway_url": f"http://{host}/gw", "user_ns": "ns", "job_id": "job", "token": "tok", "expires_at": "2099-01-01T00:00:00Z", "is_vm": False}),
        ("POST", r"/api/v1/sandbox/s1/expose$", PORT), ("GET", r"/api/v1/sandbox/s1/expose$", {"exposures": [PORT]}),
        ("GET", r"/api/v1/sandbox/expose/all$", {"exposures": [PORT]}), ("DELETE", r"/api/v1/sandbox/s1/expose/e1$", {}),
        ("POST", r"/api/v1/sandbox/s1/ssh-session$", {"session_id": "ss1", "exposure_id": "e1", "sandbox_id": "s1", "host": "h", "port": 22, "external_endpoint": "h:22", "expires_at": "2099-01-01T00:00:00Z", "ttl_seconds": 600, "gateway_url": "g", "user_ns": "ns", "job_id": "job", "token": "t"}),
        ("DELETE", r"/api/v1/sandbox/s1/ssh-session/ss1$", {}),
        ("GET", r"/api/v1/sandbox/s1/logs$", {"logs": "hello"}), ("GET", r"/api/v1/sandbox/s1/error-context$", {"status": "RUNNING"}),
        ("GET", r"/api/v1/sandbox/s1$", SB), ("DELETE", r"/api/v1/sandbox/s1$", {"status": "deleted"}),
        ("DELETE", r"/api/v1/sandbox$", {"succeeded": ["s1"], "failed": [], "message": "ok"}),
        ("POST", r"/api/v1/sandbox$", SB), ("GET", r"/api/v1/sandbox$", {"sandboxes": [SB], "total": 1, "page": 1, "perPage": 50, "hasNext": False}),
        ("POST", r"/gw/ns/job/exec$", {"stdout": "ok\n", "stderr": "", "exit_code": 0}),
        ("POST", r"/gw/ns/job/upload$", {"success": True, "path": "/tmp/a.txt", "size": 5, "timestamp": T}),
        ("GET", r"/gw/ns/job/read-file$", {"content": "hello", "size": 5}), ("GET", r"/gw/ns/job/download$", b"hello"),
        ("POST", r"/api/v1/environmentshub/resolve$", {"data": {"id": "env1", "created": True, "owner": {"name": "owner", "type": "user"}, "name": "myenv"}}),
        ("POST", r"/api/v1/environmentshub/env1/wheels$", {"data": {"wheel_id": "w1", "upload_url": f"http://{host}/upload/wheel"}}),
        ("POST", r"/api/v1/environmentshub/env1/wheels/w1/finalize$", {"data": {"success": True}}),
        ("POST", r"/api/v1/environmentshub/env1/versions$", {"data": {"version_id": "v1", "upload_url": f"http://{host}/upload/source"}}),
        ("POST", r"/api/v1/environmentshub/env1/versions/v1/finalize$", {"data": {"success": True, "message": "ok"}}),
        ("PUT", r"/upload/(wheel|source)$", {}),
        ("GET", r"/api/v1/environmentshub/$", {"data": [{"owner": {"name": "owner"}, "name": "env", "description": "sums", "visibility": "PUBLIC", "latest_version": "0.2.0", "stars": 3, "updated_at": "2026-01-02T03:04:05Z", "latest_ci_status": "SUCCESS", "tags": ["t"]}], "total_count": 41}),
        ("GET", r"/api/v1/environmentshub/owner/env/status$", {"data": {"name": "env", "visibility": "PUBLIC", "latest_version": {"semantic_version": "0.2.0", "content_hash": "abcdef0123456789", "created_at": "2026-01-02T03:04:05Z"}, "action": {"status": "FAILED", "job_id": "j1"}}}),
        ("GET", r"/api/v1/environmentshub/owner/env/versions$", {"data": {"versions": [{"version": "0.2.0", "created_at": "2026-01-02T03:04:05Z", "sha256": "a" * 64, "size": 2}, {"version": "0.1.0", "created_at": "2025-01-02", "sha256": "b" * 64, "size": 1}]}}),
        ("GET", r"/api/v1/environmentshub/owner/env/actions$", {"data": {"total": 30, "actions": [{"id": "A1", "job_type": "integration", "status": "RUNNING", "version": {"content_hash": "deadbeefcafe"}, "trigger": "push", "created_at": "2026-01-02T03:04:05Z"}]}}),
        ("GET", r"/api/v1/environmentshub/owner/env/actions/A1/logs$", {"data": {"logs": "line one\nline two"}}),
        ("GET", r"/api/v1/secrets/sec1$", {"data": {"id": "sec1", "name": "HF_TOKEN", "description": "hub", "isFile": False, "createdAt": "2026-01-02T03:04:05Z", "updatedAt": "2026-01-02T03:04:05Z"}}),
        ("GET", r"/api/v1/secrets/$", {"data": [{"id": "sec1", "name": "HF_TOKEN", "description": "hub", "isFile": False, "createdAt": "2026-01-02T03:04:05Z", "updatedAt": "2026-01-02T03:04:05Z"}]}),
        ("GET", r"/api/v1/teams/t1/members$", {"data": [{"userId": "u1", "userName": "Ada", "userEmail": "a@b.c", "role": "admin", "joinedAt": "2026-01-02T03:04:05Z"}]}),
        ("GET", r"/api/v1/template/registry-credentials$", {"credentials": [{"id": "c1", "name": "ghcr", "server": "ghcr.io", "createdAt": "2026-01-02T03:04:05Z", "updatedAt": "2026-01-02T03:04:05Z", "userId": "u", "teamId": None}]}),
        ("POST", r"/api/v1/template/check-docker-image$", {"accessible": True, "details": "pull ok"}),
        ("GET", r"/api/v1/models$", {"object": "list", "data": [{"id": "meta/llama", "created": 1767322245, "pricing": {"input_usd_per_mtok": 0.2, "output_usd_per_mtok": 0.6}}, {"id": "q/qwen"}]}),
        ("POST", r"/api/v1/hosted-evaluations$", {"evaluation_id": "ev1", "evaluation_ids": ["ev1"], "status": "PENDING"}),
        ("GET", r"/api/v1/environmentshub/owner/env2?/@latest$", {"data": {"id": "env1", "name": "env", "owner": "owner"}}),
        ("POST", r"/api/v1/environmentshub/lookup$", {"data": {"id": "env1"}}), ("GET", r"/api/v1/environmentshub/", {"data": {"id": "env1"}}),
        ("POST", r"/api/v1/evaluations/ev1/samples$", {"status": "ok"}), ("POST", r"/api/v1/evaluations/ev1/finalize$", {"evaluation_id": "ev1", "status": "COMPLETED"}),
        ("GET", r"/api/v1/evaluations/ev1/samples$", {"samples": [], "total": 0}), ("GET", r"/api/v1/evaluations/ev1$", {"evaluation_id": "ev1", "name": "n"}),
        ("PUT", r"/api/v1/evaluations/ev1$", {"evaluation_id": "ev1"}), ("POST", r"/api/v1/evaluations/$", {"evaluation_id": "ev1", "id": "ev1"}),
        ("GET", r"/api/v1/evaluations/$", {"evaluations": [], "total": 0}),
        ("GET", r"/api/v1/pods/status$", {"data": [{"podId": "p1", "providerType": "x", "status": "ACTIVE", "sshConnection": [None], "ip": "1.2.3.4"}]}),
        ("GET", r"/api/v1/pods/history$", {"total_count": 1, "offset": 0, "limit": 100, "data": [{"id": "h1", "name": "old", "providerType": "x", "type": "HOSTED", "gpuName": "H100_80GB", "count": 8, "createdAt": "2025-01-01T00:00:00Z", "terminatedAt": "2025-01-01T05:30:00Z", "priceHr": 2.5, "totalBilledPrice": 13.75, "teamId": None, "userId": "u1"}]}),
        ("GET", r"/api/v1/rft/runs/r1/logs$", {"logs": "l1\nl2"}), ("GET", r"/api/v1/rft/runs/r1/metrics$", {"metrics": [{"step": 1, "reward": 0.5}]}),
        ("GET", r"/api/v1/rft/runs/r1/rollouts$", {"samples": [], "total": 0}), ("GET", r"/api/v1/rft/runs/r1/progress$", {"latest_step": 3}),
        ("GET", r"/api/v1/rft/runs/r1/distributions$", {"bins": []}), ("GET", r"/api/v1/rft/runs/r1/checkpoints$", {"checkpoints": []}),
        ("GET", r"/api/v1/rft/runs/r1$", {"run": {"id": "r1", "name": "run", "userId": "u1", "teamId": None, "status": "RUNNING", "baseModel": "Qwen/Qwen3-4B", "environments": [{"id": "owner/env"}], "rolloutsPerExample": 8, "seqLen": 2048, "maxSteps": 10, "batchSize": 32, "createdAt": T, "updatedAt": T}}), ("PUT", r"/api/v1/rft/runs/r1/(stop|restart)$", {"run": {"id": "r1", "name": "run", "userId": "u1", "teamId": None, "status": "RUNNING", "baseModel": "Qwen/Qwen3-4B", "environments": [{"id": "owner/env"}], "rolloutsPerExample": 8, "seqLen": 2048, "maxSteps": 10, "batchSize": 32, "createdAt": T, "updatedAt": T}}),
        ("DELETE", r"/api/v1/rft/runs/r1$", {}), ("POST", r"/api/v1/rft/runs$", {"run": {"id": "r1", "name": "run", "userId": "u1", "teamId": None, "status": "RUNNING", "baseModel": "Qwen/Qwen3-4B", "environments": [{"id": "owner/env"}], "rolloutsPerExample": 8, "seqLen": 2048, "maxSteps": 10, "batchSize": 32, "createdAt": T, "updatedAt": T}}), ("GET", r"/api/v1/rft/runs$", {"runs": [{"id": "r1", "name": "run", "userId": "u1", "teamId": None, "status": "RUNNING", "baseModel": "Qwen/Qwen3-4B", "environments": [{"id": "owner/env"}], "rolloutsPerExample": 8, "seqLen": 2048, "maxSteps": 10, "batchSize": 32, "createdAt": T, "updatedAt": T}]}),
        ("GET", r"/api/v1/rft/models$", {"models": [{"name": "Qwen/Qwen3-4B", "atCapacity": False}]}),
        ("GET", r"/api/v1/rft/adapters/a1$", {"adapter": {"id": "a1", "displayName": "run-1", "userId": "u1", "teamId": None, "rftRunId": "r1", "baseModel": "Qwen/Qwen3-4B", "step": 10, "status": "READY", "deploymentStatus": "NOT_DEPLOYED", "createdAt": T, "updatedAt": T}}),
        ("POST", r"/api/v1/rft/adapters/a1/(deploy|unload)$", {"adapter": {"id": "a1", "displayName": "run-1", "userId": "u1", "teamId": None, "rftRunId": "r1", "baseModel": "Qwen/Qwen3-4B", "step": 10, "status": "READY", "deploymentStatus": "DEPLOYING", "createdAt": T, "updatedAt": T}}),
        ("GET", r"/api/v1/tunnel/t1$", {"tunnel_id": "t1", "hostname": "t1.example", "url": "https://t1.example", "frp_token": "tok", "server_host": "frp.example", "server_port": 7000, "expires_at": "2099-01-01T00:00:00Z", "status": "active", "local_port": 8080, "name": "web", "binding_secret": "b"}), ("DELETE", r"/api/v1/tunnel/t1$", {"success": True}), ("DELETE", r"/api/v1/tunnel$", {"succeeded": ["t1"], "failed": []}),
        ("POST", r"/api/v1/tunnel$", {"tunnel_id": "t1", "hostname": "t1.example", "url": "https://t1.example", "frp_token": "tok", "server_host": "frp.example", "server_port": 7000, "expires_at": "2099-01-01T00:00:00Z", "status": "active", "local_port": 8080, "name": "web", "binding_secret": "b"}), ("GET", r"/api/v1/tunnel$", {"tunnels": [{"tunnel_id": "t1", "hostname": "t1.example", "url": "https://t1.example", "frp_token": "tok", "server_host": "frp.example", "server_port": 7000, "expires_at": "2099-01-01T00:00:00Z", "status": "active", "local_port": 8080, "name": "web", "binding_secret": "b"}]}),
        ("GET", r"/api/v1/rft/adapters$", {"adapters": [{"id": "a1", "displayName": "run-1", "userId": "u1", "teamId": None, "rftRunId": "r1", "baseModel": "Qwen/Qwen3-4B", "step": 10, "status": "READY", "deploymentStatus": "NOT_DEPLOYED", "createdAt": "2025-01-01T00:00:00Z", "updatedAt": "2025-01-01T00:00:00Z"}], "total": 1}),
        ("GET", r"/api/v1/rft/deployable-models$", {"models": ["Qwen/Qwen3-4B"]}),
        ("GET", r"/api/v1/user/whoami$", {"data": {"id": "u1", "email": "a@b.c", "name": "A", "scope": {"pods": {"read": True, "write": True}}}}),
        ("GET", r"/api/v1/user/teams$", {"data": [{"teamId": "t1", "name": "Team", "slug": "team", "role": "ADMIN", "createdAt": "2025-01-01T00:00:00Z"}]}),
        ("GET", r"/api/v1/pods/p1$", POD), ("DELETE", r"/api/v1/pods/p1$", {}), ("POST", r"/api/v1/pods/?$", POD),
        ("GET", r"/api/v1/pods/?$", {"total_count": 1, "offset": 0, "limit": 100, "data": [POD]}),
        ("GET", r"/api/v1/disks/d1$", DISK), ("DELETE", r"/api/v1/disks/d1$", {"status": "deleted"}), ("PATCH", r"/api/v1/disks/d1$", {"status": "ok"}),
        ("POST", r"/api/v1/disks/?$", DISK), ("GET", r"/api/v1/disks/?$", {"total_count": 1, "offset": 0, "limit": 100, "data": [DISK]}),
        ("GET", r"/api/v1/availability/gpus$", {"items": [OFFER, {**OFFER, "cloudId": "c2", "gpuCount": 1, "dataCenter": "dc2", "prices": {"onDemand": 4.1, "currency": "USD"}}], "totalCount": 2}),
        ("GET", r"/api/v1/availability/multi-node$", {"items": [], "totalCount": 0}),
        ("GET", r"/api/v1/ssh_keys/?$", {"data": [{"id": "k1", "name": "k", "publicKey": "ssh-ed25519 AAAA test", "isPrimary": True}], "total_count": 1}),
        ("POST", r"/api/v1/ssh_keys/?$", {"id": "k2", "name": "k"}), ("DELETE", r"/api/v1/ssh_keys/k1$", {}),
        ("GET", r"/api/v1/availability/gpu-summary$", {"H100_80GB": {}}), ("GET", r"/api/v1/availability/disks$", {"items": []}),
        ("GET", r"/api/v1/availability/?", {"H100_80GB": []}),
    ]  # fmt: skip
    for m, pat, body in r:
        if m == method and re.search(pat, path):
            return body
    return {}


FLAKY: dict[str, int] = {}


LOGIN: dict[str, str] = {}


def scripted_failure(method: str, path: str, query: dict, payload):
    """Failure injection keyed by what the client asks for (both arms ask for the same things): → (status, body) or None."""
    cmd = payload.get("command") if isinstance(payload, dict) else None
    if path.endswith("/auth_challenge/generate") and isinstance(payload, dict):  # `prime login`: remember the client's ephemeral public key
        LOGIN["pem"] = payload.get("encryptionPublicKey", "")
        return 200, {"challenge": "ABCD-1234", "status_auth_token": "status-token"}
    if path.endswith("/auth_challenge/status"):  # … and hand the new API key back encrypted for it (RSA-OAEP / SHA-256), as the service does
        import base64

        from cryptography.hazmat.primitives import hashes, serialization
        from cryptography.hazmat.primitives.asymmetric import padding

        pub = serialization.load_pem_public_key(LOGIN["pem"].encode())
        blob = pub.encrypt(b"pit_new_api_key", padding.OAEP(mgf=padding.MGF1(algorithm=hashes.SHA256()), algorithm=hashes.SHA256(), label=None))
        return 200, {"result": base64.b64encode(blob).decode()}
    if path.endswith("/sandbox/missing"):
        return 404, {"detail": "Sandbox not found"}
    if path.endswith("/sandbox/unauth"):
        return 401, {"detail": "Invalid API key"}
    if path.endswith("/sandbox/broke"):
        return 402, {"detail": "Insufficient funds"}
    if path.endswith("/sandbox/invalid"):
        return 422, {"detail": [{"loc": ["body", "cpu_cores"], "msg": "too many", "type": "value_error"}]}
    if path.endswith("/read-file") and query.get("path") == "/flaky":  # idempotent: retried on 5xx
        FLAKY["read"] = FLAKY.get("read", 0) + 1
        if FLAKY["read"] % 3 != 0:
            return 503, {"detail": "try again"}
    if path.endswith("/exec") and cmd == "five-oh-three":  # not idempotent: the server may have seen it — no retry
        return 503, {"detail": "upstream"}
    if path.endswith("/exec") and cmd == "gone":
        return 502, {"error": "sandbox_not_found", "detail": "sandbox_not_found"}
    if path.endswith("/exec") and cmd == "slow":
        return 408, {"detail": "timeout"}
    if path.endswith("/exec") and cmd == "conflict":
        return 409, {"detail": "Sandbox is not running"}
    if path.endswith("/sandbox/dead/error-context"):
        return 200, {"status": "TERMINATED", "errorType": "OOM_KILLED", "errorMessage": "out of memory"}
    return None


class Recorder(BaseHTTPRequestHandler):
    protocol_version = "HTTP/1.1"
    log: list = []
    lock = threading.Lock()

    def log_message(self, *a):  # noqa: D102
        pass

    def _handle(self):
        u = urlsplit(self.path)
        n = int(self.headers.get("Content-Length") or 0)
        raw = self.rfile.read(n) if n else b""
        if u.path == "/__log":
            body = json.dumps(Recorder.log).encode()
            Recorder.log = []
        else:
            ctype = self.headers.get("Content-Type", "")
            if "json" in ctype and raw:
                payload = json.loads(raw)
            elif "multipart" in ctype:
                payload = {"multipart_bytes": "<file>", "has_hello": b"hello" in raw}
            elif "octet-stream" in ctype:
                import hashlib

                payload = {"bytes": len(raw), "sha256": hashlib.sha256(raw).hexdigest()} if u.path.endswith("/wheel") else {"bytes": "<tarball>", "gzip": raw[:2] == b"\x1f\x8b"}
            else:
                payload = raw.decode("utf-8", "replace") if raw else None
            with Recorder.lock:
                Recorder.log.append({"method": self.command, "path": u.path, "query": sorted(parse_qsl(u.query)), "body": payload,
                                     "auth": self.headers.get("Authorization")})  # fmt: skip
            code, out = scripted_failure(self.command, u.path, dict(parse_qsl(u.query)), payload) or (200, respond(self.command, u.path, self.headers.get("Host")))
            body = out if isinstance(out, bytes) else json.dumps(out).encode()
            head = f"HTTP/1.1 {code} X\r\nContent-Type: application/json\r\nContent-Length: {len(body)}\r\n\r\n".encode()
            self.wfile.write(head + body)
            self.wfile.flush()
            return
        head = f"HTTP/1.1 200 OK\r\nContent-Type: application/json\r\nContent-Length: {len(body)}\r\n\r\n".encode()
        self.wfile.write(head + body)
        self.wfile.flush()

    do_GET = do_POST = do_PUT = do_DELETE = do_PATCH = _handle  # noqa: N815


SCENARIO = r'''
import json, os, sys, tempfile
if sys.argv[1] == "ours":
    import prime_b200.compat as compat
    compat.install()
from prime_sandboxes import APIClient, CreateSandboxRequest, SandboxClient
from prime_evals import EvalsClient
from prime_evals import APIClient as EvalsAPI
from prime_cli.core import APIClient as CliAPI
from prime_cli.api.pods import PodsClient
from prime_cli.api.disks import DisksClient
from prime_cli.api.availability import AvailabilityClient

results = []
def call(label, fn):
    try:
        r = fn()
        if hasattr(r, "model_dump"):
            r = r.model_dump(mode="json")
        elif isinstance(r, list) and r and hasattr(r[0], "model_dump"):
            r = [x.model_dump(mode="json") for x in r]
        elif isinstance(r, dict):
            r = {k: (v.model_dump(mode="json") if hasattr(v, "model_dump") else ([x.model_dump(mode="json") if hasattr(x, "model_dump") else x for x in v] if isinstance(v, list) else v)) for k, v in r.items()}
        results.append([label, "ok", json.loads(json.dumps(r, default=str))])
    except Exception as e:
        results.append([label, "raised", [type(e).__name__, str(e)[:160], [k.__name__ for k in type(e).__mro__]]])

tmp = tempfile.mkdtemp()
src = os.path.join(tmp, "a.txt"); open(src, "w").write("hello")
c = SandboxClient(APIClient(api_key="k"))
call("create", lambda: c.create(CreateSandboxRequest(name="bench", docker_image="python:3.11-slim", cpu_cores=2, memory_gb=4, disk_size_gb=10, timeout_minutes=60, labels=["a", "b"], environment_vars={"X": "1"})))
call("get", lambda: c.get("s1"))
call("list", lambda: c.list(status="RUNNING", labels=["a"], page=2, per_page=10, exclude_terminated=True))
call("list_default", lambda: c.list())
call("logs", lambda: c.get_logs("s1"))
call("exec", lambda: c.execute_command("s1", "echo ok", working_dir="/w", env={"A": "1"}, timeout=7))
call("exec_default", lambda: c.execute_command("s1", "true"))
call("upload", lambda: c.upload_file("s1", "/tmp/a.txt", src))
call("upload_bytes", lambda: c.upload_bytes("s1", "/tmp/b.txt", b"hello", "b.txt"))
call("read", lambda: c.read_file("s1", "/tmp/a.txt"))
call("download", lambda: c.download_file("s1", "/tmp/a.txt", os.path.join(tmp, "out.txt")))
call("expose", lambda: c.expose("s1", 8000, name="web"))
call("list_ports", lambda: c.list_exposed_ports("s1"))
call("list_all_ports", lambda: c.list_all_exposed_ports())
call("unexpose", lambda: c.unexpose("s1", "e1"))
call("ssh_open", lambda: c.create_ssh_session("s1", ttl_seconds=600))
call("ssh_close", lambda: c.close_ssh_session("s1", "ss1"))
call("wait", lambda: c.wait_for_creation("s1", max_attempts=2))
call("bulk_wait", lambda: c.bulk_wait_for_creation(["s1"], max_attempts=2))
call("bulk_delete_ids", lambda: c.bulk_delete(sandbox_ids=["s1"]))
call("bulk_delete_labels", lambda: c.bulk_delete(labels=["a"]))
call("delete", lambda: c.delete("s1"))

def background():
    job = c.start_background_job("s1", "sleep 1 && echo done", working_dir="/w", env={"A": "1"})
    st = c.get_background_job("s1", job)
    return {"files": [job.stdout_log_file[:9], job.exit_file[-5:]], "completed": st.completed}
call("background_job", background)
call("run_background_job", lambda: {"completed": c.run_background_job("s1", "echo hi", timeout=5, poll_interval=1).completed})
call("err_404", lambda: c.get("missing"))
call("err_401", lambda: c.get("unauth"))
call("err_402", lambda: c.get("broke"))
call("err_422", lambda: c.get("invalid"))
call("retry_get_5xx", lambda: c.read_file("s1", "/flaky"))
call("no_retry_post_5xx", lambda: c.execute_command("s1", "five-oh-three"))
call("gateway_gone", lambda: c.execute_command("s1", "gone"))
call("gateway_408", lambda: c.execute_command("s1", "slow", timeout=3))
call("gateway_409", lambda: c.execute_command("s1", "conflict"))

e = EvalsClient(EvalsAPI(api_key="k"))
call("eval_create", lambda: e.create_evaluation(name="n", environments=[{"id": "env1"}], model_name="m", framework="verifiers", metadata={"k": 1}, metrics={"r": 0.5}))
call("eval_create_slug", lambda: e.create_evaluation(name="n2", environments=["owner/env"], model_name="m"))
call("eval_push", lambda: e.push_samples("ev1", [{"example_id": i, "reward": 0.5, "task": "t"} for i in range(5)]))
call("eval_finalize", lambda: e.finalize_evaluation("ev1", metrics={"r": 1.0}))
call("eval_get", lambda: e.get_evaluation("ev1"))
call("eval_list", lambda: e.list_evaluations(env_name="x", skip=5, limit=10))
call("eval_samples", lambda: e.get_samples("ev1", page=2, limit=5))
call("eval_update", lambda: e.update_evaluation("ev1", name="renamed"))

api = CliAPI(api_key="k")
pods, disks, av = PodsClient(api), DisksClient(api), AvailabilityClient(api)
call("pods_list", lambda: pods.list(offset=5, limit=10))
call("pods_get", lambda: pods.get("p1"))
call("pods_status", lambda: pods.get_status(["p1"]))
call("pods_history", lambda: pods.history())
call("pods_create", lambda: pods.create({"pod": {"name": "x", "gpuType": "H100_80GB", "gpuCount": 1}, "provider": {"type": "x"}}))
call("pods_delete", lambda: pods.delete("p1"))
call("disks_list", lambda: disks.list())
call("disks_get", lambda: disks.get("d1"))
call("disks_update", lambda: disks.update("d1", "newname"))
call("disks_delete", lambda: disks.delete("d1"))
call("avail_get", lambda: av.get(regions=["united_states"], gpu_count=8, gpu_type="H100_80GB"))
call("avail_disks", lambda: av.get_disks(regions=["united_states"]))
from prime_cli.api.rl import RLClient
from prime_cli.api.deployments import DeploymentsClient
rl, dep = RLClient(api), DeploymentsClient(api)
call("rl_list", lambda: rl.list_runs(team_id="t1"))
call("rl_models", lambda: rl.list_models())
call("rl_get", lambda: rl.get_run("r1"))
call("rl_stop", lambda: rl.stop_run("r1"))
call("rl_restart", lambda: rl.restart_run("r1"))
call("rl_delete", lambda: rl.delete_run("r1"))
call("rl_logs", lambda: rl.get_logs("r1", tail_lines=50))
call("rl_metrics", lambda: rl.get_metrics("r1", min_step=1, max_step=9, limit=5))
call("rl_rollouts", lambda: rl.get_rollouts("r1", step=3, page=2, limit=10))
call("rl_progress", lambda: rl.get_progress("r1"))
call("rl_distributions", lambda: rl.get_distributions("r1", distribution_type="reward", step=3))
call("rl_checkpoints", lambda: rl.list_checkpoints("r1"))
call("rl_env_status", lambda: rl.get_environment_status("owner", "env"))
call("rl_create", lambda: rl.create_run(model_name="Qwen/Qwen3-4B", environments=[{"id": "owner/env"}], rollouts_per_example=8, max_steps=10, batch_size=32))
call("dep_list", lambda: dep.list_adapters(team_id="t1", limit=20, offset=40))
call("dep_get", lambda: dep.get_adapter("a1"))
call("dep_deployable", lambda: dep.get_deployable_models())
call("dep_deploy", lambda: dep.deploy_adapter("a1"))
call("dep_unload", lambda: dep.unload_adapter("a1"))

import asyncio
from prime_sandboxes import AsyncSandboxClient
from prime_evals import AsyncEvalsClient
from prime_tunnel.core.client import TunnelClient

async def async_part():
    async def acall(label, coro_fn):
        try:
            r = await coro_fn()
            if hasattr(r, "model_dump"):
                r = r.model_dump(mode="json")
            elif isinstance(r, list) and r and hasattr(r[0], "model_dump"):
                r = [x.model_dump(mode="json") for x in r]
            results.append([label, "ok", json.loads(json.dumps(r, default=str))])
        except Exception as e:
            results.append([label, "raised", [type(e).__name__, str(e)[:160], [k.__name__ for k in type(e).__mro__]]])
    ac = AsyncSandboxClient(api_key="k")
    await acall("a_create", lambda: ac.create(CreateSandboxRequest(name="bench", docker_image="python:3.11-slim", cpu_cores=2, memory_gb=4)))
    await acall("a_get", lambda: ac.get("s1"))
    await acall("a_list", lambda: ac.list(labels=["a"], per_page=5))
    await acall("a_exec", lambda: ac.execute_command("s1", "echo ok", timeout=9))
    await acall("a_upload", lambda: ac.upload_file("s1", "/tmp/a.txt", src))
    await acall("a_read", lambda: ac.read_file("s1", "/tmp/a.txt"))
    await acall("a_expose", lambda: ac.expose("s1", 8000, name="web"))
    await acall("a_bulk_delete", lambda: ac.bulk_delete(sandbox_ids=["s1"]))
    await acall("a_missing", lambda: ac.get("missing"))
    await acall("a_delete", lambda: ac.delete("s1"))
    await ac.aclose()
    ae = AsyncEvalsClient(api_key="k")
    await acall("a_eval_create", lambda: ae.create_evaluation(name="n", environments=[{"id": "env1"}], model_name="m"))
    await acall("a_eval_push", lambda: ae.push_samples("ev1", [{"example_id": i, "reward": 1.0} for i in range(3)]))
    await acall("a_eval_finalize", lambda: ae.finalize_evaluation("ev1"))
    await ae.aclose()
    tc = TunnelClient(api_key="k")
    await acall("t_create", lambda: tc.create_tunnel(8080, name="web"))
    await acall("t_list", lambda: tc.list_tunnels())
    await acall("t_get", lambda: tc.get_tunnel("t1"))
    await acall("t_delete", lambda: tc.delete_tunnel("t1"))
    await acall("t_bulk_delete", lambda: tc.bulk_delete_tunnels(["t1", "t2"]))
    await tc.close()

asyncio.run(async_part())

# Tunnel lifecycle with a stand-in for the frpc binary (a script that keeps a copy of the config it is started with and prints the
# line both SDKs wait for): register -> 0600 config -> child process -> "connected" -> stop -> delete
import importlib, stat
tun_mod = importlib.import_module("prime_tunnel.tunnel")
fake = os.path.join(tmp, "frpc")
open(fake, "w").write("#!/bin/sh\ncp \"$2\" \"" + tmp + "/frpc_config_seen.toml\"\necho 'login to server success'\necho 'start proxy success'\nsleep 30\n")
os.chmod(fake, 0o755)
tun_mod.get_frpc_path = lambda *a, **k: __import__("pathlib").Path(fake)

async def tunnel_part():
    from prime_tunnel import Tunnel
    t = Tunnel(8080, name="web", connection_timeout=10.0)
    try:
        url = await t.start()
        cfg = open(os.path.join(tmp, "frpc_config_seen.toml")).read()
        lines = [ln for ln in cfg.splitlines() if ln.strip() and not ln.lstrip().startswith("#")]
        results.append(["tunnel_start", "ok", {"url": url, "tunnel_id": t.tunnel_id, "running": t.is_running, "frpc_config": lines}])
        await t.stop()
        results.append(["tunnel_stop", "ok", {"running": t.is_running}])
    except Exception as e:
        results.append(["tunnel_start", "raised", [type(e).__name__, str(e)[:300], [k.__name__ for k in type(e).__mro__]]])

asyncio.run(tunnel_part())

# MCP server: the nine tools, called as the plain async functions they are (FastMCP's decorator returns them unchanged)
try:
    import importlib
    mcp_mod = importlib.import_module("prime_mcp.mcp")  # not `import prime_mcp.mcp as m`: the package re-exports the FastMCP object under that name
except Exception as e:  # the optional `mcp` dependency is not installed
    mcp_mod = None
    results.append(["mcp_import", "raised", [type(e).__name__, str(e)[:80], [k.__name__ for k in type(e).__mro__]]])

async def mcp_part():
    async def tcall(label, coro_fn):
        try:
            r = await coro_fn()
            results.append([label, "ok", json.loads(json.dumps(r, default=str))])
        except Exception as e:
            results.append([label, "raised", [type(e).__name__, str(e)[:160], [k.__name__ for k in type(e).__mro__]]])
    m = mcp_mod
    await tcall("mcp_gpu_availability", lambda: m.check_gpu_availability(gpu_type="B200_180GB", regions="united_states", gpu_count=8))
    await tcall("mcp_cluster_availability", lambda: m.check_cluster_availability(gpu_count=16, gpu_type="B200_180GB"))
    await tcall("mcp_list_pods", lambda: m.list_pods(offset=5, limit=10))
    await tcall("mcp_pod_details", lambda: m.get_pod_details("p1"))
    await tcall("mcp_pods_status", lambda: m.get_pods_status(["p1"]))
    await tcall("mcp_pods_history", lambda: m.get_pods_history(limit=10, offset=0))
    await tcall("mcp_create_pod", lambda: m.create_pod(cloud_id="c1", gpu_type="B200_180GB", provider_type="hyperstack", data_center_id="dc1", name="mcp-pod", gpu_count=8, disk_size=2000, image="ubuntu_22_cuda_12"))
    await tcall("mcp_delete_pod", lambda: m.delete_pod("p1"))
    await tcall("mcp_ssh_keys_list", lambda: m.manage_ssh_keys(action="list"))
    await tcall("mcp_ssh_keys_add", lambda: m.manage_ssh_keys(action="add", key_name="k", public_key="ssh-ed25519 AAAA test"))
    await tcall("mcp_ssh_keys_delete", lambda: m.manage_ssh_keys(action="delete", key_id="k1"))
    await tcall("mcp_ssh_keys_primary", lambda: m.manage_ssh_keys(action="set_primary", key_id="k1"))
    await tcall("mcp_ssh_keys_bad_action", lambda: m.manage_ssh_keys(action="rotate"))
    await tcall("mcp_ssh_keys_add_missing", lambda: m.manage_ssh_keys(action="add", key_name="k"))
    await tcall("mcp_gpu_availability_all", lambda: m.check_gpu_availability())
    await tcall("mcp_pods_status_empty", lambda: m.get_pods_status([]))

if mcp_mod is not None:
    asyncio.run(mcp_part())
print(json.dumps(results))
'''


def read_json(path) -> object:
    """JSON from ``path``; gzip-compressed when the name ends in ``.gz`` (the recorded reference arms under tests/golden/)."""
    import gzip

    raw = Path(path).read_bytes()
    return json.loads(gzip.decompress(raw) if str(path).endswith(".gz") else raw)


def write_json(path, obj) -> None:
    import gzip

    raw = (json.dumps(obj, sort_keys=True, separators=(",", ":")) + "\n").encode()
    Path(path).write_bytes(gzip.compress(raw, mtime=0) if str(path).endswith(".gz") else raw)


def run_arm(arm: str, base: str) -> tuple[list, list]:
    import urllib.request

    with tempfile.TemporaryDirectory() as home:
        env = {**os.environ, "HOME": home, "PRIME_API_BASE_URL": base, "PRIME_BASE_URL": base, "PRIME_API_KEY": "k", "PRIME_DISABLE_VERSION_CHECK": "1",
               "PYTHONPATH": os.pathsep.join(REF_PATHS if arm == "reference" else [str(ROOT)])}  # fmt: skip
        env.pop("PRIME_TEAM_ID", None)
        r = subprocess.run([sys.executable, "-c", SCENARIO, arm], env=env, capture_output=True, text=True, cwd=home, timeout=600)
    if r.returncode != 0:
        raise SystemExit(f"{arm}: {r.stderr[-3000:]}")
    results = json.loads(r.stdout.strip().splitlines()[-1])
    log = json.loads(urllib.request.urlopen(base + "/__log").read())
    return results, log


def covers(ours, ref) -> bool:
    """Does ``ours`` contain everything ``ref`` says? dict: every reference key present with a covering value (extra keys allowed);
    list: same length, element-wise; scalars: equal."""
    if isinstance(ref, dict):
        return isinstance(ours, dict) and all(k in ours and covers(ours[k], v) for k, v in ref.items())
    if isinstance(ref, list):
        return isinstance(ours, list) and len(ours) == len(ref) and all(covers(a, b) for a, b in zip(ours, ref))
    return ours == ref


def normalise(log: list) -> list:
    """Drop client-generated identifiers so that two runs are comparable (request ids; the random id in a background job's file names)."""
    out = []
    for e in log:
        e = dict(e)
        if isinstance(e["body"], dict):
            e["body"] = {k: (re.sub(r"job_[0-9a-f]{8}", "job_XXXXXXXX", v) if isinstance(v, str) else v) for k, v in e["body"].items() if k not in ("request_id",)}
        e["query"] = [[k, re.sub(r"job_[0-9a-f]{8}", "job_XXXXXXXX", v) if isinstance(v, str) else v] for k, v in e.get("query", [])]
        out.append(e)
    return out


def main(reference: str | Path | None = None, record: str | Path | None = None) -> int:
    """``reference``: a JSON file with the reference arm's outcomes and normalised request log, written earlier by ``record``; the
    reference packages are then not needed. Without it the reference arm runs from REF (and ``record`` stores what it produced)."""
    srv = ThreadingHTTPServer(("127.0.0.1", 0), Recorder)
    srv.daemon_threads = True
    threading.Thread(target=srv.serve_forever, daemon=True).start()
    base = f"http://127.0.0.1:{srv.server_address[1]}"
    if reference is not None:
        rec = read_json(reference)
        ref_res, ref_log = [tuple(r) for r in rec["results"]], rec["requests"]
    else:
        ref_res, ref_log = run_arm("reference", base)
        ref_log = normalise(ref_log)
        if record is not None:
            write_json(record, {"results": ref_res, "requests": ref_log})
    our_res, our_log = run_arm("ours", base)
    our_log = normalise(our_log)
    diffs, wording = [], []
    for (la, sa, va), (lb, sb, vb) in zip(ref_res, our_res):
        if (la, sa) != (lb, sb):
            diffs.append({"call": la, "reference": [sa, va], "ours": [sb, vb]})
        elif sa == "raised":
            # same failure ⇔ what this repo raises IS-A what the reference raises (an ``except`` written for the reference still
            # catches it); the message text is informational — the reference's five packages word the same error differently
            if va[0] not in vb[2]:
                diffs.append({"call": la, "reference": va[:2], "ours": vb[:2]})
            elif va[:2] != vb[:2]:
                wording.append({"call": la, "reference": va[:2], "ours": vb[:2]})
        elif not covers(vb, va):  # parsed results: every field the reference's model has, with the same value (this repo's models may add fields)
            diffs.append({"call": la, "reference": [sa, va], "ours": [sb, vb]})
    req_diffs = []
    for i in range(max(len(ref_log), len(our_log))):
        a = ref_log[i] if i < len(ref_log) else None
        b = our_log[i] if i < len(our_log) else None
        if a != b:
            req_diffs.append({"index": i, "reference": a, "ours": b})
    out = {"calls": len(ref_res), "requests_reference": len(ref_log), "requests_ours": len(our_log), "outcome_differences": diffs,
           "same_exception_class_different_wording": wording,
           "request_differences": req_diffs[:40], "outcomes": {lab: (st if st == "ok" else f"raised {v[0]}") for lab, st, v in our_res}}  # fmt: skip
    print(json.dumps(out, indent=1))
    srv.shutdown()
    return 1 if diffs or req_diffs else 0


if __name__ == "__main__":
    import argparse

    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", default=None, help="recorded reference arm (JSON) instead of running the reference packages")
    ap.add_argument("--record", default=None, help="write the reference arm's outcomes and request log to this JSON file")
    a = ap.parse_args()
    sys.exit(main(a.reference, a.record))
