import json
import os

import httpx
import pytest

from prime_b200.platform.core import (
    APIClient,
    APIError,
    APITimeoutError,
    AsyncAPIClient,
    Config,
    PaymentRequiredError,
    RetryPolicy,
    UnauthorizedError,
    ValidationError,
)
from prime_b200.platform.core.client import IDEMPOTENT_RETRY, TRANSPORT_RETRY


def test_config_env_over_file(isolated_home, monkeypatch):
    c = Config()
    c.set_api_key("file-key")
    assert Config().api_key == "file-key"
    monkeypatch.setenv("PRIME_API_KEY", "env-key")
    assert Config().api_key == "env-key"
    monkeypatch.setenv("PRIME_API_BASE_URL", "https://x.example/api/v1/")
    assert Config().base_url == "https://x.example"


def test_config_contexts(isolated_home, monkeypatch):
    c = Config()
    c.set_api_key("k1")
    c.set_base_url("https://staging.example")
    assert c.save_environment("my staging!") == "my_staging_"
    c.set_base_url("https://other.example")
    assert "my_staging_" in c.list_environments() and "production" in c.list_environments()
    assert c.load_environment("my staging!")
    assert Config().base_url == "https://staging.example" and Config().current_environment == "my_staging_"
    # PRIME_CONTEXT selects without persisting
    c.load_environment("production")
    monkeypatch.setenv("PRIME_CONTEXT", "my_staging_")
    assert Config().base_url == "https://staging.example"
    monkeypatch.delenv("PRIME_CONTEXT")
    assert Config().base_url == "https://api.primeintellect.ai"
    with pytest.raises(ValueError):
        c.save_environment("production")


def test_sdk_config_is_read_only(isolated_home):
    c = Config(writable=False)
    assert not (isolated_home / ".prime").exists()
    with pytest.raises(PermissionError):
        c.set_api_key("x")


def _client(handler, **kw):
    return APIClient(api_key="k", transport=httpx.MockTransport(handler), **kw)


def test_prefix_auth_and_204():
    seen = {}

    def h(req):
        seen["url"], seen["auth"] = str(req.url), req.headers["authorization"]
        return httpx.Response(204)

    assert _client(h).delete("/pods/1") == {}
    assert seen["url"].endswith("/api/v1/pods/1") and seen["auth"] == "Bearer k"
    assert _client(h).get("pods") == {} and seen["url"].endswith("/api/v1/pods")


@pytest.mark.parametrize("code,exc", [(401, UnauthorizedError), (402, PaymentRequiredError)])
def test_status_mapping(code, exc):
    with pytest.raises(exc):
        _client(lambda r: httpx.Response(code, json={"detail": "no"})).get("/x")


def test_422_and_generic():
    detail = [{"loc": ["body", "model", "name"], "msg": "field required"}]
    with pytest.raises(ValidationError) as e:
        _client(lambda r: httpx.Response(422, json={"detail": detail})).post("/x", json={})
    assert "model.name: field required" in str(e.value)
    with pytest.raises(APIError, match="HTTP 500: boom"):
        _client(lambda r: httpx.Response(500, json={"detail": "boom"})).get("/x")
    with pytest.raises(APIError, match="not a dictionary"):
        _client(lambda r: httpx.Response(200, json=[1])).get("/x")


def test_timeout_and_no_key(isolated_home):
    def h(req):
        raise httpx.ReadTimeout("slow", request=req)

    with pytest.raises(APITimeoutError):
        _client(h).get("/x")
    with pytest.raises(APIError, match="No API key"):
        APIClient(transport=httpx.MockTransport(lambda r: httpx.Response(200, json={}))).get("/x")


class FlakyTransport(httpx.BaseTransport):
    """Fails N times with a connection error, then succeeds (reference idea: prime-sandboxes/tests/test_client_retry.py:9-57)."""

    def __init__(self, failures, exc=httpx.ConnectError):
        self.failures, self.calls, self.exc = failures, 0, exc

    def handle_request(self, request):
        self.calls += 1
        if self.calls <= self.failures:
            raise self.exc("nope", request=request)
        return httpx.Response(200, json={"ok": True})


def test_transport_retry_counts(monkeypatch):
    monkeypatch.setattr("time.sleep", lambda s: None)
    t = FlakyTransport(2)
    assert APIClient(api_key="k", transport=t, retry=TRANSPORT_RETRY).get("/x") == {"ok": True}
    assert t.calls == 3
    t = FlakyTransport(5)
    with pytest.raises(APIError):
        APIClient(api_key="k", transport=t, retry=TRANSPORT_RETRY).get("/x")
    assert t.calls == 3
    t = FlakyTransport(1)
    with pytest.raises(APIError):
        APIClient(api_key="k", transport=t).get("/x")  # default: no retry
    assert t.calls == 1


def test_timeouts_retry_only_for_idempotent_verbs(monkeypatch):
    monkeypatch.setattr("time.sleep", lambda s: None)
    t = FlakyTransport(1, exc=httpx.ReadTimeout)
    assert APIClient(api_key="k", transport=t, retry=IDEMPOTENT_RETRY).get("/x") == {"ok": True}
    t = FlakyTransport(1, exc=httpx.ReadTimeout)
    with pytest.raises(APITimeoutError):
        APIClient(api_key="k", transport=t, retry=IDEMPOTENT_RETRY).post("/x", json={})
    assert t.calls == 1


def test_retry_policy_delay_bounds():
    p = RetryPolicy(attempts=3, base_delay=0.1, max_delay=2.0)
    assert all(0 < p.delay(i) <= 2.0 for i in range(10))


@pytest.mark.anyio
async def test_async_client_roundtrip():
    async def h(req):
        return httpx.Response(200, json={"path": req.url.path, "body": json.loads(req.content or b"{}")})

    async with AsyncAPIClient(api_key="k", transport=httpx.MockTransport(h)) as c:
        r = await c.post("/sandbox", json={"a": 1})
    assert r == {"path": "/api/v1/sandbox", "body": {"a": 1}}


def test_reference_helper_names_are_importable():
    """Drop-in names of the reference's utils (SURVEY §2.2.1 #4-#6, #13)."""
    from prime_b200.platform.utils import display, formatters, json_help, plain

    assert formatters.obfuscate_secrets({"HF_TOKEN": "hf_abc", "K": "v"}) == {"HF_TOKEN": "***", "K": "***"}
    assert formatters.format_gpu_spec("B200_180GB", 8) == "B200_180GB x8"
    assert formatters.format_file_size(12) == "12 bytes" and formatters.format_file_size(1536) == "1.5 KB" and formatters.format_file_size(5 << 30) == "5.0 GB"
    assert json_help.json_help(".id = string").startswith("JSON output:")
    assert display.get_eval_viewer_url("ev1").endswith("/dashboard/evaluations/ev1")
    assert plain.PrimeConsole is plain.Out and plain.PlainAwareTyperGroup is plain.PlainGroup


def test_package_export_surfaces_match_the_reference():
    """Every name the five reference packages export from their __init__ resolves here too (SURVEY §2.1)."""
    import prime_b200.platform as P
    import prime_b200.platform.evals as E
    import prime_b200.platform.mcp as M
    import prime_b200.platform.sandboxes as S
    import prime_b200.platform.tunnel as Tn

    for name in ("APIClient", "APIError", "APITimeoutError", "AsyncAPIClient", "AsyncSandboxClient", "CommandRequest", "CommandResponse",
                 "CommandTimeoutError", "Config", "CreateSandboxRequest", "Sandbox", "SandboxClient", "SandboxNotRunningError", "SandboxStatus",
                 "UpdateSandboxRequest"):  # fmt: skip
        assert getattr(P, name) is not None
    assert S.TimeoutError is S.APITimeoutError
    for name in ("APIError", "APITimeoutError", "Config", "EnvironmentNotFoundError", "FinalizeEvaluationRequest", "PaymentRequiredError",
                 "PushSamplesRequest", "UnauthorizedError", "EvalsClient", "AsyncEvalsClient"):  # fmt: skip
        assert hasattr(E, name), name
    assert E.PushSamplesRequest(samples=[{"a": 1}]).model_dump() == {"samples": [{"a": 1}]}
    assert E.FinalizeEvaluationRequest().metrics is None
    assert Tn.Config is P.Config
    assert callable(M.make_prime_request) and M.pods.__name__.endswith("tools.pods") and M.ssh and M.availability


# ------------------------------------------------------------------------------------------------ drop-in import names
def test_compat_aliases_resolve_reference_import_paths():
    """Code written against the reference packages keeps its imports: the aliases are the real module objects."""
    import sys

    from prime_b200 import compat

    registered = compat.install()
    try:
        assert {"prime_sandboxes", "prime_evals", "prime_tunnel", "prime_cli", "prime_sandboxes.models", "prime_cli.api.pods"} <= set(registered)
        from prime_cli.api.pods import PodsClient, clean_connection_fields  # noqa: F401
        from prime_cli.core import Config as CliConfig
        from prime_evals import EvalsClient
        from prime_sandboxes import APIError, CreateSandboxRequest, SandboxClient
        from prime_sandboxes.models import Sandbox
        from prime_sandboxes.sandbox import SandboxAuthCache  # noqa: F401

        import prime_b200.platform.sandboxes as real

        assert SandboxClient is real.SandboxClient and Sandbox is real.Sandbox and CreateSandboxRequest is real.CreateSandboxRequest
        from prime_b200.platform.core import APIError as CoreAPIError
        from prime_b200.platform.core import Config
        from prime_b200.platform.evals import EvalsClient as RealEvals

        assert APIError is CoreAPIError and CliConfig is Config and EvalsClient is RealEvals  # ONE class hierarchy: except clauses keep matching
        from prime_cli.main import app  # the Typer root

        assert app.info.name == "prime"
    finally:
        compat.uninstall()
    assert "prime_sandboxes" not in sys.modules and "prime_cli.api.pods" not in sys.modules


def test_compat_covers_every_public_name_of_the_reference():
    """The reference side is tests/golden/reference_public_names.json, recorded from the reference packages."""
    from pathlib import Path

    from prime_b200 import compat

    ref = json.loads((Path(__file__).resolve().parents[1] / "golden" / "reference_public_names.json").read_text())
    try:
        res = compat.check(ref)
    finally:
        compat.uninstall()
    assert set(res) == {"prime_cli", "prime_sandboxes", "prime_evals", "prime_tunnel", "prime_mcp"}
    for pkg, r in res.items():
        assert "error" not in r and r["missing"] == [] and r["public_names"] >= 5, (pkg, r)


def test_reference_constructor_spellings_are_accepted(isolated_home):
    """Signature differences found by comparing 1 470 public methods with the reference: keyword names a caller may use."""
    import asyncio

    from prime_b200.platform.evals import AsyncEvalsClient
    from prime_b200.platform.sandboxes import AsyncTemplateClient, CommandTimeoutError, DownloadTimeoutError, UploadTimeoutError
    from prime_b200.platform.tunnel.client import TunnelClient

    e = CommandTimeoutError(sandbox_id="s1", command="sleep 9", timeout=5)
    assert (e.sandbox_id, e.command, e.target, e.timeout) == ("s1", "sleep 9", "sleep 9", 5) and "Command 'sleep 9' timed out after 5s" in str(e)
    assert UploadTimeoutError("s1", file_path="/a", timeout=3).file_path == "/a" and DownloadTimeoutError("s1", "/b", 2).file_path == "/b"
    with pytest.raises(TypeError):
        CommandTimeoutError("s1", timeout=5)

    async def go():
        c = AsyncEvalsClient(api_key="k1")
        assert c.client.api_key == "k1"
        await c.aclose()
        async with AsyncEvalsClient("k2") as c2:
            assert c2.client.api_key == "k2"
        async with AsyncTemplateClient() as t:
            assert hasattr(t, "check_docker_image")
        tc = TunnelClient(api_key="k", user_agent="my-agent/1.0", timeout=5)
        assert tc._headers["User-Agent"] == "my-agent/1.0"
        await tc.close()

    asyncio.run(go())


def test_compat_every_public_method_of_the_reference_exists_with_its_parameter_names():
    """The reference side is tests/golden/reference_signatures.json.gz, recorded from the reference packages."""
    from pathlib import Path

    from prime_b200 import compat

    import gzip

    ref = json.loads(gzip.decompress((Path(__file__).resolve().parents[1] / "golden" / "reference_signatures.json.gz").read_bytes()))
    try:
        res = compat.check_signatures(ref)
    finally:
        compat.uninstall()
    assert res["methods_compared"] > 1400 and res["missing"] == [] and res["parameter_name_differences"] == [] and res["errors"] == [], res


def test_wire_requests_are_identical_to_the_reference(capsys):
    """tools/wire_diff.py: one script (reference import names) against both implementations and a recording server — the HTTP
    requests (method, path, query, JSON body, auth header) and the outcomes of 108 SDK / API-client / MCP-tool calls (sync and async), injected failures and
    their retries included, must not differ. The reference arm is tests/golden/reference_wire_diff.json.gz, recorded from the reference
    packages with ``python tools/wire_diff.py --record``."""
    import sys
    from pathlib import Path

    root = Path(__file__).resolve().parents[2]
    sys.path.insert(0, str(root))
    from tools import wire_diff

    rc = wire_diff.main(reference=root / "tests" / "golden" / "reference_wire_diff.json.gz")
    out = json.loads(capsys.readouterr().out)
    assert rc == 0 and out["calls"] >= 108 and out["requests_reference"] == out["requests_ours"] >= 130
    assert out["outcome_differences"] == [] and out["request_differences"] == []
    assert sum(v == "ok" for v in out["outcomes"].values()) >= 90 and out["outcomes"]["gateway_408"] == "raised CommandTimeoutError"


@pytest.mark.slow
def test_cli_commands_behave_like_the_reference_cli(capsys):
    """tools/cli_diff.py: ``prime …`` command lines (every sixth of the 197 in the quick pass) through both CLIs against the recording server — same exit codes, same HTTP
    requests, and every key / value of the reference's ``--output json`` present in ours. The reference CLI's side is
    tests/golden/reference_cli_diff.json.gz, recorded from the reference packages with ``python tools/cli_diff.py --record``."""
    import sys
    from pathlib import Path

    root = Path(__file__).resolve().parents[2]
    sys.path.insert(0, str(root))
    from tools import cli_diff

    rc = cli_diff.main(stride=1 if os.environ.get("PRIME_B200_FULL_DIFF") else 6, reference=root / "tests" / "golden" / "reference_cli_diff.json.gz")
    out = json.loads(capsys.readouterr().out)
    assert rc == 0 and out["commands"] >= 20 and out["identical"] == out["commands"] and out["differences"] == [], [d["command"] for d in out["differences"]]


@pytest.mark.slow
def test_the_references_own_test_files_pass_against_this_package(tmp_path):
    """tools/reference_tests.py: the reference's unmodified test files, collected through the compat aliases, against the same files run
    on the reference itself.  Quick pass: the tunnel + evals SDK suites (the CLI, sandboxes and MCP suites — 334 more tests — under PRIME_B200_FULL_DIFF).
    It runs the reference's own source, so it skips where the reference packages cannot be read.  No test the reference passes may fail here."""
    import sys
    from pathlib import Path

    root = Path(__file__).resolve().parents[2]
    if not os.access("/root/reference/packages", os.R_OK | os.X_OK):
        pytest.skip("reference tree not mounted")
    sys.path.insert(0, str(root))
    from tools import reference_tests

    pkgs = list(reference_tests.PACKAGES) if os.environ.get("PRIME_B200_FULL_DIFF") else ["prime-tunnel", "prime-evals"]
    out = tmp_path / "report.json"
    assert reference_tests.main(["--packages", *pkgs, "--out", str(out)]) == 0
    report = json.loads(out.read_text())
    assert report["total_gaps"] == 0, {p: e["reference_passes_ours_does_not"] for p, e in report["packages"].items()}
    assert report["total_passed"]["ours"] == report["total_passed"]["reference"] >= 21
    for p in pkgs:
        assert report["packages"][p]["ours"]["counts"] == report["packages"][p]["reference"]["counts"]


@pytest.mark.slow
def test_the_references_example_programs_run_unchanged_on_this_package(tmp_path):
    """tools/run_reference_examples.py: /root/reference/examples/*.py, unmodified, with `prime_sandboxes` resolving to this package, against
    a local sandbox service that really runs the commands — next to the same script on the reference.  Quick pass: the two short demos
    (all six, including the 50-sandbox high-volume one, under PRIME_B200_FULL_DIFF). It runs the reference's own
    programs, so it skips where they cannot be read."""
    import sys
    from pathlib import Path

    root = Path(__file__).resolve().parents[2]
    if not os.access("/root/reference/examples", os.R_OK | os.X_OK):
        pytest.skip("reference tree not mounted")
    sys.path.insert(0, str(root))
    from tools import run_reference_examples as rre

    only = [] if os.environ.get("PRIME_B200_FULL_DIFF") else ["--only", "sandbox_demo", "sandbox_file_operations"]
    out = tmp_path / "examples.json"
    assert rre.main([*only, "--out", str(out)]) == 0
    report = json.loads(out.read_text())
    assert report["all_ok"] and len(report["examples"]) >= 2
    for name, e in report["examples"].items():
        assert e["same_exit"] and e["ours"]["exit"] == 0, (name, e)
        assert e["same_route_multiset"] and e["ours"]["requests"] == e["reference"]["requests"], (name, e)
        assert e["ours"]["sandboxes_left_running"] == 0, (name, e)


def test_plain_mode_tables_carry_no_markup():
    """`--plain` is the mode for scripts and agents: a coloured status cell must come out as the bare word."""
    from prime_b200.platform.utils.display import build_table, colorize
    from prime_b200.platform.utils.plain import to_plain

    t = build_table("Pods", [("ID", "cyan"), "Status"], [["p1", colorize("ACTIVE", {"ACTIVE": "green"})], ["p2", colorize("ERROR", {"ERROR": "red"})]])
    text = to_plain(t)
    assert "[green]" not in text and "[/]" not in text and "ACTIVE" in text and "ERROR" in text
    assert [ln.split() for ln in text.splitlines()[-2:]] == [["p1", "ACTIVE"], ["p2", "ERROR"]]


def test_unexpected_response_shapes_fail_with_one_line_not_a_traceback(isolated_home, monkeypatch):
    """A control plane that answers `{}` (or a string where an object belongs) must not crash a command with a traceback."""
    from typer.testing import CliRunner

    from prime_b200.platform.commands import registry as reg_mod
    from prime_b200.platform.main import app

    class Empty:
        def __init__(self, *a, **k):
            self.config = type("C", (), {"team_id": None})()

        def request(self, *a, **k):
            return {}

        get = post = request

    monkeypatch.setenv("PRIME_API_KEY", "k")
    monkeypatch.setattr(reg_mod, "api", lambda *a, **k: Empty(), raising=False)
    r = CliRunner().invoke(app, ["registry", "check-image", "python:3.11-slim"])
    assert r.exit_code == 1 and "Unexpected response from the API" in r.output and "Traceback" not in r.output


def test_mcp_tool_schemas_are_the_reference_schemas():
    """What an MCP client sees from `list_tools`: the nine tools with the same input schemas (parameter types, defaults, required).
    The reference side is tests/golden/reference_mcp_tool_schemas.json, recorded from the reference's MCP server."""
    import subprocess
    import sys
    from pathlib import Path

    pytest.importorskip("mcp")
    root = Path(__file__).resolve().parents[2]
    code = (
        "import asyncio, importlib, json, sys\n"
        "import prime_b200.compat as c; c.install()\n"
        "m = importlib.import_module('prime_mcp.mcp')\n"
        "print(json.dumps({t.name: t.inputSchema for t in asyncio.run(m.mcp.list_tools())}, sort_keys=True))\n"
    )
    out = {"reference": json.loads((root / "tests" / "golden" / "reference_mcp_tool_schemas.json").read_text())}
    r = subprocess.run([sys.executable, "-c", code], env={**os.environ, "PYTHONPATH": str(root)}, capture_output=True, text=True, cwd="/", timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    out["ours"] = json.loads(r.stdout.strip().splitlines()[-1])

    def shape(schema):
        props = {k: {a: b for a, b in v.items() if a not in ("title", "description")} for k, v in schema.get("properties", {}).items()}
        return {"required": sorted(schema.get("required", [])), "properties": props}

    assert sorted(out["ours"]) == sorted(out["reference"]) and len(out["ours"]) == 9
    for name, schema in out["reference"].items():
        assert shape(out["ours"][name]) == shape(schema), name


def test_every_reference_model_field_exists_with_its_wire_name():
    """53 pydantic models / 424 fields of the reference SDKs and API clients: each field exists here under the same name, with the
    same explicit wire alias, and is never stricter (required here while optional there). The reference side is
    tests/golden/reference_model_fields.json, recorded from the reference packages."""
    import subprocess
    import sys
    from pathlib import Path

    root = Path(__file__).resolve().parents[2]
    code = (
        "import importlib, inspect, json, sys, pydantic\n"
        "import prime_b200.compat as c; c.install()\n"
        "out = {}\n"
        "for mn in ['prime_sandboxes.models', 'prime_evals.models', 'prime_tunnel.models', 'prime_cli.api.pods', 'prime_cli.api.availability',\n"
        "           'prime_cli.api.disks', 'prime_cli.api.rl', 'prime_cli.api.deployments']:\n"
        "    m = importlib.import_module(mn)\n"
        "    for n, v in vars(m).items():\n"
        "        if inspect.isclass(v) and issubclass(v, pydantic.BaseModel) and v is not pydantic.BaseModel and not n.startswith('_'):\n"
        "            out[mn + '.' + n] = {fn: [f.alias, f.is_required()] for fn, f in v.model_fields.items()}\n"
        "print(json.dumps(out))\n"
    )
    got = {"reference": json.loads((root / "tests" / "golden" / "reference_model_fields.json").read_text())}
    r = subprocess.run([sys.executable, "-c", code], env={**os.environ, "PYTHONPATH": str(root)}, capture_output=True, text=True, cwd="/", timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    got["ours"] = json.loads(r.stdout.strip().splitlines()[-1])
    problems, n = [], 0
    for model, fields in got["reference"].items():
        mine = got["ours"].get(model)
        if mine is None:
            problems.append(f"missing model {model}")
            continue
        for fn, (alias, required) in fields.items():
            n += 1
            if fn not in mine:
                problems.append(f"missing field {model}.{fn}")
            elif alias is not None and mine[fn][0] != alias:
                problems.append(f"wire name of {model}.{fn}: {alias} there, {mine[fn][0]} here")
            elif mine[fn][1] and not required:
                problems.append(f"{model}.{fn} is required here, optional there")
    assert len(got["reference"]) >= 50 and n >= 400 and not problems, problems[:10]
