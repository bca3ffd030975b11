"""Drop-in import names for code written against the reference packages.

    import prime_b200.compat; prime_b200.compat.install()        # once, at program start
    from prime_sandboxes import SandboxClient, CreateSandboxRequest   # → prime_b200.platform.sandboxes
    from prime_evals import EvalsClient                               # → prime_b200.platform.evals
    from prime_cli.api.pods import PodsClient                         # → prime_b200.platform.api.pods

``install()`` registers the platform layer's modules in ``sys.modules`` under the import names of the five reference
distributions (``prime_cli``, ``prime_sandboxes``, ``prime_evals``, ``prime_tunnel``, ``prime_mcp``), package and submodules —
the module layout underneath is the same (``sandbox.py`` / ``models.py`` / ``exceptions.py`` / ``core/{client,config}.py`` …;
reference: packages/*/src/*/__init__.py), so ``from prime_sandboxes.models import Sandbox`` keeps working. The alias IS the
real module object (``prime_sandboxes.SandboxClient is prime_b200.platform.sandboxes.SandboxClient``): one class hierarchy, so
``except prime_sandboxes.APIError`` catches what this layer raises. Nothing is registered for a name whose real reference
package is already imported, and nothing is shadowed on disk — without ``install()`` the names stay free.

``python -m prime_b200.compat check [--reference /path/to/prime/packages]`` lists, per package, the public names of the reference's
``__all__`` and whether each resolves here (run against the mounted reference in ``tests/plat/test_core.py``).
"""

from __future__ import annotations

import importlib
import json
import subprocess
import sys
from pathlib import Path

_P = "prime_b200.platform"
# alias package → (real package, {alias submodule → real module})
ALIASES: dict[str, tuple[str, dict[str, str]]] = {
    "prime_sandboxes": (f"{_P}.sandboxes", {
        "sandbox": f"{_P}.sandboxes.sandbox", "models": f"{_P}.sandboxes.models", "exceptions": f"{_P}.sandboxes.exceptions",
        "rpc_command_session": f"{_P}.sandboxes.rpc_command_session", "core": f"{_P}.core", "core.client": f"{_P}.sandboxes.client",
        "core.config": f"{_P}.core.config", "_proto": f"{_P}.sandboxes.proto", "_proto.command_session": f"{_P}.sandboxes.proto",
        "_proto.command_session.command_session_pb2": f"{_P}.sandboxes.rpc_schema"}),
    "prime_evals": (f"{_P}.evals", {
        "evals": f"{_P}.evals.evals", "models": f"{_P}.evals.models", "exceptions": f"{_P}.evals.exceptions", "core": f"{_P}.core",
        "core.client": f"{_P}.core.client", "core.config": f"{_P}.core.config"}),
    "prime_tunnel": (f"{_P}.tunnel", {
        "tunnel": f"{_P}.tunnel.tunnel", "binary": f"{_P}.tunnel.binary", "models": f"{_P}.tunnel.models", "exceptions": f"{_P}.tunnel.exceptions",
        "core": f"{_P}.core", "core.client": f"{_P}.tunnel.client", "core.config": f"{_P}.core.config"}),
    "prime_mcp": (f"{_P}.mcp", {
        "mcp": f"{_P}.mcp.server", "client": f"{_P}.mcp.client", "tools": f"{_P}.mcp.tools", "tools.availability": f"{_P}.mcp.tools.availability",
        "tools.pods": f"{_P}.mcp.tools.pods", "tools.ssh": f"{_P}.mcp.tools.ssh", "core": f"{_P}.core",
        "core.client": f"{_P}.core.client", "core.config": f"{_P}.core.config"}),
    "prime_cli": (_P, {
        "main": f"{_P}.main", "api": f"{_P}.api", "commands": f"{_P}.commands", "core": f"{_P}.core", "core.client": f"{_P}.core.client",
        "core.config": f"{_P}.core.config", "utils": f"{_P}.utils", "helper": f"{_P}.helper", "verifiers_bridge": f"{_P}.verifiers_bridge",
        "verifiers_plugin": f"{_P}.verifiers_plugin", "client": f"{_P}.core.client", "config": f"{_P}.core.config",
        **{f"api.{m}": f"{_P}.api.{m}" for m in ("availability", "deployments", "disks", "inference", "pods", "rl")},
        "api.client": f"{_P}.core.client",
        **{f"commands.{m}": f"{_P}.commands.{m}" for m in ("availability", "config", "deployments", "disks", "env", "evals", "gepa", "images", "inference",
                                                              "lab", "login", "pods", "registry", "rl", "sandbox", "secrets", "switch", "teams",
                                                              "tunnel", "upgrade", "whoami")},
        **{f"utils.{m}": f"{_P}.utils.{m}" for m in ("config", "display", "env_metadata", "env_vars", "eval_push", "formatters", "hosted_eval",
                                                        "json_help", "plain", "prompt", "time_utils", "version_check")},
    }),
}  # fmt: skip


def install(packages: tuple[str, ...] | None = None, *, strict: bool = False) -> list[str]:
    """Register the aliases; returns the names registered. ``strict``: raise if a real reference package is already imported
    under one of the names (default: leave that package alone)."""
    done: list[str] = []
    for alias, (real, subs) in ALIASES.items():
        if packages is not None and alias not in packages:
            continue
        have = sys.modules.get(alias)
        if have is not None and not getattr(have, "__name__", "").startswith(_P):
            if strict:
                raise ImportError(f"{alias} is already imported from {getattr(have, '__file__', '?')}; cannot alias it")
            continue
        sys.modules[alias] = importlib.import_module(real)
        done.append(alias)
        for sub, target in subs.items():
            try:
                sys.modules[f"{alias}.{sub}"] = importlib.import_module(target)
            except ImportError:  # optional dependency of that submodule (mcp, connectrpc) is not installed: leave the name unresolved
                continue
            done.append(f"{alias}.{sub}")
    return done


def uninstall() -> None:
    for name in [n for n in sys.modules if n.split(".")[0] in ALIASES]:
        if getattr(sys.modules[name], "__name__", "").startswith(_P):
            del sys.modules[name]


_REF_DIRS = {"prime_cli": "prime", "prime_sandboxes": "prime-sandboxes", "prime_evals": "prime-evals", "prime_tunnel": "prime-tunnel",
             "prime_mcp": "prime-mcp-server"}  # fmt: skip


def reference_public_names(packages_dir: str | Path) -> dict[str, list[str]]:
    """``__all__`` (or the public attributes) of every reference package, read in a child interpreter so that the reference never
    shares a process with the aliases."""
    code = (
        "import importlib, json, sys\n"
        "out = {}\n"
        "for pkg in sys.argv[1:]:\n"
        "    try:\n"
        "        m = importlib.import_module(pkg)\n"
        "        out[pkg] = sorted(getattr(m, '__all__', [n for n in dir(m) if not n.startswith('_')]))\n"
        "    except Exception as e:\n"
        "        out[pkg] = ['!' + type(e).__name__ + ': ' + str(e)[:120]]\n"
        "print(json.dumps(out))\n"
    )
    import os

    env = {**os.environ, "PYTHONPATH": os.pathsep.join(str(Path(packages_dir) / d / "src") for d in _REF_DIRS.values())}
    r = subprocess.run([sys.executable, "-c", code, *_REF_DIRS], env=env, capture_output=True, text=True, cwd="/", timeout=300)
    if r.returncode != 0:
        raise RuntimeError(r.stderr[-2000:])
    return json.loads(r.stdout.strip().splitlines()[-1])


def check(packages_dir: str | Path | dict) -> dict[str, dict]:
    """Per reference package: how many public names, and which of them do NOT resolve through the alias. ``packages_dir`` is the
    reference tree, or the output of :func:`reference_public_names` recorded from it."""
    ref = packages_dir if isinstance(packages_dir, dict) else reference_public_names(packages_dir)
    install()
    out = {}
    for pkg, names in ref.items():
        if names and names[0].startswith("!"):
            out[pkg] = {"error": names[0][1:]}
            continue
        mod = sys.modules.get(pkg)
        out[pkg] = {"public_names": len(names), "missing": [n for n in names if mod is None or not hasattr(mod, n)]}
    return out


_SIG_CODE = r"""
import importlib, inspect, json, sys
out = {}
for modname in sys.argv[1:]:
    try:
        m = importlib.import_module(modname)
    except Exception as e:
        out[modname] = {"!": type(e).__name__ + ": " + str(e)[:100]}
        continue
    names = getattr(m, "__all__", None) or [n for n, v in vars(m).items() if not n.startswith("_") and inspect.isclass(v) and v.__module__ == m.__name__]
    d = {}
    for n in names:
        v = getattr(m, n, None)
        if inspect.isclass(v):
            meths = {}
            for mn, mv in inspect.getmembers(v):
                if (mn.startswith("_") and mn != "__init__") or not (inspect.isfunction(mv) or inspect.ismethod(mv)):
                    continue
                try:
                    meths[mn] = [p for p in inspect.signature(mv).parameters if p != "self"]
                except Exception:
                    meths[mn] = None
            d[n] = meths
        elif inspect.isfunction(v):
            d[n] = {"()": list(inspect.signature(v).parameters)}
    out[modname] = d
print(json.dumps(out))
"""
SIGNATURE_MODULES = ("prime_sandboxes", "prime_evals", "prime_tunnel", "prime_mcp", "prime_cli.api.pods", "prime_cli.api.availability",
                     "prime_cli.api.disks", "prime_cli.api.rl", "prime_cli.api.deployments", "prime_cli.api.inference", "prime_cli.core.client",
                     "prime_cli.core.config")  # fmt: skip


def reference_signatures(packages_dir: str | Path) -> dict:
    """Public classes / functions of the reference's SDK packages and API clients with their parameter names, read in a child
    interpreter."""
    import os

    env = {**os.environ, "PYTHONPATH": os.pathsep.join(str(Path(packages_dir) / d / "src") for d in _REF_DIRS.values())}
    r = subprocess.run([sys.executable, "-c", _SIG_CODE, *SIGNATURE_MODULES], env=env, capture_output=True, text=True, cwd="/", timeout=300)
    if r.returncode != 0:
        raise RuntimeError(r.stderr[-2000:])
    return json.loads(r.stdout.strip().splitlines()[-1])


def check_signatures(packages_dir: str | Path | dict) -> dict:
    """Every public class of the reference's SDK packages and API clients: do its public methods exist here, and does each
    accept the reference's parameter names? (pydantic validator methods — ``validate_*`` — are implementation detail and ignored)
    ``packages_dir`` is the reference tree, or the output of :func:`reference_signatures` recorded from it."""
    import inspect

    ref = packages_dir if isinstance(packages_dir, dict) else reference_signatures(packages_dir)
    install()
    compared, missing, param_diffs, errors = 0, [], [], []
    for modname, classes in ref.items():
        if "!" in classes:
            errors.append(f"{modname}: {classes['!']}")
            continue
        mod = sys.modules.get(modname) or importlib.import_module(modname)
        for cname, meths in classes.items():
            cls = getattr(mod, cname, None)
            if cls is None:
                missing.append(f"{modname}.{cname}")
                continue
            for mn, params in meths.items():
                if mn.startswith("validate_"):
                    continue
                compared += 1
                f = cls if mn == "()" else getattr(cls, mn, None)
                if f is None:
                    missing.append(f"{modname}.{cname}.{mn}")
                    continue
                try:
                    ours = [p for p in inspect.signature(f).parameters if p != "self"]
                except (TypeError, ValueError):
                    continue
                catch_all = any(p.kind is inspect.Parameter.VAR_KEYWORD for p in inspect.signature(f).parameters.values())
                if params is not None and not catch_all and any(p not in ours for p in params):
                    param_diffs.append(f"{modname}.{cname}.{mn}: reference {params}, here {ours}")
    return {"methods_compared": compared, "missing": missing, "parameter_name_differences": param_diffs, "errors": errors}


def main(argv: list[str] | None = None) -> int:
    import argparse

    ap = argparse.ArgumentParser(prog="python -m prime_b200.compat")
    sub = ap.add_subparsers(dest="cmd", required=True)
    c = sub.add_parser("check")
    c.add_argument("--reference", default="/root/reference/packages")
    c.add_argument("--methods", action="store_true", help="also compare the public methods and parameter names of every public class")
    sub.add_parser("list")
    a = ap.parse_args(argv)
    if a.cmd == "list":
        print(json.dumps(install(), indent=1))
        return 0
    res: dict = check(a.reference)
    bad = any(v.get("missing") or v.get("error") for v in res.values())
    if a.methods:
        res["signatures"] = check_signatures(a.reference)
        bad = bad or bool(res["signatures"]["missing"] or res["signatures"]["parameter_name_differences"] or res["signatures"]["errors"])
    print(json.dumps(res, indent=1))
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
