import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

os.environ.setdefault("PRIME_DISABLE_VERSION_CHECK", "1")
# rich reads COLUMNS / LINES when a Console is CONSTRUCTED (the package's consoles are module-level), so a narrow terminal exported by
# the caller (or by pytest-xdist: 80 × 24) would wrap the tables the CLI tests read. Pin the size before anything imports the package.
os.environ["COLUMNS"], os.environ["LINES"] = "200", "50"


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on the H100 box)")
    config.addinivalue_line("markers", "multigpu: needs >= 2 CUDA devices")
    config.addinivalue_line("markers", "slow: multi-process tests that take tens of seconds")


def pytest_collection_modifyitems(config, items):
    try:
        import torch

        n = torch.cuda.device_count() if torch.cuda.is_available() else 0
    except Exception:
        n = 0
    for item in items:
        if "gpu" in item.keywords and n == 0:
            item.add_marker(pytest.mark.skip(reason="no CUDA device"))
        if "multigpu" in item.keywords and n < 2:
            item.add_marker(pytest.mark.skip(reason="needs >= 2 CUDA devices"))
