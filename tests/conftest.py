import json
import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

GOLDEN = Path(__file__).resolve().parent / "golden"


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100 box)")


def _has_gpu() -> bool:
    try:
        from skyplane_b200 import native

        return native.device_count() > 0
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    # -m gpu on a box without a GPU must fail loudly, not skip: only auto-skip when the user did not ask for gpu tests
    if "gpu" in (config.getoption("-m") or ""):
        return
    if _has_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def golden():
    return {p.stem: json.loads(p.read_text()) for p in GOLDEN.glob("*.json")}
