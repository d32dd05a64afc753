"""pytest configuration: `gpu` marker, repo root on sys.path, shared fixtures.

`-m "not gpu"` : oracle vs golden vectors, host logic (with an oracle-backed engine double), C-ABI symbol checks,
                 world_size-2 gloo tests.  No CUDA calls.
`-m gpu`       : the parity tests proper -- every one of them goes through libsentio_b200.so (ctypes -> C ABI).
"""
import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a); skipped when no CUDA device is visible")


def _cuda_device_visible() -> bool:
    try:
        import torch

        return bool(torch.cuda.is_available())
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    """Without a CUDA device the `gpu` tests are skipped (not errors), so a plain `pytest` run is green on a CPU box."""
    if _cuda_device_visible():
        return
    skip = pytest.mark.skip(reason="needs an H100: no CUDA device visible")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def load_golden(name):
    with open(os.path.join(GOLDEN, f"{name}.json")) as f:
        return json.load(f)


@pytest.fixture(scope="session")
def built_lib():
    from sentio_b200.build import build

    return build()


@pytest.fixture(scope="session")
def engine(built_lib):
    """A real engine on cuda:0; only requested by @pytest.mark.gpu tests."""
    from sentio_b200.engine import B200Engine

    eng = B200Engine(0)
    yield eng
    eng.close()
