import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


@pytest.fixture(scope="session", autouse=True)
def _built_library():
    """The C-ABI library must exist before any test imports the package (no fallback)."""
    # load build.py by path: importing the package would dlopen a stale library first
    import importlib.util
    spec = importlib.util.spec_from_file_location(
        "_td_build", os.path.join(ROOT, "multidiffusion_upscaler_for_automatic1111_b200", "build.py"))
    build = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(build)
    if build.needs_build():
        build.build()
