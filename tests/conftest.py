import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


def pytest_collection_modifyitems(config, items):
    """GPU-marked tests SKIP (not fail) on a box without CUDA; the product itself still fails loudly
    when asked to move bytes without a GPU (tests/test_abi.py covers that)."""
    try:
        import torch

        have_gpu = torch.cuda.is_available()
    except Exception:
        have_gpu = False
    if have_gpu:
        return
    skip = pytest.mark.skip(reason="needs a CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session", autouse=True)
def _built_artifacts():
    """The native library and the C oracle are built in-tree (see __graft_entry__.build)."""
    from torchstore_b200 import _build

    if _build.needs_build():
        try:
            _build.build_native()
        except Exception as e:  # no nvcc on this box: tests that need the library will fail loudly
            print(f"[conftest] could not build libtstore_b200.so: {e}")
    from oracle import c_oracle

    c_oracle.build()
    yield
