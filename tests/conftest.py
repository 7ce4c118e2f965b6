"""Shared pytest configuration.

* registers the ``gpu`` marker (tests that need an H100; select them with ``-m gpu``)
* puts the in-tree package (``tensorflow-image-models_b200/``) and the repo root on sys.path
* makes sure the CUDA library is built (nvcc cross-compiles here without a GPU)
"""
import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
PKG = ROOT / "tensorflow-image-models_b200"
for p in (str(ROOT), str(PKG)):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (H100); run with -m gpu")


def pytest_collection_modifyitems(config, items):
    import torch

    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session", autouse=True)
def _exact_fp32_references():
    """The fp32 PyTorch references the kernels are compared with must not silently use TF32."""
    import torch

    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield


@pytest.fixture(scope="session", autouse=True)
def _built_library():
    lib = PKG / "tfimm" / "backend" / "libtfimm_b200.so"
    if not lib.exists():
        sys.path.insert(0, str(PKG))
        import importlib.util

        spec = importlib.util.spec_from_file_location("tfimm_b200_build", PKG / "build.py")
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        mod.build()
    yield
