import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "vit-prisma_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)


collect_ignore = [os.path.join("golden", "ref_tests")]     # verbatim reference test files: run only through test_reference_suite_verbatim_gpu.py


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA GPU, an H100 (sm_90a); run with `-m gpu`")


def pytest_collection_modifyitems(config, items):
    """GPU tests are skipped (not failed) when no device is visible, so a plain `pytest tests/` works anywhere."""
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
