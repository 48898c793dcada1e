import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    config.addinivalue_line("markers", "reference: needs the reference package that build() places under oracle/_ref")


def pytest_collection_modifyitems(config, items):
    import torch
    # PyTorch references used by the tests must be true fp32 (no TF32 in cuBLAS / cuDNN)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    from oracle.ref_shims import reference_available
    has_gpu = torch.cuda.is_available()
    has_ref = reference_available()
    for item in items:
        if "gpu" in item.keywords and not has_gpu:
            item.add_marker(pytest.mark.skip(reason="no CUDA device"))
        if "reference" in item.keywords and not has_ref:
            item.add_marker(pytest.mark.skip(reason="reference tree not present"))
