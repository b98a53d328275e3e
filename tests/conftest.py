import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    # GPU-side "fp32" references must be fp32: cuDNN convolutions default to TF32 (10-bit mantissa) and would be a
    # weaker oracle than the kernels under test (VERDICT r1, weak 3)
    import torch
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    config.addinivalue_line("markers", "gpu: needs a CUDA (sm_90) device")
    config.addinivalue_line("markers", "reference: needs the reference tree at /root/reference (build container only)")


def pytest_sessionstart(session):
    # A/B experiments only (tools/build_variant.py): run the GPU suite against a variant library
    variant = os.environ.get("STAR_LIB_VARIANT")
    if variant:
        import star_b200.lib as _lib
        _lib.LIB_PATH = os.path.abspath(variant)
        print(f"[conftest] using variant library {_lib.LIB_PATH}")


def pytest_collection_modifyitems(config, items):
    import torch
    has_gpu = torch.cuda.is_available()
    from oracle.ref_loader import reference_available
    has_ref = reference_available()
    for item in items:
        if "gpu" in item.keywords and not has_gpu:
            item.add_marker(pytest.mark.skip(reason="no CUDA device"))
        if "reference" in item.keywords and not has_ref:
            item.add_marker(pytest.mark.skip(reason="reference tree not present"))
