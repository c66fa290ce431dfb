import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")
    # the fp32 oracle must be fp32 on the GPU box too: TF32 (10-bit mantissa, cuDNN's default for convolutions) would make
    # the "fp32 reference" no more precise than the fp16 kernels it judges
    import torch
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(ROOT, "tests", "golden")


@pytest.fixture
def emulated_ops(monkeypatch):
    """Swap the C-ABI wrappers of anyv2v_b200.ops for their CPU contract restatements (tests/kernel_contracts.py) for the
    duration of one test, so that the host logic on top of the kernels can be exercised without a GPU."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import kernel_contracts
    from anyv2v_b200 import ops
    for name, fn in kernel_contracts.CONTRACTS.items():
        monkeypatch.setattr(ops, name, fn)
    return kernel_contracts
