import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; run with -m gpu)")
    config.addinivalue_line("markers", "reference: needs oracle/_ref (the built reference); skipped when absent")


@pytest.fixture(scope="session")
def backend():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device: the product path has no CPU fallback")
    from mnn_b200.backend import Runtime
    # one non-default stream for the whole GPU test session, current for torch AND adopted by the runtime: the tests' torch work
    # (poison fills, uploads, .cpu()) is then ordered with the backend's kernels.  (With the default stream the runtime used to
    # create its own non-blocking stream, and a fill_() could land after the kernel it was meant to precede: ~1 in 8 runs of the
    # conv-group test, every run under compute-sanitizer.)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    rt = Runtime(0)
    be = rt.onCreate()
    be._test_stream = stream
    return be
