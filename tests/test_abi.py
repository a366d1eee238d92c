"""CPU test: libmnn_b200.so loads and exports every symbol include/mnn_b200.h declares (no compute calls)."""
import ctypes
import os
import re

from mnn_b200 import _capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_symbols_exported():
    hdr = open(os.path.join(ROOT, "include", "mnn_b200.h")).read()
    declared = set(re.findall(r"MNNB200_API[^;(]*?\b(mnnb200_[a-z0-9_]+)\s*\(", hdr))
    assert len(declared) >= 25
    assert declared == set(_capi.SIGNATURES), declared ^ set(_capi.SIGNATURES)
    L = ctypes.CDLL(_capi.LIB_PATH)
    for name in declared:
        assert hasattr(L, name), f"{name} not exported"
    assert _capi.lib().mnnb200_abi_version() == 2


def test_no_cpu_fallback_without_gpu():
    """Without a CUDA device the runtime must fail loudly (status 100), never compute on the host."""
    import torch
    if torch.cuda.is_available():
        return
    h = ctypes.c_void_p()
    st = _capi.lib().mnnb200_runtime_create(0, None, ctypes.byref(h))
    assert st == 100
    assert b"no CPU fallback" in _capi.lib().mnnb200_last_error()


def test_product_does_not_import_oracle():
    for root, _, files in os.walk(os.path.join(ROOT, "mnn_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                src = open(os.path.join(root, f)).read()
                assert "import oracle" not in src and "from oracle" not in src and "oracle/" not in src, f
