"""Handle checks of libmnn_b200_gather.so's C ABI (include/mnn_b200_gather.h), whose gather execution shares libmnn_b200.so's
handles.  Every entry point of the header exists in the library with the binding's signature, and those whose first parameter
is a runtime or an execution refuse a NULL one (CPU).  Every gather entry point taking an execution refuses every other
execution type (the core library's, the Deconvolution and the Interp library's), every execution entry point of mnn_b200.h,
mnn_b200_deconv.h and mnn_b200_interp.h refuses the gather execution, and execute / plan refuse before resize (-m gpu)."""
import ctypes as C
import os
import re

import pytest

from mnn_b200 import _capi
from tests.test_exec_handles import EVERY_TYPE, INVALID_VALUE, NO_EXECUTION, create_all, handle_entry_points, zero_args
from tests.test_exec_handles_deconv import create_deconvs, deconv_entry_points
from tests.test_exec_handles_interp import create_interp, interp_entry_points

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BEFORE_RESIZE = ["mnnb200_gather_execute", "mnnb200_gather_plan"]


def gather_entry_points(kind=None):
    """entry point names of mnn_b200_gather.h (whose first parameter is mnnb200_<kind>*, when kind is given)"""
    hdr = open(os.path.join(ROOT, "include", "mnn_b200_gather.h")).read()
    first = r"\s*\(\s*mnnb200_" + kind + r"\s*\*" if kind else r"\s*\("
    return re.findall(r"MNNB200_API[^;(]*?\b(mnnb200_[a-z0-9_]+)" + first, hdr)


def test_gather_header_symbols_exported():
    declared = set(gather_entry_points())
    assert declared == set(_capi.GATHER_SIGNATURES), declared ^ set(_capi.GATHER_SIGNATURES)
    assert not declared & (set(_capi.SIGNATURES) | set(_capi.LLM_SIGNATURES) | set(_capi.DECONV_SIGNATURES) |
                           set(_capi.INTERP_SIGNATURES))
    L = _capi.gather_lib()
    for name in declared:
        assert hasattr(L, name), f"{name} not exported"


@pytest.mark.parametrize("kind", ["runtime", "exec"])
def test_gather_null_handle_refused(kind):
    L = _capi.gather_lib()
    names = gather_entry_points(kind)
    assert names
    for name in names:
        assert getattr(L, name)(*zero_args(_capi.GATHER_SIGNATURES[name][1], buffers=False)) == INVALID_VALUE, name


@pytest.mark.gpu
def test_gather_exec_entry_points_refuse_other_types_and_before_resize(backend):
    L, D, I, G = _capi.lib(), _capi.deconv_lib(), _capi.interp_lib(), _capi.gather_lib()
    rt = backend.runtime._h
    mine = gather_entry_points("exec")
    h = C.c_void_p()
    assert G.mnnb200_gather_create(rt, 0, C.byref(h)) == 0
    bad = C.c_void_p()
    assert G.mnnb200_gather_create(rt, 3, C.byref(bad)) == INVALID_VALUE
    others, keep = create_all(rt)
    deconvs = create_deconvs(rt)
    interp = create_interp(rt)
    try:
        for name in handle_entry_points("exec"):
            if name in EVERY_TYPE:
                continue
            args = zero_args(_capi.SIGNATURES[name][1][1:], buffers=True)
            want = 0 if name == "mnnb200_conv_int8_groupable" else INVALID_VALUE
            assert getattr(L, name)(h, *args) == want, name
        for name in deconv_entry_points("exec"):
            assert getattr(D, name)(h, *zero_args(_capi.DECONV_SIGNATURES[name][1][1:], buffers=True)) == INVALID_VALUE, name
        for name in interp_entry_points("exec"):
            assert getattr(I, name)(h, *zero_args(_capi.INTERP_SIGNATURES[name][1][1:], buffers=True)) == INVALID_VALUE, name
        for name in BEFORE_RESIZE:
            args = zero_args(_capi.GATHER_SIGNATURES[name][1][1:], buffers=True)
            if name.endswith("_plan"):
                args[-1] = 4
            assert getattr(G, name)(h, *args) == NO_EXECUTION, (name, L.mnnb200_last_error())
        for t, o in list(others.items()) + list(deconvs.items()) + [("interp", interp)]:
            for name in mine:
                args = zero_args(_capi.GATHER_SIGNATURES[name][1][1:], buffers=True)
                assert getattr(G, name)(o, *args) == INVALID_VALUE, (t, name)
    finally:
        for o in [h, interp] + list(deconvs.values()) + [others.pop("group")] + list(others.values()):
            L.mnnb200_exec_destroy(o)
