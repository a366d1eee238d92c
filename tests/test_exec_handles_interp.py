"""Handle checks of libmnn_b200_interp.so's C ABI (include/mnn_b200_interp.h), whose fp32 Interp execution shares libmnn_b200.so's
handles.  Every entry point of the header exists in the library with the binding's signature, and those whose first parameter
is a runtime or an execution refuse a NULL one (CPU).  Every Interp entry point taking an execution refuses every other
execution type (the core library's and the Deconvolution library's), every execution entry point of mnn_b200.h and
mnn_b200_deconv.h refuses the Interp execution, and execute / plan refuse before resize (-m gpu)."""
import ctypes as C
import os
import re

import pytest

from mnn_b200 import _capi
from tests.test_exec_handles import EVERY_TYPE, INVALID_VALUE, NO_EXECUTION, create_all, handle_entry_points, zero_args
from tests.test_exec_handles_deconv import create_deconvs, deconv_entry_points

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BEFORE_RESIZE = ["mnnb200_interp_f32_execute", "mnnb200_interp_f32_plan"]


def interp_entry_points(kind=None):
    """entry point names of mnn_b200_interp.h (whose first parameter is mnnb200_<kind>*, when kind is given)"""
    hdr = open(os.path.join(ROOT, "include", "mnn_b200_interp.h")).read()
    first = r"\s*\(\s*mnnb200_" + kind + r"\s*\*" if kind else r"\s*\("
    return re.findall(r"MNNB200_API[^;(]*?\b(mnnb200_[a-z0-9_]+)" + first, hdr)


def test_interp_header_symbols_exported():
    declared = set(interp_entry_points())
    assert declared == set(_capi.INTERP_SIGNATURES), declared ^ set(_capi.INTERP_SIGNATURES)
    assert not declared & (set(_capi.SIGNATURES) | set(_capi.LLM_SIGNATURES) | set(_capi.DECONV_SIGNATURES))
    L = _capi.interp_lib()
    for name in declared:
        assert hasattr(L, name), f"{name} not exported"


@pytest.mark.parametrize("kind", ["runtime", "exec"])
def test_interp_null_handle_refused(kind):
    L = _capi.interp_lib()
    names = interp_entry_points(kind)
    assert names
    for name in names:
        assert getattr(L, name)(*zero_args(_capi.INTERP_SIGNATURES[name][1], buffers=False)) == INVALID_VALUE, name


def create_interp(rt, resize_type=2):
    h = C.c_void_p()
    assert _capi.interp_lib().mnnb200_interp_f32_create(rt, resize_type, 0.5, 0.5, 0.0, 0.0, C.byref(h)) == 0
    return h


@pytest.mark.gpu
def test_interp_exec_entry_points_refuse_other_types_and_before_resize(backend):
    L, D, I = _capi.lib(), _capi.deconv_lib(), _capi.interp_lib()
    rt = backend.runtime._h
    mine = interp_entry_points("exec")
    h = create_interp(rt)
    others, keep = create_all(rt)
    deconvs = create_deconvs(rt)
    try:
        for name in handle_entry_points("exec"):
            if name in EVERY_TYPE:
                continue
            args = zero_args(_capi.SIGNATURES[name][1][1:], buffers=True)
            want = 0 if name == "mnnb200_conv_int8_groupable" else INVALID_VALUE
            assert getattr(L, name)(h, *args) == want, name
        for name in deconv_entry_points("exec"):
            assert getattr(D, name)(h, *zero_args(_capi.DECONV_SIGNATURES[name][1][1:], buffers=True)) == INVALID_VALUE, name
        for name in BEFORE_RESIZE:
            args = zero_args(_capi.INTERP_SIGNATURES[name][1][1:], buffers=True)
            if name.endswith("_plan"):
                args[-1] = 4
            assert getattr(I, name)(h, *args) == NO_EXECUTION, (name, L.mnnb200_last_error())
        for t, o in list(others.items()) + list(deconvs.items()):
            for name in mine:
                args = zero_args(_capi.INTERP_SIGNATURES[name][1][1:], buffers=True)
                assert getattr(I, name)(o, *args) == INVALID_VALUE, (t, name)
    finally:
        for o in [h] + list(deconvs.values()) + [others.pop("group")] + list(others.values()):
            L.mnnb200_exec_destroy(o)
