"""Handle checks of libmnn_b200_deconv.so's C ABI (include/mnn_b200_deconv.h), whose float Deconvolution executions share
libmnn_b200.so's handles.  Every entry point of the header exists in the library with the binding's signature, and those whose first parameter is a runtime or an execution refuse a
NULL one (CPU).  Every deconvolution entry point taking an execution refuses every other execution type, every execution entry
point of mnn_b200.h refuses the two deconvolution types, and execute / plan refuse before resize (-m gpu)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from mnn_b200 import _capi
from tests.test_exec_handles import EVERY_TYPE, INVALID_VALUE, NO_EXECUTION, create_all, handle_entry_points, zero_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TAKES = {"deconv_f32": {"mnnb200_deconv_f32_set_pad", "mnnb200_deconv_f32_resize", "mnnb200_deconv_f32_execute",
                        "mnnb200_deconv_f32_plan"},
         "dwdeconv_f32": {"mnnb200_deconv_f32_set_pad", "mnnb200_dwdeconv_f32_resize", "mnnb200_dwdeconv_f32_execute"}}
BEFORE_RESIZE = {"deconv_f32": ["mnnb200_deconv_f32_execute", "mnnb200_deconv_f32_plan"],
                 "dwdeconv_f32": ["mnnb200_dwdeconv_f32_execute"]}


def deconv_entry_points(kind=None):
    """entry point names of mnn_b200_deconv.h (whose first parameter is mnnb200_<kind>*, when kind is given)"""
    hdr = open(os.path.join(ROOT, "include", "mnn_b200_deconv.h")).read()
    first = r"\s*\(\s*mnnb200_" + kind + r"\s*\*" if kind else r"\s*\("
    return re.findall(r"MNNB200_API[^;(]*?\b(mnnb200_[a-z0-9_]+)" + first, hdr)


def test_deconv_header_symbols_exported():
    declared = set(deconv_entry_points())
    assert declared == set(_capi.DECONV_SIGNATURES), declared ^ set(_capi.DECONV_SIGNATURES)
    assert not declared & set(_capi.SIGNATURES) and not declared & set(_capi.LLM_SIGNATURES)
    L = _capi.deconv_lib()
    for name in declared:
        assert hasattr(L, name), f"{name} not exported"


@pytest.mark.parametrize("kind", ["runtime", "exec"])
def test_deconv_null_handle_refused(kind):
    D = _capi.deconv_lib()
    names = deconv_entry_points(kind)
    assert names
    for name in names:
        assert getattr(D, name)(*zero_args(_capi.DECONV_SIGNATURES[name][1], buffers=False)) == INVALID_VALUE, name


def create_deconvs(rt):
    L, D, P = _capi.lib(), _capi.deconv_lib(), C.c_void_p
    w, wd = np.full((16, 16, 3, 3), 0.1, np.float32), np.full((16, 3, 3), 0.1, np.float32)
    d, dd = _capi.ConvDesc(16, 16, 3, 3, 2, 2, 1, 1, 1, 1, 1, 0), _capi.ConvDesc(16, 16, 3, 3, 2, 2, 1, 1, 1, 1, 16, 0)
    ex = {}
    for name, fn, desc, wt in (("deconv_f32", D.mnnb200_deconv_f32_create, d, w),
                               ("dwdeconv_f32", D.mnnb200_dwdeconv_f32_create, dd, wd)):
        h = P()
        assert fn(rt, C.byref(desc), wt.ctypes.data_as(P), None, 0, C.byref(h)) == 0, (name, L.mnnb200_last_error())
        ex[name] = h
    return ex


@pytest.mark.gpu
def test_deconv_exec_entry_points_refuse_other_types_and_before_resize(backend):
    L, D = _capi.lib(), _capi.deconv_lib()
    rt = backend.runtime._h
    mine = deconv_entry_points("exec")
    ex = create_deconvs(rt)
    others, keep = create_all(rt)
    try:
        for t, h in ex.items():
            for name in mine:
                if name in TAKES[t]:
                    continue
                args = zero_args(_capi.DECONV_SIGNATURES[name][1][1:], buffers=True)
                assert getattr(D, name)(h, *args) == INVALID_VALUE, (t, name)
            for name in handle_entry_points("exec"):
                if name in EVERY_TYPE:
                    continue
                args = zero_args(_capi.SIGNATURES[name][1][1:], buffers=True)
                want = 0 if name == "mnnb200_conv_int8_groupable" else INVALID_VALUE
                assert getattr(L, name)(h, *args) == want, (t, name)
            for name in BEFORE_RESIZE[t]:
                args = zero_args(_capi.DECONV_SIGNATURES[name][1][1:], buffers=True)
                if name.endswith("_plan"):
                    args[-1] = 4
                assert getattr(D, name)(h, *args) == NO_EXECUTION, (t, name, L.mnnb200_last_error())
        for t, h in others.items():
            for name in mine:
                args = zero_args(_capi.DECONV_SIGNATURES[name][1][1:], buffers=True)
                assert getattr(D, name)(h, *args) == INVALID_VALUE, (t, name)
    finally:
        for h in list(ex.values()) + [others.pop("group")] + list(others.values()):
            L.mnnb200_exec_destroy(h)
