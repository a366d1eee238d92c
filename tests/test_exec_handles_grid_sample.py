"""Handle checks of libmnn_b200_grid_sample.so's C ABI (include/mnn_b200_grid_sample.h), whose fp32 GridSample execution shares
libmnn_b200.so's handles.  Every entry point of the header exists in the library with the binding's signature, and those whose
first parameter is a runtime or an execution refuse a NULL one (CPU).  Every GridSample entry point taking an execution refuses
every other execution type (the core library's, the Deconvolution, Interp, gather, scatter and RNN libraries'), every execution
entry point of those libraries refuses the GridSample execution, and execute / plan refuse before resize (-m gpu)."""
import ctypes as C
import os
import re

import pytest

from mnn_b200 import _capi
from tests.test_exec_handles import EVERY_TYPE, INVALID_VALUE, NO_EXECUTION, create_all, handle_entry_points, zero_args
from tests.test_exec_handles_deconv import create_deconvs, deconv_entry_points
from tests.test_exec_handles_gather import gather_entry_points
from tests.test_exec_handles_interp import create_interp, interp_entry_points
from tests.test_exec_handles_rnn import rnn_entry_points
from tests.test_exec_handles_scatter import scatter_entry_points

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BEFORE_RESIZE = ["mnnb200_grid_sample_f32_execute", "mnnb200_grid_sample_f32_plan"]


def grid_sample_entry_points(kind=None):
    """entry point names of mnn_b200_grid_sample.h (whose first parameter is mnnb200_<kind>*, when kind is given)"""
    hdr = open(os.path.join(ROOT, "include", "mnn_b200_grid_sample.h")).read()
    first = r"\s*\(\s*mnnb200_" + kind + r"\s*\*" if kind else r"\s*\("
    return re.findall(r"MNNB200_API[^;(]*?\b(mnnb200_[a-z0-9_]+)" + first, hdr)


def test_grid_sample_header_symbols_exported():
    declared = set(grid_sample_entry_points())
    assert declared == set(_capi.GRID_SAMPLE_SIGNATURES), declared ^ set(_capi.GRID_SAMPLE_SIGNATURES)
    assert not declared & (set(_capi.SIGNATURES) | set(_capi.LLM_SIGNATURES) | set(_capi.DECONV_SIGNATURES) |
                           set(_capi.INTERP_SIGNATURES) | set(_capi.GATHER_SIGNATURES) | set(_capi.SCATTER_SIGNATURES) |
                           set(_capi.RNN_SIGNATURES))
    L = _capi.grid_sample_lib()
    for name in declared:
        assert hasattr(L, name), f"{name} not exported"


@pytest.mark.parametrize("kind", ["runtime", "exec"])
def test_grid_sample_null_handle_refused(kind):
    L = _capi.grid_sample_lib()
    names = grid_sample_entry_points(kind)
    assert names
    for name in names:
        assert getattr(L, name)(*zero_args(_capi.GRID_SAMPLE_SIGNATURES[name][1], buffers=False)) == INVALID_VALUE, name


@pytest.mark.gpu
def test_grid_sample_exec_entry_points_refuse_other_types_and_before_resize(backend):
    L, D, I, G, S, N, GS = (_capi.lib(), _capi.deconv_lib(), _capi.interp_lib(), _capi.gather_lib(), _capi.scatter_lib(),
                            _capi.rnn_lib(), _capi.grid_sample_lib())
    rt = backend.runtime._h
    mine = grid_sample_entry_points("exec")
    h = C.c_void_p()
    assert GS.mnnb200_grid_sample_f32_create(rt, 0, 0, 0, C.byref(h)) == 0
    gather, scatter, rnn = C.c_void_p(), C.c_void_p(), C.c_void_p()
    assert G.mnnb200_gather_create(rt, 0, C.byref(gather)) == 0
    assert S.mnnb200_scatter_create(rt, 0, -1, 1, C.byref(scatter)) == 0
    assert N.mnnb200_rnn_create(rt, 0, C.byref(rnn)) == 0
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
        for lib, names, sigs in ((D, deconv_entry_points("exec"), _capi.DECONV_SIGNATURES),
                                 (I, interp_entry_points("exec"), _capi.INTERP_SIGNATURES),
                                 (G, gather_entry_points("exec"), _capi.GATHER_SIGNATURES),
                                 (S, scatter_entry_points("exec"), _capi.SCATTER_SIGNATURES),
                                 (N, rnn_entry_points("exec"), _capi.RNN_SIGNATURES)):
            for name in names:
                assert getattr(lib, name)(h, *zero_args(sigs[name][1][1:], buffers=True)) == INVALID_VALUE, name
        for name in BEFORE_RESIZE:
            args = zero_args(_capi.GRID_SAMPLE_SIGNATURES[name][1][1:], buffers=True)
            if name.endswith("_plan"):
                args[-1] = 4
            assert getattr(GS, name)(h, *args) == NO_EXECUTION, (name, L.mnnb200_last_error())
        for t, o in list(others.items()) + list(deconvs.items()) + [("interp", interp), ("gather", gather), ("scatter", scatter),
                                                                    ("rnn", rnn)]:
            for name in mine:
                args = zero_args(_capi.GRID_SAMPLE_SIGNATURES[name][1][1:], buffers=True)
                assert getattr(GS, name)(o, *args) == INVALID_VALUE, (t, name)
    finally:
        for o in [h, gather, scatter, rnn, interp] + list(deconvs.values()) + [others.pop("group")] + list(others.values()):
            L.mnnb200_exec_destroy(o)
