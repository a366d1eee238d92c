"""Handle checks of libmnn_b200_llm.so's C ABI (include/mnn_b200_llm.h), whose LayerNorm and RoPE executions share
libmnn_b200.so's handles.  Every entry point of mnn_b200_llm.h exists in the library with the binding's signature, and those
whose first parameter is a runtime or an execution refuse a NULL one (CPU).  Every LLM entry point taking an execution refuses
every other execution type, including the ten of mnn_b200.h, every execution entry point of mnn_b200.h refuses the two LLM
types, and execute refuses before resize (-m gpu)."""
import ctypes as C
import os
import re

import pytest

from mnn_b200 import _capi
from tests.test_exec_handles import EVERY_TYPE, INVALID_VALUE, NO_EXECUTION, create_all, handle_entry_points, zero_args

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TAKES = {"layernorm_f32": {"mnnb200_layernorm_f32_resize", "mnnb200_layernorm_f32_execute"},
         "rope_f32": {"mnnb200_rope_f32_resize", "mnnb200_rope_f32_execute"}}
BEFORE_RESIZE = {"layernorm_f32": ["mnnb200_layernorm_f32_execute"], "rope_f32": ["mnnb200_rope_f32_execute"]}


def llm_entry_points(kind=None):
    """entry point names of mnn_b200_llm.h (whose first parameter is mnnb200_<kind>*, when kind is given)"""
    hdr = open(os.path.join(ROOT, "include", "mnn_b200_llm.h")).read()
    first = r"\s*\(\s*mnnb200_" + kind + r"\s*\*" if kind else r"\s*\("
    return re.findall(r"MNNB200_API[^;(]*?\b(mnnb200_[a-z0-9_]+)" + first, hdr)


def test_llm_header_symbols_exported():
    declared = set(llm_entry_points())
    assert declared == set(_capi.LLM_SIGNATURES), declared ^ set(_capi.LLM_SIGNATURES)
    assert not declared & set(_capi.SIGNATURES)
    L = _capi.llm_lib()
    for name in declared:
        assert hasattr(L, name), f"{name} not exported"


@pytest.mark.parametrize("kind", ["runtime", "exec"])
def test_llm_null_handle_refused(kind):
    L = _capi.llm_lib()
    names = llm_entry_points(kind)
    assert names
    for name in names:
        got = getattr(L, name)(*zero_args(_capi.LLM_SIGNATURES[name][1], buffers=False))
        assert got == INVALID_VALUE, name


def create_llm_ops(rt):
    L, P = _capi.llm_lib(), C.c_void_p
    ex = {}
    for name, fn, args in (("layernorm_f32", L.mnnb200_layernorm_f32_create, (rt, 64, 1e-6, 1, None, None, 0)),
                           ("rope_f32", L.mnnb200_rope_f32_create, (rt, 2, 1, 64, 0, None, None))):
        h = P()
        assert fn(*args, C.byref(h)) == 0, (name, _capi.lib().mnnb200_last_error())
        ex[name] = h
    return ex


@pytest.mark.gpu
def test_llm_exec_entry_points_refuse_other_types_and_before_resize(backend):
    core, L = _capi.lib(), _capi.llm_lib()
    llm_names = llm_entry_points("exec")
    assert set().union(*TAKES.values()) == set(llm_names)
    core_names = [n for n in handle_entry_points("exec") if n not in EVERY_TYPE]
    ex, keep = create_all(backend.runtime._h)
    llm = create_llm_ops(backend.runtime._h)
    try:
        for t, h in list(ex.items()) + list(llm.items()):
            for name in llm_names:
                if name in TAKES.get(t, ()):
                    continue
                args = zero_args(_capi.LLM_SIGNATURES[name][1][1:], buffers=True)
                assert getattr(L, name)(h, *args) == INVALID_VALUE, (t, name)
        for t, h in llm.items():
            for name in core_names:
                args = zero_args(_capi.SIGNATURES[name][1][1:], buffers=True)
                want = 0 if name == "mnnb200_conv_int8_groupable" else INVALID_VALUE
                assert getattr(core, name)(h, *args) == want, (t, name)
            for name in BEFORE_RESIZE[t]:
                args = zero_args(_capi.LLM_SIGNATURES[name][1][1:], buffers=True)
                assert getattr(L, name)(h, *args) == NO_EXECUTION, (t, name, core.mnnb200_last_error())
            cost = (C.c_double(), C.c_double())
            assert core.mnnb200_exec_cost(h, C.byref(cost[0]), C.byref(cost[1])) == 0
    finally:
        for h in [ex.pop("group")] + list(ex.values()) + list(llm.values()):
            core.mnnb200_exec_destroy(h)
