"""Handle checks of the C ABI.  Every entry point whose first parameter is a runtime or an execution refuses a NULL one
without touching it (CPU).  Every entry point taking an execution refuses the types it does not take, and execute / plan
refuse before resize (-m gpu).  A conv group whose member was resized since bind refuses to launch until it is bound again:
the resize rewrote the tables the group's layer table points at (-m gpu)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from mnn_b200 import _capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NO_EXECUTION, INVALID_VALUE = 4, 5


def handle_entry_points(kind):
    """{name: first parameter type} of the header's entry points whose first parameter is mnnb200_<kind>*"""
    hdr = open(os.path.join(ROOT, "include", "mnn_b200.h")).read()
    names = re.findall(r"MNNB200_API[^;(]*?\b(mnnb200_[a-z0-9_]+)\s*\(\s*mnnb200_" + kind + r"\s*\*", hdr)
    assert names and set(names) <= set(_capi.SIGNATURES)
    return names


def zero_args(argtypes, buffers):
    """zero / NULL for every argument; `buffers` gives int and pointer arrays for the int* / void** ones instead"""
    out = []
    for t in argtypes:
        if t in (C.c_float, C.c_double):
            out.append(0.0)
        elif t in (C.POINTER(C.c_int), C.POINTER(C.c_void_p), C.POINTER(C.c_double)) and buffers:
            out.append(C.cast((C.c_int64 * 64)(), t))
        elif t is C.c_void_p or hasattr(t, "contents"):
            out.append(None)
        else:
            out.append(0)
    return out


# what a NULL handle gets from the entry points that do not return a status
NOT_STATUS = {"mnnb200_runtime_destroy": None, "mnnb200_exec_destroy": None, "mnnb200_runtime_stream": None,
              "mnnb200_runtime_last_gpu_ms": -1.0, "mnnb200_conv_int8_groupable": 0}


@pytest.mark.parametrize("kind", ["runtime", "exec"])
def test_null_handle_refused(kind):
    L = _capi.lib()
    for name in handle_entry_points(kind):
        argtypes = _capi.SIGNATURES[name][1]
        got = getattr(L, name)(*zero_args(argtypes, buffers=False))
        assert got == NOT_STATUS.get(name, INVALID_VALUE), name


# ---- one execution of each type ----------------------------------------------------------------------------------------
def conv_desc(ic, oc, k, group=1):
    return _capi.ConvDesc(ic, oc, k, k, 1, 1, k // 2, k // 2, 1, 1, group, 0)


def create_all(rt):
    """{type: handle} for the ten execution types, none resized"""
    L, P = _capi.lib(), C.c_void_p
    rng = np.random.default_rng(3)
    ptr = lambda a: a.ctypes.data_as(P)
    w8, f32 = (lambda *s: rng.integers(-8, 8, s).astype(np.int8)), (lambda *s: rng.random(s).astype(np.float32) + 0.5)
    keep, ex = [], {}

    def make(name, fn, *args):
        h = P()
        assert fn(*args, C.byref(h)) == 0, (name, L.mnnb200_last_error())
        ex[name] = h

    d3, dw, d1 = conv_desc(16, 16, 3), conv_desc(16, 16, 3, group=16), conv_desc(16, 16, 1)
    keep += [d3, dw, d1]
    arrays = dict(w=w8(16, 16, 3, 3), wdw=w8(16, 1, 3, 3), s=f32(16), wl=w8(16, 32), wf=f32(16, 16, 3, 3), wfdw=f32(16, 1, 3, 3))
    keep.append(arrays)
    a = arrays
    make("conv", L.mnnb200_conv_int8_create, rt, C.byref(d3), ptr(a["w"]), ptr(a["s"]), None)
    make("dwconv", L.mnnb200_dwconv_int8_create, rt, C.byref(dw), ptr(a["wdw"]), ptr(a["s"]), None)
    make("linear", L.mnnb200_linear_w8_create, rt, 32, 16, ptr(a["wl"]), ptr(a["s"]), None, None, 0, 0)
    from mnn_b200.backend import encode_winograd_attr
    attr = encode_winograd_attr([(0, 0, 3, 3, 2, 2, np.full(16, 0.1), np.zeros(16), np.full(16 * 16, 0.01))])
    keep.append(attr)
    make("wino", L.mnnb200_conv_int8_wino_create, rt, C.byref(d3), ptr(a["w"]), ptr(a["s"]), None, ptr(attr), attr.size)
    make("matmul", L.mnnb200_matmul_create, rt, 1, 8, 16, 16, 0, 0, 0)
    members = (P * 1)(ex["conv"].value)
    make("group", L.mnnb200_conv_group_create, rt, members, 1)
    make("scale_int8", L.mnnb200_scale_int8_create, rt, 16, ptr(a["s"]), None)
    make("conv_f32", L.mnnb200_conv_f32_create, rt, C.byref(d3), ptr(a["wf"]), None, 0)
    make("dwconv_f32", L.mnnb200_dwconv_f32_create, rt, C.byref(dw), ptr(a["wfdw"]), None, 0)
    make("scale_f32", L.mnnb200_scale_f32_create, rt, 16, ptr(a["s"]), None)
    return ex, keep


# entry point -> the execution types it takes (exec_cost and exec_destroy take every type)
TAKES = {
    "conv": {"mnnb200_conv_int8_resize", "mnnb200_conv_int8_execute", "mnnb200_conv_int8_groupable",
             "mnnb200_conv_int8_group_plan", "mnnb200_conv_int8_set_pad", "mnnb200_conv_int8_set_variant"},
    "dwconv": {"mnnb200_dwconv_int8_resize", "mnnb200_dwconv_int8_execute", "mnnb200_conv_int8_set_pad"},
    "linear": {"mnnb200_linear_w8_resize", "mnnb200_linear_w8_execute", "mnnb200_linear_w8_plan", "mnnb200_conv_int8_set_variant"},
    "wino": {"mnnb200_conv_int8_wino_resize", "mnnb200_conv_int8_wino_execute", "mnnb200_conv_int8_wino_execute_phases",
             "mnnb200_conv_int8_wino_plan", "mnnb200_conv_int8_set_pad"},
    "matmul": {"mnnb200_matmul_execute"},
    "group": {"mnnb200_conv_group_bind", "mnnb200_conv_group_execute"},
    "scale_int8": {"mnnb200_scale_int8_resize", "mnnb200_scale_int8_execute"},
    "conv_f32": {"mnnb200_conv_f32_resize", "mnnb200_conv_f32_execute", "mnnb200_conv_f32_plan", "mnnb200_conv_f32_set_pad"},
    "dwconv_f32": {"mnnb200_dwconv_f32_resize", "mnnb200_dwconv_f32_execute", "mnnb200_conv_f32_set_pad"},
    "scale_f32": {"mnnb200_scale_f32_resize", "mnnb200_scale_f32_execute"},
}
EVERY_TYPE = {"mnnb200_exec_cost", "mnnb200_exec_destroy"}
# execute and plan of a type before its resize (the group: before bind); matmul has no resize
BEFORE_RESIZE = {
    "conv": ["mnnb200_conv_int8_execute", "mnnb200_conv_int8_group_plan"], "dwconv": ["mnnb200_dwconv_int8_execute"],
    "linear": ["mnnb200_linear_w8_execute", "mnnb200_linear_w8_plan"],
    "wino": ["mnnb200_conv_int8_wino_execute", "mnnb200_conv_int8_wino_execute_phases", "mnnb200_conv_int8_wino_plan"],
    "group": ["mnnb200_conv_group_execute"], "scale_int8": ["mnnb200_scale_int8_execute"],
    "conv_f32": ["mnnb200_conv_f32_execute", "mnnb200_conv_f32_plan"], "dwconv_f32": ["mnnb200_dwconv_f32_execute"],
    "scale_f32": ["mnnb200_scale_f32_execute"],
}


@pytest.mark.gpu
def test_exec_entry_points_refuse_wrong_type_and_before_resize(backend):
    L = _capi.lib()
    names = handle_entry_points("exec")
    assert set().union(*TAKES.values()) | EVERY_TYPE == set(names)
    ex, keep = create_all(backend.runtime._h)
    try:
        for t, h in ex.items():
            for name in names:
                if name in TAKES[t] or name in EVERY_TYPE:
                    continue
                args = zero_args(_capi.SIGNATURES[name][1][1:], buffers=True)
                want = 0 if name == "mnnb200_conv_int8_groupable" else INVALID_VALUE
                assert getattr(L, name)(h, *args) == want, (t, name)
            for name in BEFORE_RESIZE.get(t, []):
                args = zero_args(_capi.SIGNATURES[name][1][1:], buffers=True)
                if name.endswith("_plan"):
                    args[-1] = 4
                assert getattr(L, name)(h, *args) == NO_EXECUTION, (t, name, L.mnnb200_last_error())
    finally:
        for h in [ex.pop("group")] + list(ex.values()):
            L.mnnb200_exec_destroy(h)


@pytest.mark.gpu
def test_conv_group_stale_after_member_resize(backend):
    from tests.test_gpu_conv_group import Layer, case, run_group
    rng = np.random.default_rng(17)
    layers = [Layer(backend, case(rng, 24, 40, (3, 3), 1, (10, 10), pad=(1, 1), z_in=0)),
              Layer(backend, case(rng, 32, 48, (1, 1), 2, (8, 8)))]
    grp = run_group(backend, layers)
    for L in layers:
        L.check()
    # a larger batch and a non-zero input zero point: the member's epilogue table is rewritten and its border tables appear
    before = layers[0].plan()
    c = layers[0].c
    c["x"] = rng.integers(-128, 128, (3,) + c["x"].shape[1:]).astype(np.int8)
    c["z_in"] = 5
    layers[0].resize()
    assert layers[0].plan()["m_tiles"] > before["m_tiles"]
    assert grp.onExecute() == NO_EXECUTION
    assert b"resized since bind" in _capi.lib().mnnb200_last_error()
    assert grp.bind([L.xin for L in layers], [L.yout for L in layers]) == 0
    for L in layers:
        L.poison()
    assert grp.onExecute() == 0
    backend.onSync()
    for L in layers:
        L.check()
