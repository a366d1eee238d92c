"""The plugin's fp32 neighbour ops one op at a time (-m gpu): BinaryOp, Eltwise, ReLU, UnaryOp, Pooling, Reduction, Softmax, ArgMax /
ArgMin, Scale and the Raster that Transpose, Concat, Slice, StridedSlice, Pad, Tile, BroadcastTo and layout changes lower to.
Every case of oracle/ops_oracle.all_cases() runs through the reference's Express executor (oracle/_ref/refdump_ops) on
MNN_FORWARD_CPU and on MNN_FORWARD_CUDA = the plugin, all cases in one process each.

Nothing but the declined forms may be handed to the CPU backup backend.  The CPU is matched bit for bit (every NaN counted equal)
wherever the kernel restates the CPU's float path; the transcendental UnaryOps, Softmax and the SUM / MEAN / PROD reductions are
held to bounds against float64 (oracle/ops_oracle.py), and to the same bound plus the CPU's own error against the CPU.  Cases
with several runs go through one executor: new values (the second run is captured into a CUDA graph, the third replays it), then
other shapes, so that what an execution derives from shapes at resize is derived again."""
import os

import numpy as np
import pytest

from oracle import ops_oracle as O
from tests.test_plugin import PLUGIN

pytestmark = pytest.mark.gpu
CASES = O.all_cases()
# ulp bounds of the GPU's transcendental UnaryOps against float64, from the CUDA math library's documented maxima (expf 2 ulp,
# logf 1, tanhf 2, erfcf 4) plus half an ulp per further rounded operation; GELU and GELU_STANDARD add their inner argument's
# rounding times the outer function's condition number (gelu_condition)
UNARY_ULPS = {"EXP": 2, "LOG": 1, "TANH": 2, "SIGMOID": 4, "SILU": 5, "GELU": 5, "GELU_STANDARD": 5}
# the plugin's declined count of each declined form: one per op it has no execution for
DECLINED = {"declined_unary_FLOOR": 1, "declined_unary_SIN": 1, "declined_unary_ERF": 1, "declined_binary_POW": 1,
            "declined_binary_FLOORDIV": 1, "declined_eltwise_coeff": 1, "declined_argmax_top2": 1,
            "declined_softmax_nhwc_4d": 1}


@pytest.fixture(scope="module")
def results():
    if not O.have_refdump():
        pytest.skip("oracle/_ref/refdump_ops is built by build() where the reference sources are")
    if not os.path.exists(PLUGIN):
        pytest.fail("mnn_b200/libmnn_b200_plugin.so is missing although the reference harness is present")
    cases = list(CASES.values())
    cpu, gpu = O.run(cases), O.run(cases, plugin=PLUGIN)
    return {n: (c, g) for n, c, g in zip(CASES, cpu, gpu)}


def gelu_condition(op, x):
    """the condition number of x sigmoid(t) in its inner argument t = 2 sqrt(2/pi) (x + 0.044715 x^3) (GELU), and of
    0.5 x erfc(u) in u = -x / sqrt 2 (GELU_STANDARD), in float64"""
    x = np.asarray(x, np.float64)
    with np.errstate(all="ignore"):
        if op == "GELU":
            t = 2 * np.sqrt(2 / np.pi) * (x + 0.044715 * x ** 3)
            return np.abs(t) * (1 - O.unary64("SIGMOID", t))
        if op == "GELU_STANDARD":
            from scipy.special import erfcx
            u = -x / np.sqrt(2)
            return np.abs(2 * u / np.sqrt(np.pi) / erfcx(u))
    return np.zeros_like(x)


def unary_bound(op, x):
    """the GPU's bound in ulps per element.  An inner argument off by a relative error r moves the result by condition * r, which
    is at most condition * r / 2^-24 ulps.  GELU's t = 2 * 0.79788458 (x + 0.044715 x^3): five roundings (5 * 2^-24) and the two
    constants' own errors (4.9e-8 and 2.8e-8); GELU_STANDARD's u = -0.70710678 x: one rounding and 1.7e-8"""
    r = {"GELU": 5 * 2.0 ** -24 + 7.7e-8, "GELU_STANDARD": 2.0 ** -24 + 1.7e-8}.get(op, 0.0)
    return UNARY_ULPS[op] + gelu_condition(op, x) * r / 2.0 ** -24


def _kind_checks(name):
    c = CASES[name]
    if c["kind"] == "unary":
        op = [k for k, v in O.UNARY.items() if v == c["ip"][0]][0]
        return "bound_unary" if op in O.UNARY_TRANSCENDENTAL else "bits", op
    if c["kind"] == "reduce":
        op = [k for k, v in O.REDUCE.items() if v == c["ip"][0]][0]
        return ("bits" if op in ("MAXIMUM", "MINIMUM") else "bound_reduce"), op
    if c["kind"] == "softmax":
        return "bound_softmax", None
    return "bits", None


def _nan_positions(y, ref):
    return y.shape == ref.shape and np.array_equal(np.isnan(y), np.isnan(ref))


@pytest.mark.parametrize("name", [n for n in CASES if not n.startswith("declined_")])
def test_op_on_plugin_matches_cpu(results, name):
    cpu, gpu = results[name]
    c = CASES[name]
    assert cpu["ok"], "the CPU could not run the case"
    assert gpu["ok"] and gpu["declined"] == 0 and gpu["created"] >= 1, gpu
    mode, op = _kind_checks(name)
    special = "special" in name
    for run, (xs, y, ref) in enumerate(zip(c["runs"], gpu["ys"], cpu["ys"])):
        where = f"{name} run {run}"
        assert y.shape == ref.shape and y.dtype == ref.dtype, where
        if mode == "bits":
            if c["kind"] in ("transpose", "concat", "slice", "strided_slice", "pad", "tile", "broadcast_to", "reshape", "convert"):
                assert np.array_equal(O.bits(y), O.bits(ref)), where   # a copy: NaN payloads too
            else:
                assert O.same_bits(y, ref), f"{where}: {np.flatnonzero(O.bits(y) != O.bits(ref))[:8]}"
            continue
        if special:
            # no finite bound through an infinity or NaN: the NaN positions agree with float64's.  Not with the CPU's: its
            # polynomial TANH, SIGMOID and EXP clamp their argument, so NaN gives 1, 1 and 1.6e-38 there, and its Softmax of a
            # row holding +inf or NaN is not NaN
            x = xs[0]
            y64 = O.unary64(op, x) if mode == "bound_unary" else (
                O.softmax64(x, c["ip"][0]) if mode == "bound_softmax" else O.reduce64(x, op, c["ip"][2:], c["ip"][1]))
            with np.errstate(all="ignore"):
                assert _nan_positions(y, y64.astype(np.float32)), where
            continue
        if mode == "bound_unary":
            x = xs[0]
            y64 = O.unary64(op, x)
            e_gpu, e_cpu = O.ulp_error(y, y64), O.ulp_error(ref, y64)
            bound = unary_bound(op, x)
            print(f"{op}: GPU max {e_gpu.max():.3g} ulp (bound {UNARY_ULPS[op]}+), CPU max {e_cpu.max():.3g} ulp vs float64")
            worst = np.argmax(e_gpu - bound)
            assert (e_gpu <= bound).all(), f"{where}: x={x[worst]!r} gpu={y[worst]!r} f64={y64[worst]!r} {e_gpu[worst]} ulp"
            # against the CPU: the same bound plus the CPU's own error, in ulps of float64's result (where the GPU is finite:
            # past FLT_MAX the CPU's EXP clamps)
            e_gc = np.abs(y.astype(np.float64) - ref) / O.ulp32(y64)
            fin = np.isfinite(y)
            assert (e_gc[fin] <= bound[fin] + e_cpu[fin] + 1e-9).all(), where
        elif mode == "bound_softmax":
            axis = c["ip"][0]
            x = xs[0] if c["inputs"][0][1] == O.NCHW else xs[0]
            y64 = O.softmax64(x, axis)
            b = O.softmax_bound(x, axis)
            print(f"{name}: GPU {np.abs(y - y64).max():.3g}, CPU {np.abs(ref - y64).max():.3g}, bound {b.max():.3g}")
            assert (np.abs(y - y64) <= b).all(), where
            assert (np.abs(y.astype(np.float64) - ref) <= b + np.abs(ref - y64)).all(), where
        else:
            axes, keep = c["ip"][2:], c["ip"][1]
            x = xs[0]
            y64 = O.reduce64(x, op, axes, keep)
            b = O.sum_bound(x, axes, op).reshape(y64.shape)
            print(f"{name}: GPU {np.abs(y - y64).max():.3g}, CPU {np.abs(ref - y64).max():.3g}, bound {b.max():.3g}")
            assert (np.abs(y - y64) <= b).all(), where
            assert (np.abs(y.astype(np.float64) - ref) <= b + np.abs(ref - y64)).all(), where


@pytest.mark.parametrize("name", list(DECLINED))
def test_declined_form_runs_on_cpu_backup(results, name):
    cpu, gpu = results[name]
    assert cpu["ok"] and gpu["ok"]
    assert gpu["declined"] == DECLINED[name], gpu
    for y, ref in zip(gpu["ys"], cpu["ys"]):
        assert O.same_bits(y, ref), name


def test_every_family_is_rerun_and_resized():
    kinds = {CASES[n]["kind"] for n in CASES if "rerun_resize" in n}
    assert kinds >= {"binary", "eltwise", "relu", "unary", "pool", "reduce", "softmax", "argmax", "scale", "concat", "pad"}
    for n in CASES:
        if "rerun_resize" in n:
            shapes = [tuple(a.shape for a in r) for r in CASES[n]["runs"]]
            assert len(shapes) >= 4 and shapes[0] == shapes[1] == shapes[2] != shapes[3], n
