"""Grouped fp32 Convolution through the MNN plugin (-m gpu).  The unmodified reference core runs grouped Convolution ops and two
ResNeXt bottlenecks through its Express executor on MNN_FORWARD_CUDA = mnn_b200/libmnn_b200_plugin.so (oracle/_ref/refdump_gconv),
and ResNeXt-50 32x4d (oracle/_ref/resnext50_f32.mnn, seeded weights, written by build()) through its Interpreter.  Nothing may be
declined to the CPU backup backend, and every output must be within 1e-3 of MNN_FORWARD_CPU (max|d| / max|ref|)."""
import os
import tempfile

import numpy as np
import pytest

from oracle import gconv_oracle as D
from tests.golden import make_gconv_golden as G
from tests.test_plugin import PLUGIN, _run
from tests.test_plugin_f32 import _compare

pytestmark = pytest.mark.gpu


def _need_harness():
    if not D.have_refdump():
        pytest.skip("oracle/_ref/refdump_gconv is built by build() where the reference sources are")
    if not os.path.exists(PLUGIN):
        pytest.fail("mnn_b200/libmnn_b200_plugin.so is missing although the reference harness is present")


def _rel(a, b):
    return float(np.abs(np.asarray(a, np.float64) - b).max() / max(np.abs(b).max(), 1e-12))


@pytest.mark.parametrize("name", list(G.CASES))
def test_golden_op_on_plugin(name):
    """each recorded grouped op (the inputCount form included) on the plugin: created there, within 1e-3 of the recorded CPU
    outputs"""
    _need_harness()
    n, ic, oc, hw, k, s, pads, d, group, input_count, relu, relu6 = G.CASES[name]
    x, w, b = G.case_inputs(name)
    y, stats = D.ref_gconv(x, w, b, group, input_count, s, pads, d, bool(relu), bool(relu6), plugin=PLUGIN)
    assert stats is not None and stats["plugin_declined"] == 0 and stats["plugin_created"] >= 1, stats
    rec, idx, shape = G.load()[name]
    assert y.shape == shape
    flat = y.astype(np.float64).reshape(-1)
    assert _rel(flat if idx is None else flat[idx], rec) <= 1e-3


def test_resnext_bottlenecks_on_plugin():
    """a stride-2 bottleneck with a projection shortcut, then one with an identity shortcut, run twice on one executor with two
    inputs: every op on the plugin, both runs' grouped-conv and graph outputs within 1e-3 of the CPU backend's"""
    _need_harness()
    cpu, _ = D.ref_block(2, 5)
    gpu, stats = D.ref_block(2, 5, plugin=PLUGIN)
    assert stats is not None and stats["plugin_declined"] == 0 and stats["plugin_created"] >= 8, stats
    assert sorted(cpu) == sorted(gpu) == ["grouped_0", "grouped_1", "output_0", "output_1"]
    assert not np.array_equal(cpu["output_0"], cpu["output_1"])
    for k in cpu:
        assert _rel(gpu[k], cpu[k]) <= 1e-3, k


def _resnext():
    _need_harness()
    if not os.path.exists(D.RESNEXT):
        pytest.skip("oracle/_ref/resnext50_f32.mnn is written by build() where the reference sources are")
    return D.RESNEXT


def test_resnext50_on_plugin_matches_cpu_backend():
    """ResNeXt-50 at batch 2 through the Interpreter: every command on the plugin, every fp32 tensor within 1e-3 of the CPU's"""
    model = _resnext()
    with tempfile.TemporaryDirectory() as d:
        cpu, _, _ = _run(os.path.join(d, "cpu"), 2, False, model)
        gpu, stats, r = _run(os.path.join(d, "gpu"), 2, True, model)
        kinds = _compare(d, cpu, gpu, stats, r)
    assert kinds["Convolution"] >= 53, kinds


def test_resnext50_graph_replay_matches_cpu_backend():
    """4 plain forwards first (eager, capture, replay, replay): the replayed output equals the CPU backend's within 1e-3"""
    model = _resnext()
    keep = os.environ.get("REFDUMP_RUN_REPEATS")
    os.environ["REFDUMP_RUN_REPEATS"] = "4"
    try:
        with tempfile.TemporaryDirectory() as d:
            cpu, _, _ = _run(os.path.join(d, "cpu"), 2, False, model)
            gpu, stats, r = _run(os.path.join(d, "gpu"), 2, True, model)
            _compare(d, cpu, gpu, stats, r)
            oc = np.fromfile(os.path.join(d, "cpu", "output_plain.f32"), np.float32)
            og = np.fromfile(os.path.join(d, "gpu", "output_plain.f32"), np.float32)
            assert _rel(og, oc) <= 1e-3, "graph-replayed forward differs"
    finally:
        if keep is None:
            os.environ.pop("REFDUMP_RUN_REPEATS", None)
        else:
            os.environ["REFDUMP_RUN_REPEATS"] = keep
