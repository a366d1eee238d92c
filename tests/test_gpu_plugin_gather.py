"""Gather, GatherV2, GatherND, GatherElements, Cast, broadcast MatMul and BatchMatMul through the MNN plugin (-m gpu).  The unmodified
reference core runs each recorded op through its Express executor on MNN_FORWARD_CUDA = mnn_b200/libmnn_b200_plugin.so
(oracle/_ref/refdump_gather), four input sets on one executor (eager, then captured and replayed as a graph): created there,
gathers and casts bit for bit, MatMuls within 1e-3.  Every case of matmul_golden.npz, the batched ones included, runs the same
way.  The BERT- and ViT-style fixtures (oracle/_ref/{bert,vit}_f32.mnn) run through the Interpreter at batch 2 with nothing
declined: the CPU runs the gathers and the broadcast / batched MatMuls as While loops, which are matched with the plugin's
commands by name.  Every compute command's fp32 output and the session output are within 1e-3 of the CPU's (max|d| / max|ref|),
and a graph-replayed forward equals the eager one bit for bit."""
import os
import re
import tempfile

import numpy as np
import pytest

from oracle import gather_oracle as G
from tests.golden import make_gather_golden as M
from tests.test_plugin import PLUGIN

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _need_harness():
    if not G.have_refdump():
        pytest.skip("oracle/_ref/refdump_gather is built by build() where the reference sources are")
    if not os.path.exists(PLUGIN):
        pytest.fail("mnn_b200/libmnn_b200_plugin.so is missing although the reference harness is present")


def _rel(a, ref):
    return float(np.abs(np.asarray(a, np.float64) - ref).max() / max(np.abs(ref).max(), 1e-12))


def _more_sets(name, n=3):
    """further input sets of a case's shapes and index ranges"""
    rng = np.random.default_rng(len(name))
    base = M.case_inputs(name)
    sets = []
    for _ in range(n):
        s = []
        for a in base:
            if a.dtype == np.int32 and name not in M.MATMUL_CASES and len(s) == 1:
                s.append(rng.permutation(a.reshape(-1)).reshape(a.shape).astype(np.int32))   # the same index values, moved
            elif a.dtype == np.int32:
                s.append(rng.integers(-1000, 1000, a.shape).astype(np.int32))
            else:
                s.append(rng.standard_normal(a.shape).astype(np.float32))
        sets.append(s)
    return sets


@pytest.mark.parametrize("name", list(M.CASES))
def test_golden_op_on_plugin(name):
    _need_harness()
    more = _more_sets(name)
    ys, stats = M.case_reference(name, more=more, plugin=PLUGIN)
    assert stats is not None and stats["plugin_declined"] == 0 and stats["plugin_created"] >= 1, stats
    shape, sha = M.load()[0][name]
    assert ys[0].shape == shape and M.digest(ys[0]) == sha
    c = M.CASES[name]
    for inputs, y in zip([M.case_inputs(name)] + more, ys):
        if c["kind"] == "Cast":
            ref = G.cast_i32_f32(inputs[0]) if c["cast_to"] == "float32" else G.cast_f32_i32(inputs[0])
        elif c["kind"] == "GatherND":
            ref = G.gather_nd(*inputs, c["axis"] or 0)
        elif c["kind"] == "GatherElements":
            ref = G.gather_elements(*inputs, c["axis"] or 0)
        else:
            ref = G.gather(*inputs, c["axis"] or 0)
        assert np.array_equal(np.ascontiguousarray(y).view(np.uint32), np.ascontiguousarray(ref).view(np.uint32))


@pytest.mark.parametrize("name", list(M.MATMUL_CASES))
def test_broadcast_matmul_golden_on_plugin(name):
    """within 1e-3 of the recorded CPU on the eager run, and the captured and replayed runs of the same inputs equal to it"""
    _need_harness()
    ys, stats = M.case_reference(name, more=[M.case_inputs(name)] * 3, plugin=PLUGIN)
    assert stats is not None and stats["plugin_declined"] == 0 and stats["plugin_created"] >= 1, stats
    ref = M.load()[1][name]
    assert ys[0].shape == ref.shape and _rel(ys[0], ref) <= 1e-3
    for y in ys[1:]:
        assert np.array_equal(y.view(np.uint32), ys[0].view(np.uint32))


def test_every_matmul_golden_through_reference_executor_on_plugin():
    """matmul_golden.npz's cases, batched ones included, as MatMul ops on the plugin: none declined, each within 1e-3"""
    _need_harness()
    g = np.load(os.path.join(ROOT, "tests", "golden", "matmul_golden.npz"))
    batched = 0
    for i in range(int(g["ncase"])):
        a, b, ta, tb, ref = g[f"m{i}_a"], g[f"m{i}_b"], bool(g[f"m{i}_ta"]), bool(g[f"m{i}_tb"]), g[f"m{i}_y"]
        y, stats = G.ref_op("MatMul", [a, b], ta=ta, tb=tb, plugin=PLUGIN)
        assert stats is not None and stats["plugin_declined"] == 0 and stats["plugin_created"] >= 1, (i, stats)
        assert y.shape == ref.shape and _rel(y, ref) <= 1e-3, (i, _rel(y, ref))
        batched += a.ndim > 2
    assert batched >= 3


def _norm(name):
    return re.sub(r"_raster_\d+$", "", name)


# every compute command and the session output, MatMuls and all they feed included
MODEL_REL = 1e-3


def _compare_models(d, cpu, gpu, stats, r):
    """every plugin compute command against the CPU's last command of the same name (the CPU's While for a gather or a
    broadcast MatMul)"""
    assert stats is not None and stats["plugin_declined"] == 0, f"commands fell back to the CPU backend: {stats}\n{r.stdout[-2500:]}"
    cpu_by = {}
    for f, n, t in cpu:
        if not t.startswith("Raster"):
            cpu_by[_norm(n)] = f
    compared, worst = 0, {}
    for f, n, t in gpu:
        if t.startswith("Raster"):
            continue
        if _norm(n) not in cpu_by:
            # a Gather of fewer than 3 constant indices is a Raster region on the CPU (GeometryGather.cpp:45-71), folded into
            # its consumer's input: no command of its own; its consumer's output is compared
            assert t in ("Gather", "GatherV2"), f"plugin command {n} ({t}) has no CPU command of that name"
            continue
        a = np.fromfile(os.path.join(d, "cpu", cpu_by[_norm(n)]), np.float32)
        b = np.fromfile(os.path.join(d, "gpu", f), np.float32)
        assert a.shape == b.shape, n
        err = _rel(b, a)
        assert err <= MODEL_REL, f"{n} ({t}) rel err {err}"
        compared += 1
        worst[t] = max(worst.get(t, 0.0), err)
    oc = np.fromfile(os.path.join(d, "cpu", "output.f32"), np.float32)
    og = np.fromfile(os.path.join(d, "gpu", "output.f32"), np.float32)
    assert oc.shape == og.shape and _rel(og, oc) <= MODEL_REL, f"session output differs: {_rel(og, oc)}"
    worst["session output"] = _rel(og, oc)
    replayed = np.fromfile(os.path.join(d, "gpu", "output_plain.f32"), np.float32)
    assert np.array_equal(replayed.view(np.uint32), og.view(np.uint32)), "the graph-replayed forward differs from the eager one"
    return compared, worst


@pytest.mark.parametrize("model", ["bert", "vit"])
def test_transformer_fixture_on_plugin_matches_cpu_backend(model):
    _need_harness()
    path = G.BERT if model == "bert" else G.VIT
    if not os.path.exists(path):
        pytest.skip(f"{path} is written by build() where the reference sources are")
    with tempfile.TemporaryDirectory() as d:
        cpu, _, _ = G.run_model(path, 2, 3, os.path.join(d, "cpu"))
        gpu, stats, r = G.run_model(path, 2, 3, os.path.join(d, "gpu"), plugin=PLUGIN, repeats=4)
        compared, worst = _compare_models(d, cpu, gpu, stats, r)
    types = {t for _, _, t in gpu}
    assert {"MatMul", "BatchMatMul"} <= types and ({"GatherV2", "Cast"} <= types if model == "bert" else "Gather" in types)
    assert sum(t == "While" for _, _, t in cpu) >= 10
    print(f"{model}: {compared} plugin commands compared, created {stats['plugin_created']}, worst rel err per type "
          + ", ".join(f"{t} {e:.2e}" for t, e in sorted(worst.items())))
