"""ScatterNd and ScatterElements through the MNN plugin (-m gpu).  The unmodified reference core runs each recorded op through its
Express executor on MNN_FORWARD_CUDA = mnn_b200/libmnn_b200_plugin.so (oracle/_ref/refdump_scatter), four input sets on one
executor (eager, then captured and replayed as a graph with the new indices and updates): every case is created on the plugin
with nothing declined, and each output equals the golden or the sequential loop bit for bit.  The PointPillars- and
GraphSAGE-style fixtures (oracle/_ref/{pillars,gnn}_f32.mnn) run through the Interpreter with nothing declined, within 1e-3 of
the CPU backend command by command, and a graph-replayed forward equals the eager one bit for bit."""
import os
import tempfile

import numpy as np
import pytest

from oracle import scatter_oracle as S
from tests.golden import make_scatter_golden as M
from tests.test_gpu_plugin_gather import _compare_models
from tests.test_plugin import PLUGIN

pytestmark = pytest.mark.gpu


def _need_harness():
    if not S.have_refdump():
        pytest.skip("oracle/_ref/refdump_scatter is built by build() where the reference sources are")
    if not os.path.exists(PLUGIN):
        pytest.fail("mnn_b200/libmnn_b200_plugin.so is missing although the reference harness is present")


def _more_sets(name, n=3):
    """further (indices, updates[, data]) of a case's shapes: the same index values moved, fresh updates and data"""
    rng = np.random.default_rng(len(name) + 7)
    idx, upd, data = M.case_inputs(name)
    sets = []
    for _ in range(n):
        if M.CASES[name]["kind"] == "ScatterNd":
            i = idx.reshape(-1, idx.shape[-1])[rng.permutation(idx.reshape(-1, idx.shape[-1]).shape[0])].reshape(idx.shape)
        else:
            i = rng.permutation(idx.reshape(-1)).reshape(idx.shape)
        fresh = (lambda a: rng.integers(-1000, 1000, a.shape).astype(np.int32)) if upd.dtype == np.int32 else \
                (lambda a: rng.standard_normal(a.shape).astype(np.float32))
        s = (i.astype(np.int32), fresh(upd))
        sets.append(s + ((fresh(data),) if data is not None else ()))
    return sets


@pytest.mark.parametrize("name", sorted(M.CASES))
def test_golden_op_on_plugin(name):
    _need_harness()
    c = M.CASES[name]
    more = _more_sets(name)
    ys, stats = M.case_reference(name, more=more, plugin=PLUGIN)
    assert stats is not None and stats["plugin_declined"] == 0 and stats["plugin_created"] >= 1, stats
    shape, sha = M.load()[name]
    assert ys[0].shape == shape and M.digest(ys[0]) == sha
    red = M.reduction(name)
    for k, s in enumerate(more, 1):
        idx, upd = s[0], s[1]
        data = s[2] if len(s) > 2 else None
        ref = S.scatter(c["kind"], c["out"], idx, upd, data, red, c.get("axis") or 0)
        assert np.array_equal(S.canonical(ys[k]), S.canonical(ref)), f"input set {k}"
        if red is None:
            assert np.array_equal(ys[k].view(np.uint32), ref.view(np.uint32)), f"input set {k}: NaN payloads"


@pytest.mark.parametrize("model", ["pillars", "gnn"])
def test_scatter_fixture_on_plugin_matches_cpu_backend(model):
    """the PointPillars- and GraphSAGE-style fixtures through the Interpreter at batch 1: nothing declined, every compute
    command and the session output within 1e-3 of MNN_FORWARD_CPU (matched by name), a graph-replayed forward equal to the
    eager one"""
    _need_harness()
    path = S.PILLARS if model == "pillars" else S.GNN
    if not os.path.exists(path):
        pytest.skip(f"{path} is written by build() where the reference sources are")
    with tempfile.TemporaryDirectory() as d:
        cpu, _, _ = S.run_model(path, 1, 3, os.path.join(d, "cpu"))
        gpu, stats, r = S.run_model(path, 1, 3, os.path.join(d, "gpu"), plugin=PLUGIN, repeats=4)
        compared, worst = _compare_models(d, cpu, gpu, stats, r)
    types = {t for _, _, t in gpu}
    want = {"ScatterNd", "Convolution", "Deconvolution"} if model == "pillars" else {"ScatterElements", "GatherV2", "BinaryOp"}
    assert want <= types, types
    print(f"{model}: {compared} plugin commands compared, created {stats['plugin_created']}, worst rel err per type "
          + ", ".join(f"{t} {e:.2e}" for t, e in sorted(worst.items())))
