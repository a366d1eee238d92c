"""fp32 GridSample through the MNN plugin (-m gpu).  The unmodified reference core runs the recorded GridSample ops through its
Express executor on MNN_FORWARD_CUDA = mnn_b200/libmnn_b200_plugin.so (oracle/_ref/refdump_grid_sample), and the flow-warp and
3D-LUT fixtures (oracle/_ref/flow_f32.mnn, lut_f32.mnn, seeded weights, written by build()) through its Interpreter.  Nothing may
be declined to the CPU backup backend.  The one-op models equal the restatement bit for bit (a NaN by its position), on the first (eager) run and on the
runs the plugin captures and replays as a graph, and the first equals the recorded CPU golden.  Every compute command of the two
fixtures is within 1e-3 of MNN_FORWARD_CPU (max|d| / max|ref|), and a graph-replayed forward equals the eager one."""
import os
import tempfile

import numpy as np
import pytest

from oracle import grid_sample_oracle as S
from tests.golden import make_grid_sample_golden as G
from tests.test_gpu_grid_sample_f32 import bits, golden_digest
from tests.test_plugin import PLUGIN, _run
from tests.test_plugin_f32_models import _compare

pytestmark = pytest.mark.gpu


def _need_harness():
    if not S.have_refdump():
        pytest.skip("oracle/_ref/refdump_grid_sample is built by build() where the reference sources are")
    if not os.path.exists(PLUGIN):
        pytest.fail("mnn_b200/libmnn_b200_plugin.so is missing although the reference harness is present")


@pytest.mark.parametrize("name", list(G.CASES))
def test_golden_op_on_plugin(name):
    """each recorded GridSample on the plugin, run four times on one executor (eager, then captured and replayed) with four input
    sets: created there, every output bit-exact to the restatement, the first to the recorded CPU"""
    _need_harness()
    c = G.CASES[name]
    x, g = G.case_inputs(name)
    rng = np.random.default_rng(len(name))
    more = [(rng.standard_normal(x.shape).astype(np.float32), rng.uniform(-1.1, 1.1, g.shape).astype(np.float32))
            for _ in range(3)]
    ys, stats = G.case_reference(name, more=more, plugin=PLUGIN)
    assert stats is not None and stats["plugin_declined"] == 0 and stats["plugin_created"] >= 1, stats
    shape, sha = G.load()[name]
    assert ys[0].shape == shape and golden_digest(ys[0], G.case_oracle(name)) == sha
    for (xi, gi), y in zip([(x, g)] + more, ys):
        ref = S.grid_sample(xi, gi, c["mode"], c["padding"], c["align"])
        assert np.array_equal(bits(y), bits(ref))


def _fixture(model):
    _need_harness()
    path = S.FLOW if model == "flow" else S.LUT
    if not os.path.exists(path):
        pytest.skip(f"{path} is written by build() where the reference sources are")
    return path


@pytest.mark.parametrize("model", ["flow", "lut"])
def test_fixture_on_plugin_matches_cpu_backend(model, monkeypatch):
    """the flow-warp / 3D-LUT net at batch 2 through the Interpreter: every command on the plugin (the GridSample among them),
    every compute command within 1e-3 of the CPU's, and the fourth (graph-replayed) forward equal to the eager one"""
    path = _fixture(model)
    with tempfile.TemporaryDirectory() as d:
        cpu, _, _ = _run(os.path.join(d, "cpu"), 2, False, path)
        monkeypatch.setenv("REFDUMP_RUN_REPEATS", "4")
        gpu, stats, r = _run(os.path.join(d, "gpu"), 2, True, path)
        _compare(d, f"{model}_f32.mnn", cpu, gpu, stats, r)
        eager = np.fromfile(os.path.join(d, "gpu", "output.f32"), np.float32)
        replayed = np.fromfile(os.path.join(d, "gpu", "output_plain.f32"), np.float32)
        assert np.array_equal(replayed.view(np.uint32), eager.view(np.uint32)), "the graph-replayed forward differs from the eager one"
    assert sum(t == "GridSample" for _, _, t, _, _ in gpu) == 1
