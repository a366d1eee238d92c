"""fp32 Interp and Resize through the MNN plugin (-m gpu).  The unmodified reference core runs the recorded Interp ops through its
Express executor on MNN_FORWARD_CUDA = mnn_b200/libmnn_b200_plugin.so (oracle/_ref/refdump_interp), and the DeepLab-v3-style and
FPN fixtures (oracle/_ref/deeplab_f32.mnn, fpn_f32.mnn, seeded weights, written by build()) through its Interpreter.  Nothing may
be declined to the CPU backup backend.  The one-op models equal the CPU bit for bit, on the first (eager) run and on the runs the
plugin captures and replays as a graph; every compute command's output of the two models is within 1e-3 of MNN_FORWARD_CPU
(max|d| / max|ref|).  Layout Rasters are not compared: the two backends insert different ones."""
import os
import tempfile

import numpy as np
import pytest

from oracle import interp_oracle as I
from tests.golden import make_interp_golden as G
from tests.test_plugin import PLUGIN, _run
from tests.test_plugin_f32_models import _compare, _compute

pytestmark = pytest.mark.gpu


def _need_harness():
    if not I.have_refdump():
        pytest.skip("oracle/_ref/refdump_interp is built by build() where the reference sources are")
    if not os.path.exists(PLUGIN):
        pytest.fail("mnn_b200/libmnn_b200_plugin.so is missing although the reference harness is present")


def _rel(a, b):
    return float(np.abs(np.asarray(a, np.float64) - b).max() / max(np.abs(b).max(), 1e-12))


@pytest.mark.parametrize("name", list(G.CASES))
def test_golden_op_on_plugin(name):
    """each recorded Interp on the plugin, run four times on one executor (eager, then captured and replayed) with four inputs:
    created there, every output bit-exact to the restatement, the first to the recorded CPU"""
    _need_harness()
    x = G.case_inputs(name)
    rng = np.random.default_rng(len(name))
    more = [rng.standard_normal(x.shape).astype(np.float32) for _ in range(3)]
    ys, stats = G.case_reference(name, x2=more, plugin=PLUGIN)
    assert stats is not None and stats["plugin_declined"] == 0 and stats["plugin_created"] >= 1, stats
    shape, sha = G.load()[name]
    assert ys[0].shape == shape and G.digest(ys[0]) == sha
    c = G.CASES[name]
    for xi, y in zip([x] + more, ys):
        ref = I.interp(xi, c["resize_type"], *G.case_transform(name), G.case_out_hw(name))
        assert np.array_equal(y.view(np.uint32), ref.view(np.uint32))


def _model(path):
    _need_harness()
    if not os.path.exists(path):
        pytest.skip(f"{path} is written by build() where the reference sources are")
    return path


def test_fpn_neck_on_plugin_matches_cpu_backend():
    """the nearest x2 FPN neck with one Resize at batch 2 through the Interpreter: every command on the plugin, every fp32
    tensor within 1e-3 of the CPU's"""
    model = _model(I.FPN)
    with tempfile.TemporaryDirectory() as d:
        cpu, _, _ = _run(os.path.join(d, "cpu"), 2, False, model)
        gpu, stats, r = _run(os.path.join(d, "gpu"), 2, True, model)
        _compare(d, "fpn_f32.mnn", cpu, gpu, stats, r)
    assert sum(t == "Interp" for _, _, t, _, _ in cpu) >= 3


def test_deeplab_on_plugin_matches_cpu_backend():
    """the DeepLab-v3-style net at batch 2: every command on the plugin, every compute command's output before the ArgMax within
    1e-3 of the CPU's, and the class map equal wherever the CPU's best class is clear of the runner-up (near-ties may go either way)"""
    model = _model(I.DEEPLAB)
    with tempfile.TemporaryDirectory() as d:
        cpu, _, _ = _run(os.path.join(d, "cpu"), 2, False, model)
        gpu, stats, r = _run(os.path.join(d, "gpu"), 2, True, model)
        assert stats is not None and stats["plugin_declined"] == 0, f"commands fell back to the CPU backend: {stats}\n{r.stdout[-2500:]}"
        cc, gc = _compute(cpu), _compute(gpu)
        assert [c[1:] for c in cc] == [g[1:] for g in gc], "command lists differ"
        for (fc, name, typ), (fg, _, _) in zip(cc, gc):
            if typ.startswith("ArgMax"):
                continue
            a = np.fromfile(os.path.join(d, "cpu", fc), np.float32)
            b = np.fromfile(os.path.join(d, "gpu", fg), np.float32)
            assert a.shape == b.shape and _rel(b, a) <= 1e-3, f"{name} ({typ})"
        assert sum(t == "Interp" for _, _, t in cc) >= 3
        # the logits: the last Raster (the NCHW conversion in front of the ArgMax)
        last = [l.split("|") for l in open(os.path.join(d, "cpu", "index.txt")).read().splitlines() if l.split("|")[2] == "Raster"][-1]
        dims = [int(v) for v in last[3].split(",")]
        xc = np.fromfile(os.path.join(d, "cpu", last[0]), np.float32).reshape(dims)
        oc = np.fromfile(os.path.join(d, "cpu", "output.f32"), np.int32).reshape(dims[0], *dims[2:])
        og = np.fromfile(os.path.join(d, "gpu", "output.f32"), np.int32).reshape(oc.shape)
        assert np.array_equal(oc, np.argmax(xc, axis=1)), "the CPU's ArgMax is not the first maximum of the dumped logits"
        top = np.sort(xc, axis=1)
        clear = (top[:, -1] - top[:, -2]) > 2e-3 * np.abs(xc).max()
        assert clear.mean() > 0.9 and np.array_equal(oc[clear], og[clear]), "class map differs where the maximum is clear"
