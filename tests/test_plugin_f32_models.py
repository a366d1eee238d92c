"""The other fp32 benchmark graphs end to end (-m gpu): MobileNet-v3, NASNet, Inception-v3, SqueezeNet v1.0 / v1.1 and
MobileNet-v1 with seeded float weights (oracle/_ref/*_f32.mnn, written by build()) on MNN_FORWARD_CUDA =
mnn_b200/libmnn_b200_plugin.so against MNN_FORWARD_CPU's default session.

The plugin reports Compiler_Geometry, so its session runs with GEOMETRY_COMPUTE_MASK 0: a one-sided broadcast BinaryOp reaches
it as a layout Raster plus an equal-size BinaryOp, where the CPU runs one While loop command of the same name.  Raster commands
are ignored and each CPU While is matched with the plugin's BinaryOp of that name (names are compared without the `_raster_<k>`
suffix the geometry gives a decomposed op's commands); the compute command lists must then be equal,
nothing may be declined, and every compute command's fp32 output and the session output must be within 1e-3 of the CPU
(max|d| / max|ref|).  SqueezeNet v1.0 ends in an ArgMax over the batch axis of its logits: its int32 output must be the first
maximum of the plugin's own logits, and equal to the CPU's wherever the maximum is clear of the 1e-3 gate."""
import os
import re
import tempfile

import numpy as np
import pytest

from oracle import oracle as O
from tests.test_plugin import PLUGIN, _run

pytestmark = pytest.mark.gpu

INT32_OUTPUT = {"squeezenet_v10_f32.mnn"}


def _model(name):
    if not O.have_reference():
        pytest.skip("the reference core (oracle/_ref) is not in this snapshot")
    if not os.path.exists(PLUGIN):
        pytest.fail("mnn_b200/libmnn_b200_plugin.so is missing although the reference core is present")
    path = os.path.join(O.REF_DIR, name)
    if not os.path.exists(path):
        pytest.skip(f"{name} not generated (build() writes it where the reference exists)")
    return path


def _rel(a, b):
    return float(np.abs(a.astype(np.float64) - b).max() / max(np.abs(a).max(), 1e-12))


def _norm(name):
    # the geometry names a decomposed op's commands after its helper Rasters, which differ between the two masks
    return re.sub(r"_raster_\d+$", "", name)


def _compute(recs):
    return [(f, _norm(n), "BinaryOp" if t == "While" else t) for f, n, t, _, _ in recs if not t.startswith("Raster")]


def _argmax_input(outdir):
    """file and dims of SqueezeNet v1.0's logits: the flatten Raster that feeds both its Softmax and its ArgMax"""
    last = [l.split("|") for l in open(os.path.join(outdir, "index.txt")).read().splitlines() if l.split("|")[2] == "Raster"][-1]
    return last[0], [int(v) for v in last[3].split(",")]


def _compare(d, name, cpu, gpu, stats, r, output="output.f32"):
    assert stats is not None and stats["plugin_declined"] == 0, f"commands fell back to the CPU backend: {stats}\n{r.stdout[-2500:]}"
    cc, gc = _compute(cpu), _compute(gpu)
    assert [c[1:] for c in cc] == [g[1:] for g in gc], "command lists differ"
    # Raster outputs are layout helpers whose names and shapes depend on the mask; every compute output after them is compared
    worst, worst_at = 0.0, ""
    for (fc, cname, typ), (fg, _, _) in zip(cc, gc):
        a = np.fromfile(os.path.join(d, "cpu", fc), np.float32)
        b = np.fromfile(os.path.join(d, "gpu", fg), np.float32)
        assert a.shape == b.shape, cname
        err = _rel(a, b)
        assert err <= 1e-3, f"{cname} ({typ}) rel err {err}"
        if err > worst:
            worst, worst_at = err, f"{cname} ({typ})"
    if name in INT32_OUTPUT:
        # ArgMax over axis 0 (the batch) of the logits: each side's indices are the first maximum of its own logits, and they
        # agree wherever the CPU's two rows are further apart than twice the 1e-3 gate (with these weights the rows of the two
        # images differ by ~2e-6 of max|logit|, so that is rarely the case: the kernel's tie rule is tested directly in
        # tests/test_gpu_float_elementwise.py)
        oc = np.fromfile(os.path.join(d, "cpu", output), np.int32)
        og = np.fromfile(os.path.join(d, "gpu", output), np.int32)
        (fc, dc), (fg, dg) = _argmax_input(os.path.join(d, "cpu")), _argmax_input(os.path.join(d, "gpu"))
        assert dc == dg, (dc, dg)
        xc = np.fromfile(os.path.join(d, "cpu", fc), np.float32).reshape(dc[0], -1)
        xg = np.fromfile(os.path.join(d, "gpu", fg), np.float32).reshape(dg[0], -1)
        assert _rel(xc, xg) <= 1e-3, "logits differ"
        assert og.size == xg.shape[1] and oc.size == xc.shape[1]
        assert np.array_equal(oc, np.argmax(xc, axis=0)), "the CPU's ArgMax is not the first maximum of the dumped logits"
        assert np.array_equal(og, np.argmax(xg, axis=0)), "plugin ArgMax differs from the first maximum of its input"
        top = np.sort(xc, axis=0)
        clear = (top[-1] - top[-2]) > 2e-3 * np.abs(xc).max()
        assert np.array_equal(oc[clear], og[clear]), "ArgMax indices differ where the maximum is clear"
        print(f"{name}: ArgMax {og.size} indices, {int(clear.sum())} with a clear maximum, {int((oc != og).sum())} near-ties differ")
    else:
        oc = np.fromfile(os.path.join(d, "cpu", output), np.float32)
        og = np.fromfile(os.path.join(d, "gpu", output), np.float32)
        assert oc.shape == og.shape and _rel(oc, og) <= 1e-3, "session output differs"
    whiles = sum(t == "While" for _, _, t, _, _ in cpu)
    print(f"{name}: {len(cpu)} / {len(gpu)} commands (cpu / plugin), {whiles} CPU While, plugin_created {stats['plugin_created']}, "
          f"worst per-tensor rel err {worst:.2e} at {worst_at}")
    return whiles


CASES = [("mbv3_f32.mnn", 1), ("mbv3_f32.mnn", 4), ("nasnet_f32.mnn", 2), ("inception_v3_f32.mnn", 2),
         ("squeezenet_v10_f32.mnn", 2), ("squeezenet_v11_f32.mnn", 2), ("mbv1_f32.mnn", 2)]


@pytest.mark.parametrize("model_name,batch", CASES)
def test_float_benchmark_model_on_plugin_matches_cpu_backend(model_name, batch):
    model = _model(model_name)
    with tempfile.TemporaryDirectory() as d:
        cpu, _, _ = _run(os.path.join(d, "cpu"), batch, False, model)
        gpu, stats, r = _run(os.path.join(d, "gpu"), batch, True, model)
        whiles = _compare(d, model_name, cpu, gpu, stats, r)
    if model_name.startswith("mbv3"):
        assert whiles >= 9, "the squeeze-excite multiplies are While loops on the CPU"


def test_float_benchmark_model_graph_replay_matches_cpu_backend():
    """MobileNet-v3 at batch 2, 4 plain forwards first (eager, capture, replay, replay): the replayed output equals the CPU's"""
    model = _model("mbv3_f32.mnn")
    keep = os.environ.get("REFDUMP_RUN_REPEATS")
    os.environ["REFDUMP_RUN_REPEATS"] = "4"
    try:
        with tempfile.TemporaryDirectory() as d:
            cpu, _, _ = _run(os.path.join(d, "cpu"), 2, False, model)
            gpu, stats, r = _run(os.path.join(d, "gpu"), 2, True, model)
            _compare(d, "mbv3_f32.mnn", cpu, gpu, stats, r)
            _compare(d, "mbv3_f32.mnn", cpu, gpu, stats, r, output="output_plain.f32")
    finally:
        if keep is None:
            os.environ.pop("REFDUMP_RUN_REPEATS", None)
        else:
            os.environ["REFDUMP_RUN_REPEATS"] = keep
