"""CPU check of the generated fp32 model fixtures (oracle/_ref/mbv2_f32.mnn, r50_f32.mnn; skipped when absent): every conv has
seeded, non-zero float weights, relu6 is kept, and the reference CPU backend's forward is finite and not saturated."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from mnn_b200 import mnn_file
from oracle import oracle as O

pytestmark = pytest.mark.reference


def _model(name):
    path = os.path.join(O.REF_DIR, name)
    if not O.have_reference() or not os.path.exists(path):
        pytest.skip(f"{name} not generated (oracle/float_models.py, run by build() where the reference exists)")
    return path


def _conv_float_weights(path):
    """(op type, relu6, fp32 weights) of every conv: Convolution2D field 1 is the float weight vector"""
    buf = open(path, "rb").read()
    root = mnn_file.Table(buf, int.from_bytes(buf[:4], "little"))
    out = []
    for o in root.table_vector(3):
        if o.scalar(1, "B", 0) != mnn_file.PARAM_CONV2D:
            continue
        main = o.table(2)
        w = main.vector(1, "<f4")
        out.append((mnn_file.OP_NAMES.get(o.scalar(5, "i", 0)), bool(main.table(0).scalar(13, "b", 0)),
                    np.zeros(0, np.float32) if w is None else w))
    return out


@pytest.mark.parametrize("name,convs,relu6", [("mbv2_f32.mnn", 53, True), ("r50_f32.mnn", 54, False)])
def test_float_fixture_weights_and_cpu_forward(name, convs, relu6):
    path = _model(name)
    cv = _conv_float_weights(path)
    assert len(cv) == convs
    for typ, _, w in cv:
        assert w.size > 0 and np.count_nonzero(w) >= 0.999 * w.size, f"{typ}: zero weights"   # seeded, not Revert's zeros
        assert np.abs(w).max() <= 1.2 + 1e-6
    assert any(r6 for _, r6, _ in cv) == relu6, "relu6 flags changed"
    env = dict(os.environ, LD_LIBRARY_PATH=O.REF_DIR + ":" + os.environ.get("LD_LIBRARY_PATH", ""))
    env.pop("REFDUMP_PLUGIN", None)
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run([O.REFDUMP, "run", path, "1", "3", d, "4"], env=env, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-1500:]
        peaks = []
        for line in open(os.path.join(d, "index.txt")):
            f = line.split("|")[0]
            t = np.fromfile(os.path.join(d, f), np.float32)
            assert np.isfinite(t).all(), line
            peaks.append(float(np.abs(t).max()))
        out = np.fromfile(os.path.join(d, "output.f32"), np.float32)
    # O(1) activations: no tensor blows up, and the ReLU6 ceiling does not hold whole tensors
    assert 0.5 < max(peaks) < 100, max(peaks)
    assert np.isfinite(out).all() and out.std() > 0 and abs(out.sum() - 1.0) < 1e-3
