"""GPU: the whole MobileNet-v2 int8 .mnn on the CUDA path (no CPU fallback) against the outputs of the REAL reference CPU
backend, recorded under tests/golden (committed checkpoints at batch 1, every op at batch 2)."""
import hashlib
import os

import numpy as np
import pytest

from oracle import oracle as O

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
MODEL = os.path.join(GOLD, "mbv2_int8.mnn")
# Softmax runs an fp32 exp internally (the reference uses its own polynomial): +-1 LSB there, bit-exact elsewhere
FP_INTERNAL = ("MobilenetV2/Predictions/Softmax",)


def test_wholenet_checkpoints_vs_reference_golden():
    from mnn_b200.session import WholeNetSession
    g = np.load(os.path.join(GOLD, "mbv2_int8_checkpoints.npz"))
    sess = WholeNetSession(MODEL, 1)
    sess.set_input(g["input"])
    sess.run()
    names = [str(n) for n in g["names"]]
    assert len(names) >= 10
    for i, name in enumerate(names):
        got = sess.read_int8(name)
        ref = g[f"t{i}"].reshape(got.shape)
        d = np.abs(got.astype(int) - ref.astype(int)).max()
        assert d <= (1 if name in FP_INTERNAL else 0), f"{name}: max |diff| = {d}"
    out = sess.get_output()
    ref = g["output"].reshape(out.shape)
    assert np.abs(out - ref).max() <= 1e-3 * max(np.abs(ref).max(), 1e-6) + 0.05   # one softmax LSB = scale ~0.03


def check_vs_reference_b2(sess, tag=""):
    """every int8 checkpoint of a batch-2 forward on refdump's seed-11 input against the reference CPU backend's output, recorded
    by tests/golden/make_config_golden.py (sha256 of each tensor; the softmax output in full, +-1 LSB)"""
    g = np.load(os.path.join(GOLD, "config_golden.npz"))
    full = {n: g[f"b2_full{i}"] for i, n in enumerate(FP_INTERNAL)}
    checked = 0
    for name, h in zip((str(n) for n in g["b2_names"]), (str(h) for h in g["b2_sha256"])):
        if name not in sess.checkpoints:
            continue
        got = sess.read_int8(name)
        if name in full:
            dmax = np.abs(got.astype(int) - full[name].reshape(got.shape).astype(int)).max()
            assert dmax <= 1, f"{tag}{name}: max |diff| = {dmax}"
        else:
            assert hashlib.sha256(np.ascontiguousarray(got).tobytes()).hexdigest() == h, f"{tag}{name} differs from the reference"
        checked += 1
    assert checked >= 60, checked       # 36 conv + 17 depthwise + 10 add + pool + softmax


@pytest.mark.parametrize("batch", [2])
def test_wholenet_every_op_vs_live_reference(batch):
    from mnn_b200.session import WholeNetSession
    x = O.refdump_input(11, (batch, 3, 224, 224))
    sess = WholeNetSession(MODEL, batch)
    sess.capture()                      # CUDA-graph replay is the product path
    sess.set_input(x)
    sess.run()
    check_vs_reference_b2(sess)

