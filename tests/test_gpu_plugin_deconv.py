"""fp32 Deconvolution through the MNN plugin (-m gpu): the unmodified reference core runs Deconvolution and DeconvolutionDepthwise
ops through its Express executor on MNN_FORWARD_CUDA = mnn_b200/libmnn_b200_plugin.so (oracle/_ref/refdump_deconv).  Nothing
may be declined to the CPU backup backend, and every output must be within 1e-3 of MNN_FORWARD_CPU (max|d| / max|ref|)."""
import os

import numpy as np
import pytest

from oracle import deconv_oracle as D

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PLUGIN = os.path.join(ROOT, "mnn_b200", "libmnn_b200_plugin.so")


def _need_harness():
    if not D.have_refdump():
        pytest.skip("oracle/_ref/refdump_deconv is built by build() where the reference sources are")
    if not os.path.exists(PLUGIN):
        pytest.fail("mnn_b200/libmnn_b200_plugin.so is missing although the reference harness is present")


def _rel(a, b):
    return float(np.abs(np.asarray(a, np.float64) - b).max() / max(np.abs(b).max(), 1e-12))


def test_deconv_between_convs_on_plugin():
    """conv -> deconv -> depthwise deconv -> conv, run twice on one executor with two inputs: every op on the plugin, both runs'
    deconvolution and graph outputs within 1e-3 of the CPU backend's"""
    _need_harness()
    cpu, _ = D.ref_chain(2, 7)
    gpu, stats = D.ref_chain(2, 7, plugin=PLUGIN)
    assert stats is not None and stats["plugin_declined"] == 0 and stats["plugin_created"] >= 4, stats
    assert sorted(cpu) == sorted(gpu) == ["deconv_0", "deconv_1", "output_0", "output_1"]
    assert not np.array_equal(cpu["output_0"], cpu["output_1"])
    for k in cpu:
        assert _rel(gpu[k], cpu[k]) <= 1e-3, k


# (stride, pads [t, l, b, r], dilation, out_pads, same, output shape, depthwise, relu, relu6)
FORMS = {
    "k4_s2_p1_relu": (2, (1, 1, 1, 1), 1, (0, 0), 0, None, 0, 1, 0),
    "s3_d2_outpads_relu6": (3, (0, 2, 1, 0), 2, (1, 2), 0, None, 0, 0, 1),
    "same_output_shape": (2, (0, 0, 0, 0), 1, (0, 0), 1, (11, 9), 0, 0, 0),
    "depthwise_asym": (2, (1, 0, 1, 0), 1, (1, 0), 0, None, 1, 0, 0),
}


@pytest.mark.parametrize("name", list(FORMS))
def test_deconv_forms_on_plugin(name):
    _need_harness()
    s, pads, d, op, same, out, dw, relu, relu6 = FORMS[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    ic, oc, k = 12, 12 if dw else 10, 4
    x = rng.standard_normal((2, ic, 6, 5)).astype(np.float32)
    w = (rng.standard_normal((ic, k, k) if dw else (ic, oc, k, k)) * 0.3).astype(np.float32)
    b = rng.standard_normal(oc).astype(np.float32)
    args = (x, w, b, s, pads, d, op, bool(same), out, bool(dw), bool(relu), bool(relu6))
    y_cpu = D.ref_deconv(*args)
    y_gpu, stats = D.ref_deconv(*args, plugin=PLUGIN)
    assert stats is not None and stats["plugin_declined"] == 0 and stats["plugin_created"] >= 1, stats
    assert y_gpu.shape == y_cpu.shape
    assert _rel(y_gpu, y_cpu) <= 1e-3
