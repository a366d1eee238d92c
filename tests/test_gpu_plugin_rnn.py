"""LSTM and RNN through the MNN plugin (-m gpu).  The unmodified reference core runs each recorded op through its Express
executor on MNN_FORWARD_CUDA = mnn_b200/libmnn_b200_plugin.so (oracle/_ref/refdump_rnn), four input sets on one executor (eager,
then captured and replayed as a graph with new inputs and new weights): every case is created on the plugin with nothing
declined and each output is within 1e-3 of the reference CPU.  The CRNN- and KWS-style fixtures (oracle/_ref/{crnn,kws}_f32.mnn)
run through the Interpreter with nothing declined, every compute command within 1e-3 of the CPU backend, and a graph-replayed
forward equal to the eager one; the KWS chunk runs four chained chunks with its states fed back."""
import os
import tempfile

import numpy as np
import pytest

from oracle import rnn_oracle as R
from tests.golden import make_rnn_golden as M
from tests.test_plugin import PLUGIN

pytestmark = pytest.mark.gpu


def _need_harness():
    if not R.have_refdump():
        pytest.skip("oracle/_ref/refdump_rnn is built by build() where the reference sources are")
    if not os.path.exists(PLUGIN):
        pytest.fail("mnn_b200/libmnn_b200_plugin.so is missing although the reference harness is present")


def _rel(a, b):
    return float(np.abs(np.asarray(a, np.float64) - b).max() / max(1e-6, float(np.abs(b).max())))


def _fresh_sets(name, n=3):
    """further input sets of a case's shapes: fresh values for every input, weights included"""
    rng = np.random.default_rng(len(name) + 17)
    first = [a for a in M.case_inputs(name)[1:] if a is not None]
    return [tuple((rng.standard_normal(a.shape) * float(np.abs(a).max()) / 2).astype(np.float32) for a in first) for _ in range(n)]


@pytest.mark.parametrize("name", sorted(M.CASES))
def test_golden_op_on_plugin(name):
    _need_harness()
    cell, x, w, r, b, h0, c0 = M.case_inputs(name)
    more = _fresh_sets(name)
    outs, stats = R.ref_op(cell, x, w, r, b, h0, c0, more=more, plugin=PLUGIN)
    assert stats is not None and stats["plugin_declined"] == 0 and stats["plugin_created"] >= 1, stats
    gold = np.load(M.PATH)
    for k, y in zip(("y", "y_h", "y_c"), outs[0]):
        assert _rel(y, gold[f"{name}/{k}"]) <= 1e-3, (name, k)
    cpu = R.ref_op(cell, x, w, r, b, h0, c0, more=more)
    for s in range(1, len(outs)):
        for k, (g, c) in enumerate(zip(outs[s], cpu[s])):
            assert _rel(g, c) <= 1e-3, (name, "input set", s, k)


def _compare(d, cpu, gpu, stats, r):
    """every plugin compute command against the CPU.  Commands the CPU has by name are compared directly; the CPU runs an
    LSTM / RNN as While loops named <op>_raster_<k>, so the plugin's Y is compared with the last of those outputs of Y's shape,
    and its Y_h with that Y at T - 1 (direction 0) and 0 (direction 1)"""
    assert stats is not None and stats["plugin_declined"] == 0, f"commands fell back to the CPU backend: {stats}\n{r.stdout[-2500:]}"
    load = lambda side, f: np.fromfile(os.path.join(d, side, f), np.float32)
    shapes = {}
    by_name = {}
    for f, n, t in cpu:
        by_name[n] = f
    with open(os.path.join(d, "cpu", "index.txt")) as fi:
        for line in fi:
            f, n, _, dims = line.rstrip("\n").split("|")[:4]
            shapes.setdefault(n, []).append((f, tuple(int(v) for v in dims.split(",") if v)))
    gshape = {}
    with open(os.path.join(d, "gpu", "index.txt")) as fi:
        for line in fi:
            f, n, _, dims = line.rstrip("\n").split("|")[:4]
            gshape[f] = tuple(int(v) for v in dims.split(",") if v)
    compared, worst = 0, {}
    for f, n, t in gpu:
        if t.startswith("Raster"):
            continue
        g = load("gpu", f)
        if t in ("LSTM", "RNN"):
            out = int(f.split("_")[1].split(".")[0])
            if out == 2:
                continue          # Y_c: checked through the session outputs (KWS's c_n)
            ycands = [(cf, s) for k, lst in shapes.items() if k.startswith(n + "_raster_") for cf, s in lst if len(s) == 4]
            yf, ys = max(ycands)
            y = load("cpu", yf).reshape(ys)
            ref = y if out == 0 else np.stack([y[-1, 0]] + ([y[0, 1]] if ys[1] > 1 else [])).reshape(-1)
        else:
            assert n in by_name, f"plugin command {n} ({t}) has no CPU command of that name"
            ref = load("cpu", by_name[n])
        err = _rel(g.reshape(-1), np.asarray(ref, np.float64).reshape(-1))
        assert err <= 1e-3, f"{n} ({t}) rel err {err}"
        compared += 1
        worst[t] = max(worst.get(t, 0.0), err)
    oc, og = load("cpu", "output.f32"), load("gpu", "output.f32")
    assert oc.shape == og.shape and _rel(og, oc) <= 1e-3, f"session output differs: {_rel(og, oc)}"
    replayed = load("gpu", "output_plain.f32")
    assert np.array_equal(replayed.view(np.uint32), og.view(np.uint32)), "the graph-replayed forward differs from the eager one"
    return compared, worst


@pytest.mark.parametrize("model", ["crnn", "kws"])
def test_rnn_fixture_on_plugin_matches_cpu_backend(model):
    _need_harness()
    path = R.CRNN if model == "crnn" else R.KWS
    if not os.path.exists(path):
        pytest.skip(f"{path} is written by build() where the reference sources are")
    batch = 4 if model == "crnn" else 2
    with tempfile.TemporaryDirectory() as d:
        cpu, _, _ = R.run_model(path, batch, 3, os.path.join(d, "cpu"))
        gpu, stats, r = R.run_model(path, batch, 3, os.path.join(d, "gpu"), plugin=PLUGIN, repeats=4)
        compared, worst = _compare(d, cpu, gpu, stats, r)
    types = {t for _, _, t in gpu}
    assert ({"LSTM"} if model == "crnn" else {"LSTM", "RNN"}) <= types, types
    print(f"{model}: {compared} plugin commands compared, created {stats['plugin_created']}, worst rel err per type "
          + ", ".join(f"{t} {e:.2e}" for t, e in sorted(worst.items())))


def test_kws_four_chained_chunks_on_plugin():
    """four chunks of 16 frames, each chunk's final h_n, c_n, hr_n fed back as the next one's h0, c0, h0r: every chunk's logits
    and states within 1e-3 of the CPU backend, nothing declined"""
    _need_harness()
    if not os.path.exists(R.KWS):
        pytest.skip(f"{R.KWS} is written by build() where the reference sources are")
    with tempfile.TemporaryDirectory() as d:
        cpu, _ = R.run_chunks(3, 9, 4, os.path.join(d, "cpu"))
        gpu, stats = R.run_chunks(3, 9, 4, os.path.join(d, "gpu"), plugin=PLUGIN)
    assert stats is not None and stats["plugin_declined"] == 0, stats
    for key, ref in cpu.items():
        assert _rel(gpu[key], ref) <= 1e-3, key
    assert not np.array_equal(cpu[(0, "h_n")], cpu[(3, "h_n")])
