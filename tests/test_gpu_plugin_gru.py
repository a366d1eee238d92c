"""GRU through the MNN plugin (-m gpu).  The unmodified reference core runs each recorded op through its Express executor on
MNN_FORWARD_CUDA = mnn_b200/libmnn_b200_plugin.so (oracle/_ref/refdump_gru), four input sets on one executor (eager, then
captured and replayed as a graph with new inputs and new weights): every case is created on the plugin with nothing declined
and each output is within 1e-3 of the reference CPU, except the backward Y_h the CPU takes from its scratch (checked against
the restatement).  The denoiser and tagger fixtures (oracle/_ref/{denoise,tagger}_f32.mnn) run through the Interpreter with
nothing declined, every compute command within 1e-3 of the CPU backend, and a graph-replayed forward equal to the eager one;
the denoiser runs four chained chunks with its states fed back."""
import os
import tempfile

import numpy as np
import pytest

from oracle import gru_oracle as G
from tests.golden import make_gru_golden as M
from tests.test_plugin import PLUGIN

pytestmark = pytest.mark.gpu


def _need_harness():
    if not G.have_refdump():
        pytest.skip("oracle/_ref/refdump_gru is built by build() where the reference sources are")
    if not os.path.exists(PLUGIN):
        pytest.fail("mnn_b200/libmnn_b200_plugin.so is missing although the reference harness is present")


def _rel(a, b):
    return float(np.abs(np.asarray(a, np.float64) - b).max() / max(1e-6, float(np.abs(b).max())))


def _fresh_sets(name, n=3):
    """further input sets of a case's shapes: fresh values for every input, weights included"""
    rng = np.random.default_rng(len(name) + 17)
    _, _, _, x, params, h0 = M.case_inputs(name)
    fresh = lambda a: None if a is None else (rng.standard_normal(a.shape) * float(np.abs(a).max()) / 2).astype(np.float32)
    return [(fresh(x), [fresh(p) for p in params], fresh(h0)) for _ in range(n)]


def _check(name, lbr, keep, n_out, x, params, h0, got, cpu, what):
    """the plugin's outputs against the CPU's, the CPU's scratch-backed backward Y_h against the restatement instead"""
    names = ("y", "y_h")[:n_out] if keep else ("y_h",)
    for k, g, c in zip(names, got, cpu):
        if k == "y_h" and keep and g.shape[0] == 2:
            assert _rel(g[0], c[0]) <= 1e-3, (name, what, "y_h forward")
            _, yh64 = G.run64(lbr, x, params, h0)
            assert _rel(g[1], yh64[1]) <= 1e-3, (name, what, "y_h backward")
        else:
            assert _rel(g, c) <= 1e-3, (name, what, k)


@pytest.mark.parametrize("name", sorted(M.CASES))
def test_golden_op_on_plugin(name):
    _need_harness()
    lbr, keep, n_out, x, params, h0 = M.case_inputs(name)
    more = _fresh_sets(name)
    outs, stats = G.ref_op(lbr, x, params, h0, keep, n_out, more=more, plugin=PLUGIN)
    assert stats is not None and stats["plugin_declined"] == 0 and stats["plugin_created"] >= 1, stats
    gold = np.load(M.PATH)
    names = ("y", "y_h")[:n_out] if keep else ("y_h",)
    _check(name, lbr, keep, n_out, x, params, h0, outs[0],
           [gold[f"{name}/{k}"] if f"{name}/{k}" in gold else np.zeros_like(y) for k, y in zip(names, outs[0])], "golden")
    cpu = G.ref_op(lbr, x, params, h0, keep, n_out, more=more)
    for s in range(1, len(outs)):
        xs, ps, hs = more[s - 1]
        _check(name, lbr, keep, n_out, xs, ps, hs, outs[s], cpu[s], f"input set {s}")


def _compare(d, cpu, gpu, stats, r):
    """every plugin compute command against the CPU command of the same name, the session output too, and the graph-replayed
    forward against the eager one"""
    assert stats is not None and stats["plugin_declined"] == 0, f"commands fell back to the CPU backend: {stats}\n{r.stdout[-2500:]}"
    load = lambda side, f: np.fromfile(os.path.join(d, side, f), np.float32)
    by_name = {}
    for f, n, t in cpu:
        by_name.setdefault(n, []).append(f)
    compared, worst = 0, {}
    for f, n, t in gpu:
        if t.startswith("Raster"):
            continue
        assert n in by_name, f"plugin command {n} ({t}) has no CPU command of that name"
        out = int(f.split("_")[1].split(".")[0])
        ref = load("cpu", sorted(by_name[n])[out] if len(by_name[n]) > out else by_name[n][0])
        err = _rel(load("gpu", f), np.asarray(ref, np.float64))
        assert err <= 1e-3, f"{n} ({t}) rel err {err}"
        compared += 1
        worst[t] = max(worst.get(t, 0.0), err)
    oc, og = load("cpu", "output.f32"), load("gpu", "output.f32")
    assert oc.shape == og.shape and _rel(og, oc) <= 1e-3, f"session output differs: {_rel(og, oc)}"
    replayed = load("gpu", "output_plain.f32")
    assert np.array_equal(replayed.view(np.uint32), og.view(np.uint32)), "the graph-replayed forward differs from the eager one"
    return compared, worst


@pytest.mark.parametrize("model", ["denoise", "tagger"])
def test_gru_fixture_on_plugin_matches_cpu_backend(model):
    _need_harness()
    path = G.DENOISE if model == "denoise" else G.TAGGER
    if not os.path.exists(path):
        pytest.skip(f"{path} is written by build() where the reference sources are")
    batch = 3 if model == "denoise" else 4
    with tempfile.TemporaryDirectory() as d:
        cpu, _, _ = G.run_model(path, batch, 3, os.path.join(d, "cpu"))
        gpu, stats, r = G.run_model(path, batch, 3, os.path.join(d, "gpu"), plugin=PLUGIN, repeats=4)
        compared, worst = _compare(d, cpu, gpu, stats, r)
    types = {t for _, _, t in gpu}
    assert "RNNSequenceGRU" in types, types
    print(f"{model}: {compared} plugin commands compared, created {stats['plugin_created']}, worst rel err per type "
          + ", ".join(f"{t} {e:.2e}" for t, e in sorted(worst.items())))


def test_denoiser_four_chained_chunks_on_plugin():
    """four chunks of 16 frames, each chunk's final h1_n, h2_n, h3_n fed back as the next one's h1_0, h2_0, h3_0: every chunk's
    gains and states within 1e-3 of the CPU backend, nothing declined"""
    _need_harness()
    if not os.path.exists(G.DENOISE):
        pytest.skip(f"{G.DENOISE} is written by build() where the reference sources are")
    with tempfile.TemporaryDirectory() as d:
        cpu, _ = G.run_chunks(3, 9, 4, os.path.join(d, "cpu"))
        gpu, stats = G.run_chunks(3, 9, 4, os.path.join(d, "gpu"), plugin=PLUGIN)
    assert stats is not None and stats["plugin_declined"] == 0, stats
    for key, ref in cpu.items():
        assert _rel(gpu[key], ref) <= 1e-3, key
    assert not np.array_equal(cpu[(0, "h3_n")], cpu[(3, "h3_n")])
