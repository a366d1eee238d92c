"""The GRU restatement (oracle/gru_oracle.py) and the launch plans of the recurrences, on the CPU.

The restatement equals torch.nn.GRU in float64 for linear_before_reset = 1 (torch's form, weights permuted); a missing h0 is a
zero h0; the per-step bound covers an fp32 step.  The C++ plan searches of gru.cu and rnn.cu (recur_common.cuh), compiled
into a host program, equal the Python restatements of both over the census shapes and more, so the LSTM / RNN plans did not
move when the search became shared.  The GRU kernels compile without spills.  With the reference built: the restatement equals
the goldens and the live reference CPU on fresh seeds, and the CPU's backward Y_h with both outputs and no h0 is zeros."""
import os
import subprocess

import numpy as np
import pytest

from oracle import gru_oracle as G
from oracle import rnn_oracle as R

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


@pytest.mark.parametrize("D", [1, 2])
def test_oracle_equals_torch_in_float64(D):
    import torch
    rng = np.random.default_rng(40 + D)
    T, B, I, H = 5, 3, 7, 11
    x = rng.standard_normal((T, B, I)).astype(np.float32)
    params = G.random_params(rng, D, I, H)
    h0 = rng.standard_normal((D, B, H)).astype(np.float32)
    Y, Yh = G.run64(1, x, params, h0)
    gru = torch.nn.GRU(I, H, bidirectional=D == 2).double()
    with torch.no_grad():
        for d in range(D):
            sfx = "_reverse" if d else ""
            w_ih, w_hh, b_ih, b_hh = G.torch_gru_weights(params[5 * d:5 * d + 5], I)
            getattr(gru, "weight_ih_l0" + sfx).copy_(torch.from_numpy(w_ih))
            getattr(gru, "weight_hh_l0" + sfx).copy_(torch.from_numpy(w_hh))
            getattr(gru, "bias_ih_l0" + sfx).copy_(torch.from_numpy(b_ih))
            getattr(gru, "bias_hh_l0" + sfx).copy_(torch.from_numpy(b_hh))
        out, hn = gru(torch.from_numpy(x.astype(np.float64)), torch.from_numpy(h0.astype(np.float64)))
    out = out.numpy().reshape(T, B, D, H).transpose(0, 2, 1, 3)
    assert np.abs(out - Y).max() < 1e-12 and np.abs(hn.numpy() - Yh).max() < 1e-12


@pytest.mark.parametrize("lbr", [0, 1])
def test_no_initial_state_is_zero_state(lbr):
    rng = np.random.default_rng(9 + lbr)
    x = rng.standard_normal((4, 2, 5)).astype(np.float32)
    params = G.random_params(rng, 2, 5, 6)
    a, b = G.run64(lbr, x, params), G.run64(lbr, x, params, np.zeros((2, 2, 6), np.float32))
    assert all(np.array_equal(u, v) for u, v in zip(a, b))


def _sig32(z):
    return (np.float32(1) / (np.float32(1) + np.exp(-z))).astype(np.float32)


def fp32_step(lbr, x_t, p, h_prev):
    """one step rounded in fp32 throughout, in the reference's order (numpy's fp32 dot products: another summation order)"""
    f = np.float32
    x = np.asarray(x_t, f)
    I = x.shape[1]
    wg, bg, wc, bc, rb = (np.asarray(a, f) for a in p)
    bg, bc, rb = bg.reshape(-1), bc.reshape(-1), rb.reshape(-1)
    H = wc.shape[1]
    h = np.zeros((x.shape[0], H), f) if h_prev is None else np.asarray(h_prev, f)
    g = (((x @ wg[:I]) + bg) + (h @ wg[I:])) + rb[:2 * H]
    z, r = _sig32(g[:, :H]), _sig32(g[:, H:])
    if lbr:
        pre = ((r * ((h @ wc[I:]) + rb[2 * H:])) + x @ wc[:I]) + bc
    else:
        pre = ((x @ wc[:I]) + ((r * h) @ wc[I:])) + (rb[2 * H:] + bc)
    n = np.tanh(pre).astype(f)
    return ((h - n) * z) + n


@pytest.mark.parametrize("lbr", [0, 1])
def test_step_bound_covers_fp32_rounding_of_the_step(lbr):
    for seed, (B, I, H, scale) in enumerate([(3, 20, 33, None), (5, 64, 256, None), (2, 12, 17, 4.0), (4, 300, 100, None)]):
        rng = np.random.default_rng(70 + seed + 10 * lbr)
        x = rng.standard_normal((B, I)).astype(np.float32)
        p = G.random_params(rng, 1, I, H, scale)
        h0 = rng.standard_normal((B, H)).astype(np.float32)
        for hp in (None, h0):
            h64, e = G.step_check_bounds(lbr, x, p, hp)
            got = fp32_step(lbr, x, p, hp).astype(np.float64)
            assert (np.abs(got - h64) <= e).all(), (seed, np.max(np.abs(got - h64) / e))


def test_plan_census():
    for sms in (114, 132):
        cells = G.census(sms)
        assert {k[1] for k in cells} == {1, 2, 4, 8, 16} and {k[2] for k in cells} == {0, 1}
        assert {(k[0], k[2], k[6]) for k in cells} == {(lbr, res, ks) for lbr in (0, 1) for res in (0, 1)
                                                      for ks in (1, 2, 4, 8) if (res, ks) != (0, 8)}
        for (lbr, b, h, d) in cells.values():
            assert G.choose_plan(lbr, b, h, d, sms)["smem"] <= G.SMEM_CAP


def test_plan_of_the_user_sizes():
    """the plans of the sizes tools/gru_bench.py times, on 132 SMs: R resident below H 512, streamed at 1024, and at 512 resident
    unless the LBR = 0 form's r * h_prev of 8 rows takes the room; a cluster per (direction, batch group) of at most 8 rows"""
    for lbr in (0, 1):
        for d in (1, 2):
            for h in (64, 128, 256, 512, 1024):
                for b in (1, 8, 64):
                    pl = G.choose_plan(lbr, b, h, d, 132)
                    assert pl is not None and pl["rows"] == min(b, 8) and pl["groups"] == -(-b // 8)
                    assert pl["resident"] == int(h < 512 or (h == 512 and (lbr == 1 or b == 1))), (lbr, d, h, b, pl)
    assert G.choose_plan(0, 1, 4096, 1, 132)["rows"] == 1 and G.choose_plan(0, 9, 4096, 1, 132)["rows"] == 3


PLAN_MAIN = r"""
#include <atomic>
#include <cstdio>
#include "gru_ops.h"
#include "rnn_ops.h"
namespace mnnb200 { std::atomic<unsigned long long> g_launch_count; }
using namespace mnnb200;
int main() {
    char kind[8];
    int c, b, h, d, sms;
    while (scanf("%7s %d %d %d %d %d", kind, &c, &b, &h, &d, &sms) == 6) {
        RnnPlan p;
        const bool ok = kind[0] == 'g' ? gru_choose_plan(c, b, h, d, sms, 232448, nullptr, nullptr, &p)
                                       : rnn_choose_plan(c, b, h, d, sms, 232448, nullptr, nullptr, &p);
        if (!ok) printf("none\n");
        else printf("%d %d %d %d %d %d %d %d\n", p.cs, p.groups, p.rows, p.hs, p.ks, p.threads, p.resident, p.smem);
    }
    return 0;
}
"""


def test_cpp_plan_search_equals_the_restatements(tmp_path):
    """gru_choose_plan and rnn_choose_plan (one shared search) against gru_oracle / rnn_oracle.choose_plan"""
    from mnn_b200 import build as B
    main = tmp_path / "plan_main.cu"
    main.write_text(PLAN_MAIN)
    exe = tmp_path / "plan_main"
    subprocess.run([NVCC, "-o", str(exe), str(main), os.path.join(B.CSRC, "gru.cu"), os.path.join(B.CSRC, "rnn.cu"),
                    "-I" + B.CSRC] + [f for f in B.NVCC_FLAGS if f != "-lineinfo"], check=True, capture_output=True)
    hs = sorted(set(R.CENSUS_H) | set(G.CENSUS_H) | {2048, 3000, 4096})
    bs = sorted(set(R.CENSUS_B) | {200, 1000})
    cases = [(k, c, b, h, d, sms) for k, cells in (("gru", (0, 1)), ("rnn", (0, 1))) for c in cells for h in hs for b in bs
             for d in (1, 2) for sms in (114, 132)]
    out = subprocess.run([str(exe)], input="".join(f"{k} {c} {b} {h} {d} {s}\n" for k, c, b, h, d, s in cases),
                         capture_output=True, text=True, check=True).stdout.split("\n")
    keys = ("cs", "groups", "rows", "hs", "ks", "threads", "resident", "smem")
    for (k, c, b, h, d, sms), line in zip(cases, out):
        want = (G if k == "gru" else R).choose_plan(c, b, h, d, sms)
        got = None if line == "none" else dict(zip(keys, map(int, line.split())))
        assert got == want, (k, c, b, h, d, sms, got, want)


def test_gru_kernels_compile_without_spills(tmp_path):
    from mnn_b200 import build as B
    src = os.path.join(B.CSRC, "gru.cu")
    out = subprocess.run([NVCC, "-c", src, "-o", str(tmp_path / "gru.o"), "-Xptxas", "-v"] + B.NVCC_FLAGS,
                         capture_output=True, text=True, check=True).stderr
    spills = [l for l in out.splitlines() if "spill" in l and not l.strip().startswith("0 bytes stack frame, 0 bytes spill")]
    assert "gru_recur_f32_kernel" in out and not spills, spills


# ---- the restatement against the recorded and the live reference CPU ----------------------------------------------------
from tests.golden import make_gru_golden as M  # noqa: E402

needs_ref = pytest.mark.skipif(not G.have_refdump(), reason="oracle/_ref/refdump_gru not built (no reference sources)")


def close(got, ref, what):
    """the project's rule for the CPU's fp32 (polynomial sigmoid / tanh): within 1e-3 of max |ref|"""
    assert got.shape == ref.shape, what
    assert np.abs(np.asarray(got, np.float64) - ref).max() <= 1e-3 * max(1e-6, float(np.abs(ref).max())), what


@pytest.mark.parametrize("name", sorted(M.CASES))
def test_oracle_matches_golden(name):
    lbr, keep, n_out, x, params, h0 = M.case_inputs(name)
    gold = np.load(M.PATH)
    Y, Yh = G.run64(lbr, x, params, h0)
    if keep:
        close(Y, gold[f"{name}/y"].astype(np.float64), (name, "y"))
    cpu = G.cpu_y_h(Y, Yh, h0 is not None, keep, n_out)
    if f"{name}/y_h" in gold:
        close(cpu, gold[f"{name}/y_h"].astype(np.float64), (name, "y_h"))
    else:
        assert cpu is None or not (keep and n_out > 1), name


@needs_ref
@pytest.mark.parametrize("lbr", [0, 1])
@pytest.mark.parametrize("D", [1, 2])
def test_oracle_matches_live_reference_on_fresh_seeds(lbr, D):
    """fresh seeds with B != H != I, with and without h0: the gate order (z, r), the bias split and both candidate forms"""
    rng = np.random.default_rng(2000 + 2 * lbr + D)
    for hh in (False, True):
        T, B, I, H = 7, 5, 11, 3
        x = rng.standard_normal((T, B, I)).astype(np.float32)
        params = G.random_params(rng, D, I, H, 0.8)
        h0 = rng.standard_normal((D, B, H)).astype(np.float32) if hh else None
        Y, Yh = G.run64(lbr, x, params, h0)
        y, = G.ref_op(lbr, x, params, h0, n_out=1)
        close(y, Y, (hh, "y"))
        assert np.abs(y - Y).max() < 1e-5, hh                # far inside the rule: the same arithmetic
        yh, = G.ref_op(lbr, x, params, h0, keep_all=False, n_out=1)
        close(yh, Yh, (hh, "y_h without keepAllOutputs"))
        assert np.abs(yh - Yh).max() < 1e-5, hh


@needs_ref
@pytest.mark.parametrize("lbr", [0, 1])
def test_reference_backward_y_h_is_its_zeroed_scratch(lbr):
    """with keepAllOutputs, Y and Y_h both requested and no h0, the reference CPU copies the backward Y_h from the op's scratch
    (memset to zero), not from the last backward step: Y_h[1] is zeros where ONNX's value is Y[0][1].  Its forward half and Y
    are right.  (With h0 that scratch is never written, so its contents are not tested.)"""
    rng = np.random.default_rng(3000 + lbr)
    x = rng.standard_normal((4, 3, 5)).astype(np.float32)
    params = G.random_params(rng, 2, 5, 6)
    y, yh = G.ref_op(lbr, x, params, None)
    Y, Yh = G.run64(lbr, x, params)
    assert np.array_equal(yh[1].view(np.uint32), np.zeros_like(yh[1]).view(np.uint32))
    assert np.abs(Yh[1]).min() > 0 and np.array_equal(Yh[1], Y[0, 1])
    close(yh[0], Yh[0], "forward Y_h")
    close(y, Y, "Y")
    close(yh, G.cpu_y_h(Y, Yh, False, True, 2), "the CPU's Y_h")
