"""The numpy restatement of LSTM / RNN (oracle/rnn_oracle.py) on the CPU: against torch.nn.LSTM / nn.RNN in float64 (an
independent implementation, with ONNX's i, o, f, c gate rows permuted to torch's i, f, g, o), the conventions of the
reference's lowering that torch does not share (no h_prev R^T term and no f * c term at the first step without initial states,
direction 1 writing Y at T - 1 - s, Y_h of direction 1 at position 0), and the launch plan's census on 114 and 132 SMs."""
import subprocess

import numpy as np
import pytest

from oracle import rnn_oracle as R
from tests.golden import make_rnn_golden as M

needs_ref = pytest.mark.skipif(not R.have_refdump(), reason="oracle/_ref/refdump_rnn not built (no reference sources)")


def close(got, ref, what):
    """the project's rule for the CPU's fp32 (polynomial sigmoid / tanh): within 1e-3 of max |ref|"""
    assert got.shape == ref.shape, what
    assert np.abs(np.asarray(got, np.float64) - ref).max() <= 1e-3 * max(1e-6, float(np.abs(ref).max())), what


@pytest.mark.parametrize("name", sorted(M.CASES))
def test_oracle_matches_golden(name):
    cell, x, w, r, b, h0, c0 = M.case_inputs(name)
    gold = np.load(M.PATH)
    for k, y in zip(("y", "y_h", "y_c"), R.run64(cell, x, w, r, b, h0, c0)):
        if y is not None:
            close(y, gold[f"{name}/{k}"].astype(np.float64), (name, k))


@needs_ref
@pytest.mark.parametrize("cell", [0, 1])
@pytest.mark.parametrize("D", [1, 2])
def test_oracle_matches_live_reference_on_fresh_seeds(cell, D):
    """fresh seeds, B != H and I != H (the reference's HR MatMul reads R and h_prev densely at their view offsets, whatever its
    view strides {B, 1, 0} say), with and without initial states; gate rows in ONNX order i, o, f, c"""
    rng = np.random.default_rng(1000 + 2 * cell + D)
    for init in ("none", "h0c0" if cell == 0 else "h0"):
        T, B, I, H = 7, 5, 11, 3
        G = R.GATES[cell]
        x = rng.standard_normal((T, B, I)).astype(np.float32)
        w = (rng.standard_normal((D, G * H, I)) * 0.5).astype(np.float32)
        r = (rng.standard_normal((D, G * H, H)) * 0.5).astype(np.float32)
        b = (rng.standard_normal((D, G * H)) * 0.5).astype(np.float32)
        h0 = rng.standard_normal((D, B, H)).astype(np.float32) if init != "none" else None
        c0 = rng.standard_normal((D, B, H)).astype(np.float32) if init == "h0c0" else None
        for k, (got, ref) in enumerate(zip(R.ref_op(cell, x, w, r, b, h0, c0), R.run64(cell, x, w, r, b, h0, c0))):
            close(got, ref, (init, k))
            assert np.abs(got - ref).max() < 1e-5, (init, k)   # far inside the rule: the same arithmetic


@needs_ref
def test_reference_ignores_the_lstm_clip_parameter():
    """the geometry never reads the LSTM parameter beyond outputCount (the converter drops ONNX's activations, clip and
    input_forget): a clippingThreshold changes nothing even where the cell state passes it"""
    rng = np.random.default_rng(12)
    x = rng.standard_normal((4, 2, 5)).astype(np.float32)
    w, r = (rng.standard_normal((1, 16, 5)) * 3).astype(np.float32), (rng.standard_normal((1, 16, 4)) * 3).astype(np.float32)
    b = rng.standard_normal((1, 16)).astype(np.float32)
    clipped, plain = R.ref_op(0, x, w, r, b, clip=0.01), R.ref_op(0, x, w, r, b)
    assert np.abs(plain[2]).max() > 0.01
    for a, p in zip(clipped, plain):
        assert np.array_equal(a, p)


@needs_ref
def test_reference_crashes_on_lstm_h0_without_c0():
    """an LSTM with h0 but no c0 takes the geometry's "has init" branch with a null cell input: the reference CPU dies with
    SIGSEGV, so it has no result there.  The kernel starts the cell at zeros then (ONNX's meaning)"""
    rng = np.random.default_rng(13)
    x = rng.standard_normal((2, 2, 3)).astype(np.float32)
    w, r = rng.standard_normal((1, 16, 3)).astype(np.float32), rng.standard_normal((1, 16, 4)).astype(np.float32)
    b, h0 = rng.standard_normal((1, 16)).astype(np.float32), rng.standard_normal((1, 2, 4)).astype(np.float32)
    with pytest.raises(subprocess.CalledProcessError) as e:
        R.ref_op(0, x, w, r, b, h0)
    assert e.value.returncode == -11


def data(rng, cell, T, B, I, H, D):
    g = R.GATES[cell]
    x = rng.standard_normal((T, B, I))
    w, r = rng.standard_normal((D, g * H, I)) * 0.4, rng.standard_normal((D, g * H, H)) * 0.4
    b = rng.standard_normal((D, g * H)) * 0.3
    h0, c0 = rng.standard_normal((D, B, H)), rng.standard_normal((D, B, H))
    return x, w, r, b, h0, c0


@pytest.mark.parametrize("cell", [0, 1])
@pytest.mark.parametrize("D", [1, 2])
def test_oracle_equals_torch_in_float64(cell, D):
    import torch
    rng = np.random.default_rng(cell * 2 + D)
    T, B, I, H = 5, 3, 7, 6
    x, w, r, b, h0, c0 = data(rng, cell, T, B, I, H, D)
    mod = (torch.nn.LSTM if cell == 0 else torch.nn.RNN)(I, H, bidirectional=D == 2).double()
    with torch.no_grad():
        for d in range(D):
            sfx = "_reverse" if d else ""
            wd, rd, bd = R.torch_lstm_weights(w[d], r[d], b[d]) if cell == 0 else (w[d], r[d], b[d])
            getattr(mod, "weight_ih_l0" + sfx).copy_(torch.from_numpy(wd))
            getattr(mod, "weight_hh_l0" + sfx).copy_(torch.from_numpy(rd))
            getattr(mod, "bias_ih_l0" + sfx).copy_(torch.from_numpy(bd))
            getattr(mod, "bias_hh_l0" + sfx).zero_()
        st = (torch.from_numpy(h0), torch.from_numpy(c0)) if cell == 0 else torch.from_numpy(h0)
        y, hn = mod(torch.from_numpy(x), st)
    Y, Yh, Yc = R.run64(cell, x, w, r, b, h0, c0 if cell == 0 else None)
    np.testing.assert_allclose(Y, y.numpy().reshape(T, B, D, H).transpose(0, 2, 1, 3), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(Yh, (hn[0] if cell == 0 else hn).numpy(), rtol=1e-12, atol=1e-12)
    if cell == 0:
        np.testing.assert_allclose(Yc, hn[1].numpy(), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("cell", [0, 1])
def test_no_initial_state_is_zero_state(cell):
    """without h0 / c0 the first step drops the h_prev R^T and f * c terms: the same values as zero states (ONNX's default)"""
    rng = np.random.default_rng(9)
    x, w, r, b, _, _ = data(rng, cell, 4, 2, 5, 3, 2)
    Y, Yh, Yc = R.run64(cell, x, w, r, b)
    z = np.zeros((2, 2, 3))
    Y0, Yh0, Yc0 = R.run64(cell, x, w, r, b, z, z if cell == 0 else None)
    np.testing.assert_array_equal(Y, Y0)
    np.testing.assert_array_equal(Yh, Yh0)
    # direction 1 runs from t = T - 1 down: its Y_h is Y at position 0, direction 0's at T - 1
    np.testing.assert_array_equal(Yh[0], Y[-1, 0])
    np.testing.assert_array_equal(Yh[1], Y[0, 1])


def test_step_bound_covers_fp32_rounding_of_the_step():
    """the step bound exceeds an fp32 evaluation of the same step (numpy float32 arithmetic in the reference's order)"""
    rng = np.random.default_rng(4)
    B, I, H = 4, 9, 33
    x = rng.standard_normal((B, I)).astype(np.float32)
    w, r = (rng.standard_normal((4 * H, I)) * 0.3).astype(np.float32), (rng.standard_normal((4 * H, H)) * 0.3).astype(np.float32)
    b = rng.standard_normal(4 * H).astype(np.float32)
    hp, cp = rng.standard_normal((B, H)).astype(np.float32), rng.standard_normal((B, H)).astype(np.float32)
    gate, gabs = R.gates64(x, w, b)
    h64, c64, eh, ec = R.step_check_bounds(0, gate, gabs, I, b, r, hp, cp)
    z = ((x @ w.T + b) + hp @ r.T).astype(np.float32)
    sig = lambda v: (1 / (1 + np.exp(-v.astype(np.float64)))).astype(np.float32)
    i, o, f, g = sig(z[:, :H]), sig(z[:, H:2 * H]), sig(z[:, 2 * H:3 * H]), np.tanh(z[:, 3 * H:])
    c = i * g + f * cp
    h = np.tanh(c) * o
    assert (np.abs(h - h64) <= eh).all() and (np.abs(c - c64) <= ec).all()
    assert eh.max() < 1e-4 and ec.max() < 1e-4


@pytest.mark.parametrize("sms", [114, 132])
def test_plan_census(sms):
    """every launch cell the chooser reaches on the SM count has a representative, and the cells span every cluster size,
    resident and streamed R, one and several batch groups, a ragged last group, both D and every threads-per-dot-product"""
    cells = R.census(sms)
    assert {k[1] for k in cells} == {1, 2, 4, 8, 16} and {k[2] for k in cells} == {0, 1}
    assert {k[3] for k in cells} == {0, 1} and {k[4] for k in cells} == {0, 1} and {k[5] for k in cells} == {1, 2}
    assert {k[6] for k in cells} == {1, 2, 4, 8} and {k[0] for k in cells} == {0, 1}
    for key, (cell, b, h, d) in cells.items():
        pl = R.choose_plan(cell, b, h, d, sms)
        assert R.cell_of(cell, b, d, pl) == key
        assert pl["smem"] <= R.SMEM_CAP and pl["cs"] * (pl["hs"] - 1) < h + pl["hs"]
        assert pl["groups"] * pl["rows"] >= b > (pl["groups"] - 1) * pl["rows"]


def test_plan_of_the_user_sizes():
    """the plans of the sizes tools/rnn_bench.py times, on 132 SMs"""
    want = {(0, 32, 256, 2): (16, 4, 8, 1), (0, 16, 512, 1): (16, 2, 8, 0), (0, 1, 128, 1): (4, 1, 1, 1),
            (0, 64, 1024, 1): (16, 8, 8, 0)}
    for (cell, b, h, d), (cs, groups, rows, resident) in want.items():
        pl = R.choose_plan(cell, b, h, d, 132)
        assert (pl["cs"], pl["groups"], pl["rows"], pl["resident"]) == (cs, groups, rows, resident), (b, h, d, pl)
