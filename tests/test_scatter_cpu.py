"""The ScatterNd / ScatterElements restatement (oracle/scatter_oracle.py) against the recorded goldens, and, where
oracle/_ref/refdump_scatter exists, against the live reference CPU on fresh seeds (CPU).  This is where the rules the kernels
build on are pinned: S is the product of the updates' dims from index D on (not the slice length when the indices' rank is not
D + 1); without a reduction a destination outside the output is skipped, a negative index is not wrapped, a component past its
axis whose total lands inside writes there, and the last writer wins; with ADD / SUB / MUL the updates fold in index order."""
import numpy as np
import pytest

from oracle import scatter_oracle as S
from tests.golden import make_scatter_golden as M

needs_ref = pytest.mark.skipif(not S.have_refdump(), reason="oracle/_ref/refdump_scatter not built (no reference sources)")


@pytest.mark.parametrize("name", sorted(M.CASES))
def test_oracle_matches_golden(name):
    y = M.case_oracle(name)
    shape, sha = M.load()[name]
    assert y.shape == shape and M.digest(y) == sha


def test_s_rule_when_indices_rank_is_not_d_plus_1():
    # indices [4, 2] into [3, 5, 768]: S = prod(updates.shape[2:]) = 1, so each update writes one element
    n, d, s, r, _ = S.geometry("ScatterNd", (3, 5, 768), (4, 2), (4, 768))
    assert (n, d, s, r) == (4, 2, 1, 768)
    y = M.case_oracle("nd3_rank_not_d_plus_1_s1")
    assert np.count_nonzero(y) <= 4


def test_last_writer_and_index_order():
    idx = np.array([[1], [1], [0], [1]], np.int32)
    upd = np.array([[1.0], [2.0], [3.0], [4.0]], np.float32)
    assert S.scatter("ScatterNd", (2, 1), idx, upd).reshape(-1).tolist() == [3.0, 4.0]
    big = np.array([1e8, 1.0, -1e8, 1.0], np.float32).reshape(4, 1)
    y = S.scatter("ScatterNd", (2, 1), np.array([[0]] * 4, np.int32), big, reduction="add")
    assert y[0, 0] == np.float32(1.0)            # ((0 + 1e8) + 1) - 1e8 + 1: the 1 lost to 1e8 stays lost


def test_index_terms_past_int32_are_skipped():
    # (2^24 + 5) * 256 and -(2^24 - 5) * 256 leave int32: skipped (test_reference_skips_index_terms_past_int32 pins the CPU)
    d, ok = S.destinations("ScatterNd", (16, 256), np.array([[(1 << 24) + 5], [-(1 << 24) + 5], [5]], np.int32))
    assert ok.tolist() == [False, False, True] and d[2] == 5 * 256


@needs_ref
@pytest.mark.reference
@pytest.mark.parametrize("name", sorted(M.CASES))
def test_reference_matches_golden(name):
    y = M.case_reference(name)
    shape, sha = M.load()[name]
    assert y.shape == shape and M.digest(y) == sha


@needs_ref
@pytest.mark.reference
@pytest.mark.parametrize("seed", range(4))
def test_reference_matches_oracle_fresh_seeds(seed):
    rng = np.random.default_rng(9100 + seed)
    # ScatterNd, every D up to the rank, with and without data, skipped and landing-inside indices
    out = (int(rng.integers(2, 6)), int(rng.integers(2, 5)), int(rng.integers(1, 9)))
    for d in (1, 2, 3):
        n = int(rng.integers(1, 30))
        idx = np.stack([rng.integers(-1, out[k] + 2, n) for k in range(d)], -1).astype(np.int32)
        upd = rng.standard_normal((n,) + out[d:]).astype(np.float32)
        data = rng.standard_normal(out).astype(np.float32) if seed % 2 else None
        ref = S.ref_op("ScatterNd", out, idx, upd, data)
        assert np.array_equal(ref.view(np.uint32), S.scatter("ScatterNd", out, idx, upd, data).view(np.uint32)), d
        idx = np.stack([rng.integers(0, out[k], n) for k in range(d)], -1).astype(np.int32)
        for red in ("add", "sub", "mul"):
            ref = S.ref_op("ScatterNd", out, idx, upd, data, red)
            assert np.array_equal(S.canonical(ref), S.canonical(S.scatter("ScatterNd", out, idx, upd, data, red))), (d, red)
    # ScatterElements on every axis with every reduction
    shape = (3, 4, 5)
    data = rng.standard_normal(shape).astype(np.float32)
    for axis in (0, 1, 2, -1):
        ishape = list(shape)
        ishape[axis] = int(rng.integers(1, 12))
        idx = rng.integers(0, shape[axis], ishape).astype(np.int32)
        upd = rng.standard_normal(ishape).astype(np.float32)
        for red in (None, "add", "sub", "mul"):
            ref = S.ref_op("ScatterElements", shape, idx, upd, data, red if red else -1, axis=axis)
            want = S.scatter("ScatterElements", shape, idx, upd, data, red, axis)
            assert np.array_equal(S.canonical(ref), S.canonical(want)), (axis, red)


@needs_ref
@pytest.mark.reference
def test_reference_skips_index_terms_past_int32():
    # index * stride past int32: int32 wraparound would put (2^24 + 5) * 256 and -(2^24 - 5) * 256 on row 5, but the CPU
    # writes neither, as the oracle and the kernel skip them (no reduction only: with one the CPU has no bounds check)
    idx = np.array([[(1 << 24) + 5], [-(1 << 24) + 5], [2]], np.int32)
    upd = np.arange(3 * 256, dtype=np.float32).reshape(3, 256)
    data = np.full((16, 256), -1.0, np.float32)
    ref = S.ref_op("ScatterNd", (16, 256), idx, upd, data)
    assert (ref[5] == -1).all()
    assert np.array_equal(ref.view(np.uint32), S.scatter("ScatterNd", (16, 256), idx, upd, data).view(np.uint32))


@needs_ref
@pytest.mark.reference
def test_reference_drops_updates_for_other_reductions():
    # MAXIMUM (9) is not ADD / SUB / MUL: the CPU's fold falls into `default: break` and y stays data (the GPU refuses it)
    data = np.arange(6, dtype=np.float32).reshape(2, 3)
    idx = np.array([[1, 0, 1]], np.int32)
    upd = np.full((1, 3), 100.0, np.float32)
    assert np.array_equal(S.ref_op("ScatterElements", (2, 3), idx, upd, data, 9, axis=0), data)
