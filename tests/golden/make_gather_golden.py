"""Writes tests/golden/gather_golden.npz: Gather, GatherV2, GatherND, GatherElements and Cast outputs, and broadcast MatMul /
BatchMatMul outputs, recorded from the reference CPU backend (oracle/_ref/refdump_gather op, built by build() where the reference
sources are).

Each case's inputs are rebuilt from its seed by `case_inputs` (numpy's PCG64 generator, the same on every machine).  Gather and
Cast outputs are bit-exact targets, so the file holds only their shape and the sha256 of their bytes; the MatMul outputs are
held to 1e-3 of max|ref| and are stored whole.  Out-of-range indices appear only where the CPU's zero-fill rule is the kernels'
(oracle/gather_oracle.py: cpu_defined).
Run: python tests/golden/make_gather_golden.py"""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
PATH = os.path.join(ROOT, "tests", "golden", "gather_golden.npz")
F, I = "float32", "int32"

# name -> kind, params (shape, dtype), indices (shape, low, high), axis (None: none), axis_input (a constant third input)
CASES = {
    "gatherv2_embedding_inside768": dict(kind="GatherV2", params=((64, 768), F), indices=((4, 16), 0, 64), axis=0, axis_input=True),
    "gatherv2_axis1_inside3": dict(kind="GatherV2", params=((4, 9, 3), F), indices=((5,), 0, 9), axis=1, axis_input=True),
    "gatherv2_axis_last_inside1": dict(kind="GatherV2", params=((3, 4, 10), F), indices=((2, 3), 0, 10), axis=-1),
    "gatherv2_one_index": dict(kind="GatherV2", params=((2, 17, 12), F), indices=((1,), 0, 1), axis=1, axis_input=True),
    "gatherv2_negative_out_of_range": dict(kind="GatherV2", params=((12, 5), F), indices=((6, 4), -4, 16), axis=0),
    "gatherv2_int32_params": dict(kind="GatherV2", params=((20, 6), I), indices=((7,), 0, 20), axis=0, axis_input=True),
    "gather_axis0": dict(kind="Gather", params=((30, 8), F), indices=((3, 5), -2, 33), axis=None),
    "gather_axis1_op": dict(kind="Gather", params=((3, 8, 4), F), indices=((6,), 0, 8), axis=1),
    "gathernd_d2_inside768": dict(kind="GatherND", params=((3, 5, 768), F), indices=((4, 2), 0, (3, 5)), axis=None),
    "gathernd_d1_inside3_out_of_range": dict(kind="GatherND", params=((10, 3), F), indices=((2, 6, 1), -2, 12), axis=None),
    "gathernd_d3_inside1": dict(kind="GatherND", params=((3, 4, 5), F), indices=((2, 3, 3), 0, (3, 4, 5)), axis=None),
    "gathernd_batch1": dict(kind="GatherND", params=((3, 5, 4), F), indices=((3, 2, 1), 0, 5), axis=1),
    "gathernd_batch1_d2": dict(kind="GatherND", params=((2, 4, 3, 2), F), indices=((2, 5, 2), 0, (4, 3)), axis=1),
    "gatherelements_axis0_out_of_range": dict(kind="GatherElements", params=((4, 3, 5), F), indices=((6, 3, 5), -3, 7), axis=0,
                                              axis_input=True),
    "gatherelements_axis1": dict(kind="GatherElements", params=((5, 6), F), indices=((5, 9), 0, 6), axis=1, axis_input=True),
    "gatherelements_topk_smaller": dict(kind="GatherElements", params=((2, 3, 50), F), indices=((2, 3, 5), 0, 50), axis=-1,
                                        axis_input=True),
    "cast_i32_f32": dict(kind="Cast", params=((1000,), I), cast_to=F),
    "cast_f32_i32": dict(kind="Cast", params=((1000,), F), cast_to=I),
}
# name -> kind, A shape, B shape, ta, tb: the broadcasts ShapeMatMul takes, and 1-D operands
MATMUL_CASES = {
    "matmul_bsd_de": ("MatMul", (2, 16, 64), (64, 48), 0, 0),
    "batchmatmul_1hsd_bhds": ("BatchMatMul", (1, 4, 32, 16), (2, 4, 16, 32), 0, 0),
    "batchmatmul_adjy": ("BatchMatMul", (2, 3, 24, 16), (2, 3, 24, 16), 0, 1),
    "batchmatmul_adjx_b1": ("BatchMatMul", (3, 16, 20), (1, 16, 12), 1, 0),
    "matmul_ta_tb_both_broadcast": ("MatMul", (2, 1, 32, 10), (1, 3, 12, 32), 1, 1),
    "matmul_1d_a": ("MatMul", (64,), (3, 64, 20), 0, 0),
    "matmul_1d_b": ("MatMul", (2, 5, 64), (64,), 0, 0),
}


def seed_of(name):
    return sorted(list(CASES) + list(MATMUL_CASES)).index(name) + 2000


def case_inputs(name):
    """[params, indices] of a gather case, [x] of a Cast case, [A, B] of a MatMul case"""
    rng = np.random.default_rng(seed_of(name))
    if name in MATMUL_CASES:
        _, sa, sb, _, _ = MATMUL_CASES[name]
        return [rng.standard_normal(sa).astype(np.float32), rng.standard_normal(sb).astype(np.float32)]
    c = CASES[name]
    shape, dt = c["params"]
    if c["kind"] == "Cast":
        if dt == I:
            x = rng.integers(-2**31, 2**31, shape, dtype=np.int64).astype(np.int32)
            x[:8] = [0, 1, -1, 16777217, -16777217, 2**31 - 1, -2**31, 33554435]
            return [x]
        x = (rng.standard_normal(shape) * np.exp2(rng.integers(0, 40, shape))).astype(np.float32)
        x[:10] = [0.5, -0.5, 1.9999999, -2.5, np.nan, np.inf, -np.inf, 2147483520.0, -2147483648.0, 3e9]
        return [x]
    p = rng.standard_normal(shape).astype(np.float32) if dt == F else rng.integers(-1000, 1000, shape).astype(np.int32)
    ishape, lo, hi = c["indices"]
    if isinstance(hi, tuple):       # a GatherND tuple: each component in its own dim
        idx = np.stack([rng.integers(0, h, ishape[:-1]) for h in hi], -1)
    else:
        idx = rng.integers(lo, hi, ishape)
    return [p, np.asarray(idx, np.int32)]


def case_oracle(name):
    from oracle import gather_oracle as G
    c = CASES[name]
    x = case_inputs(name)
    if c["kind"] == "Cast":
        return G.cast_i32_f32(x[0]) if c["cast_to"] == F else G.cast_f32_i32(x[0])
    axis = c["axis"] or 0
    if c["kind"] in ("Gather", "GatherV2"):
        return G.gather(*x, axis)
    if c["kind"] == "GatherND":
        return G.gather_nd(*x, axis)
    return G.gather_elements(*x, axis)


def case_reference(name, **kw):
    from oracle import gather_oracle as G
    if name in MATMUL_CASES:
        kind, _, _, ta, tb = MATMUL_CASES[name]
        return G.ref_op(kind, case_inputs(name), ta=ta, tb=tb, **kw)
    c = CASES[name]
    if c["kind"] == "Cast":
        return G.ref_op("Cast", case_inputs(name), cast_to=c["cast_to"], **kw)
    return G.ref_op(c["kind"], case_inputs(name), axis=c["axis"], axis_input=c.get("axis_input", False), **kw)


def matmul_oracle(name):
    """float64 C = op(A) op(B) over the broadcast batches, with numpy's squeeze of 1-D operands"""
    _, _, _, ta, tb = MATMUL_CASES[name]
    a, b = (v.astype(np.float64) for v in case_inputs(name))
    if ta and a.ndim > 1:
        a = np.swapaxes(a, -1, -2)
    if tb and b.ndim > 1:
        b = np.swapaxes(b, -1, -2)
    return a @ b


def digest(y):
    return hashlib.sha256(np.ascontiguousarray(y).tobytes()).hexdigest()


def load():
    """{gather / cast case: (shape, sha256)}, {matmul case: y}"""
    g = np.load(PATH)
    out = {n: (tuple(int(v) for v in g[f"{n}__shape"]), str(g[f"{n}__sha"])) for n in CASES}
    return out, {n: g[f"{n}__y"] for n in MATMUL_CASES}


def main():
    sys.path.insert(0, ROOT)
    from oracle import gather_oracle as G
    if not G.have_refdump():
        sys.exit("needs oracle/_ref/refdump_gather (run build() where the reference sources are)")
    arrays = {}
    for name in CASES:
        y = case_reference(name)
        c = CASES[name]
        if c["kind"] != "Cast":
            assert G.cpu_defined(c["kind"], *case_inputs(name), c["axis"] or 0), name
        arrays[f"{name}__shape"] = np.array(y.shape, np.int64)
        arrays[f"{name}__sha"] = np.array(digest(y))
    for name in MATMUL_CASES:
        arrays[f"{name}__y"] = case_reference(name)
    np.savez_compressed(PATH, **arrays)
    print("wrote", PATH, len(CASES) + len(MATMUL_CASES), "cases")


if __name__ == "__main__":
    main()
