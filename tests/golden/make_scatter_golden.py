"""Writes tests/golden/scatter_golden.npz: ScatterNd and ScatterElements outputs recorded from the reference CPU backend
(oracle/_ref/refdump_scatter op, built by build() where the reference sources are).

Each case's inputs are rebuilt from its seed by `case_inputs` (numpy's PCG64 generator, the same on every machine).  Outputs are
bit-exact targets, so the file holds only their shape and the sha256 of their bytes; with a reduction every NaN is hashed as
0x7fc00000 (oracle/scatter_oracle.py: canonical), since fp32 arithmetic keeps a NaN but not its payload.  With a reduction,
every destination lies inside the output: the CPU does no bounds check there.
Run: python tests/golden/make_scatter_golden.py"""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
PATH = os.path.join(ROOT, "tests", "golden", "scatter_golden.npz")
F, I = "float32", "int32"

# name -> kind, out (the output's shape), idx (shape, low, high; a tuple of highs: one ScatterNd component per dim), upd (the
# updates' shape), data (a data input), red (None, 'add', 'sub', 'mul'), axis (ScatterElements' fourth input; None: none),
# torch (a BinaryOp parameter with opType left at ADD), dtype, values ('order': 1e8 and 1 mixed, 'special': NaN and +-Inf)
CASES = {
    "nd3_zero_d1_s768": dict(kind="ScatterNd", out=(6, 768), idx=((4, 1), 0, 6), upd=(4, 768)),
    "nd4_d2_s3_duplicates": dict(kind="ScatterNd", out=(5, 4, 3), idx=((10, 2), 0, (2, 2)), upd=(10, 3), data=True),
    "nd4_d3_rank_s1": dict(kind="ScatterNd", out=(3, 4, 5), idx=((2, 6, 3), 0, (3, 4, 5)), upd=(2, 6), data=True),
    "nd4_negative_and_past_end_skipped": dict(kind="ScatterNd", out=(8, 3), idx=((12, 1), -3, 11), upd=(12, 3), data=True),
    "nd3_component_past_axis_lands_inside": dict(kind="ScatterNd", out=(4, 5), idx=((6, 2), 0, (3, 9)), upd=(6,)),
    "nd4_int32": dict(kind="ScatterNd", out=(20, 6), idx=((7, 1), 0, 20), upd=(7, 6), data=True, dtype=I),
    "nd3_rank_not_d_plus_1_s1": dict(kind="ScatterNd", out=(3, 5, 768), idx=((4, 2), 0, (3, 5)), upd=(4, 768)),
    "nd4_batched_indices_d2": dict(kind="ScatterNd", out=(4, 5, 6), idx=((2, 3, 2), 0, (4, 5)), upd=(2, 3, 6), data=True),
    "nd4_add_duplicates": dict(kind="ScatterNd", out=(6, 3), idx=((40, 1), 0, 6), upd=(40, 3), data=True, red="add"),
    "nd3_mul_zero_canvas": dict(kind="ScatterNd", out=(5, 4), idx=((9, 1), 0, 5), upd=(9, 4), red="mul"),
    "nd4_special_values_copied": dict(kind="ScatterNd", out=(9, 8), idx=((6, 1), 0, 9), upd=(6, 8), data=True, values="special"),
    "el_axis0_none": dict(kind="ScatterElements", out=(5, 4), idx=((3, 4), 0, 5), upd=(3, 4), axis=0),
    "el_axis1_none_negative_lands_inside": dict(kind="ScatterElements", out=(4, 5), idx=((4, 5), -2, 5), upd=(4, 5), axis=1),
    "el_axis0_no_axis_input_add": dict(kind="ScatterElements", out=(6, 3), idx=((8, 3), 0, 6), upd=(8, 3), red="add"),
    "el_axis1_add": dict(kind="ScatterElements", out=(4, 6), idx=((4, 9), 0, 6), upd=(4, 9), axis=1, red="add"),
    "el_axis_neg1_sub": dict(kind="ScatterElements", out=(2, 3, 7), idx=((2, 3, 10), 0, 7), upd=(2, 3, 10), axis=-1, red="sub"),
    "el_axis1_mul": dict(kind="ScatterElements", out=(3, 5), idx=((3, 12), 0, 5), upd=(3, 12), axis=1, red="mul"),
    "el_axis_neg1_none": dict(kind="ScatterElements", out=(3, 2, 6), idx=((3, 2, 4), 0, 6), upd=(3, 2, 4), axis=-1),
    "el_add_order_changes_sum": dict(kind="ScatterElements", out=(3, 4), idx=((3, 200), 0, 4), upd=(3, 200), axis=1, red="add",
                                     values="order"),
    "el_add_special_values": dict(kind="ScatterElements", out=(4, 8), idx=((4, 30), 0, 8), upd=(4, 30), axis=1, red="add",
                                  values="special"),
    "el_mul_special_values": dict(kind="ScatterElements", out=(16,), idx=((64,), 0, 16), upd=(64,), axis=0, red="mul",
                                  values="special"),
    "el_torch_scatter_default_add": dict(kind="ScatterElements", out=(5, 3), idx=((7, 3), 0, 5), upd=(7, 3), axis=0, torch=True),
    "el_updates_read_flat": dict(kind="ScatterElements", out=(4, 4), idx=((2, 3), 0, 4), upd=(3, 5), axis=1),
}


def seed_of(name):
    return sorted(CASES).index(name) + 3000


def _values(rng, shape, kind):
    v = rng.standard_normal(shape).astype(np.float32)
    if kind == "order":
        v = np.where(rng.random(shape) < 0.2, np.float32(1e8) * np.sign(v), np.float32(1.0)).astype(np.float32)
    elif kind == "special":
        flat = v.reshape(-1)
        pick = rng.choice(flat.size, min(flat.size, 9), replace=False)
        flat[pick] = np.array([np.nan, np.inf, -np.inf] * 3, np.float32)[:pick.size]
    return v


def case_inputs(name):
    """(indices, updates, data or None) of a case"""
    c = CASES[name]
    rng = np.random.default_rng(seed_of(name))
    ishape, lo, hi = c["idx"]
    if isinstance(hi, tuple):
        idx = np.stack([rng.integers(lo, h, ishape[:-1]) for h in hi], -1)
    else:
        idx = rng.integers(lo, hi, ishape)
    idx = np.asarray(idx, np.int32)
    if c.get("dtype") == I:
        upd = rng.integers(-1000, 1000, c["upd"]).astype(np.int32)
        data = rng.integers(-1000, 1000, c["out"]).astype(np.int32) if c.get("data") else None
    else:
        upd = _values(rng, c["upd"], c.get("values"))
        need_data = c.get("data") or c["kind"] == "ScatterElements"
        data = rng.standard_normal(c["out"]).astype(np.float32) if need_data else None
    return idx, upd, data


def reduction(name):
    c = CASES[name]
    return "add" if c.get("torch") else c.get("red")


def case_oracle(name):
    from oracle import scatter_oracle as S
    c = CASES[name]
    idx, upd, data = case_inputs(name)
    return S.scatter(c["kind"], c["out"], idx, upd, data, reduction(name), c.get("axis") or 0)


def case_reference(name, **kw):
    from oracle import scatter_oracle as S
    c = CASES[name]
    idx, upd, data = case_inputs(name)
    red = c.get("red")
    if c["kind"] == "ScatterElements" and red is None and not c.get("torch"):
        red = -1                         # ONNX ScatterElements without a reduction: opType -1
    return S.ref_op(c["kind"], c["out"], idx, upd, data, red, axis=c.get("axis"), torch_style=c.get("torch", False), **kw)


def digest(y):
    from oracle import scatter_oracle as S
    return hashlib.sha256(np.ascontiguousarray(S.canonical(y)).tobytes()).hexdigest()


def load():
    """{case: (shape, sha256)}"""
    g = np.load(PATH)
    return {n: (tuple(int(v) for v in g[f"{n}__shape"]), str(g[f"{n}__sha"])) for n in CASES}


def main():
    sys.path.insert(0, ROOT)
    from oracle import scatter_oracle as S
    if not S.have_refdump():
        sys.exit("needs oracle/_ref/refdump_scatter (run build() where the reference sources are)")
    arrays = {}
    for name in CASES:
        y = case_reference(name)
        arrays[f"{name}__shape"] = np.array(y.shape, np.int64)
        arrays[f"{name}__sha"] = np.array(digest(y))
    np.savez_compressed(PATH, **arrays)
    print("wrote", PATH, len(CASES), "cases")


if __name__ == "__main__":
    main()
