"""Restatement of the reference CPU's ScatterNd and ScatterElements.

GeometryScatter.cpp:13-152 lowers both ops to one While loop (buildScatterND) that the CPU runs in index order
(parallel = false, CPURaster.cpp:1194-1197).  y starts as a copy of data, or zeros for a 3-input ScatterNd.  Update i has a
destination dst_i = sum_d c[i][d] * stride[d], stride being the output's element strides (the CPU computes it with a MUL and a
SUM reduce; where a term c * stride leaves int32 its result is its own arithmetic's, and this restatement, like the GPU, skips
the update: tests/test_scatter_cpu.py pins the cases where the CPU skips it too):
  - ScatterNd(indices, updates, shape[, data]): N = prod(indices.shape[:-1]), D = indices.shape[-1], c[i] = indices[i, :],
    and S = prod(updates.shape[D:]).  S is the product of the updates' dims from *index D* on, as the CPU computes it: that is
    the slice length only when indices.ndim == D + 1 (indices [4, 2] into [3, 5, 768] give S = 1, not 768).  Pinned on the
    live reference by tests/test_scatter_cpu.py.
  - ScatterElements(data, indices, updates[, axis]): N = indices.size, S = 1, c[i] = i's coordinate in indices' shape with the
    axis component replaced by indices[i]; updates are read flat (their first N elements).
Without a reduction (fuse < 0, CPURaster.cpp:911-962) slice i is copied to y[dst_i : dst_i + S] when 0 <= dst_i < y.size
and skipped otherwise; negative indices are not wrapped; the last writer wins.  With ADD / SUB / MUL (fuse >= 0,
CPURaster.cpp:964-1186) y[dst_i + w] = y[dst_i + w] op updates[i][w] in plain fp32, in update order, and the CPU has no bounds
check; this restatement, like the GPU, skips an out-of-range destination there (the CPU's result is undefined).  Any other
reduction code drops the updates on the CPU (y = data); the GPU refuses it."""
import json
import os
import struct
import subprocess
import tempfile

import numpy as np

KINDS = {"ScatterNd": 0, "ScatterElements": 1}
REDUCTIONS = {None: -1, "add": 0, "sub": 1, "mul": 2}


def geometry(kind, out_shape, idx_shape, upd_shape, axis=0):
    """(N, D, S, R, strides) as GeometryScatter.cpp computes them"""
    out_shape = tuple(int(v) for v in out_shape)
    strides = [int(np.prod(out_shape[k + 1:], dtype=np.int64)) for k in range(len(out_shape))]
    if kind == "ScatterNd":
        d = int(idx_shape[-1])
        n = int(np.prod(idx_shape[:-1], dtype=np.int64))
        s = int(np.prod(upd_shape[d:], dtype=np.int64))
        r = int(np.prod(out_shape[d:], dtype=np.int64))
        return n, d, s, r, strides[:d]
    return int(np.prod(idx_shape, dtype=np.int64)), len(out_shape), 1, 1, strides


def destinations(kind, out_shape, indices, axis=0):
    """(dst_i, ok_i) for every update: the exact destination, and whether every term c * stride of it lies in int32"""
    indices = np.asarray(indices, np.int64)
    if kind == "ScatterNd":
        n, d, _, _, strides = geometry(kind, out_shape, indices.shape, (), axis)
        terms = indices.reshape(n, d) * np.array(strides, np.int64)
        return terms.sum(1), np.all((terms >= -2 ** 31) & (terms < 2 ** 31), 1)
    rank = len(out_shape)
    if axis < 0:
        axis += rank
    strides = geometry(kind, out_shape, indices.shape, (), axis)[4]
    coords = np.indices(indices.shape, dtype=np.int64).reshape(rank, -1)
    coords[axis] = indices.reshape(-1)
    terms = coords * np.array(strides, np.int64)[:, None]
    return terms.sum(0), np.all((terms >= -2 ** 31) & (terms < 2 ** 31), 0)


def scatter(kind, out_shape, indices, updates, data=None, reduction=None, axis=0):
    """the sequential loop: y = data (zeros when None), then every update in index order.  reduction: None, 'add', 'sub', 'mul'"""
    updates = np.asarray(updates)
    dtype = updates.dtype if data is None else np.asarray(data).dtype
    y = np.zeros(int(np.prod(out_shape)), dtype) if data is None else np.asarray(data).reshape(-1).copy()
    n, d, s, r, _ = geometry(kind, out_shape, np.asarray(indices).shape, updates.shape, axis)
    if n == 0 or s == 0:
        return y.reshape(out_shape)
    dst, ok = destinations(kind, out_shape, indices, axis)
    upd = updates.reshape(-1)[:n * s].reshape(n, s).astype(dtype)
    ok = ok & (dst >= 0) & (dst < y.size)
    if reduction is None:
        for i in np.nonzero(ok)[0]:
            y[dst[i]:dst[i] + s] = upd[i]
        return y.reshape(out_shape)
    assert dtype == np.float32, "a reduction is fp32 arithmetic"
    fn = {"add": np.add, "sub": np.subtract, "mul": np.multiply}[reduction]
    keep = np.nonzero(ok)[0]
    order = keep[np.argsort(dst[keep], kind="stable")]
    if order.size == 0:
        return y.reshape(out_shape)
    ds = dst[order]
    starts = np.r_[0, np.nonzero(np.diff(ds))[0] + 1, ds.size]
    for a, b in zip(starts[:-1], starts[1:]):
        o = ds[a]
        seq = np.concatenate([y[o:o + s][None, :], upd[order[a:b]]], 0)
        y[o:o + s] = fn.accumulate(seq, axis=0, dtype=np.float32)[-1]     # sequential, one rounding per step
    return y.reshape(out_shape)


def canonical(y):
    """y's bits with every NaN made 0x7fc00000: an ADD / SUB / MUL keeps a NaN a NaN but not its payload"""
    y = np.asarray(y)
    if y.dtype != np.float32:
        return y.view(np.uint32) if y.dtype.itemsize == 4 else y
    b = y.view(np.uint32).copy()
    b[np.isnan(y)] = 0x7fc00000
    return b


# ---- the live reference: oracle/_ref/refdump_scatter (oracle/refdump_scatter.cpp over oracle/_ref/libMNN.so), built by build()
HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(HERE, "_ref")
REFDUMP_SCATTER = os.path.join(REF_DIR, "refdump_scatter")
PILLARS = os.path.join(REF_DIR, "pillars_f32.mnn")
GNN = os.path.join(REF_DIR, "gnn_f32.mnn")
PILLARS_SEED, GNN_SEED = 51, 52


def have_refdump():
    return os.path.exists(REFDUMP_SCATTER)


def build_refdump():
    """compile oracle/refdump_scatter.cpp against the reference build of oracle/build_ref.py and write the PointPillars- and
    GraphSAGE-style fixtures with it"""
    from oracle import build_ref as B
    src = os.path.join(HERE, "refdump_scatter.cpp")
    lib = os.path.join(REF_DIR, "libMNN.so")
    fresh = have_refdump() and all(os.path.getmtime(REFDUMP_SCATTER) > os.path.getmtime(d) for d in (src, lib))
    if not fresh:
        cmd = ["g++", "-O2", "-std=gnu++11", "-w", "-o", REFDUMP_SCATTER, src] + ["-I" + os.path.join(B.REF, i) for i in B.INCLUDES] + \
              ["-L" + REF_DIR, "-lMNN", "-Wl,-rpath,$ORIGIN", "-pthread", "-ldl"]
        subprocess.check_call(cmd)
    for path, cmd, seed in ((PILLARS, "pillars", PILLARS_SEED), (GNN, "gnn", GNN_SEED)):
        if not fresh or not os.path.exists(path):
            _run([cmd, path, seed])


def _run(args, plugin=None, env_more=None):
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = REF_DIR + ":" + env.get("LD_LIBRARY_PATH", "")
    env.pop("REFDUMP_PLUGIN", None)
    if plugin:
        env["REFDUMP_PLUGIN"] = plugin
    env.update(env_more or {})
    return subprocess.run([REFDUMP_SCATTER] + [str(a) for a in args], env=env, capture_output=True, text=True, timeout=900,
                          check=True)


def ref_op(kind, out_shape, indices, updates, data=None, reduction=None, axis=None, torch_style=False, more=None, plugin=None):
    """outputs of one reference op through the Express executor on MNN_FORWARD_CPU.  kind: 'ScatterNd' or 'ScatterElements'
    (whose out_shape is data's); reduction: None, 'add', 'sub', 'mul' or a BinaryOpOperation code; axis: ScatterElements' constant
    fourth input (None: no fourth input); torch_style: a BinaryOp parameter whose opType is left at its default (ADD).  more:
    further (indices, updates[, data]) tuples run through the same executor (all outputs returned, stacked).  plugin: run on
    MNN_FORWARD_CUDA with that plugin, and (ys, the plugin's stats) returned"""
    first = (indices, updates) + ((data,) if data is not None else ())
    sets = [first] + [tuple(m) for m in (more or [])]
    arrs = [[np.ascontiguousarray(a) for a in s] for s in sets]
    if kind == "ScatterElements":              # the op's input order: data, indices, updates
        arrs = [[s[2], s[0], s[1]] for s in arrs]
    red = reduction if isinstance(reduction, int) else REDUCTIONS[reduction]
    hdr = struct.pack("<6i", KINDS[kind], red, int(torch_style), 0 if axis is None else 1, 0 if axis is None else int(axis),
                      len(out_shape)) + struct.pack(f"<{len(out_shape)}i", *out_shape)
    hdr += struct.pack("<i", len(arrs[0]))
    for a in arrs[0]:
        hdr += struct.pack(f"<2i{a.ndim}i", 1 if a.dtype == np.int32 else 0, a.ndim, *a.shape)
    body = b"".join(a.astype(np.int32 if a.dtype == np.int32 else np.float32).tobytes() for s in arrs for a in s)
    with tempfile.TemporaryDirectory() as d:
        req, out = os.path.join(d, "req"), os.path.join(d, "out")
        open(req, "wb").write(hdr + struct.pack("<i", len(arrs)) + body)
        r = _run(["op", req, out], plugin)
        raw = open(out, "rb").read()
    dtype, rank = struct.unpack("<2i", raw[:8])
    dims = struct.unpack(f"<{rank}i", raw[8:8 + 4 * rank])
    ys = np.frombuffer(raw[8 + 4 * rank:], np.int32 if dtype == 1 else np.float32).reshape((len(arrs),) + dims).copy()
    ys = ys[0] if more is None else ys
    if plugin is None:
        return ys
    stats = [json.loads(line) for line in r.stdout.splitlines() if line.startswith('{"plugin_')]
    return ys, (stats[-1] if stats else None)


def run_model(model, batch, seed, outdir, plugin=None, repeats=None):
    """`refdump_scatter run`: every command's fp32 outputs under outdir (index.txt); returns (records, plugin stats, process)"""
    os.makedirs(outdir, exist_ok=True)
    r = _run(["run", model, batch, seed, outdir], plugin, {"REFDUMP_RUN_REPEATS": str(repeats)} if repeats else None)
    recs = []
    for line in open(os.path.join(outdir, "index.txt")):
        f, name, typ = line.rstrip("\n").split("|")[:3]
        recs.append((f, name, typ.strip()))
    stats = [json.loads(line) for line in r.stdout.splitlines() if line.startswith('{"plugin_')]
    return recs, (stats[-1] if stats else None), r
