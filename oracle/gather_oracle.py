"""Restatement of the reference CPU's Gather, GatherV2, GatherND and GatherElements, and of its int32 <-> fp32 Cast.

The CPU runs the gathers as the While loops GeometryGather.cpp builds for Compiler_Loop: one region copy per index (tuple),
whose source offset is the index times the slice stride plus the sum of the other coordinates' strides (CPURaster.cpp's loop
for a single UnaryOp command).  When that offset lies outside the params the slice is zero-filled; a negative index is not
wrapped.  An index past its axis whose offset still lies inside the params (possible when outside > 1, or for one component
of a GatherND tuple) makes the CPU read another row, or past the end of the params; the GPU kernels zero-fill every index
outside [0, the axis length) instead.  The restatements here zero-fill by the kernels' rule, and the tests compare them with
the CPU only where the CPU's result is defined by the same rule (index in range, or offset outside the params).

GatherND over batch dims: buildGatherND strides each tuple over the params' dims batch_dims .. batch_dims + d and adds no
offset for the batch, so every batch reads from the first batch of params (out[b, j] = params[0][tuple]).  Pinned on the live
reference by tests/test_gather_cpu.py.

Axis: Gather / GatherV2 take the op's Axis when it has one, else a third input, else 0; GatherND's batch dims are the op's
Axis; GatherElements' axis is a third input, else 0 (GeometryGather.cpp:15-29, 420-440)."""
import json
import os
import struct
import subprocess
import tempfile

import numpy as np

KINDS = {"Gather": 0, "GatherV2": 1, "GatherND": 2, "GatherElements": 3, "Cast": 4, "MatMul": 5, "BatchMatMul": 6}


def gather(params, indices, axis=0):
    """Gather / GatherV2: out = params[:axis] + indices.shape + params[axis+1:]; indices outside [0, len) give zeros"""
    params = np.asarray(params)
    indices = np.asarray(indices, np.int32)
    if axis < 0:
        axis += params.ndim
    n = params.shape[axis]
    ok = (indices >= 0) & (indices < n)
    out = np.take(params, np.where(ok, indices, 0), axis=axis)
    mask = ok.reshape((1,) * axis + indices.shape + (1,) * (params.ndim - axis - 1))
    return np.where(mask, out, np.zeros((), params.dtype)).astype(params.dtype)


def gather_nd(params, indices, batch_dims=0):
    """GatherND as the CPU computes it: each tuple indexes the params' dims batch_dims .. batch_dims + d from the start of params
    (no batch offset); a tuple with a component outside its dim gives a zero slice"""
    params = np.asarray(params)
    indices = np.asarray(indices, np.int32)
    d = indices.shape[-1]
    sub = params.reshape((-1,) + params.shape[batch_dims:])[0]            # the first batch
    tup = indices.reshape(-1, d)
    ok = np.all((tup >= 0) & (tup < np.array(sub.shape[:d])), axis=1)
    safe = np.where(ok[:, None], tup, 0)
    out = sub[tuple(safe[:, k] for k in range(d))]                       # [N] + sub.shape[d:]
    out = np.where(ok.reshape((-1,) + (1,) * (out.ndim - 1)), out, np.zeros((), params.dtype))
    return out.reshape(indices.shape[:-1] + params.shape[batch_dims + d:]).astype(params.dtype)


def gather_elements(params, indices, axis=0):
    """GatherElements: out[i] = params[i with i[axis] = indices[i]], zero for an index outside [0, params.shape[axis])"""
    params = np.asarray(params)
    indices = np.asarray(indices, np.int32)
    if axis < 0:
        axis += params.ndim
    ok = (indices >= 0) & (indices < params.shape[axis])
    sub = params[tuple(slice(0, s) for s in indices.shape[:axis]) + (slice(None),) +
                 tuple(slice(0, s) for s in indices.shape[axis + 1:])]
    out = np.take_along_axis(sub, np.where(ok, indices, 0).astype(np.int64), axis=axis)
    return np.where(ok, out, np.zeros((), params.dtype)).astype(params.dtype)


def cast_i32_f32(x):
    return np.asarray(x, np.int32).astype(np.float32)


def cast_f32_i32(x):
    """truncation; NaN and values outside the int32 range give INT32_MIN (x86's cvttss2si)"""
    x = np.asarray(x, np.float32)
    ok = (x >= np.float32(-2147483648.0)) & (x < np.float32(2147483648.0))
    return np.where(ok, np.trunc(np.where(ok, x, 0)).astype(np.int64), -2147483648).astype(np.int32)


def cpu_defined(kind, params, indices, axis=0):
    """True where the CPU's zero-fill rule is this module's: every index in range, or its source offset outside the params"""
    params = np.asarray(params)
    indices = np.asarray(indices, np.int64)
    if kind in ("Gather", "GatherV2"):
        if axis < 0:
            axis += params.ndim
        inside = int(np.prod(params.shape[axis + 1:], dtype=np.int64))
        off = indices * inside
        return bool(np.all(((indices >= 0) & (indices < params.shape[axis])) | (off < 0) | (off >= params.size)))
    if kind == "GatherND":
        b = axis
        d = indices.shape[-1]
        dims = np.array(params.shape[b:b + d])
        strides = np.array([int(np.prod(params.shape[b + k + 1:], dtype=np.int64)) for k in range(d)])
        tup = indices.reshape(-1, d)
        off = (tup * strides).sum(1)
        return bool(np.all(np.all((tup >= 0) & (tup < dims), 1) | (off < 0) | (off >= params.size)))
    if axis < 0:
        axis += params.ndim
    strides = [int(np.prod(params.shape[k + 1:], dtype=np.int64)) for k in range(params.ndim)]
    coords = np.indices(indices.shape, dtype=np.int64)
    off = sum((indices if k == axis else coords[k]) * strides[k] for k in range(params.ndim))
    return bool(np.all(((indices >= 0) & (indices < params.shape[axis])) | (off < 0) | (off >= params.size)))


# ---- the live reference: oracle/_ref/refdump_gather (oracle/refdump_gather.cpp over oracle/_ref/libMNN.so), built by build()
HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(HERE, "_ref")
REFDUMP_GATHER = os.path.join(REF_DIR, "refdump_gather")
BERT = os.path.join(REF_DIR, "bert_f32.mnn")
VIT = os.path.join(REF_DIR, "vit_f32.mnn")
BERT_SEED, VIT_SEED = 41, 42


def have_refdump():
    return os.path.exists(REFDUMP_GATHER)


def build_refdump():
    """compile oracle/refdump_gather.cpp against the reference build of oracle/build_ref.py and write the BERT- and ViT-style
    fixtures with it"""
    from oracle import build_ref as B
    src = os.path.join(HERE, "refdump_gather.cpp")
    lib = os.path.join(REF_DIR, "libMNN.so")
    fresh = have_refdump() and all(os.path.getmtime(REFDUMP_GATHER) > os.path.getmtime(d) for d in (src, lib))
    if not fresh:
        cmd = ["g++", "-O2", "-std=gnu++11", "-w", "-o", REFDUMP_GATHER, src] + ["-I" + os.path.join(B.REF, i) for i in B.INCLUDES] + \
              ["-L" + REF_DIR, "-lMNN", "-Wl,-rpath,$ORIGIN", "-pthread", "-ldl"]
        subprocess.check_call(cmd)
    for path, cmd, seed in ((BERT, "bert", BERT_SEED), (VIT, "vit", VIT_SEED)):
        if not fresh or not os.path.exists(path):
            _run([cmd, path, seed])


def _run(args, plugin=None, env_more=None):
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = REF_DIR + ":" + env.get("LD_LIBRARY_PATH", "")
    env.pop("REFDUMP_PLUGIN", None)
    if plugin:
        env["REFDUMP_PLUGIN"] = plugin
    env.update(env_more or {})
    return subprocess.run([REFDUMP_GATHER] + [str(a) for a in args], env=env, capture_output=True, text=True, timeout=900,
                          check=True)


def ref_op(kind, inputs, axis=None, axis_input=False, ta=False, tb=False, cast_to=None, more=None, plugin=None):
    """outputs of one reference op on MNN_FORWARD_CPU.  kind: a KINDS name; inputs: arrays (float32 or int32); axis: the op's
    Axis parameter (or, with axis_input, a constant int32 third input); ta / tb: (Batch)MatMul's transposes; cast_to: 'float32' or
    'int32'.  more: further input lists run through the same executor (all outputs returned, stacked).  plugin: run on
    MNN_FORWARD_CUDA with that plugin, and (ys, the plugin's stats) returned"""
    sets = [inputs] + list(more or [])
    arrs = [[np.ascontiguousarray(a) for a in s] for s in sets]
    mode = 0 if axis is None else (2 if axis_input else 1)
    hdr = struct.pack("<7i", KINDS[kind], mode, 0 if axis is None else int(axis), int(ta), int(tb),
                      1 if cast_to == "int32" else 0, len(arrs[0]))
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
    """`refdump_gather run`: every command's fp32 outputs under outdir (index.txt); returns (records, plugin stats, process)"""
    os.makedirs(outdir, exist_ok=True)
    r = _run(["run", model, batch, seed, outdir], plugin, {"REFDUMP_RUN_REPEATS": str(repeats)} if repeats else None)
    recs = []
    for line in open(os.path.join(outdir, "index.txt")):
        f, name, typ = line.rstrip("\n").split("|")[:3]
        recs.append((f, name, typ.strip()))
    stats = [json.loads(line) for line in r.stdout.splitlines() if line.startswith('{"plugin_')]
    return recs, (stats[-1] if stats else None), r
