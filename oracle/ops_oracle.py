"""The fp32 neighbour ops one op at a time: the cases the plugin tests run on the reference CPU and on the plugin, their seeded
inputs, and float64 restatements of the ops whose CPU and GPU results are compared by a bound rather than bit for bit.

run() writes every case into one request for oracle/_ref/refdump_ops (oracle/refdump_ops.cpp over oracle/_ref/libMNN.so), which
builds each op with the reference's Express API and runs it on MNN_FORWARD_CPU, or on the plugin when given one, in a single
process.  A case is a dict: kind (KIND), ip / fp (the op's int and float parameters, see refdump_ops.cpp), inputs
[(dtype, format)], runs [[array per input]] (several runs: one executor, new values, and a resize when the shapes change)."""
import os
import struct
import subprocess
import tempfile

import numpy as np

F = np.float32
KIND = {k: i for i, k in enumerate(
    ["binary", "eltwise", "relu", "unary", "pool", "reduce", "softmax", "argmax", "scale", "transpose", "concat",
     "strided_slice", "slice", "pad", "tile", "broadcast_to", "reshape", "convert"])}
BINARY = {"ADD": 0, "SUB": 1, "MUL": 2, "POW": 6, "REALDIV": 7, "MINIMUM": 8, "MAXIMUM": 9, "FLOORDIV": 13,
          "SquaredDifference": 14}
UNARY = {"ABS": 0, "NEG": 1, "FLOOR": 2, "SQUARE": 4, "SQRT": 5, "RSQRT": 6, "EXP": 7, "LOG": 8, "SIN": 9, "RECIPROCAL": 15,
         "ERF": 25, "SIGMOID": 29, "TANH": 30, "HARDSWISH": 31, "GELU": 32, "GELU_STANDARD": 33, "SILU": 34}
UNARY_EXACT = ("ABS", "NEG", "SQUARE", "SQRT", "RSQRT", "RECIPROCAL", "HARDSWISH")
UNARY_TRANSCENDENTAL = ("EXP", "LOG", "SIGMOID", "TANH", "GELU", "GELU_STANDARD", "SILU")
ELTWISE = {"PROD": 0, "SUM": 1, "MAXIMUM": 2, "SUB": 3}
REDUCE = {"SUM": 0, "MEAN": 3, "MAXIMUM": 4, "MINIMUM": 5, "PROD": 6}
POOL_MAX, POOL_AVG = 0, 1
PAD_CAFFE, PAD_VALID, PAD_SAME = 0, 1, 2
NCHW, NHWC = 0, 1
FLT_MAX = np.finfo(F).max
SPECIALS = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, FLT_MAX, -FLT_MAX, 1e-40, -1e-40, 3e-42, -3e-42], F)


# ---- the live reference: oracle/_ref/refdump_ops, built by build()
HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(HERE, "_ref")
REFDUMP_OPS = os.path.join(REF_DIR, "refdump_ops")


def have_refdump():
    return os.path.exists(REFDUMP_OPS)


def build_refdump():
    """compile oracle/refdump_ops.cpp against the reference build of oracle/build_ref.py (where the reference sources are)"""
    from oracle import build_ref as B
    src = os.path.join(HERE, "refdump_ops.cpp")
    lib = os.path.join(REF_DIR, "libMNN.so")
    if have_refdump() and all(os.path.getmtime(REFDUMP_OPS) > os.path.getmtime(d) for d in (src, lib)):
        return
    cmd = ["g++", "-O2", "-std=gnu++11", "-w", "-o", REFDUMP_OPS, src] + ["-I" + os.path.join(B.REF, i) for i in B.INCLUDES] + \
          ["-L" + REF_DIR, "-lMNN", "-Wl,-rpath,$ORIGIN", "-pthread", "-ldl"]
    subprocess.check_call(cmd)


def case(kind, runs, ip=(), fp=(), fmt=None):
    """a case of `kind` whose runs are lists of input arrays (float32 or int32); fmt: the inputs' formats (default NCHW)"""
    runs = [[np.ascontiguousarray(a) for a in r] for r in runs]
    fmt = fmt or [NCHW] * len(runs[0])
    inputs = [(1 if a.dtype == np.int32 else 0, f) for a, f in zip(runs[0], fmt)]
    return {"kind": kind, "ip": [int(v) for v in ip], "fp": [float(v) for v in fp], "inputs": inputs, "runs": runs}


def _request(cases):
    out = [struct.pack("<i", len(cases))]
    for c in cases:
        out.append(struct.pack("<2i", KIND[c["kind"]], len(c["ip"])) + struct.pack(f"<{len(c['ip'])}i", *c["ip"]))
        out.append(struct.pack("<i", len(c["fp"])) + np.asarray(c["fp"], F).tobytes())
        out.append(struct.pack("<i", len(c["inputs"])) + b"".join(struct.pack("<2i", t, f) for t, f in c["inputs"]))
        out.append(struct.pack("<i", len(c["runs"])))
        for r in c["runs"]:
            for a in r:
                assert a.dtype in (np.float32, np.int32), a.dtype
                out.append(struct.pack(f"<{a.ndim + 1}i", a.ndim, *a.shape) + a.tobytes())
    return b"".join(out)


def run(cases, plugin=None, env=None):
    """run every case in one refdump_ops process: a list of {"ok", "created", "declined", "ys"} (ys: one array per run).
    plugin: the plugin's .so, run on MNN_FORWARD_CUDA; env: more environment variables"""
    e = dict(os.environ)
    e["LD_LIBRARY_PATH"] = REF_DIR + ":" + e.get("LD_LIBRARY_PATH", "")
    e.pop("REFDUMP_PLUGIN", None)
    if plugin:
        e["REFDUMP_PLUGIN"] = plugin
    e.update(env or {})
    with tempfile.TemporaryDirectory() as d:
        req, out = os.path.join(d, "req"), os.path.join(d, "out")
        with open(req, "wb") as f:
            f.write(_request(cases))
        p = subprocess.run([REFDUMP_OPS, req, out], env=e, capture_output=True, text=True, timeout=1200)
        if p.returncode != 0:
            raise RuntimeError(f"refdump_ops exited {p.returncode}: {p.stderr[-2000:]}")
        raw = open(out, "rb").read()
    res, at = [], 0

    def words(k):
        nonlocal at
        v = struct.unpack_from(f"<{k}i", raw, at)
        at += 4 * k
        return v
    for _ in cases:
        ok, created, declined, runs = words(4)
        ys = []
        for _ in range(runs):
            t, nd = words(2)
            dims = words(nd)
            n = int(np.prod(dims)) if nd else 1
            ys.append(np.frombuffer(raw, np.int32 if t else F, n, at).reshape(dims).copy())
            at += 4 * n
        res.append({"ok": bool(ok), "created": created, "declined": declined, "ys": ys})
    return res


# ---- inputs
def rng(seed):
    return np.random.default_rng(seed)


def uniform(seed, shape, lo=-4.0, hi=4.0):
    return rng(seed).uniform(lo, hi, shape).astype(F)


def salted(seed, shape, lo=-4.0, hi=4.0):
    """uniform values with every special value (signed zeros, infinities, NaN, +-FLT_MAX, denormals) at seeded positions, about
    one element in four, and each special value at least once"""
    x = uniform(seed, shape, lo, hi).reshape(-1)
    r = rng(seed + 1)
    pos = r.permutation(x.size)[: max(x.size // 4, min(x.size, SPECIALS.size))]
    x[pos] = SPECIALS[np.arange(pos.size) % SPECIALS.size]
    return x.reshape(shape)


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def same_bits(a, b):
    """equal shapes and bits, every NaN counted equal to every NaN"""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.dtype != F:
        return np.array_equal(a, b)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(bits(a)[~na], bits(b)[~nb])


# ---- float64 restatements (bounds only)
def unary64(op, x):
    x = np.asarray(x, np.float64)
    with np.errstate(all="ignore"):
        if op == "EXP":
            return np.exp(x)
        if op == "LOG":
            return np.log(x)
        if op == "TANH":
            return np.tanh(x)
        if op == "SIGMOID":
            return np.where(x >= 0, 1 / (1 + np.exp(-np.abs(x))), np.exp(-np.abs(x)) / (1 + np.exp(-np.abs(x))))
        if op == "SILU":
            return x * unary64("SIGMOID", x)
        if op == "GELU":       # the tanh form: 0.5 x (1 + tanh(sqrt(2 / pi) (x + 0.044715 x^3)))
            z = np.sqrt(2 / np.pi) * (x + 0.044715 * x ** 3)
            return x * unary64("SIGMOID", 2 * z)
        if op == "GELU_STANDARD":
            from scipy.special import erfc
            return 0.5 * x * erfc(-x / np.sqrt(2))
    raise ValueError(op)


def ulp32(y):
    """the float32 ulp at |y| (float64), 2^-149 for zero and denormals"""
    y = np.abs(np.asarray(y, np.float64))
    e = np.floor(np.log2(np.maximum(y, np.finfo(F).tiny)))
    return np.exp2(np.maximum(e, -126) - 23)


def ulp_error(y, y64):
    """|y - y64| in float32 ulps of y64 (both infinite with one sign, or y64 beyond FLT_MAX and y infinite: 0)"""
    y, y64 = np.asarray(y, np.float64), np.asarray(y64, np.float64)
    with np.errstate(all="ignore"):
        d = np.abs(y - y64) / ulp32(np.clip(y64, -FLT_MAX, FLT_MAX))
    d[(y == y64)] = 0
    big = np.abs(y64) > FLT_MAX * (1 + 2.0 ** -24)
    d[big & np.isinf(y) & (np.sign(y) == np.sign(y64))] = 0
    return d


def softmax64(x, axis):
    x = np.asarray(x, np.float64)
    e = np.exp(x - x.max(axis=axis, keepdims=True))
    return e / e.sum(axis=axis, keepdims=True)


def reduce64(x, op, axes, keep):
    x = np.asarray(x, np.float64)
    f = {"SUM": np.sum, "MEAN": np.mean, "MAXIMUM": np.max, "MINIMUM": np.min, "PROD": np.prod}[op]
    return f(x, axis=tuple(axes), keepdims=bool(keep))


def sum_bound(x, axes, op):
    """the rounding bound of any order of float32 summation over `axes`: (n - 1) u sum|x| (Higham 2002, eq. 4.4), u = 2^-24;
    MEAN adds the division's rounding; PROD: (n - 1) u |prod| relative"""
    n = int(np.prod([x.shape[a] for a in axes]))
    u = 2.0 ** -24
    if op == "PROD":
        return 1.01 * n * u * np.abs(reduce64(x, "PROD", axes, True))
    s = np.abs(np.asarray(x, np.float64)).sum(axis=tuple(axes), keepdims=True)
    if op == "MEAN":
        return 1.01 * (n * u * s / n + u * s / n)
    return 1.01 * (n - 1) * u * s


def softmax_bound(x, axis):
    """|y - y64| bound of a float32 softmax with expf (2 ulp): each exp(x - max) is off by 4u + |x - max| u relative (the
    subtraction rounds, the exponential amplifies it), the sum of n such terms by (n + 4 + max|x - max|) u, the division or
    reciprocal-multiply by 2u; u = 2^-24.  Twice that, plus one subnormal ulp"""
    x = np.asarray(x, np.float64)
    d = x.max(axis=axis, keepdims=True) - x
    n = x.shape[axis]
    u = 2.0 ** -24
    rel = u * (4 + d + n + 4 + d.max(axis=axis, keepdims=True) + 2)
    return 2 * rel * softmax64(x, axis) + 2.0 ** -149


# ---- the cases
def _log_uniform(seed, n, lo, hi, signed=False):
    r = rng(seed)
    v = np.exp(r.uniform(np.log(lo), np.log(hi), n))
    if signed:
        v *= r.choice([-1.0, 1.0], n)
    return v.astype(F)


UNARY_DOMAIN = {   # inputs of each UnaryOp: its whole useful range, saturation included
    "ABS": (-1e6, 1e6), "NEG": (-1e6, 1e6), "SQUARE": (-1e15, 1e15), "SQRT": "pos", "RSQRT": "pos", "RECIPROCAL": "signed",
    "HARDSWISH": (-8, 8), "EXP": (-104, 89), "LOG": "pos", "SIGMOID": (-110, 100), "TANH": (-100, 100),
    "GELU": (-100, 100), "GELU_STANDARD": (-100, 100), "SILU": (-110, 100)}


def unary_input(op, seed, n=65539):
    d = UNARY_DOMAIN[op]
    if d == "pos":
        return _log_uniform(seed, n, 1e-38, 1e38)
    if d == "signed":
        return _log_uniform(seed, n, 1e-37, 1e37, signed=True)
    x = uniform(seed, n, *d)
    x[: n // 4] = uniform(seed + 1, n // 4, -12, 12)   # the bends of the curves, densely
    return x


def _binary_pair(seed, op, shape_a, shape_b):
    a, b = uniform(seed, shape_a), uniform(seed + 1, shape_b)
    if op == "REALDIV":
        b = (np.sign(b) * (np.abs(b) + 0.25)).astype(F)
    if a.shape == b.shape and a.size > 7:
        a.reshape(-1)[: a.size // 7] = b.reshape(-1)[: a.size // 7]   # ties and exact zeros
    return a, b


BIG = (1 << 20) + 5


def binary_cases():
    out = {}
    for k, op in enumerate(("ADD", "SUB", "MUL", "REALDIV", "MINIMUM", "MAXIMUM", "SquaredDifference")):
        s = 100 * k
        for n in (1, 3, 4099):
            for form in ("equal", "left1", "right1"):
                for act in (0, 1):
                    sa, sb = ((1,) if form == "left1" else (n,)), ((1,) if form == "right1" else (n,))
                    a, b = _binary_pair(s + n + len(form) + act, op, sa, sb)
                    out[f"binary_{op}_{form}_{n}_act{act}"] = case("binary", [[a, b]], ip=[BINARY[op], act])
        a, b = _binary_pair(s + 1, op, (BIG,), (BIG,))
        out[f"binary_{op}_equal_big_act1"] = case("binary", [[a, b]], ip=[BINARY[op], 1])
        a, b = _binary_pair(s + 2, op, (1,), (1,))
        out[f"binary_{op}_both1"] = case("binary", [[a, b]], ip=[BINARY[op], 0])
        a, b = _binary_pair(s + 3, op, (2, 5, 6, 7), (1, 5, 1, 1))
        out[f"binary_{op}_bcast_1c11"] = case("binary", [[a, b]], ip=[BINARY[op], k % 2])
        a, b = _binary_pair(s + 4, op, (5, 1, 1), (2, 5, 6, 7))
        out[f"binary_{op}_bcast_c11_left"] = case("binary", [[a, b]], ip=[BINARY[op], (k + 1) % 2])
        a, b = salted(s + 5, 4099), salted(s + 6, 4099)
        out[f"binary_{op}_special_act0"] = case("binary", [[a, b]], ip=[BINARY[op], 0])
        out[f"binary_{op}_special_act1"] = case("binary", [[a, b]], ip=[BINARY[op], 1])
    a1, b1 = uniform(7, (2, 3, 5, 7)), uniform(8, (2, 3, 5, 7))
    a2, b2 = uniform(9, (2, 3, 5, 7)), uniform(10, (2, 3, 5, 7))
    a3, b3 = uniform(11, (3, 4, 9, 2)), uniform(12, (3, 4, 9, 2))
    out["binary_MAXIMUM_rerun_resize"] = case("binary", [[a1, b1], [a2, b2], [a1, b2], [a3, b3]], ip=[BINARY["MAXIMUM"], 1])
    return out


def eltwise_cases():
    out = {}
    shape = (2, 7, 9, 13)
    for k, t in enumerate(ELTWISE):
        for m in (2, 3, 4):
            xs = [uniform(1000 + 10 * k + m + i, shape) for i in range(m)]
            if t == "PROD":
                xs = [(1 + x / 8).astype(F) for x in xs]
            out[f"eltwise_{t}_{m}"] = case("eltwise", [xs], ip=[ELTWISE[t]])
        out[f"eltwise_{t}_special"] = case("eltwise", [[salted(1100 + k + i, shape) for i in range(3)]], ip=[ELTWISE[t]])
    r = [[uniform(1200 + i + 3 * j, (2, 3, 5, 7) if j < 3 else (1, 4, 3, 5)) for i in range(3)] for j in range(4)]
    out["eltwise_SUB_rerun_resize"] = case("eltwise", r, ip=[ELTWISE["SUB"]])
    return out


def relu_cases():
    out = {}
    for slope in (0.0, 0.1):
        for n in (3, 4099, BIG - 2):
            out[f"relu_{slope}_{n}"] = case("relu", [[uniform(int(n + 10 * slope), (n,))]], fp=[slope])
        out[f"relu_{slope}_special"] = case("relu", [[salted(77, (4099,))]], fp=[slope])
    r = [[uniform(1300 + j, (2, 3, 5, 7) if j < 3 else (3, 2, 7, 3))] for j in range(4)]
    out["relu_0.1_rerun_resize"] = case("relu", r, fp=[0.1])
    return out


def unary_cases():
    out = {}
    for k, op in enumerate(UNARY_EXACT + UNARY_TRANSCENDENTAL):
        out[f"unary_{op}"] = case("unary", [[unary_input(op, 2000 + k)]], ip=[UNARY[op]])
        out[f"unary_{op}_special"] = case("unary", [[salted(2100 + k, (4099,))]], ip=[UNARY[op]])
    r = [[uniform(2200 + j, (2, 3, 5, 7) if j < 3 else (5, 3, 3, 3), -10, 10)] for j in range(4)]
    out["unary_TANH_rerun_resize"] = case("unary", r, ip=[UNARY["TANH"]])
    return out


def _pool(kind, k, s, pad_type=PAD_CAFFE, pad=(0, 0), glob=False, ceil=False, count=0, pads=()):
    return [kind, k[0], k[1], s[0], s[1], pad_type, pad[0], pad[1], int(glob), int(ceil), count, len(pads)] + list(pads)


POOL_FORMS = {   # name: (Pool parameters but the type, input shape)
    "pads_k3s2p1": (dict(k=(3, 3), s=(2, 2), pad=(1, 1)), (2, 3, 13, 11)),
    "same_k3s2": (dict(k=(3, 3), s=(2, 2), pad_type=PAD_SAME), (2, 3, 14, 11)),
    "valid_k3s2": (dict(k=(3, 3), s=(2, 2), pad_type=PAD_VALID), (2, 3, 13, 12)),
    "caffe_pads4": (dict(k=(3, 3), s=(2, 2), pads=(1, 2, 1, 2)), (2, 3, 12, 13)),
    "global": (dict(k=(1, 1), s=(1, 1), glob=True), (2, 5, 9, 7)),
    "ceil_k3s2p1": (dict(k=(3, 3), s=(2, 2), pad=(1, 1), ceil=True), (2, 3, 12, 10)),
    "count_incl": (dict(k=(3, 3), s=(2, 2), pad=(1, 1), count=1), (2, 3, 13, 11)),
    "count_excl": (dict(k=(3, 3), s=(2, 2), pad=(1, 1), count=2), (2, 3, 13, 11)),
    "in_padding": (dict(k=(2, 2), s=(1, 1), pad=(2, 2)), (1, 3, 5, 6)),
    "nonsquare": (dict(k=(3, 2), s=(2, 1), pad=(1, 0)), (2, 4, 11, 9)),
}


def pool_cases():
    out = {}
    for j, (name, (kw, shape)) in enumerate(POOL_FORMS.items()):
        for kind, tag in ((POOL_MAX, "max"), (POOL_AVG, "avg")):
            out[f"pool_{tag}_{name}"] = case("pool", [[uniform(3000 + 2 * j + kind, shape)]], ip=_pool(kind, **kw))
    for kind, tag in ((POOL_MAX, "max"), (POOL_AVG, "avg")):
        out[f"pool_{tag}_special"] = case("pool", [[salted(3100 + kind, (2, 3, 13, 11))]], ip=_pool(kind, (3, 3), (2, 2), pad=(1, 1)))
        r = [[uniform(3200 + j, (2, 3, 13, 11) if j < 3 else (1, 3, 8, 17))] for j in range(4)]
        out[f"pool_{tag}_rerun_resize"] = case("pool", r, ip=_pool(kind, (3, 3), (2, 2), pad_type=PAD_SAME))
    return out


REDUCE_SHAPES = ((7, 33), (3, 5, 37), (2, 3, 4, 5))


def reduce_input(op, seed, shape):
    if op == "PROD":
        r = rng(seed)
        return (r.uniform(0.8, 1.25, shape) * r.choice([-1, 1], shape)).astype(F)
    return uniform(seed, shape)


def reduce_cases():
    out = {}
    for k, op in enumerate(REDUCE):
        for shape in REDUCE_SHAPES:
            nd = len(shape)
            axes_list = [(a,) for a in range(nd)] + [(0, nd - 1), tuple(range(nd))]
            for j, axes in enumerate(axes_list):
                keep = (j + k) % 2
                x = reduce_input(op, 4000 + 100 * k + 10 * nd + j, shape)
                out[f"reduce_{op}_{nd}d_axes{''.join(map(str, axes))}_keep{keep}"] = \
                    case("reduce", [[x]], ip=[REDUCE[op], keep] + list(axes))
    for op in ("MAXIMUM", "MINIMUM"):
        inf = -np.inf if op == "MAXIMUM" else np.inf
        x = uniform(4500, (6, 8))
        x[1], x[3, :5] = inf, inf   # a row of -inf (+inf for MIN), the masked-attention pattern
        out[f"reduce_{op}_inf_rows"] = case("reduce", [[x]], ip=[REDUCE[op], 0, 1])
        x = uniform(4501, (4, 100))
        x[0], x[2, 1:] = inf, inf
        out[f"reduce_{op}_inf_long_rows"] = case("reduce", [[x]], ip=[REDUCE[op], 0, 1])
        out[f"reduce_{op}_special_rows"] = case("reduce", [[salted(4502, (40, 8))]], ip=[REDUCE[op], 0, 1])
        out[f"reduce_{op}_special_cols"] = case("reduce", [[salted(4503, (3, 20, 5))]], ip=[REDUCE[op], 0, 1])
    out["reduce_SUM_special"] = case("reduce", [[salted(4504, (3, 20, 5))]], ip=[REDUCE["SUM"], 0, 1])
    r = [[uniform(4600 + j, (3, 5, 37) if j < 3 else (2, 9, 4))] for j in range(4)]
    out["reduce_MAXIMUM_rerun_resize"] = case("reduce", r, ip=[REDUCE["MAXIMUM"], 1, 1])
    return out


def softmax_cases():
    out = {}
    for shape in ((9, 37), (3, 5, 37), (2, 3, 5, 7), (2, 40, 3, 1)):
        for axis in range(len(shape)):
            out[f"softmax_{len(shape)}d_{'x'.join(map(str, shape))}_axis{axis}"] = \
                case("softmax", [[uniform(5000 + axis + 10 * len(shape), shape, -20, 20)]], ip=[axis])
    out["softmax_2d_axis_neg1"] = case("softmax", [[uniform(5100, (5, 1000), -20, 20)]], ip=[-1])
    out["softmax_2d_nhwc"] = case("softmax", [[uniform(5101, (6, 33), -20, 20)]], ip=[1], fmt=[NHWC])
    out["softmax_special"] = case("softmax", [[salted(5102, (16, 12))]], ip=[1])
    r = [[uniform(5200 + j, (3, 5, 37) if j < 3 else (4, 6, 11), -20, 20)] for j in range(4)]
    out["softmax_rerun_resize"] = case("softmax", r, ip=[1])
    return out


def argmax_cases():
    out = {}
    for shape in ((9, 37), (3, 5, 37), (2, 3, 5, 7)):
        for axis in list(range(len(shape))) + [-1]:
            for is_min in (0, 1):
                x = rng(6000 + axis + len(shape) + 10 * is_min).integers(-3, 4, shape).astype(F)   # heavy ties
                out[f"arg{'min' if is_min else 'max'}_{len(shape)}d_axis{axis}"] = \
                    case("argmax", [[x]], ip=[is_min, axis, 1, 0])
    out["argmax_special"] = case("argmax", [[salted(6100, (16, 12))]], ip=[0, 1, 1, 0])
    out["argmin_special"] = case("argmax", [[salted(6101, (16, 12))]], ip=[1, 1, 1, 0])
    r = [[rng(6200 + j).integers(-3, 4, (3, 5, 37) if j < 3 else (2, 7, 4)).astype(F)] for j in range(4)]
    out["argmax_rerun_resize"] = case("argmax", r, ip=[0, 1, 1, 0])
    return out


def scale_cases():
    out = {}
    c = 5
    s, b = uniform(7000, c), uniform(7001, c)
    for bias in (0, 1):
        out[f"scale_bias{bias}"] = case("scale", [[uniform(7002 + bias, (2, c, 7, 9))]], ip=[c, bias],
                                        fp=list(s) + (list(b) if bias else []))
    out["scale_special"] = case("scale", [[salted(7004, (2, c, 7, 9))]], ip=[c, 1], fp=list(s) + list(b))
    r = [[uniform(7100 + j, (2, c, 7, 9) if j < 3 else (3, c, 4, 13))] for j in range(4)]
    out["scale_rerun_resize"] = case("scale", r, ip=[c, 1], fp=list(s) + list(b))
    return out


def _ints(seed, shape):
    return rng(seed).integers(-2 ** 31, 2 ** 31 - 1, shape, dtype=np.int64).astype(np.int32)


def raster_cases():
    out = {}
    shape = (2, 3, 4, 5)
    for j, perm in enumerate(((0, 2, 3, 1), (0, 3, 1, 2), (3, 2, 1, 0), (1, 0, 3, 2), (2, 0, 3, 1), (0, 1, 3, 2))):
        out[f"transpose_{''.join(map(str, perm))}"] = case("transpose", [[uniform(8000 + j, shape)]], ip=perm)
    out["transpose_int32"] = case("transpose", [[_ints(8010, shape)]], ip=(0, 2, 3, 1))
    out["transpose_special"] = case("transpose", [[salted(8011, shape)]], ip=(3, 1, 0, 2))
    for axis in range(4):
        for m in (2, 3, 5):
            xs = []
            for i in range(m):
                sh = list(shape)
                sh[axis] = 1 + (i * 3 + axis) % 4
                xs.append(uniform(8100 + 10 * axis + i, tuple(sh)))
            out[f"concat_axis{axis}_{m}"] = case("concat", [xs], ip=[axis])
    out["concat_int32"] = case("concat", [[_ints(8200, (2, 3, 4, 5)), _ints(8201, (2, 1, 4, 5))]], ip=[1])
    out["slice"] = case("slice", [[uniform(8300, (3, 6, 7, 8))]], ip=[4, 1, 2, 0, 3, 2, 3, 7, 4])
    out["strided_slice_neg_step"] = case("strided_slice", [[uniform(8301, (3, 6, 7, 8))]],
                                         ip=[4, 0, 5, 6, 1, 3, 0, 0, 7, 1, -2, -1, 2, 0, 0])
    out["strided_slice_step2"] = case("strided_slice", [[uniform(8302, (3, 6, 7, 8))]],
                                      ip=[4, 0, 1, 0, 0, 3, 6, 7, 8, 1, 2, 3, 1, 0, 0])
    out["pad"] = case("pad", [[uniform(8400, (2, 3, 4, 5))]], ip=[0, 1, 1, 0, 2, 1, 0, 3])
    out["pad_int32"] = case("pad", [[_ints(8401, (2, 3, 4, 5))]], ip=[1, 0, 0, 2, 0, 0, 1, 1])
    out["tile"] = case("tile", [[uniform(8500, (2, 3, 4, 5))]], ip=[2, 1, 3, 2])
    out["broadcast_to"] = case("broadcast_to", [[uniform(8600, (1, 3, 1, 5))]], ip=[4, 3, 6, 5])
    out["broadcast_to_int32"] = case("broadcast_to", [[_ints(8601, (3, 1))]], ip=[2, 3, 7])
    out["reshape_nchw_to_nhwc"] = case("reshape", [[uniform(8700, (2, 3, 4, 5))]], ip=[NHWC, 2, 4, 5, 3])
    out["convert_nchw_to_nhwc"] = case("convert", [[uniform(8701, (2, 3, 4, 5))]], ip=[NHWC])
    out["convert_nhwc_to_nchw"] = case("convert", [[uniform(8702, (2, 4, 5, 3))]], ip=[NCHW], fmt=[NHWC])
    r = [[uniform(8800 + 2 * j, (2, 3, 4, 5) if j < 3 else (3, 2, 6, 1)),
          uniform(8801 + 2 * j, (2, 1, 4, 5) if j < 3 else (3, 4, 6, 1))] for j in range(4)]
    out["concat_rerun_resize"] = case("concat", r, ip=[1])
    r = [[uniform(8900 + j, (2, 3, 4, 5) if j < 3 else (1, 4, 2, 3))] for j in range(4)]
    out["pad_rerun_resize"] = case("pad", r, ip=[0, 0, 1, 1, 0, 2, 2, 0])
    return out


def declined_cases():
    """forms the plugin hands back to the CPU backup backend"""
    out = {}
    for op in ("FLOOR", "SIN", "ERF"):
        out[f"declined_unary_{op}"] = case("unary", [[uniform(9000 + UNARY[op], (2, 3, 5, 7))]], ip=[UNARY[op]])
    a, b = rng(9100).uniform(0.5, 3, (2, 3, 5, 7)).astype(F), uniform(9101, (2, 3, 5, 7))
    out["declined_binary_POW"] = case("binary", [[a, b]], ip=[BINARY["POW"], 0])
    out["declined_binary_FLOORDIV"] = case("binary", [[b, a]], ip=[BINARY["FLOORDIV"], 0])
    # of the coefficient forms the CPU runs only {1, 0}, a copy of the first input (CPUEltwise.cpp:35-45)
    out["declined_eltwise_coeff"] = case("eltwise", [[a, b]], ip=[ELTWISE["SUM"]], fp=[1.0, 0.0])
    out["declined_argmax_top2"] = case("argmax", [[uniform(9200, (3, 8, 5))]], ip=[0, 1, 2, 0])
    out["declined_softmax_nhwc_4d"] = case("softmax", [[uniform(9300, (2, 5, 6, 7))]], ip=[3], fmt=[NHWC])
    return out


def all_cases():
    out = {}
    for f in (binary_cases, eltwise_cases, relu_cases, unary_cases, pool_cases, reduce_cases, softmax_cases, argmax_cases,
              scale_cases, raster_cases, declined_cases):
        out.update(f())
    return out
