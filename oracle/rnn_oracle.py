"""LSTM / RNN (OpType_LSTM / OpType_RNN of ONNX models) restated in numpy, with the error bound of one GPU step.

The reference lowers the op in GeometryLSTM.cpp (_ComputeLSTMOnnx): Gate = X W^T + B over all T * B rows (one MatMul per
direction; direction 1 on X reversed in time), then per step HR = h_prev R^T, z = Gate_t + HR and
    LSTM (gate rows in ONNX order i, o, f, c): i = sigmoid(z_i), g = tanh(z_c), f = sigmoid(z_f), o = sigmoid(z_o),
          Temp = i * g, I = f * c_prev, c = Temp + I, h = tanh(c) * o;
    RNN:  h = tanh(z).
Without initial states the first step has no HR term and no f * c term.  Direction 1 writes Y at T - 1 - s; Y_h is Y at T - 1
for direction 0 and at 0 for direction 1; Y_c the last cell state.  Layouts: X [T, B, I], W [D, G*H, I], R [D, G*H, H],
B [D, G*H], h0 / c0 [D, B, H]; Y [T, D, B, H], Y_h / Y_c [D, B, H]; G = 4 (LSTM) or 1 (RNN).

`step64` is one step in float64 from given fp32 inputs, and `step_bound` the per-element bound of the GPU's fp32 step against
it, computed from the step's own inputs: the projection by the split-TF32 MatMul's model, the h_prev . R term by
gamma_H sum |r||h|, sigmoid and tanh by UnaryOp's ulp bounds carried through their derivatives, and one rounding per operation
of the cell update and h.  `choose_plan` restates the launch plan of rnn.cu (rnn_choose_plan) for a device of a given SM count.
"""
import numpy as np

U = 2.0 ** -24                           # unit roundoff of fp32
SIGMOID_ULPS, TANH_ULPS = 4, 2           # UnaryOp's bounds (tests/test_gpu_plugin_float_ops.py UNARY_ULPS)
GATES = {0: 4, 1: 1}                     # cell 0 LSTM, 1 RNN
SMEM_CAP = 232448                        # dynamic shared memory per CTA on an H100 (cudaDevAttrMaxSharedMemoryPerBlockOptin)
THREADS, MAX_CLUSTER, MAX_ROWS, MAX_HIDDEN, PARTIALS = 256, 16, 8, 4096, 8


def sigmoid64(z):
    z = np.asarray(z, np.float64)
    with np.errstate(over="ignore"):
        return np.where(z >= 0, 1.0 / (1.0 + np.exp(-np.abs(z))), np.exp(-np.abs(z)) / (1.0 + np.exp(-np.abs(z))))


def gates64(x, w, b):
    """Gate = x W^T + b in float64 for one direction: x [N, I], w [G*H, I], b [G*H]; and sum |x||w| (the split-TF32 model's S)"""
    x64, w64 = np.asarray(x, np.float64), np.asarray(w, np.float64)
    return x64 @ w64.T + np.asarray(b, np.float64), np.abs(x64) @ np.abs(w64).T


def step64(cell, gate, r, h_prev, c_prev):
    """one step of one direction in float64: gate [B, G*H] (the projection row of this step), r [G*H, H], h_prev / c_prev [B, H]
    or None (the first step without initial states).  Returns (h, c, z, hr_abs) with z the pre-activations [B, G*H] and
    hr_abs = sum |h_prev||r| [B, G*H]"""
    gate = np.asarray(gate, np.float64)
    if h_prev is None:
        hr, hr_abs = 0.0, np.zeros_like(gate)
    else:
        h64, r64 = np.asarray(h_prev, np.float64), np.asarray(r, np.float64)
        hr, hr_abs = h64 @ r64.T, np.abs(h64) @ np.abs(r64).T
    z = gate + hr
    if cell == 1:
        return np.tanh(z), None, z, hr_abs
    H = z.shape[1] // 4
    i, o, f, g = sigmoid64(z[:, :H]), sigmoid64(z[:, H:2 * H]), sigmoid64(z[:, 2 * H:3 * H]), np.tanh(z[:, 3 * H:])
    c = i * g if c_prev is None else i * g + f * np.asarray(c_prev, np.float64)
    return np.tanh(c) * o, c, z, hr_abs


def matmul_tolerance(s, l, bias):
    """the split-TF32 MatMul's per-element bound (tests/test_gpu_matmul_f32.py::tolerance): S = sum |a||b| over l terms"""
    tau = 2.0 ** -20 + 3 * -(-l // 8) * (8 + 2) * 2.0 ** -23
    return tau * s + 2.0 ** -23 * (s + np.abs(np.asarray(bias, np.float64)))


def _ulp(v):
    return np.spacing(np.abs(np.asarray(v, np.float64)).astype(np.float32)).astype(np.float64)


def bound_from(cell, z, ez, c_prev):
    """propagate the pre-activation bound ez [B, G*H] through the activations and the cell update at z (float64)"""
    if cell == 1:
        t = np.tanh(z)
        return (1 - t * t) * ez + TANH_ULPS * _ulp(t), None
    H = z.shape[1] // 4
    zi, zo, zf, zg = z[:, :H], z[:, H:2 * H], z[:, 2 * H:3 * H], z[:, 3 * H:]
    ei, eo, ef, eg = ez[:, :H], ez[:, H:2 * H], ez[:, 2 * H:3 * H], ez[:, 3 * H:]
    i, o, f, g = sigmoid64(zi), sigmoid64(zo), sigmoid64(zf), np.tanh(zg)
    e_i = i * (1 - i) * ei + SIGMOID_ULPS * _ulp(i)
    e_o = o * (1 - o) * eo + SIGMOID_ULPS * _ulp(o)
    e_f = f * (1 - f) * ef + SIGMOID_ULPS * _ulp(f)
    e_g = (1 - g * g) * eg + TANH_ULPS * _ulp(g)
    temp = i * g
    e_temp = np.abs(g) * e_i + np.abs(i) * e_g + e_i * e_g + _ulp(temp) / 2
    if c_prev is None:
        c, e_c = temp, e_temp
    else:
        cp = np.asarray(c_prev, np.float64)
        fc = f * cp
        e_fc = np.abs(cp) * e_f + _ulp(fc) / 2
        c = temp + fc
        e_c = e_temp + e_fc + _ulp(c) / 2 + 2 * U * (np.abs(temp) + np.abs(fc))
    tc = np.tanh(c)
    e_tc = (1 - tc * tc) * e_c + TANH_ULPS * _ulp(tc) + _ulp(tc) / 2
    h = tc * o
    e_h = np.abs(o) * e_tc + np.abs(tc) * e_o + e_tc * e_o + _ulp(h) / 2
    return e_h, e_c


def step_check_bounds(cell, gate, gate_abs, n_in, bias, r, h_prev, c_prev, slack=1.05):
    """(h64, c64, e_h, e_c): float64's step and the GPU's bound per element, from the step's fp32 inputs"""
    h64, c64, z, hr_abs = step64(cell, gate, r, h_prev, c_prev)
    H = r.shape[1]
    gam = H * U / (1 - H * U)
    ez = matmul_tolerance(gate_abs, n_in, bias) + gam * hr_abs + (0.0 if h_prev is None else 2 * U * np.abs(z))   # + the add z = G + HR
    e_h, e_c = bound_from(cell, z, ez * slack, c_prev)
    return h64, c64, e_h * slack, None if e_c is None else e_c * slack


def run64(cell, x, w, r, b, h0=None, c0=None):
    """the whole op in float64: (Y [T, D, B, H], Y_h [D, B, H], Y_c [D, B, H] or None)"""
    T, B, I = x.shape
    D, GH, _ = w.shape
    H = r.shape[2]
    Y = np.zeros((T, D, B, H))
    Yh, Yc = np.zeros((D, B, H)), np.zeros((D, B, H))
    for d in range(D):
        g, _ = gates64(x.reshape(T * B, I), w[d], b[d])
        g = g.reshape(T, B, GH)
        h = None if h0 is None else np.asarray(h0[d], np.float64)
        c = None if c0 is None else np.asarray(c0[d], np.float64)
        if cell == 0 and h is not None and c is None:
            c = np.zeros((B, H))
        for s in range(T):
            t = T - 1 - s if d else s
            h, c, _, _ = step64(cell, g[t], r[d], h, c)
            Y[t, d] = h
        Yh[d] = h
        if cell == 0:
            Yc[d] = c
    return Y, Yh, (Yc if cell == 0 else None)


def torch_lstm_weights(w, r, b):
    """ONNX-order (i, o, f, c) gate rows to torch.nn.LSTM's (i, f, g, o) for one direction: the permutation of row blocks"""
    H = w.shape[0] // 4
    perm = np.concatenate([np.arange(0, H), np.arange(2 * H, 3 * H), np.arange(3 * H, 4 * H), np.arange(H, 2 * H)])
    return w[perm], r[perm], b[perm]


# ---- the launch plan (rnn.cu rnn_choose_plan), for a device whose every cluster fits ------------------------------------
def _ks(items):
    ks = PARTIALS
    while ks > 1 and items * ks > THREADS:
        ks >>= 1
    return ks


def _shape(cell, h, rows, groups, cs, resident):
    hs = -(-h // cs)
    ks = _ks(rows * hs)
    rstride = h + ((ks - h) % 32)
    smem = 16 + 4 * (2 * rows * h + rows * hs) + (4 * GATES[cell] * hs * rstride if resident else 0)
    return dict(cs=cs, groups=groups, rows=rows, hs=hs, ks=ks, resident=int(resident), smem=smem,
                threads=min(THREADS, (rows * hs * ks + 31) // 32 * 32))


def choose_plan(cell, b, h, d, sms, smem_cap=SMEM_CAP, max_cluster=MAX_CLUSTER):
    """the plan of (cell, B, H, D) on a device of `sms` SMs; max_cluster: the largest cluster that fits (16 on an H100)"""
    max_rows = max(1, min(MAX_ROWS, 24576 // h))
    groups = -(-b // max_rows)
    rows = -(-b // groups)
    top = 1
    while top * 2 <= min(h, MAX_CLUSTER):
        top *= 2
    cs = 1
    while cs < top and rows * -(-h // cs) > 32:
        cs *= 2
    while cs > 1 and cs * groups * d > sms:
        cs //= 2
    while True:
        pl = _shape(cell, h, rows, groups, cs, False)
        c = cs
        while c <= top:
            r = _shape(cell, h, rows, groups, c, True)
            if r["smem"] <= smem_cap:
                pl = r
                break
            c *= 2
        if pl["smem"] <= smem_cap and pl["cs"] <= max_cluster:
            return pl
        if cs == 1:
            return None
        cs //= 2
        top = cs


def cell_of(cell, b, d, pl):
    """the launch cell a plan runs: (cell, cluster size, resident, several batch groups, ragged last group, D, KS)"""
    return (cell, pl["cs"], pl["resident"], int(pl["groups"] > 1), int(pl["groups"] * pl["rows"] != b), d, pl["ks"])


# candidate shapes of the census: every launch cell one of them reaches on a device is a cell the kernel has there
CENSUS_H = (1, 2, 3, 4, 5, 8, 9, 16, 17, 31, 32, 33, 64, 65, 100, 128, 200, 256, 300, 384, 440, 512, 700, 1024)
CENSUS_B = (1, 2, 3, 5, 8, 9, 11, 16, 17, 24, 33, 64, 65, 100, 128)


def census(sms, smem_cap=SMEM_CAP, max_cluster=MAX_CLUSTER):
    """{launch cell: the cheapest (cell, B, H, D) reaching it} over CENSUS_H x CENSUS_B x D x cell"""
    out = {}
    for cell in (0, 1):
        for d in (1, 2):
            for h in CENSUS_H:
                for b in CENSUS_B:
                    pl = choose_plan(cell, b, h, d, sms, smem_cap, max_cluster)
                    if pl is None:
                        continue
                    key = cell_of(cell, b, d, pl)
                    cost = b * h * h * GATES[cell] * d
                    if key not in out or cost < out[key][0]:
                        out[key] = (cost, (cell, b, h, d))
    return {k: v[1] for k, v in out.items()}


# ---- the live reference: oracle/_ref/refdump_rnn (oracle/refdump_rnn.cpp over oracle/_ref/libMNN.so), built by build() ------
import json  # noqa: E402
import os  # noqa: E402
import struct  # noqa: E402
import subprocess  # noqa: E402
import tempfile  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(HERE, "_ref")
REFDUMP_RNN = os.path.join(REF_DIR, "refdump_rnn")
CRNN = os.path.join(REF_DIR, "crnn_f32.mnn")
KWS = os.path.join(REF_DIR, "kws_f32.mnn")
CRNN_SEED, KWS_SEED = 61, 62


def have_refdump():
    return os.path.exists(REFDUMP_RNN)


def build_refdump():
    """compile oracle/refdump_rnn.cpp against the reference build of oracle/build_ref.py and write the CRNN- and KWS-style
    fixtures with it"""
    from oracle import build_ref as B
    src = os.path.join(HERE, "refdump_rnn.cpp")
    lib = os.path.join(REF_DIR, "libMNN.so")
    fresh = have_refdump() and all(os.path.getmtime(REFDUMP_RNN) > os.path.getmtime(d) for d in (src, lib))
    if not fresh:
        cmd = ["g++", "-O2", "-std=gnu++11", "-w", "-o", REFDUMP_RNN, src] + ["-I" + os.path.join(B.REF, i) for i in B.INCLUDES] + \
              ["-L" + REF_DIR, "-lMNN", "-Wl,-rpath,$ORIGIN", "-pthread", "-ldl"]
        subprocess.check_call(cmd)
    for path, cmd, seed in ((CRNN, "crnn", CRNN_SEED), (KWS, "kws", KWS_SEED)):
        if not fresh or not os.path.exists(path):
            _run([cmd, path, seed])


def _run(args, plugin=None, env_more=None):
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = REF_DIR + ":" + env.get("LD_LIBRARY_PATH", "")
    env.pop("REFDUMP_PLUGIN", None)
    if plugin:
        env["REFDUMP_PLUGIN"] = plugin
    env.update(env_more or {})
    return subprocess.run([REFDUMP_RNN] + [str(a) for a in args], env=env, capture_output=True, text=True, timeout=900,
                          check=True)


def _stats(r):
    stats = [json.loads(line) for line in r.stdout.splitlines() if line.startswith('{"plugin_')]
    return stats[-1] if stats else None


def ref_op(cell, x, w, r, b, h0=None, c0=None, more=None, clip=0.0, plugin=None):
    """outputs (Y, Y_h[, Y_c]) of one reference op through the Express executor on MNN_FORWARD_CPU.  The inputs given (c0 only
    with h0) are the op's inputs; more: further input tuples of the same shapes through the same executor (a list of output
    tuples returned); clip: the LSTM parameter's clippingThreshold.  plugin: run on MNN_FORWARD_CUDA with that plugin, and
    (outputs, the plugin's stats) returned"""
    first = tuple(a for a in (x, w, r, b, h0, c0) if a is not None)
    sets = [first] + [tuple(m) for m in (more or [])]
    T, B, I = x.shape
    D, GH, _ = w.shape
    H = r.shape[2]
    hdr = struct.pack("<7ifi", cell, T, B, I, H, D, len(first), clip, len(sets))
    body = b"".join(np.ascontiguousarray(a, np.float32).tobytes() for s in sets for a in s)
    with tempfile.TemporaryDirectory() as d:
        req, out = os.path.join(d, "req"), os.path.join(d, "out")
        open(req, "wb").write(hdr + body)
        res = _run(["op", req, out], plugin)
        raw = np.frombuffer(open(out, "rb").read(), np.float32)
    shapes = [(T, D, B, H), (D, B, H)] + ([(D, B, H)] if cell == 0 else [])
    outs, pos = [], 0
    for _ in sets:
        one = []
        for s in shapes:
            n = int(np.prod(s))
            one.append(raw[pos:pos + n].reshape(s).copy())
            pos += n
        outs.append(tuple(one))
    outs = outs[0] if more is None else outs
    return outs if plugin is None else (outs, _stats(res))


def run_model(model, batch, seed, outdir, plugin=None, repeats=None):
    """`refdump_rnn run`: every command's fp32 outputs under outdir (index.txt); returns (records, plugin stats, process)"""
    os.makedirs(outdir, exist_ok=True)
    r = _run(["run", model, batch, seed, outdir], plugin, {"REFDUMP_RUN_REPEATS": str(repeats)} if repeats else None)
    recs = []
    for line in open(os.path.join(outdir, "index.txt")):
        f, name, typ = line.rstrip("\n").split("|")[:3]
        recs.append((f, name, typ.strip()))
    return recs, _stats(r), r


def run_chunks(batch, seed, chunks, outdir, plugin=None):
    """`refdump_rnn chunks` over kws_f32.mnn: {(chunk, output name): array}, plugin stats"""
    os.makedirs(outdir, exist_ok=True)
    r = _run(["chunks", KWS, batch, seed, chunks, outdir], plugin)
    out = {}
    for k in range(chunks):
        for name in ("output", "h_n", "c_n", "hr_n"):
            out[(k, name)] = np.fromfile(os.path.join(outdir, f"chunk{k}_{name}.f32"), np.float32)
    return out, _stats(r)
