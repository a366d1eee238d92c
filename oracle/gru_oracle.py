"""GRU (OpType_RNNSequenceGRU) restated in numpy, with the error bound of one GPU step, the launch plan of gru.cu and a census
of its launch cells.

The reference (CPURNNSequenceGRU.cpp, runRNNStep) runs per step and batch row, every line rounded in fp32:
    g = [x_t, h] Wg + bg;  g = g + rb[0:2H];  z = sigmoid(g[0:H]);  r = sigmoid(g[H:2H])
    linear_before_reset 0: n_pre = [x_t, r * h] Wc + (rb[2H:3H] + bc)
    linear_before_reset 1: n_pre = ((r * (h Wc[I:] + rb[2H:3H])) + x_t Wc[0:I]) + bc
    n = tanh(n_pre);  h' = ((h - n) * z) + n
Layouts: X [T, B, I]; per direction Wg [I + H, 2H] (rows 0 .. I - 1 the x part; columns z, then r), bg [2H], Wc [I + H, H],
bc [H], rb [3H]; h0 [D, B, H]; Y [T, D, B, H], Y_h [D, B, H].  Without h0, h starts at zeros.  Direction 1 walks t from T - 1
down to 0 and writes Y[t][1].  `run64` gives ONNX's Y_h (each direction's last h); `cpu_y_h` the reference CPU's, whose backward
half is its scratch when Y and Y_h are both requested (zeros without h0).

`step_check_bounds` is one step in float64 from given fp32 inputs and the per-element bound of the GPU's fp32 step against it:
the x terms by the split-TF32 MatMul's model, each h . R row by gamma_H sum |r||h| (rnn_oracle's helpers), sigmoid and tanh
by UnaryOp's ulp bounds carried through their derivatives, and one rounding per operation of the rest.
"""
import numpy as np

from oracle.rnn_oracle import (MAX_CLUSTER, MAX_HIDDEN, MAX_ROWS, PARTIALS, SIGMOID_ULPS, SMEM_CAP, TANH_ULPS, THREADS, U,  # noqa: F401
                               _ulp, matmul_tolerance, sigmoid64)


def split(p, I):
    """one direction's five tensors (Wg, bg, Wc, bc, rb) in float64, split into x and h parts"""
    wg, bg, wc, bc, rb = (np.asarray(a, np.float64).reshape(np.shape(a)) for a in p)
    bg, bc, rb = bg.reshape(-1), bc.reshape(-1), rb.reshape(-1)
    return wg[:I], wg[I:], bg, wc[:I], wc[I:], bc, rb


def step64(lbr, x_t, p, h_prev):
    """one step of one direction in float64: x_t [B, I], p the five tensors, h_prev [B, H] or None (zeros).  Returns h'"""
    x = np.asarray(x_t, np.float64)
    I = x.shape[1]
    wgx, wgh, bg, wcx, wch, bc, rb = split(p, I)
    H = wch.shape[1]
    h = np.zeros((x.shape[0], H)) if h_prev is None else np.asarray(h_prev, np.float64)
    g = x @ wgx + h @ wgh + bg + rb[:2 * H]
    z, r = sigmoid64(g[:, :H]), sigmoid64(g[:, H:])
    if lbr:
        pre = r * (h @ wch + rb[2 * H:]) + x @ wcx + bc
    else:
        pre = x @ wcx + (r * h) @ wch + (rb[2 * H:] + bc)
    n = np.tanh(pre)
    return (h - n) * z + n


def run64(lbr, x, params, h0=None):
    """the whole op in float64: (Y [T, D, B, H], Y_h [D, B, H]) with ONNX's Y_h; params: 5 * D tensors in the op's order"""
    T, B, I = x.shape
    D = len(params) // 5
    H = np.shape(params[3])[-1]
    Y, Yh = np.zeros((T, D, B, H)), np.zeros((D, B, H))
    for d in range(D):
        p = params[5 * d:5 * d + 5]
        h = None if h0 is None else h0[d]
        for s in range(T):
            t = T - 1 - s if d else s
            h = step64(lbr, x[t], p, h)
            Y[t, d] = h
        Yh[d] = h
    return Y, Yh


def cpu_y_h(Y, Yh, has_h0, keep_all, n_out):
    """the reference CPU's Y_h: with keepAllOutputs and two outputs its backward half is the op's scratch -- zeros without h0,
    unset (None here) with h0"""
    if not (keep_all and n_out > 1) or Yh.shape[0] == 1:
        return Yh
    if has_h0:
        return None
    out = Yh.copy()
    out[1] = 0.0
    return out


def torch_gru_weights(p, I):
    """one direction's tensors as torch.nn.GRU's (weight_ih [3H, I], weight_hh [3H, H], bias_ih, bias_hh), gate rows r, z, n:
    the linear_before_reset = 1 form is torch's"""
    wgx, wgh, bg, wcx, wch, bc, rb = split(p, I)
    H = wch.shape[1]
    w_ih = np.concatenate([wgx[:, H:].T, wgx[:, :H].T, wcx.T])
    w_hh = np.concatenate([wgh[:, H:].T, wgh[:, :H].T, wch.T])
    b_ih = np.concatenate([bg[H:], bg[:H], bc])
    b_hh = np.concatenate([rb[H:2 * H], rb[:H], rb[2 * H:]])
    return w_ih, w_hh, b_ih, b_hh


def step_check_bounds(lbr, x_t, p, h_prev, slack=1.05):
    """(h64, e_h): float64's step and the GPU's bound per element [B, H], from the step's fp32 inputs (h_prev None: zeros)"""
    x = np.asarray(x_t, np.float64)
    I = x.shape[1]
    wgx, wgh, bg, wcx, wch, bc, rb = split(p, I)
    H = wch.shape[1]
    h = np.zeros((x.shape[0], H)) if h_prev is None else np.asarray(h_prev, np.float64)
    gam = H * U / (1 - H * U)
    ax = np.abs(x)
    # z, r: g = (P_zr + h . R_zr) + rb, P_zr = x Wg_x + bg by the MatMul
    pzr, pzr_abs = x @ wgx + bg, ax @ np.abs(wgx)
    hzr = h @ wgh
    s = pzr + hzr
    g = s + rb[:2 * H]
    eg = matmul_tolerance(pzr_abs, I, bg) + gam * (np.abs(h) @ np.abs(wgh)) + U * np.abs(s) + U * np.abs(g)
    z, r = sigmoid64(g[:, :H]), sigmoid64(g[:, H:])
    ez = z * (1 - z) * eg[:, :H] + SIGMOID_ULPS * _ulp(z)
    er = r * (1 - r) * eg[:, H:] + SIGMOID_ULPS * _ulp(r)
    pn, pn_abs = x @ wcx, ax @ np.abs(wcx)
    epn = matmul_tolerance(pn_abs, I, 0.0)
    if lbr:
        hn = h @ wch + rb[2 * H:]
        ehn = gam * (np.abs(h) @ np.abs(wch)) + U * np.abs(hn)
        a = r * hn
        ea = np.abs(hn) * er + r * ehn + er * ehn + _ulp(a) / 2
        b = a + pn
        pre = b + bc
        epre = ea + epn + U * np.abs(b) + U * np.abs(pre)
    else:
        rh = r * h
        erh = np.abs(h) * er + _ulp(rh) / 2
        d = rh @ wch
        ed = gam * (np.abs(rh) @ np.abs(wch)) + erh @ np.abs(wch)
        bsum = rb[2 * H:] + bc
        s2 = pn + d
        pre = s2 + bsum
        epre = epn + ed + U * np.abs(s2) + U * np.abs(pre) + U * np.abs(bsum)
    n = np.tanh(pre)
    en = (1 - n * n) * epre * slack + TANH_ULPS * _ulp(n)
    dlt = h - n
    m = dlt * z
    h1 = m + n
    eh = (1 + np.abs(z)) * en + np.abs(dlt) * ez * slack + en * ez + np.abs(z) * _ulp(dlt) / 2 + _ulp(m) / 2 + _ulp(h1) / 2
    return h1, eh * slack


# ---- the launch plan (gru.cu gru_choose_plan over recur_common.cuh recur_choose_plan), for a device whose every cluster fits --
def _ks(items):
    ks = PARTIALS
    while ks > 1 and items * ks > THREADS:
        ks >>= 1
    return ks


def _shape(lbr, h, rows, groups, cs, resident):
    hs = -(-h // cs)
    ks = _ks(rows * hs)
    rstride = h + ((ks - h) % 32)
    head, extra = (16, 0) if lbr else (32, h)
    smem = head + 4 * (2 * rows * h + rows * hs + rows * extra) + (4 * 3 * hs * rstride if resident else 0)
    return dict(cs=cs, groups=groups, rows=rows, hs=hs, ks=ks, resident=int(resident), smem=smem,
                threads=min(THREADS, (rows * hs * ks + 31) // 32 * 32))


def choose_plan(lbr, b, h, d, sms, smem_cap=SMEM_CAP, max_cluster=MAX_CLUSTER):
    """the plan of (linear_before_reset, B, H, D) on a device of `sms` SMs; max_cluster: the largest cluster that fits"""
    extra = 0 if lbr else h
    max_rows = max(1, min(MAX_ROWS, 49152 // (2 * h + extra)))
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
        pl = _shape(lbr, h, rows, groups, cs, False)
        c = cs
        while c <= top:
            r = _shape(lbr, h, rows, groups, c, True)
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


def cell_of(lbr, b, d, pl):
    """the launch cell a plan runs: (LBR, cluster size, resident, several batch groups, ragged last group, D, KS)"""
    return (lbr, pl["cs"], pl["resident"], int(pl["groups"] > 1), int(pl["groups"] * pl["rows"] != b), d, pl["ks"])


# candidate shapes of the census: every launch cell one of them reaches on a device is a cell the kernel has there
CENSUS_H = (1, 2, 3, 4, 5, 8, 9, 16, 17, 31, 32, 33, 64, 65, 100, 128, 200, 256, 300, 384, 440, 512, 600, 700, 1024)
CENSUS_B = (1, 2, 3, 5, 8, 9, 11, 16, 17, 24, 33, 64, 65, 100, 128)


def census(sms, smem_cap=SMEM_CAP, max_cluster=MAX_CLUSTER):
    """{launch cell: the cheapest (LBR, B, H, D) reaching it} over CENSUS_H x CENSUS_B x D x LBR"""
    out = {}
    for lbr in (0, 1):
        for d in (1, 2):
            for h in CENSUS_H:
                for b in CENSUS_B:
                    pl = choose_plan(lbr, b, h, d, sms, smem_cap, max_cluster)
                    if pl is None:
                        continue
                    key = cell_of(lbr, b, d, pl)
                    cost = b * h * h * 3 * d
                    if key not in out or cost < out[key][0]:
                        out[key] = (cost, (lbr, b, h, d))
    return {k: v[1] for k, v in out.items()}


def random_params(rng, d, i, h, scale=None):
    """5 * d fp32 tensors in the op's order, the op's shapes: Wg [I + H, 2H], bg [1, 2H], Wc [I + H, H], bc [1, H], rb [1, 3H]"""
    s = scale if scale is not None else 1.0 / np.sqrt(h)
    out = []
    for _ in range(d):
        out += [(rng.standard_normal((i + h, 2 * h)) * s).astype(np.float32),
                (rng.standard_normal((1, 2 * h)) * 0.5).astype(np.float32),
                (rng.standard_normal((i + h, h)) * s).astype(np.float32),
                (rng.standard_normal((1, h)) * 0.5).astype(np.float32),
                (rng.standard_normal((1, 3 * h)) * 0.5).astype(np.float32)]
    return out


# ---- the live reference: oracle/_ref/refdump_gru (oracle/refdump_gru.cpp over oracle/_ref/libMNN.so), built by build() ------
import os  # noqa: E402
import struct  # noqa: E402
import subprocess  # noqa: E402
import tempfile  # noqa: E402

from oracle.rnn_oracle import _stats  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(HERE, "_ref")
REFDUMP_GRU = os.path.join(REF_DIR, "refdump_gru")
DENOISE = os.path.join(REF_DIR, "denoise_f32.mnn")
TAGGER = os.path.join(REF_DIR, "tagger_f32.mnn")
DENOISE_SEED, TAGGER_SEED = 71, 72


def have_refdump():
    return os.path.exists(REFDUMP_GRU)


def build_refdump():
    """compile oracle/refdump_gru.cpp against the reference build of oracle/build_ref.py and write the denoiser and tagger
    fixtures with it"""
    from oracle import build_ref as B
    src = os.path.join(HERE, "refdump_gru.cpp")
    lib = os.path.join(REF_DIR, "libMNN.so")
    fresh = have_refdump() and all(os.path.getmtime(REFDUMP_GRU) > os.path.getmtime(d) for d in (src, lib))
    if not fresh:
        cmd = ["g++", "-O2", "-std=gnu++11", "-w", "-o", REFDUMP_GRU, src] + ["-I" + os.path.join(B.REF, i) for i in B.INCLUDES] + \
              ["-L" + REF_DIR, "-lMNN", "-Wl,-rpath,$ORIGIN", "-pthread", "-ldl"]
        subprocess.check_call(cmd)
    for path, cmd, seed in ((DENOISE, "denoise", DENOISE_SEED), (TAGGER, "tagger", TAGGER_SEED)):
        if not fresh or not os.path.exists(path):
            _run([cmd, path, seed])


def _run(args, plugin=None, env_more=None):
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = REF_DIR + ":" + env.get("LD_LIBRARY_PATH", "")
    env.pop("REFDUMP_PLUGIN", None)
    if plugin:
        env["REFDUMP_PLUGIN"] = plugin
    env.update(env_more or {})
    return subprocess.run([REFDUMP_GRU] + [str(a) for a in args], env=env, capture_output=True, text=True, timeout=900,
                          check=True)


def ref_op(lbr, x, params, h0=None, keep_all=True, n_out=2, more=None, plugin=None):
    """outputs of one reference op through the Express executor on MNN_FORWARD_CPU: (Y, Y_h) with keep_all and two outputs,
    (Y,) with one, (Y_h,) without keep_all.  more: further (x, params, h0) sets through the same executor (a list of output
    tuples returned).  plugin: run on MNN_FORWARD_CUDA with that plugin, and (outputs, the plugin's stats) returned"""
    sets = [(x, params, h0)] + list(more or [])
    T, B, I = x.shape
    D = len(params) // 5
    H = np.shape(params[3])[-1]
    hdr = struct.pack("<10i", lbr, T, B, I, H, D, int(h0 is not None), int(keep_all), n_out, len(sets))
    body = b"".join(np.ascontiguousarray(a, np.float32).tobytes() for xs, ps, hs in sets
                    for a in [xs] + list(ps) + ([] if hs is None else [hs]))
    with tempfile.TemporaryDirectory() as d:
        req, out = os.path.join(d, "req"), os.path.join(d, "out")
        open(req, "wb").write(hdr + body)
        res = _run(["op", req, out], plugin)
        raw = np.frombuffer(open(out, "rb").read(), np.float32)
    shapes = ([(T, D, B, H), (D, B, H)][:n_out]) if keep_all else [(D, B, H)]
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
    """`refdump_gru run`: every command's fp32 outputs under outdir (index.txt); returns (records, plugin stats, process)"""
    os.makedirs(outdir, exist_ok=True)
    r = _run(["run", model, batch, seed, outdir], plugin, {"REFDUMP_RUN_REPEATS": str(repeats)} if repeats else None)
    recs = []
    for line in open(os.path.join(outdir, "index.txt")):
        f, name, typ = line.rstrip("\n").split("|")[:3]
        recs.append((f, name, typ.strip()))
    return recs, _stats(r), r


def run_chunks(batch, seed, chunks, outdir, plugin=None):
    """`refdump_gru chunks` over denoise_f32.mnn: {(chunk, output name): array}, plugin stats"""
    os.makedirs(outdir, exist_ok=True)
    r = _run(["chunks", DENOISE, batch, seed, chunks, outdir], plugin)
    out = {}
    for k in range(chunks):
        for name in ("output", "h1_n", "h2_n", "h3_n"):
            out[(k, name)] = np.fromfile(os.path.join(outdir, f"chunk{k}_{name}.f32"), np.float32)
    return out, _stats(r)
