"""Restatement of the reference CPU's fp32 GridSample (CPUGridSample, source/backend/cpu/CPUGridSample.cpp).

Finding (the live reference, x86 with AVX2 / AVX512): OpCommonUtils::opCompabilityForLowp lists GridSample, so an
MNN_FORWARD_CPU session runs it on AVX2Backend, packed by 8 (AVX2) or 16 (AVX-512), not on the pack-4 backup CPUBackend that
Interp uses.  The functions that run on an AVX-512 host are _AVX512_MNNGridSampleComputeCord (4-D), _AVX_MNNGridSampleComputeCord3D
(5-D: the avx512 table does not replace it) and the avx512 copy of GridSampler.hpp's MNNGridSampleInterp / MNNGridSampleInterp3D.
oracle/build_ref.py compiles the avx512/ sources with -mfma and the avx/ ones without; GCC 13 at -O3 contracts the intrinsic
chains where it may.  The disassembly of the reference built here shows:
  _AVX512_MNNGridSampleComputeCord    vaddps (1 + g), vfmsub132ps, vmulps 0.5: c = 0.5 * fmsub(1 + g, in - a, b)
  MNNGridSampleInterp (avx512 copy)   vmulps then vfmadd132ps per pair: i00 * f0 + i01 * f1 = fma(i01, f1, i00 * f0), and so
                                      for every pair and axis, in MNNGridSampleInterp3D too
  _AVX_MNNGridSampleComputeCord3D     vmulps / vaddps and vmulss / vaddss only: c = k * g + k0, two roundings
On an AVX2-only host both interpolation tables are the avx/ ones, without FMA, and the 4-D coordinate is unfused as well
(fused=False here).  tests/golden/grid_sample_golden.npz was recorded on an AVX-512 host through oracle/refdump_grid_sample.cpp
and equals grid_sample(..., fused=True) bit for bit; the kernel (mnn_b200/csrc/grid_sample_f32.cu) computes the fused form.

Other facts restated: taps floor(c) and ceil(c) (equal on an integral c, weights 0 and 1), f0 = (float)ceil - c, f1 = 1 - f0;
nearest floor(c + 0.5f); every float -> int conversion is x86's cvttss2si, NaN / +-Inf / |c| >= 2^31 -> INT_MIN, whose weight
then follows from (float)INT_MIN - c; ZEROS reads +0 for an outside tap (still multiplied by its weight), CLAMP and REFLECTION
clamp the tap (REFLECTION is not PyTorch's / ONNX's reflection).  grid_sample64() is the same sampling with float64 weights and
sums, for a sanity bound.

Finding (layout): CPUGridSample reads x and writes y in the CPU backend's packed NC4HW4 layout ([c / pack][n][spatial][pack])
without looking at the tensors' format.  The model converter always gives a GridSample's first input and its output NC4HW4
(AddTensorFormatConverter.cpp: NC4HW4_SINGLE), and then the CPU is right.  A graph that hands it an NCHW x (an Express graph
can: a conv output that Express converts back to NCHW) gets its linear buffer misread as packed -- a result that depends on
the host's pack (16 with AVX-512, 8 with AVX2) and, when c is not a multiple of the pack, reads and writes past both buffers
(a SIGSEGV in the one-op harness).  grid_sample_linear_misread() restates the misreading where it is defined; the kernel does
not follow it: it samples the tensors as their format says, which is what the CPU computes for every converted model."""
import json
import os
import struct
import subprocess
import tempfile

import numpy as np

F = np.float32
INT_MIN = -2 ** 31
MODES = {"bilinear": 0, "nearest": 1}
PADDINGS = {"zeros": 0, "border": 1, "reflection": 2}


def fma32(a, b, c):
    """float32 fma(a, b, c), rounded once: the exact float64 product, TwoSum with c, round to odd in float64, then to float32"""
    a, b, c = (np.asarray(v, F).astype(np.float64) for v in (a, b, c))
    p = a * b                                  # exact: 24 + 24 significant bits
    with np.errstate(invalid="ignore", over="ignore"):
        s = p + c
        bp = s - p
        err = (p - (s - bp)) + (c - bp)        # s + err == p + c exactly
        bits = s.view(np.int64)
        fix = np.isfinite(s) & np.isfinite(err) & (err != 0) & ((bits & 1) == 0)
        odd = np.nextafter(s, np.where(err > 0, np.inf, -np.inf))
        s = np.where(fix, odd, s)
        return s.astype(F)


def cvt_x86(v):
    """cvttss2si of float32 values v (already integral): int64 values, INT_MIN for NaN, +-Inf and out-of-range"""
    v = np.asarray(v, F)
    with np.errstate(invalid="ignore"):
        ok = (v >= F(-2.0 ** 31)) & (v < F(2.0 ** 31))
    return np.where(ok, np.where(ok, v, F(0)).astype(np.int64), INT_MIN)


def coords(grid, in_sizes, align_corners, fused=True):
    """float32 coordinates [..., axes] (x, y[, z] = W, H[, D]) of a grid [..., axes]; in_sizes (W, H[, D])"""
    g = np.asarray(grid, F)
    a, b = (F(1), F(0)) if align_corners else (F(0), F(1))
    out = np.empty_like(g)
    with np.errstate(invalid="ignore", over="ignore"):
        for i, n in enumerate(in_sizes):
            gi = g[..., i]
            if g.shape[-1] == 2:
                ina = F(n) - a
                one_g = F(1) + gi
                t = fma32(one_g, ina, -b) if fused else one_g * ina - b
                out[..., i] = F(0.5) * t
            else:
                k, k0 = F(0.5) * (F(n) - a), F(0.5) * (F(n) - a - b)
                out[..., i] = k * gi + k0
    return out


def _axis(c, n, nearest, zeros):
    """taps [..., s] (clamped for indexing), valid flags and weights [..., s] (bilinear) of one axis of size n"""
    with np.errstate(invalid="ignore", over="ignore"):
        if nearest:
            t = cvt_x86(np.floor(c + F(0.5)))[..., None]
            w = None
        else:
            t0, t1 = cvt_x86(np.floor(c)), cvt_x86(np.ceil(c))
            f0 = t1.astype(F) - c
            f1 = F(1) - f0
            t, w = np.stack([t0, t1], -1), np.stack([f0, f1], -1)
    valid = (t >= 0) & (t < n) if zeros else np.ones(t.shape, bool)
    return np.clip(t, 0, n - 1), valid, w


def _lerp(v0, v1, f0, f1, fused, f64=False):
    if f64:
        return v0 * f0 + v1 * f1
    with np.errstate(invalid="ignore", over="ignore"):
        return fma32(v1, f1, v0 * f0) if fused else v0 * f0 + v1 * f1


def grid_sample(x, grid, mode="bilinear", padding="zeros", align_corners=False, fused=True, f64=False):
    """y float32 of CPUGridSample: x [n, c, (d,) h, w], grid [n, (od,) oh, ow, rank - 2] -> y [n, c, (od,) oh, ow], bit for bit
    (fused=True: an AVX-512 host; False: AVX2).  f64: the same taps and weights, the sums in float64 (grid_sample64)"""
    x = np.asarray(x, np.float64 if f64 else F)
    grid = np.asarray(grid, F)
    nearest, zeros = mode in ("nearest", 1), padding in ("zeros", 0)
    d3 = x.ndim == 5
    xs = x if d3 else x[:, :, None]
    n, c, D, H, W = xs.shape
    ax = grid.shape[-1]
    cord = coords(grid, (W, H, D)[:ax], align_corners, fused)
    out_sp = grid.shape[1:-1]
    cord = cord.reshape(n, -1, ax)
    P = cord.shape[1]
    y = np.empty((n, c, P), xs.dtype)
    for bi in range(n):
        taps = [_axis(cord[bi, :, i], (W, H, D)[i], nearest, zeros) for i in range(ax)]
        if not d3:
            taps.append((np.zeros((P, 1), np.int64), np.ones((P, 1), bool), None))
        (tx, vx, wx), (ty, vy, wy), (tz, vz, wz) = taps
        xb = xs[bi]

        def tap(sz, sy, sx):
            v = xb[:, tz[:, sz], ty[:, sy], tx[:, sx]]
            ok = vz[:, sz] & vy[:, sy] & vx[:, sx]
            return np.where(ok[None], v, xs.dtype.type(0))
        if nearest:
            y[bi] = tap(0, 0, 0)
            continue
        wxs = [w.astype(xs.dtype)[None] for w in (wx[:, 0], wx[:, 1])]
        wys = [w.astype(xs.dtype)[None] for w in (wy[:, 0], wy[:, 1])]

        def plane(sz):
            i0 = _lerp(tap(sz, 0, 0), tap(sz, 0, 1), *wxs, fused, f64)
            i1 = _lerp(tap(sz, 1, 0), tap(sz, 1, 1), *wxs, fused, f64)
            return _lerp(i0, i1, *wys, fused, f64)
        if d3:
            wzs = [w.astype(xs.dtype)[None] for w in (wz[:, 0], wz[:, 1])]
            y[bi] = _lerp(plane(0), plane(1), *wzs, fused, f64)
        else:
            y[bi] = plane(0)
    return y.reshape((n, c) + tuple(out_sp))


def grid_sample_linear_misread(x, grid, mode="bilinear", padding="zeros", align_corners=False, pack=16, fused=True):
    """what CPUGridSample computes when x and y reach it in a linear NCHW layout instead of NC4HW4: it reads x's buffer as
    [c / pack][n][spatial][pack] and writes y's the same way, whatever the tensors' format says.  Defined for c % pack == 0 only
    (otherwise it reads and writes past both buffers).  pack is the CPU backend's: 16 on an AVX-512 host, 8 on AVX2"""
    x = np.asarray(x, F)
    n, c = x.shape[:2]
    assert c % pack == 0
    sp = x.shape[2:]
    mem = x.reshape(-1)
    seen = mem.reshape((c // pack, n) + sp + (pack,))
    xr = np.moveaxis(seen, -1, 2).swapaxes(0, 1).reshape(x.shape)          # the logical x the packed reading sees
    yr = grid_sample(xr, grid, mode, padding, align_corners, fused)
    osp = yr.shape[2:]
    packed = np.moveaxis(yr.reshape((n, c // pack, pack) + osp), 2, -1).swapaxes(0, 1)
    return np.ascontiguousarray(packed).reshape(yr.shape)                   # its packed bytes, read back as NCHW


def grid_sample64(x, grid, mode="bilinear", padding="zeros", align_corners=False):
    """the same sampling with float64 values and sums (the coordinates, taps and weights as the CPU's)"""
    return grid_sample(x, grid, mode, padding, align_corners, f64=True)


# ---- the live reference: oracle/_ref/refdump_grid_sample (oracle/refdump_grid_sample.cpp over oracle/_ref/libMNN.so), built by build()
HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(HERE, "_ref")
REFDUMP_GRID_SAMPLE = os.path.join(REF_DIR, "refdump_grid_sample")
FLOW = os.path.join(REF_DIR, "flow_f32.mnn")
LUT = os.path.join(REF_DIR, "lut_f32.mnn")
FLOW_SEED, LUT_SEED = 41, 42


def have_refdump():
    return os.path.exists(REFDUMP_GRID_SAMPLE)


def host_fused():
    """whether the reference CPU of this host runs the AVX-512 (fused) GridSample tables"""
    try:
        flags = open("/proc/cpuinfo").read()
    except OSError:
        return False
    return all(f in flags.split() for f in ("avx512f", "avx512bw", "avx512dq", "avx512vl"))


def build_refdump():
    """compile oracle/refdump_grid_sample.cpp against the reference build of oracle/build_ref.py (where the reference sources are)
    and write the flow-warp and 3D-LUT fixtures with it"""
    from oracle import build_ref as B
    src = os.path.join(HERE, "refdump_grid_sample.cpp")
    lib = os.path.join(REF_DIR, "libMNN.so")
    fresh = have_refdump() and all(os.path.getmtime(REFDUMP_GRID_SAMPLE) > os.path.getmtime(d) for d in (src, lib))
    if not fresh:
        cmd = ["g++", "-O2", "-std=gnu++11", "-w", "-o", REFDUMP_GRID_SAMPLE, src] + \
              ["-I" + os.path.join(B.REF, i) for i in B.INCLUDES] + ["-L" + REF_DIR, "-lMNN", "-Wl,-rpath,$ORIGIN", "-pthread", "-ldl"]
        subprocess.check_call(cmd)
    for path, cmd, seed in ((FLOW, "flow", FLOW_SEED), (LUT, "lut", LUT_SEED)):
        if not fresh or not os.path.exists(path):
            _run([cmd, path, seed])


def _run(args, plugin=None):
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = REF_DIR + ":" + env.get("LD_LIBRARY_PATH", "")
    env.pop("REFDUMP_PLUGIN", None)
    if plugin:
        env["REFDUMP_PLUGIN"] = plugin
    return subprocess.run([REFDUMP_GRID_SAMPLE] + [str(a) for a in args], env=env, capture_output=True, text=True, timeout=600,
                          check=True)


def ref_grid_sample(x, grid, mode="bilinear", padding="zeros", align_corners=False, more=None, plugin=None, linear_x=False):
    """y (NCHW float32) of one reference GridSample op on MNN_FORWARD_CPU.  linear_x: hand x to the op in its NCHW layout instead
    of the NC4HW4 the model converter gives it.  more: a list of further (x, grid) pairs run through
    the same executor after the first (all outputs returned, stacked).  plugin: run on MNN_FORWARD_CUDA with that plugin, and
    (ys, the plugin's stats) returned"""
    x, grid = np.ascontiguousarray(x, F), np.ascontiguousarray(grid, F)
    rank = x.ndim
    xd = x.shape if rank == 5 else x.shape[:2] + (1,) + x.shape[2:]
    gd = grid.shape[1:-1] if rank == 5 else (1,) + grid.shape[1:-1]
    sets = [(x, grid)] + [(np.ascontiguousarray(a, F), np.ascontiguousarray(g, F)) for a, g in (more or [])]
    hdr = struct.pack("<14i", rank, xd[0], xd[1], xd[2], xd[3], xd[4], gd[0], gd[1], gd[2], MODES.get(mode, mode),
                      PADDINGS.get(padding, padding), int(align_corners), len(sets), int(linear_x))
    body = b"".join(a.tobytes() + g.tobytes() for a, g in sets)
    with tempfile.TemporaryDirectory() as d:
        req, out = os.path.join(d, "req"), os.path.join(d, "out")
        open(req, "wb").write(hdr + body)
        r = _run(["op", req, out], plugin)
        raw = open(out, "rb").read()
    rk = struct.unpack("<i", raw[:4])[0]
    dims = struct.unpack(f"<{rk}i", raw[4:4 + 4 * rk])
    ys = np.frombuffer(raw[4 + 4 * rk:], F).reshape((len(sets),) + dims).copy()
    ys = ys[0] if more is None else ys
    if plugin is None:
        return ys
    stats = [json.loads(line) for line in r.stdout.splitlines() if line.startswith('{"plugin_')]
    return ys, (stats[-1] if stats else None)
