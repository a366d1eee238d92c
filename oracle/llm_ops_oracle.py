"""Restatement of MNN-LLM's LayerNorm / RMSNorm and fused RoPE (CPULayerNorm, CPURoPE + MNNRoPEComputeBasic), the error bound
of their fp32 arithmetic, and the front-end of the reference harness oracle/_ref/refdump_llm (oracle/refdump_llm.cpp).

TEST INFRASTRUCTURE ONLY, like oracle/oracle.py: mnn_b200 (the product) never imports this module.

Norms reduce in another order on every implementation (the CPU in SIMD lanes, the kernels in a tree), so they are compared with
`norm_bound`.  The RoPE rotation is a fixed sequence of rounded fp32 operations: `rope_f32` repeats it bit for bit.
"""
import os
import struct
import subprocess
import tempfile

import numpy as np

from oracle import oracle as O

REFDUMP_LLM = os.path.join(O.REF_DIR, "refdump_llm")
U = 2.0 ** -24   # unit roundoff of fp32


def have_reference():
    return os.path.exists(REFDUMP_LLM) and os.path.exists(os.path.join(O.REF_DIR, "libMNN_fuse.so"))


def rope_dim(head_dim, rope_cut):
    """CPURoPE.cpp:176-180: rope_cut_head_dim in (0, head_dim], else head_dim, rounded down to even"""
    return (rope_cut if 0 < rope_cut <= head_dim else head_dim) // 2 * 2


# ---------------------------------------------------------------------------------------------------------------- inputs
def codes(shape, seed):
    """int8 codes in [-127, 127] from an integer hash of (element index, seed): the same on every machine and numpy version, so
    the recorded cases keep only their seed"""
    i = np.arange(int(np.prod(shape)), dtype=np.uint64)
    m = np.uint64(0xFFFFFFFF)
    h = (i * np.uint64(0x9E3779B1) + np.uint64(seed) * np.uint64(0x85EBCA77)) & m
    for mul, sh in ((0x2C1B3C6D, 12), (0x297A2D39, 15), (0x7FEB352D, 13)):
        h ^= h >> np.uint64(sh)
        h = (h * np.uint64(mul)) & m
    return ((h % np.uint64(255)).astype(np.int64) - 127).astype(np.int8).reshape(shape)


def norm_inputs(dims, inner, seed, offset, residual, rms, has_gamma, has_beta):
    """x (codes / 32 + offset), r (codes / 64, the residual form), gamma (1 + codes / 256) and beta (codes / 256, zeros for
    RMSNorm): exact in fp32"""
    x = codes(dims, seed).astype(np.float32) * np.float32(2.0 ** -5) + np.float32(offset)
    r = codes(dims, seed + 1).astype(np.float32) * np.float32(2.0 ** -6) if residual else None
    gamma = 1 + codes(inner, seed + 2).astype(np.float32) * np.float32(2.0 ** -8) if has_gamma else None
    beta = None
    if has_beta:
        beta = np.zeros(inner, np.float32) if rms else codes(inner, seed + 3).astype(np.float32) * np.float32(2.0 ** -8)
    return x, r, gamma, beta


def rope_inputs(seq, heads, kv_heads, head_dim, seed):
    """q, k (codes / 16) and the q / k norm gammas (1 + codes / 256)"""
    q = codes((seq, heads * head_dim), seed).astype(np.float32) * np.float32(2.0 ** -4)
    k = codes((seq, kv_heads * head_dim), seed + 1).astype(np.float32) * np.float32(2.0 ** -4)
    qg = 1 + codes(head_dim, seed + 2).astype(np.float32) * np.float32(2.0 ** -8)
    kg = 1 + codes(head_dim, seed + 3).astype(np.float32) * np.float32(2.0 ** -8)
    return q, k, qg, kg


def digest(a):
    """sha256 of an fp32 array's bytes: a bit-exact output recorded without its values"""
    import hashlib
    return hashlib.sha256(np.ascontiguousarray(a, np.float32).tobytes()).hexdigest()


# ---------------------------------------------------------------------------------------------------------------- LayerNorm
def norm64(x, eps, rms, gamma=None, beta=None):
    """MNNNorm over the last axis of x in float64: mean (0 for RMSNorm), var = mean((x - mean)^2), y = (x - mean) / sqrt(var + eps),
    then y * gamma + beta only when both are given (CPULayerNorm.cpp:35)"""
    x = np.asarray(x, np.float64)
    mean = np.zeros(x.shape[:-1] + (1,)) if rms else x.mean(-1, keepdims=True)
    var = ((x - mean) ** 2).mean(-1, keepdims=True)
    y = (x - mean) / np.sqrt(var + float(np.float32(eps)))
    if gamma is not None and beta is not None:
        y = y * np.asarray(gamma, np.float64) + np.asarray(beta, np.float64)
    return y


def norm_bound(x, eps, rms, gamma=None, beta=None, terms=None):
    """Per-element bound on |y_fp32 - y_exact| for an fp32 norm whose sums carry at most `terms` rounded additions in a chain
    (the kernels: 4V per thread + 10 tree levels; the CPU: one per element of the row, `terms` = inner).  With L = terms + 2:
      mean:   |m - m*| <= dm = L u sum|x| / n                               (sum, then the division)
      inv:    relative error rho = (L + 9) u / 2 + dm^2 / (2 (var* + eps))  (sum of squares of rounded differences, / n, + eps,
              sqrt, reciprocal; a mean off by dm adds n dm^2 to the sum of squares)
      t = (x - m) inv:  |t - t*| <= inv* dm + |t*| (rho + 3u)
      y = t g + b:      |y - y*| <= |g| |t - t*| + 2u (|t* g| + |b|)
    doubled for the second-order terms this drops."""
    x = np.asarray(x, np.float64)
    n = x.shape[-1]
    L = (n if terms is None else terms) + 2
    mean = np.zeros(x.shape[:-1] + (1,)) if rms else x.mean(-1, keepdims=True)
    var = ((x - mean) ** 2).mean(-1, keepdims=True)
    e = float(np.float32(eps))
    inv = 1.0 / np.sqrt(var + e)
    dm = 0.0 if rms else L * U * np.abs(x).sum(-1, keepdims=True) / n
    rho = (L + 9) * U / 2 + dm ** 2 / (2 * (var + e))
    t = (x - mean) * inv
    dt = inv * dm + np.abs(t) * (rho + 3 * U)
    if gamma is not None and beta is not None:
        g, b = np.abs(np.asarray(gamma, np.float64)), np.abs(np.asarray(beta, np.float64))
        return 2 * (g * dt + 2 * U * (np.abs(t) * g + b))
    return 2 * (dt + 2 * U * np.abs(t))


def kernel_terms(inner):
    """the longest chain of rounded additions in layernorm_f32_kernel's reductions: 4V values per thread, then 5 + 5 tree levels"""
    n4, v = (inner + 3) // 4, 1
    while v < 16 and (n4 + v - 1) // v > 256:
        v *= 2
    return 4 * v + 10


# ---------------------------------------------------------------------------------------------------------------- RoPE
def rope64(x, cos, sin, head_dim, rope_cut, norm=None):
    """x [seq][heads * head_dim] -> [seq][heads][head_dim] in float64; norm = (gamma, beta or None, eps, rms) applied per head first
    (beta None: zeros, CPURoPE.cpp:43-47)"""
    seq = x.shape[0]
    h = np.asarray(x, np.float64).reshape(seq, -1, head_dim)
    if norm is not None:
        g, b, eps, rms = norm
        h = norm64(h, eps, rms, g, np.zeros(head_dim) if b is None else b)
    rd = rope_dim(head_dim, rope_cut)
    half = rd // 2
    c = np.asarray(cos, np.float64).reshape(seq, 1, rd)
    s = np.asarray(sin, np.float64).reshape(seq, 1, rd)
    out = h.copy()
    x0, x1 = h[..., :half], h[..., half:rd]
    out[..., :half] = x0 * c[..., :half] - x1 * s[..., :half]
    out[..., half:rd] = x1 * c[..., half:] + x0 * s[..., half:]
    return out


def rope_f32(x, cos, sin, head_dim, rope_cut):
    """MNNRoPEComputeBasic in fp32, the CPU's operation order (each product rounded, then the difference / sum): bit-exact"""
    seq = x.shape[0]
    h = np.asarray(x, np.float32).reshape(seq, -1, head_dim)
    rd = rope_dim(head_dim, rope_cut)
    half = rd // 2
    c = np.asarray(cos, np.float32).reshape(seq, 1, rd)
    s = np.asarray(sin, np.float32).reshape(seq, 1, rd)
    out = h.copy()
    x0, x1 = h[..., :half], h[..., half:rd]
    out[..., :half] = (x0 * c[..., :half]) - (x1 * s[..., :half])
    out[..., half:rd] = (x1 * c[..., half:]) + (x0 * s[..., half:])
    return out


def rope_norm_bound(x, cos, sin, head_dim, rope_cut, norm, terms=None):
    """bound on |out_fp32 - out_exact| of a normalised RoPE: the norm's bound on each operand carried through the rotation, plus
    the rotation's own rounding 2u (|x0 c| + |x1 s|) (and the copied dims' norm bound)"""
    seq = x.shape[0]
    h = np.asarray(x, np.float64).reshape(seq, -1, head_dim)
    g, b, eps, rms = norm
    b = np.zeros(head_dim) if b is None else b
    e = norm_bound(h, eps, rms, g, b, terms)
    v = np.abs(norm64(h, eps, rms, g, b))
    rd = rope_dim(head_dim, rope_cut)
    half = rd // 2
    c = np.abs(np.asarray(cos, np.float64)).reshape(seq, 1, rd)
    s = np.abs(np.asarray(sin, np.float64)).reshape(seq, 1, rd)
    out = e.copy()
    e0, e1, v0, v1 = e[..., :half], e[..., half:rd], v[..., :half], v[..., half:rd]
    out[..., :half] = e0 * c[..., :half] + e1 * s[..., :half] + 2 * U * (v0 * c[..., :half] + v1 * s[..., :half]) * 2
    out[..., half:rd] = e1 * c[..., half:] + e0 * s[..., half:] + 2 * U * (v1 * c[..., half:] + v0 * s[..., half:]) * 2
    return out


# ---------------------------------------------------------------------------------------------------------------- harness
def layernorm_request(runs, dims, eps, rms, form=0, axis=1, group=1, gamma=None, beta=None):
    """refdump_llm request for a LayerNorm; runs = [x] or [x, r] per run (form 2: the NC4HW4 residual form)"""
    affine = len(gamma) if gamma is not None else (len(beta) if beta is not None else 0)
    dims = list(dims) + [0] * (4 - len(dims))
    hdr = struct.pack("<14if", 0, len(runs), form, len([d for d in dims if d]), *dims, axis, group, int(rms),
                      int(gamma is not None), int(beta is not None), affine, eps)
    hdr += struct.pack("<9if", *([0] * 9), 0.0)
    body = b"".join(np.ascontiguousarray(a, np.float32).tobytes() for a in (gamma, beta) if a is not None)
    for run in runs:
        body += b"".join(np.ascontiguousarray(a, np.float32).tobytes() for a in run)
    return hdr + body


def rope_request(runs, heads, kv_heads, head_dim, rope_cut, q_norm=None, k_norm=None, norm_rms=1, norm_eps=1e-6):
    """refdump_llm request for a RoPE; runs = [(q, k, cos, sin)]; q_norm / k_norm = (gamma, beta or None); the two tables share
    rms and eps, and beta is present in both or neither"""
    seq = runs[0][0].shape[0]
    has_beta = any(n is not None and n[1] is not None for n in (q_norm, k_norm))
    hdr = struct.pack("<14if", 1, len(runs), *([0] * 12), 0.0)
    hdr += struct.pack("<9if", seq, heads, kv_heads, head_dim, rope_cut, int(q_norm is not None), int(k_norm is not None),
                       int(norm_rms), int(has_beta), norm_eps)
    body = b""
    for n in (q_norm, k_norm):
        if n is not None:
            body += np.ascontiguousarray(n[0], np.float32).tobytes()
            if has_beta:
                body += np.ascontiguousarray(n[1], np.float32).tobytes()
    for run in runs:
        body += b"".join(np.ascontiguousarray(a, np.float32).tobytes() for a in run)
    return hdr + body


def run_refdump(payload, env=None, model=None):
    """refdump_llm on a request: (every run's outputs as one float32 array, stdout)"""
    if env is None:
        env = dict(os.environ)
        env["LD_LIBRARY_PATH"] = O.REF_DIR + ":" + env.get("LD_LIBRARY_PATH", "")
    with tempfile.TemporaryDirectory() as d:
        req, out = os.path.join(d, "req.bin"), os.path.join(d, "out.bin")
        open(req, "wb").write(payload)
        r = subprocess.run([REFDUMP_LLM, req, out] + ([model] if model else []), env=env, capture_output=True, text=True,
                           timeout=600)
        assert r.returncode == 0, r.stderr[-1500:]
        return np.fromfile(out, np.float32), r.stdout
