"""LayerNorm / RMSNorm and the fused RoPE on the GPU (-m gpu): the C ABI against float64, and the plugin under the reference's
unmodified Interpreter against the outputs recorded from its CPU backend.

Every norm output must lie within norm_bound (oracle/llm_ops_oracle.py) of float64 for the kernel's chain of rounded additions
(kernel_terms: 4V values per thread, then 10 tree levels); RoPE without q / k norms must equal the fp32 restatement in the CPU's
operation order bit for bit, and a normalised RoPE lie within rope_norm_bound.  Inputs sit between NaN guard bands, 4 bytes past
16-byte alignment where a case asks for the scalar path; outputs sit in NaN-filled buffers with guard bands, so an unwritten
element or a write outside the tensor shows."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from oracle import llm_ops_oracle as L
from oracle import oracle as O
from tests.test_llm_ops_cpu import norm_cases, rope_cases

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PLUGIN = os.path.join(ROOT, "mnn_b200", "libmnn_b200_plugin.so")
NOT_SUPPORT, NO_EXECUTION, INVALID_VALUE = 2, 4, 5
GUARD = 1024   # NaN floats either side of every tensor (+1 for a misaligned one)


def lib():
    """libmnn_b200_llm.so (include/mnn_b200_llm.h)"""
    from mnn_b200 import _capi
    return _capi.llm_lib()


def core():
    """libmnn_b200.so, whose handles and error message the LLM ops share"""
    from mnn_b200 import _capi
    return _capi.lib()


def err_msg():
    return core().mnnb200_last_error().decode()


class Guarded:
    """a device fp32 tensor in a NaN-filled buffer with GUARD floats either side; misalign puts it 4 bytes past 16-byte alignment"""

    def __init__(self, host=None, n=None, misalign=False):
        import torch
        self.n = int(host.size if host is not None else n)
        self.off = GUARD + (1 if misalign else 0)
        self.buf = torch.full((self.off + self.n + GUARD,), float("nan"), dtype=torch.float32, device="cuda")
        if host is not None:
            self.buf[self.off:self.off + self.n] = torch.from_numpy(np.ascontiguousarray(host, np.float32).ravel()).cuda()

    @property
    def ptr(self):
        return C.c_void_p(self.buf.data_ptr() + 4 * self.off)

    def get(self):
        """the tensor's values; the guard bands must still be NaN"""
        h = self.buf.cpu().numpy()
        assert np.isnan(h[:self.off]).all() and np.isnan(h[self.off + self.n:]).all(), "a write outside the tensor"
        return h[self.off:self.off + self.n]


def sync(backend):
    backend.onSync()


# ---------------------------------------------------------------------------------------------------------------- LayerNorm
def norm_create(backend, inner, eps, rms, gamma=None, beta=None):
    h = C.c_void_p()
    g = np.ascontiguousarray(gamma, np.float32) if gamma is not None else None
    b = np.ascontiguousarray(beta, np.float32) if beta is not None else None
    size = len(g) if g is not None else 0
    st = lib().mnnb200_layernorm_f32_create(backend.runtime._h, inner, eps, rms, g.ctypes.data if g is not None else None,
                                            b.ctypes.data if b is not None else None, size, C.byref(h))
    return st, h


def norm_run(backend, h, x, r=None, misalign=False):
    """execute an already resized execution on x (and r): (y, sum or None) as host arrays, guard bands checked"""
    dx = Guarded(x, misalign=misalign)
    dr = Guarded(r, misalign=misalign) if r is not None else None
    ds = Guarded(n=x.size, misalign=misalign) if r is not None else None
    dy = Guarded(n=x.size, misalign=misalign)
    st = lib().mnnb200_layernorm_f32_execute(h, dx.ptr, dr.ptr if dr else None, ds.ptr if ds else None, dy.ptr)
    assert st == 0, err_msg()
    sync(backend)
    return dy.get().reshape(x.shape), (ds.get().reshape(x.shape) if ds else None)


def norm_check(x, y, eps, rms, gamma, beta, what, s=None, r=None):
    inner = x.shape[-1]
    if r is not None:
        exact = (x + r).astype(np.float32)
        assert np.array_equal(s, exact), f"{what}: the sum x + r"
        x = exact
    assert np.isfinite(y).all(), f"{what}: an output left unwritten"
    ref = L.norm64(x, eps, rms, gamma, beta)
    bound = L.norm_bound(x, eps, rms, gamma, beta, terms=L.kernel_terms(inner))
    err = np.abs(y - ref)
    assert (err <= bound).all(), f"{what}: worst {float((err - bound).max())} past the bound, max err {float(err.max())}"


def norm_data(rng, rows, inner, offset=0.0, affine=True, rms=True):
    x = (rng.standard_normal((rows, inner)) * 1.5 + offset).astype(np.float32)
    gamma = rng.uniform(0.5, 1.5, inner).astype(np.float32) if affine else None
    beta = (np.zeros(inner, np.float32) if rms else rng.uniform(-0.5, 0.5, inner).astype(np.float32)) if affine else None
    return x, gamma, beta


# inner, rows, rms, affine, residual, misalign
NORM_SWEEP = [
    (2048, 1, 1, True, False, False), (2048, 8, 1, True, True, False), (2048, 4096, 1, True, False, False),
    (2048, 4096, 1, True, True, False), (2048, 3, 0, True, False, True), (5504, 5, 1, True, False, False),
    (5504, 2, 0, False, True, True), (8192, 4, 1, True, True, False), (8192, 64, 0, True, False, False),
    (16384, 3, 1, True, False, False), (16384, 2, 0, True, True, True), (2050, 7, 1, True, False, False),
    (2050, 5, 0, True, True, False), (768, 9, 0, True, False, True), (33, 17, 0, False, False, False),
    (1, 6, 1, False, False, False), (32768, 2, 1, True, False, False), (4096, 3, 0, True, True, False),
    (1024, 5, 1, True, False, False),
]


@pytest.mark.parametrize("inner,rows,rms,affine,residual,misalign", NORM_SWEEP)
def test_layernorm_against_float64(backend, inner, rows, rms, affine, residual, misalign):
    rng = np.random.default_rng(inner * 7 + rows)
    x, gamma, beta = norm_data(rng, rows, inner, offset=0.0 if rms else 2.0, affine=affine, rms=rms)
    r = (rng.standard_normal((rows, inner)) * 0.5).astype(np.float32) if residual else None
    st, h = norm_create(backend, inner, 1e-6 if rms else 1e-5, rms, gamma, beta)
    assert st == 0, err_msg()
    try:
        assert lib().mnnb200_layernorm_f32_resize(h, rows) == 0, err_msg()
        y, s = norm_run(backend, h, x, r, misalign)
        norm_check(x, y, 1e-6 if rms else 1e-5, rms, gamma, beta, f"inner {inner} rows {rows}", s, r)
    finally:
        core().mnnb200_exec_destroy(h)


def test_layernorm_gamma_without_beta_is_ignored(backend):
    rng = np.random.default_rng(5)
    x, gamma, _ = norm_data(rng, 4, 256)
    st, h = norm_create(backend, 256, 1e-6, 1, gamma, None)
    assert st == 0, err_msg()
    try:
        assert lib().mnnb200_layernorm_f32_resize(h, 4) == 0
        y, _ = norm_run(backend, h, x)
        norm_check(x, y, 1e-6, 1, None, None, "gamma alone")
    finally:
        core().mnnb200_exec_destroy(h)


def test_layernorm_one_execution_resized_across_row_counts(backend):
    rng = np.random.default_rng(11)
    x, gamma, beta = norm_data(rng, 4096, 2048)
    r = (rng.standard_normal(x.shape) * 0.5).astype(np.float32)
    st, h = norm_create(backend, 2048, 1e-6, 1, gamma, beta)
    assert st == 0
    try:
        for rows in (1, 4096, 7, 512, 1):
            assert lib().mnnb200_layernorm_f32_resize(h, rows) == 0, err_msg()
            y, s = norm_run(backend, h, x[:rows], r[:rows])
            norm_check(x[:rows], y, 1e-6, 1, gamma, beta, f"resized to {rows}", s, r[:rows])
    finally:
        core().mnnb200_exec_destroy(h)


def test_layernorm_refusals_keep_the_previous_plan(backend):
    rng = np.random.default_rng(12)
    x, gamma, beta = norm_data(rng, 3, 2048)
    assert norm_create(backend, 2048, 1e-6, 1, gamma[:2047], beta[:2047])[0] == NOT_SUPPORT       # gamma size != inner
    assert norm_create(backend, 32772, 1e-6, 1)[0] == NOT_SUPPORT                                  # the row does not fit
    st, h = norm_create(backend, 2048, 1e-6, 1, gamma, beta)
    assert st == 0
    try:
        y0 = Guarded(n=x.size)
        assert lib().mnnb200_layernorm_f32_execute(h, Guarded(x).ptr, None, None, y0.ptr) == NO_EXECUTION
        assert lib().mnnb200_layernorm_f32_resize(h, 3) == 0
        assert lib().mnnb200_layernorm_f32_resize(h, 0) == NOT_SUPPORT                             # zero rows
        assert lib().mnnb200_layernorm_f32_resize(h, (1 << 31) // 2048 + 1) == NOT_SUPPORT          # past 32-bit indexing
        dx = Guarded(x)
        assert lib().mnnb200_layernorm_f32_execute(h, dx.ptr, dx.ptr, None, y0.ptr) == INVALID_VALUE  # residual without sum
        y, _ = norm_run(backend, h, x)                                                             # the plan of resize(3)
        norm_check(x, y, 1e-6, 1, gamma, beta, "after refusals")
    finally:
        core().mnnb200_exec_destroy(h)


# ---------------------------------------------------------------------------------------------------------------- RoPE
def rope_create(backend, heads, kvh, hd, cut, q_norm=None, k_norm=None):
    from mnn_b200 import _capi
    keep, tabs = [], []
    for n in (q_norm, k_norm):
        if n is None:
            tabs.append(None)
            continue
        g = np.ascontiguousarray(n[0], np.float32)
        b = np.ascontiguousarray(n[1], np.float32) if n[1] is not None else None
        keep += [g, b]
        t = _capi.RopeNorm(g.ctypes.data, b.ctypes.data if b is not None else None, len(g), n[2], n[3])
        keep.append(t)
        tabs.append(C.byref(t))
    h = C.c_void_p()
    st = lib().mnnb200_rope_f32_create(backend.runtime._h, heads, kvh, hd, cut, tabs[0], tabs[1], C.byref(h))
    return st, h


def rope_run(backend, h, q, k, cos, sin, misalign=False):
    dq, dk, dc, ds = (Guarded(a, misalign=misalign) for a in (q, k, cos, sin))
    qo, ko = Guarded(n=q.size, misalign=misalign), Guarded(n=k.size, misalign=misalign)
    assert lib().mnnb200_rope_f32_execute(h, dq.ptr, dk.ptr, dc.ptr, ds.ptr, qo.ptr, ko.ptr) == 0, err_msg()
    sync(backend)
    return qo.get(), ko.get()


def rope_check(side, x, cos, sin, hd, cut, norm, got, what):
    seq = x.shape[0]
    got = got.reshape(seq, -1, hd)
    assert np.isfinite(got).all(), f"{what} {side}: an output left unwritten"
    if norm is None:
        ref = L.rope_f32(x, cos, sin, hd, cut)
        assert np.array_equal(got.view(np.int32), ref.view(np.int32)), f"{what} {side}: not bit-exact"
    else:
        ref = L.rope64(x, cos, sin, hd, cut, norm)
        bound = L.rope_norm_bound(x, cos, sin, hd, cut, norm, terms=(hd + 31) // 32 + 5)
        assert (np.abs(got - ref) <= bound).all(), f"{what} {side}: past the bound"


def rope_data(rng, seq, heads, kvh, hd, cut, first=0):
    rd = L.rope_dim(hd, cut)
    inv = 10000.0 ** (-np.arange(0, rd, 2, dtype=np.float64) / max(rd, 1))
    ang = np.arange(first, first + seq, dtype=np.float64)[:, None] * inv[None, :]
    ang = np.concatenate([ang, ang], 1)
    q = rng.standard_normal((seq, heads * hd)).astype(np.float32)
    k = rng.standard_normal((seq, kvh * hd)).astype(np.float32)
    return q, k, np.cos(ang).astype(np.float32), np.sin(ang).astype(np.float32)


@pytest.mark.parametrize("name,c", rope_cases(), ids=lambda v: v if isinstance(v, str) else "")
def test_rope_golden_cases(backend, name, c):
    """the recorded cases through the C ABI: the CPU's outputs bit for bit without norms, within the bound with them"""
    st, h = rope_create(backend, c["heads"], c["kv_heads"], c["head_dim"], c["rope_cut"], c["q_norm"], c["k_norm"])
    assert st == 0, err_msg()
    try:
        hd = c["head_dim"]
        assert lib().mnnb200_rope_f32_resize(h, c["seq"], c["heads"] * hd, c["kv_heads"] * hd) == 0, err_msg()
        qo, ko = rope_run(backend, h, c["q"], c["k"], c["cos"], c["sin"])
        for side, got in (("q", qo), ("k", ko)):
            rope_check(side, c[side], c["cos"], c["sin"], hd, c["rope_cut"], c[f"{side}_norm"], got, name)
            if c[f"{side}_norm"] is None:
                assert L.digest(got) == c[f"{side}_sha256"], f"{name} {side}: differs from the CPU"
    finally:
        core().mnnb200_exec_destroy(h)


# seq, heads, kv_heads, head_dim, rope_cut, norms (None / "rms" / "ln"), misalign
ROPE_SWEEP = [
    (4096, 16, 16, 128, 0, None, False), (4096, 12, 2, 128, 0, None, False), (3, 16, 16, 128, 0, None, True),
    (5, 12, 2, 128, 63, None, True), (9, 4, 4, 64, 32, None, False), (7, 8, 2, 96, 0, None, False),
    (2, 4, 1, 80, 0, None, False), (1, 2, 1, 256, 0, "rms", False), (33, 16, 8, 128, 0, "rms", True),
    (6, 8, 4, 128, 64, "ln", False), (4096, 16, 8, 128, 0, "rms", False), (3, 2, 2, 130, 0, "ln", True),
]


@pytest.mark.parametrize("seq,heads,kvh,hd,cut,norm,misalign", ROPE_SWEEP)
def test_rope_against_restatement(backend, seq, heads, kvh, hd, cut, norm, misalign):
    rng = np.random.default_rng(seq * 31 + hd)
    q, k, cos, sin = rope_data(rng, seq, heads, kvh, hd, cut, first=5)
    nq = nk = None
    if norm:
        rms = 1 if norm == "rms" else 0
        nq = (rng.uniform(0.5, 1.5, hd).astype(np.float32), None if rms else rng.uniform(-0.5, 0.5, hd).astype(np.float32), 1e-6, rms)
        nk = (rng.uniform(0.5, 1.5, hd).astype(np.float32), None, 1e-6, rms)
    st, h = rope_create(backend, heads, kvh, hd, cut, nq, nk)
    assert st == 0, err_msg()
    try:
        assert lib().mnnb200_rope_f32_resize(h, seq, heads * hd, kvh * hd) == 0, err_msg()
        qo, ko = rope_run(backend, h, q, k, cos, sin, misalign)
        rope_check("q", q, cos, sin, hd, cut, nq, qo, f"seq {seq} {heads}/{kvh}x{hd}")
        rope_check("k", k, cos, sin, hd, cut, nk, ko, f"seq {seq} {heads}/{kvh}x{hd}")
    finally:
        core().mnnb200_exec_destroy(h)


def test_rope_resized_and_refusals_keep_the_previous_plan(backend):
    rng = np.random.default_rng(21)
    assert rope_create(backend, 0, 2, 128, 0)[0] == NOT_SUPPORT
    assert rope_create(backend, 12, 0, 128, 0)[0] == NOT_SUPPORT
    assert rope_create(backend, 12, 2, 0, 0)[0] == NOT_SUPPORT
    assert rope_create(backend, 12, 2, 128, 0, (np.ones(64, np.float32), None, 1e-6, 1))[0] == NOT_SUPPORT   # norm size != head_dim
    st, h = rope_create(backend, 12, 2, 128, 0)
    assert st == 0
    try:
        for seq in (1, 37, 4096, 2):
            q, k, cos, sin = rope_data(rng, seq, 12, 2, 128, 0, first=seq)
            assert lib().mnnb200_rope_f32_resize(h, seq, 12 * 128, 2 * 128) == 0, err_msg()
            qo, ko = rope_run(backend, h, q, k, cos, sin)
            rope_check("q", q, cos, sin, 128, 0, None, qo, f"resized to {seq}")
            rope_check("k", k, cos, sin, 128, 0, None, ko, f"resized to {seq}")
        assert lib().mnnb200_rope_f32_resize(h, 0, 12 * 128, 2 * 128) == NOT_SUPPORT                # zero tokens
        assert lib().mnnb200_rope_f32_resize(h, 2, 16 * 128, 2 * 128) == NOT_SUPPORT                # a q width of 16 heads
        assert lib().mnnb200_rope_f32_resize(h, 2, 12 * 128, 4 * 128) == NOT_SUPPORT                # a k width of 4 heads
        assert lib().mnnb200_rope_f32_resize(h, (1 << 31) // 1536 + 1, 12 * 128, 2 * 128) == NOT_SUPPORT
        qo, ko = rope_run(backend, h, q, k, cos, sin)                                               # still the seq 2 plan
        rope_check("q", q, cos, sin, 128, 0, None, qo, "after refusals")
        rope_check("k", k, cos, sin, 128, 0, None, ko, "after refusals")
    finally:
        core().mnnb200_exec_destroy(h)


# ---------------------------------------------------------------------------------------------------------------- plugin
def plugin_env():
    if not L.have_reference():
        pytest.skip("the reference core with the fused ops and its harness (oracle/_ref) are not in this snapshot")
    if not os.path.exists(PLUGIN):
        pytest.fail("mnn_b200/libmnn_b200_plugin.so is missing although the reference core is present")
    env = dict(os.environ, REFDUMP_PLUGIN=PLUGIN)
    env["LD_LIBRARY_PATH"] = O.REF_DIR + ":" + os.path.join(ROOT, "mnn_b200") + ":" + env.get("LD_LIBRARY_PATH", "")
    return env


def run_plugin(payload):
    res, out = L.run_refdump(payload, env=plugin_env())
    stats = [json.loads(l) for l in out.splitlines() if l.startswith("{\"plugin_")]
    assert stats, out[-500:]
    assert stats[-1]["plugin_created"] >= 1 and stats[-1]["plugin_declined"] == 0, stats
    return res


@pytest.mark.parametrize("name,c", norm_cases(), ids=lambda v: v if isinstance(v, str) else "")
def test_layernorm_golden_model_on_plugin(name, c):
    """the one-op model through the Interpreter on the plugin, three runSessions: the recorded input (eager), a second input
    (captured into the plugin's CUDA graph) and the recorded input again (graph replay)"""
    rng = np.random.default_rng(len(name))
    x1, r1 = c["x"], c["r"]
    x2 = (c["x"] + rng.standard_normal(c["x"].shape).astype(np.float32)).astype(np.float32)
    r2 = (c["r"] * -0.5).astype(np.float32) if c["r"] is not None else None
    runs = [[a for a in (x, r) if a is not None] for x, r in ((x1, r1), (x2, r2), (x1, r1))]
    res = run_plugin(L.layernorm_request(runs, c["dims"], c["eps"], c["rms"], c["form"], c["axis"], c["group"], c["gamma"], c["beta"]))
    n, per = x1.size, x1.size * (2 if c["form"] == 2 else 1)
    assert res.size == 3 * per
    rows, inner = c["rows"], c["inner"]
    for i, (x, r) in enumerate(((x1, r1), (x2, r2), (x1, r1))):
        out = res[i * per:(i + 1) * per]
        s, y = (out[:n].reshape(rows, inner), out[n:].reshape(rows, inner)) if c["form"] == 2 else (None, out.reshape(rows, inner))
        norm_check(x.reshape(rows, inner), y, c["eps"], c["rms"], c["gamma"], c["beta"], f"{name} run {i + 1}", s,
                   r.reshape(rows, inner) if r is not None else None)
    # run 1 against the recorded CPU values: both within their bounds of float64
    y1 = res[n:per] if c["form"] == 2 else res[:per]
    xs = x1 + r1 if r1 is not None else x1
    xs = xs.reshape(rows, inner).astype(np.float32)
    bound = L.norm_bound(xs, c["eps"], c["rms"], c["gamma"], c["beta"], terms=inner) + \
        L.norm_bound(xs, c["eps"], c["rms"], c["gamma"], c["beta"], terms=L.kernel_terms(inner))
    assert (np.abs(y1.reshape(rows, inner)[c["keep"]] - c["y"]) <= bound[c["keep"]]).all(), f"{name}: vs the CPU"
    assert np.array_equal(res[:per], res[2 * per:]), f"{name}: the replayed run differs from the eager one"


@pytest.mark.parametrize("name,c", rope_cases(), ids=lambda v: v if isinstance(v, str) else "")
def test_rope_golden_model_on_plugin(name, c):
    rng = np.random.default_rng(len(name) + 1)
    hd, cut = c["head_dim"], c["rope_cut"]
    q2 = rng.standard_normal(c["q"].shape).astype(np.float32)
    k2 = rng.standard_normal(c["k"].shape).astype(np.float32)
    inputs = [(c["q"], c["k"]), (q2, k2), (c["q"], c["k"])]
    runs = [(q, k, c["cos"], c["sin"]) for q, k in inputs]
    norm = lambda n: (n[0], n[1]) if n is not None else None
    res = run_plugin(L.rope_request(runs, c["heads"], c["kv_heads"], hd, cut, norm(c["q_norm"]), norm(c["k_norm"]), 1, 1e-6))
    nq, nk = c["q"].size, c["k"].size
    assert res.size == 3 * (nq + nk)
    for i, (q, k) in enumerate(inputs):
        out = res[i * (nq + nk):(i + 1) * (nq + nk)]
        rope_check("q", q, c["cos"], c["sin"], hd, cut, c["q_norm"], out[:nq], f"{name} run {i + 1}")
        rope_check("k", k, c["cos"], c["sin"], hd, cut, c["k_norm"], out[nq:], f"{name} run {i + 1}")
        if i == 0 and c["q_norm"] is None:
            for side, got in (("q", out[:nq]), ("k", out[nq:])):
                assert L.digest(got) == c[f"{side}_sha256"], f"{name} {side}: differs from the CPU"
    assert np.array_equal(res[:nq + nk], res[2 * (nq + nk):]), f"{name}: the replayed run differs from the eager one"
