"""MNN-LLM's LayerNorm / RMSNorm and fused RoPE without a device: the restatement (oracle/llm_ops_oracle.py) against the outputs
recorded from the reference CPU backend (tests/golden/llm_norm_rope_golden.npz), and the C ABI's refusals of NULL handles
(libmnn_b200_llm.so).

Every recorded norm output lies within norm_bound of the float64 restatement, with the CPU's chain of one rounded addition per
element of the row; the residual form's sum x + r is exact; RoPE without q / k norms equals the fp32 restatement in the CPU's
operation order bit for bit, and with norms lies within rope_norm_bound."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import llm_ops_oracle as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "llm_norm_rope_golden.npz")
INVALID_VALUE = 5


def _golden():
    return np.load(GOLDEN)


def norm_cases():
    """[(name, dict)] of the recorded norms: x (inputs rebuilt from the case's seed), r, dims, form, axis, group, rms, eps,
    gamma, beta, the rows kept and their recorded y, the sha256 of the recorded sum x + r"""
    g = _golden()
    out = []
    for name in sorted({k.split("/")[0] for k in g.files if "/" in k and not k.startswith("rope")}):
        form, axis, group, rms, hg, hb, rows, inner, seed = (int(v) for v in g[f"{name}/meta"][:9])
        dims = tuple(int(d) for d in g[f"{name}/meta"][9:] if d)
        x, r, gamma, beta = L.norm_inputs(dims, inner, seed, float(g[f"{name}/offset"]), form == 2, rms, hg, hb)
        out.append((name, dict(form=form, axis=axis, group=group, rms=rms, rows=rows, inner=inner, dims=dims,
                               eps=float(g[f"{name}/eps"]), gamma=gamma, beta=beta, keep=g[f"{name}/rows"], y=g[f"{name}/y"],
                               x=x, r=r, sum_sha256=str(g[f"{name}/sum_sha256"]) if form == 2 else None)))
    return out


def rope_cases():
    """[(name, dict)] of the recorded RoPEs: q, k (rebuilt from the seed), cos, sin, seq, heads, kv_heads, head_dim, rope_cut,
    q / k norms; without norms the sha256 of the recorded q_out / k_out, with them the tokens kept and their outputs"""
    g = _golden()
    out = []
    for name in sorted({k.split("/")[0] for k in g.files if k.startswith("rope")}):
        seq, heads, kvh, hd, cut, norm, seed = (int(v) for v in g[f"{name}/meta"])
        q, k, qg, kg = L.rope_inputs(seq, heads, kvh, hd, seed)
        rd = L.rope_dim(hd, cut)
        c = dict(seq=seq, heads=heads, kv_heads=kvh, head_dim=hd, rope_cut=cut, q=q, k=k, cos=g[f"cos_{rd}"][:seq],
                 sin=g[f"sin_{rd}"][:seq], q_norm=(qg, None, 1e-6, 1) if norm else None, k_norm=(kg, None, 1e-6, 1) if norm else None)
        if norm:
            c.update(keep=g[f"{name}/rows"], q_out=g[f"{name}/q_out"], k_out=g[f"{name}/k_out"])
        else:
            c.update(q_sha256=str(g[f"{name}/q_sha256"]), k_sha256=str(g[f"{name}/k_sha256"]))
        out.append((name, c))
    return out


def test_golden_covers_the_cases():
    names = [n for n, _ in norm_cases()] + [n for n, _ in rope_cases()]
    assert len(names) == 18
    forms = {c["form"] for _, c in norm_cases()}
    assert forms == {0, 1, 2}
    assert {c["inner"] for _, c in norm_cases() if c["rms"]} >= {2048, 256}


@pytest.mark.parametrize("name,c", norm_cases(), ids=lambda v: v if isinstance(v, str) else "")
def test_norm_restatement_within_bound_of_reference(name, c):
    x = c["x"].reshape(c["rows"], c["inner"])
    if c["form"] == 2:
        s = (x + c["r"].reshape(c["rows"], c["inner"])).astype(np.float32)
        assert L.digest(s) == c["sum_sha256"], "the residual sum is one rounded addition"
        x = s
    ref = L.norm64(x, c["eps"], c["rms"], c["gamma"], c["beta"])[c["keep"]]
    bound = L.norm_bound(x, c["eps"], c["rms"], c["gamma"], c["beta"], terms=c["inner"])[c["keep"]]
    err = np.abs(c["y"] - ref)
    assert (err <= bound).all(), f"{name}: worst {float((err - bound).max())} past the bound"


def test_gamma_without_beta_is_ignored():
    """rms_gamma_only carries a gamma and no beta: the CPU normalises without the affine transform"""
    c = dict(norm_cases())["rms_gamma_only"]
    assert c["gamma"] is not None and c["beta"] is None
    x = c["x"].reshape(c["rows"], c["inner"])
    plain = L.norm64(x, c["eps"], 1)
    scaled = plain * c["gamma"]
    assert np.abs(c["y"] - plain).max() < 1e-5 < np.abs(c["y"] - scaled).max()


@pytest.mark.parametrize("name,c", rope_cases(), ids=lambda v: v if isinstance(v, str) else "")
def test_rope_restatement_matches_reference(name, c):
    hd, cut = c["head_dim"], c["rope_cut"]
    for side in ("q", "k"):
        if c[f"{side}_norm"] is None:
            got = L.rope_f32(c[side], c["cos"], c["sin"], hd, cut)
            assert L.digest(got) == c[f"{side}_sha256"], f"{name} {side}: not bit-exact"
            assert np.abs(L.rope64(c[side], c["cos"], c["sin"], hd, cut) - got).max() < 1e-5
        else:
            rec = c[f"{side}_out"]
            nm = c[f"{side}_norm"]
            ref = L.rope64(c[side], c["cos"], c["sin"], hd, cut, nm)[c["keep"]]
            bound = L.rope_norm_bound(c[side], c["cos"], c["sin"], hd, cut, nm, terms=hd)[c["keep"]]
            assert (np.abs(rec - ref) <= bound).all(), f"{name} {side}"


def test_rope_dim_rule():
    assert [L.rope_dim(128, c) for c in (0, -1, 64, 63, 128, 129, 1)] == [128, 128, 64, 62, 128, 128, 0]


def test_null_handles_refused_without_a_device():
    from mnn_b200 import _capi
    lib = _capi.llm_lib()
    h = C.c_void_p()
    assert lib.mnnb200_layernorm_f32_create(None, 2048, 1e-6, 1, None, None, 0, C.byref(h)) == INVALID_VALUE
    assert lib.mnnb200_rope_f32_create(None, 16, 16, 128, 0, None, None, C.byref(h)) == INVALID_VALUE
    assert lib.mnnb200_layernorm_f32_resize(None, 4) == INVALID_VALUE
    assert lib.mnnb200_layernorm_f32_execute(None, None, None, None, None) == INVALID_VALUE
    assert lib.mnnb200_rope_f32_resize(None, 4, 2048, 2048) == INVALID_VALUE
    assert lib.mnnb200_rope_f32_execute(None, None, None, None, None, None, None) == INVALID_VALUE
