"""Writes tests/golden/llm_norm_rope_golden.npz: MNN-LLM's LayerNorm / RMSNorm and fused RoPE recorded from the reference CPU
backend (oracle/_ref/refdump_llm over libMNN_fuse.so, oracle/build_ref_fuse.py), each case a one-op .mnn run by its Interpreter.

Inputs are not stored: oracle/llm_ops_oracle.py's norm_inputs / rope_inputs rebuild them from each case's seed (int8 codes from
an integer hash, times a power of two: exact in fp32).  Stored per case: the parameters, the norm output of the rows in
`<case>/rows` (every row, except every 64th of the 512-token norm), the sha256 of the residual form's sum (exact), the sha256 of
every RoPE output without q / k norms (bit-exact), and the tokens in `<case>/rows` of a normalised RoPE (every 9th of 37).
cos / sin are stored once per rotary width (positions 3..39, theta base 10000).

    python tests/golden/make_llm_ops_golden.py      (from the repository root, after __graft_entry__.build())
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import llm_ops_oracle as L  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "llm_norm_rope_golden.npz")

# name: dims, eps, rms, form (0 plain, 1 NC4HW4, 2 NC4HW4 residual), axis, group, affine (gamma+beta / gamma only / none), offset
NORMS = {
    "rms_qwen_t1": ((1, 2048), 1e-6, 1, 0, 1, 1, "gb", 0.0),
    "rms_qwen_t7": ((7, 2048), 1e-6, 1, 0, 1, 1, "gb", 0.0),
    "rms_qwen_t512": ((512, 2048), 1e-6, 1, 0, 1, 1, "gb", 0.0),
    "ln_affine_768": ((9, 768), 1e-5, 0, 0, 1, 1, "gb", 3.0),
    "ln_no_affine": ((5, 3, 40), 1e-5, 0, 0, 2, 1, "", -1.5),
    "rms_gamma_only": ((4, 256), 1e-6, 1, 0, 1, 1, "g", 0.0),
    "ln_group2": ((3, 4, 6, 5), 1e-5, 0, 0, 0, 2, "gb", 0.5),
    "ln_c4": ((6, 1002, 1, 1), 1e-5, 0, 1, 1, 1, "gb", 0.25),
    "rms_residual_t1": ((1, 2048, 1, 1), 1e-6, 1, 2, 1, 1, "gb", 0.0),
    "rms_residual_t5": ((5, 2048, 1, 1), 1e-6, 1, 2, 1, 1, "gb", 0.0),
}
# name: seq, heads, kv_heads, head_dim, rope_cut, q/k RMSNorm
ROPES = {
    "rope_16x128_s1": (1, 16, 16, 128, 0, False),
    "rope_16x128_s37": (37, 16, 16, 128, 0, False),
    "rope_gqa_12_2_s1": (1, 12, 2, 128, 0, False),
    "rope_gqa_12_2_s37": (37, 12, 2, 128, 0, False),
    "rope_cut64_s37": (37, 16, 2, 128, 64, False),
    "rope_cut63_s37": (37, 16, 2, 128, 63, False),
    "rope_qknorm_s1": (1, 16, 8, 128, 0, True),
    "rope_qknorm_s37": (37, 16, 8, 128, 0, True),
}
TABLE_SEQ = 37


def rope_tables(seq, rd, first_pos):
    """rotate-half cos / sin of positions first_pos.. (theta base 10000), as MNN-LLM's cos / sin inputs hold them"""
    inv = 10000.0 ** (-np.arange(0, rd, 2, dtype=np.float64) / rd)
    ang = np.arange(first_pos, first_pos + seq, dtype=np.float64)[:, None] * inv[None, :]
    ang = np.concatenate([ang, ang], 1)
    return np.cos(ang).astype(np.float32), np.sin(ang).astype(np.float32)


def inner_of(dims, form, axis, group):
    n = int(np.prod(dims))
    return dims[1] if form else (n // (dims[0] * group) if group > 1 else int(np.prod(dims[len(dims) - axis:])))


def main():
    assert L.have_reference(), "build oracle/_ref/refdump_llm first (python __graft_entry__.py)"
    out = {}
    for seed, (name, (dims, eps, rms, form, axis, group, affine, offset)) in enumerate(NORMS.items()):
        seed = 100 + 10 * seed
        n, inner = int(np.prod(dims)), inner_of(dims, form, axis, group)
        x, r, gamma, beta = L.norm_inputs(dims, inner, seed, offset, form == 2, rms, "g" in affine, "b" in affine)
        y, _ = L.run_refdump(L.layernorm_request([[x] + ([r] if r is not None else [])], dims, eps, rms, form, axis, group, gamma, beta))
        rows = n // inner
        keep = np.arange(0, rows, 64) if rows >= 512 else np.arange(rows)
        if form == 2:
            s, y = y[:n], y[n:]
            out[f"{name}/sum_sha256"] = np.array(L.digest(s))
        out[f"{name}/y"], out[f"{name}/rows"] = y.reshape(rows, inner)[keep], keep
        out[f"{name}/meta"] = np.array([form, axis, group, rms, int(gamma is not None), int(beta is not None), rows, inner, seed] +
                                       list(dims) + [0] * (4 - len(dims)), np.int64)
        out[f"{name}/eps"], out[f"{name}/offset"] = np.float32(eps), np.float32(offset)
        print(name, rows, inner)
    tables = {}
    for seed, (name, (seq, heads, kvh, hd, cut, norm)) in enumerate(ROPES.items()):
        seed = 500 + 10 * seed
        rd = L.rope_dim(hd, cut)
        if rd not in tables:
            tables[rd] = rope_tables(TABLE_SEQ, rd, 3)
            out[f"cos_{rd}"], out[f"sin_{rd}"] = tables[rd]
        cos, sin = (t[:seq] for t in tables[rd])
        q, k, qg, kg = L.rope_inputs(seq, heads, kvh, hd, seed)
        qn, kn = ((qg, None), (kg, None)) if norm else (None, None)
        res, _ = L.run_refdump(L.rope_request([(q, k, cos, sin)], heads, kvh, hd, cut, qn, kn, 1, 1e-6))
        qout, kout = res[:q.size].reshape(seq, heads, hd), res[q.size:].reshape(seq, kvh, hd)
        out[f"{name}/meta"] = np.array([seq, heads, kvh, hd, cut, int(norm), seed], np.int64)
        if norm:
            keep = np.arange(0, seq, 9)
            out[f"{name}/q_out"], out[f"{name}/k_out"], out[f"{name}/rows"] = qout[keep], kout[keep], keep
        else:
            out[f"{name}/q_sha256"], out[f"{name}/k_sha256"] = np.array(L.digest(qout)), np.array(L.digest(kout))
        print(name, seq, heads, kvh, hd, cut, norm)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
