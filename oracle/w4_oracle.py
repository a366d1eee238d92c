"""ctypes front-end for oracle/w4_oracle.c (the 4-bit LLM linear layer) and for the reference harness oracle/_ref/refdump_w4.

TEST INFRASTRUCTURE ONLY, like oracle/oracle.py: mnn_b200 (the product) never imports this module.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle import oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libmnn_oracle_w4.so")
REFDUMP_W4 = os.path.join(O.REF_DIR, "refdump_w4")


def build(force=False):
    """Compile the C restatement.  -ffp-contract=off: the reference epilogues are unfused."""
    src = os.path.join(HERE, "w4_oracle.c")
    if force or not os.path.exists(LIB_PATH) or os.path.getmtime(LIB_PATH) < os.path.getmtime(src):
        subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fno-fast-math", "-shared", "-fPIC",
                               "-fvisibility=hidden", src, "-o", LIB_PATH, "-lm"])
    return LIB_PATH


def build_refdump():
    """oracle/_ref/refdump_w4 from oracle/refdump_w4.cpp, with the recipe and flags oracle/build_ref.py uses for refdump
    (needs the reference tree and oracle/_ref/libMNN.so)."""
    from oracle import build_ref as B
    src = [os.path.join(HERE, "refdump_w4.cpp"), os.path.join(B.REF, "tools/cpp/revertMNNModel.cpp")]
    deps = src[:1] + [os.path.join(HERE, "refdump.cpp")]
    if os.path.exists(REFDUMP_W4) and all(os.path.getmtime(REFDUMP_W4) > os.path.getmtime(d) for d in deps):
        return REFDUMP_W4
    cmd = ["g++", "-O2", "-std=gnu++11", "-w", "-o", REFDUMP_W4] + src + \
          ["-I" + HERE] + ["-I" + os.path.join(B.REF, i) for i in B.INCLUDES] + ["-I" + os.path.join(B.REF, "tools/cpp")] + \
          ["-L" + O.REF_DIR, "-lMNN", "-Wl,-rpath,$ORIGIN", "-pthread", "-ldl", "-rdynamic"]
    subprocess.check_call(cmd)
    return REFDUMP_W4


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(LIB_PATH)
    return _lib


def have_reference():
    return O.have_reference() and os.path.exists(REFDUMP_W4)


def pack_w4(q):
    """int8 weights in [-8, 7], [oc][ic] -> the buffer ConvolutionCommon::load(..., forceInt8) returns for a 4-bit layer:
    u = q + 8, two per byte, the even index in the high nibble (ConvolutionCommon.cpp:367-371)."""
    u = (np.ascontiguousarray(q, np.int16).reshape(-1) + 8).astype(np.uint8)
    return ((u[0::2] << 4) | u[1::2]).astype(np.uint8)


def unpack_w4(wpacked, oc):
    """pack_w4's inverse: [oc][ic] int8 in [-8, 7]"""
    wpacked = np.ascontiguousarray(wpacked, np.uint8).reshape(-1)
    u = np.empty(wpacked.size * 2, np.int16)
    u[0::2], u[1::2] = wpacked >> 4, wpacked & 15
    return (u - 8).astype(np.int8).reshape(oc, -1)


def linear_w4_dynamic_blocks(x, wpacked, oc, alpha, wzero=None, bias=None, blocks=1, relu=False, relu6=False):
    """4-bit weights (w4_oracle.c: mnn_oracle_linear_w4_dynamic_blocks): wpacked as pack_w4 returns it, alpha / wzero
    [oc][blocks] with wzero as load() returns it (wire min + 8 * alpha) or None."""
    x = np.ascontiguousarray(x, np.float32)
    tokens, ic = x.shape
    wpacked = np.ascontiguousarray(wpacked, np.uint8).reshape(-1)
    assert ic % blocks == 0 and wpacked.size * 2 == oc * ic
    alpha = np.ascontiguousarray(alpha, np.float32).reshape(oc, blocks)
    wzero = None if wzero is None else np.ascontiguousarray(wzero, np.float32).reshape(oc, blocks)
    bias = None if bias is None else np.ascontiguousarray(bias, np.float32)
    y = np.empty((tokens, oc), np.float32)
    p = O._p
    lib().mnn_oracle_linear_w4_dynamic_blocks(p(x, C.c_float), tokens, ic, p(wpacked, C.c_uint8), oc, p(alpha, C.c_float),
                                              p(wzero, C.c_float), p(bias, C.c_float), int(blocks), int(relu), int(relu6),
                                              p(y, C.c_float))
    return y


def ref_linear(x, q, alpha, asym=False, bias=None, blocks=1, threads=1):
    """the reference CPU backend's 4-bit linear layer: q [oc][ic] in [-8, 7], alpha as the wire holds it"""
    payload = O.linear_request(x, q, alpha, asym, bias, blocks)
    return O.run_linear_request(payload, np.shape(x)[0], np.shape(q)[0], REFDUMP_W4, threads=threads)[0]
