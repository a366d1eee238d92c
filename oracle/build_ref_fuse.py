#!/usr/bin/env python3
"""Build a variant of the UNMODIFIED reference CPU backend with MNN_SUPPORT_TRANSFORMER_FUSE into oracle/_ref/libMNN_fuse.so,
and the LayerNorm / RoPE harness oracle/_ref/refdump_llm over it (source: oracle/refdump_llm.cpp).

TEST INFRASTRUCTURE ONLY, like oracle/build_ref.py, whose source groups, per-group ISA flags and definitions it takes unchanged.

Without the define the reference core registers no shape computer for the fused RoPE op (source/shape/ShapeRegister.cpp:246-254),
so a RoPE op cannot run through its Interpreter.  In the core and the x86 CPU backend the define only adds the fused ops' shape
computers, the CPU Attention creators and the flash-attention block size: the main libMNN.so, which every other golden and test
is pinned on, stays as it is, and this library is a second build next to it (as libMNN_avx2.so is).

Usage: python oracle/build_ref_fuse.py [-j N]
"""
import argparse
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
if os.path.dirname(HERE) not in sys.path:
    sys.path.insert(0, os.path.dirname(HERE))
from oracle import build_ref as B  # noqa: E402

NAME = "libMNN_fuse.so"
LIB = os.path.join(B.OUT, NAME)
REFDUMP_LLM = os.path.join(B.OUT, "refdump_llm")
DEFS = B.DEFS + ["-DMNN_SUPPORT_TRANSFORMER_FUSE"]


def compile_one(args):
    src, flags, objdir = args
    obj = os.path.join(objdir, os.path.relpath(src, B.REF).replace("/", "__") + ".o")
    if os.path.exists(obj) and os.path.getmtime(obj) > os.path.getmtime(src):
        return obj, 0, ""
    cmd = ["g++", "-c", src, "-o", obj] + B.BASE + DEFS + flags + ["-I" + os.path.join(B.REF, i) for i in B.INCLUDES]
    p = subprocess.run(cmd, capture_output=True, text=True)
    return obj, p.returncode, p.stderr[-2000:]


def build_lib(jobs):
    objdir = os.path.join(B.OUT, "objfuse")
    os.makedirs(objdir, exist_ok=True)
    work = [(s, f, objdir) for s, f in B.sources(True)]
    print(f"[build_ref_fuse] {NAME}: {len(work)} translation units, -j{jobs}", flush=True)
    objs, failed = [], 0
    with ThreadPoolExecutor(jobs) as ex:
        for obj, rc, err in ex.map(compile_one, work):
            objs.append(obj)
            if rc:
                failed += 1
                print(f"[build_ref_fuse] FAILED {obj}\n{err}", flush=True)
    if failed:
        sys.exit(f"[build_ref_fuse] {failed} translation units failed")
    subprocess.check_call(["g++", "-shared", "-fPIC", "-o", LIB, "-Wl,-soname," + NAME] + objs + ["-pthread", "-ldl"])
    print(f"[build_ref_fuse] wrote {LIB}", flush=True)


def build_refdump():
    src = [os.path.join(HERE, "refdump_llm.cpp"), os.path.join(B.REF, "tools/cpp/revertMNNModel.cpp")]
    deps = src[:1] + [os.path.join(HERE, "refdump.cpp"), LIB]
    if os.path.exists(REFDUMP_LLM) and all(os.path.getmtime(REFDUMP_LLM) > os.path.getmtime(d) for d in deps):
        return
    cmd = ["g++", "-O2", "-std=gnu++11", "-w", "-o", REFDUMP_LLM] + src + ["-I" + HERE] + \
          ["-I" + os.path.join(B.REF, i) for i in B.INCLUDES] + ["-I" + os.path.join(B.REF, "tools/cpp")] + \
          ["-L" + B.OUT, "-lMNN_fuse", "-Wl,-rpath,$ORIGIN", "-pthread", "-ldl", "-rdynamic"]
    subprocess.check_call(cmd)
    print(f"[build_ref_fuse] wrote {REFDUMP_LLM}", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("-j", type=int, default=os.cpu_count() or 4)
    a = ap.parse_args()
    if not os.path.isdir(B.REF):
        sys.exit(f"[build_ref_fuse] {B.REF} not present (GPU box uses the prebuilt oracle/_ref)")
    os.makedirs(B.OUT, exist_ok=True)
    if not os.path.exists(LIB):
        build_lib(a.j)
    build_refdump()


if __name__ == "__main__":
    main()
