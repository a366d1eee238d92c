#!/usr/bin/env python3
"""fp32 model fixtures: MobileNet-v2 and ResNet-50 v2 with seeded float weights, from the reference's weight-less benchmark graphs.

TEST INFRASTRUCTURE ONLY.  Builds oracle/_ref/revert_float (oracle/revert_float.cpp + the reference's Revert tool, linked
against oracle/_ref/libMNN.so) and writes oracle/_ref/mbv2_f32.mnn and oracle/_ref/r50_f32.mnn (about 14 MB and 100 MB of
fp32 weights: git-ignored, generated where the reference exists)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle.build_ref import INCLUDES, OUT, REF  # noqa: E402

MODELS = (("MobileNetV2_224.mnn", "mbv2_f32.mnn", 21), ("resnet-v2-50.mnn", "r50_f32.mnn", 22))


def build_tool():
    exe = os.path.join(OUT, "revert_float")
    src = [os.path.join(HERE, "revert_float.cpp"), os.path.join(REF, "tools/cpp/revertMNNModel.cpp")]
    if os.path.exists(exe) and all(os.path.getmtime(exe) > os.path.getmtime(s) for s in src):
        return exe
    cmd = ["g++", "-O2", "-std=gnu++11", "-w", "-o", exe] + src + ["-I" + os.path.join(REF, i) for i in INCLUDES] + \
          ["-I" + os.path.join(REF, "tools/cpp"), "-L" + OUT, "-lMNN", "-Wl,-rpath,$ORIGIN", "-pthread", "-ldl"]
    subprocess.check_call(cmd)
    return exe


def main():
    if not os.path.isdir(REF) or not os.path.exists(os.path.join(OUT, "libMNN.so")):
        sys.exit("[float_models] needs the reference and oracle/_ref/libMNN.so (oracle/build_ref.py)")
    exe = build_tool()
    for src, dst, seed in MODELS:
        out = os.path.join(OUT, dst)
        if not os.path.exists(out):
            subprocess.check_call([exe, os.path.join(REF, "benchmark", "models", src), out, str(seed)])
            print(f"[float_models] wrote {out}", flush=True)


if __name__ == "__main__":
    main()
