"""Builds libmnn_b200.so (CUDA kernels + C ABI) in-tree for sm_90a (H100) with nvcc.  No torch involvement."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libmnn_b200.so")
SOURCES = ["capi.cu", "conv_int8_mma.cu", "elementwise.cu", "gemm_i8_wgmma.cu", "winograd_int8.cu", "gemm_f16_wgmma.cu", "conv_int8_stem.cu", "conv_group_wgmma.cu", "linear_w8_gemv.cu", "conv_f32_wgmma.cu"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + ["-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC,-ffp-contract=off,-fvisibility=hidden", "--expt-relaxed-constexpr"]
# every float operation in that file is an explicit intrinsic / PTX instruction: no implicit contraction wanted anywhere in it
PER_FILE_FLAGS = {"conv_group_wgmma.cu": ["--fmad=false"]}


def build(force=False, verbose=False):
    srcs = [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    deps = srcs + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))] + \
           [os.path.join(HERE, "..", "include", "mnn_b200.h")]
    if not force and os.path.exists(LIB) and all(os.path.getmtime(LIB) > os.path.getmtime(d) for d in deps):
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objs = []
    procs = []
    for s in srcs:
        o = s[:-3] + ".o"
        objs.append(o)
        cmd = [nvcc, "-c", s, "-o", o] + NVCC_FLAGS + PER_FILE_FLAGS.get(os.path.basename(s), []) + (["-Xptxas", "-v"] if verbose else [])
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for s, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode:
            sys.stderr.write(out)
        if p.returncode:
            failed = True
    if failed:
        raise RuntimeError("nvcc failed")
    subprocess.check_call([nvcc, "-shared", "-o", LIB] + objs + ARCH + ["-lcudart"])
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
