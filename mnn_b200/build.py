"""Builds libmnn_b200.so (CUDA kernels + C ABI), libmnn_b200_llm.so (the MNN-LLM LayerNorm / RoPE ops, include/mnn_b200_llm.h)
libmnn_b200_deconv.so (the float Deconvolution, include/mnn_b200_deconv.h), libmnn_b200_interp.so (the float Interp,
include/mnn_b200_interp.h), libmnn_b200_gather.so (the gathers and the int32 / fp32 Cast, include/mnn_b200_gather.h) and
libmnn_b200_scatter.so (ScatterNd and ScatterElements, include/mnn_b200_scatter.h), libmnn_b200_rnn.so (LSTM and RNN,
include/mnn_b200_rnn.h) and libmnn_b200_grid_sample.so (the float GridSample, include/mnn_b200_grid_sample.h), the last seven
linked against libmnn_b200.so, and libmnn_b200_shallow.so (the shallow conv-group
kernel, which libmnn_b200.so launches and links against), in-tree for sm_90a (H100) with nvcc.  No torch involvement."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libmnn_b200.so")
LLM_LIB = os.path.join(HERE, "libmnn_b200_llm.so")
DECONV_LIB = os.path.join(HERE, "libmnn_b200_deconv.so")
INTERP_LIB = os.path.join(HERE, "libmnn_b200_interp.so")
GATHER_LIB = os.path.join(HERE, "libmnn_b200_gather.so")
SCATTER_LIB = os.path.join(HERE, "libmnn_b200_scatter.so")
RNN_LIB = os.path.join(HERE, "libmnn_b200_rnn.so")
GRID_SAMPLE_LIB = os.path.join(HERE, "libmnn_b200_grid_sample.so")
SHALLOW_LIB = os.path.join(HERE, "libmnn_b200_shallow.so")
SOURCES = ["capi.cu", "conv_int8_mma.cu", "elementwise.cu", "gemm_i8_wgmma.cu", "winograd_int8.cu", "gemm_f16_wgmma.cu", "conv_int8_stem.cu", "conv_group_wgmma.cu", "linear_w8_gemv.cu", "conv_f32_wgmma.cu"]
LLM_SOURCES = ["llm_ops.cu", "llm_capi.cu"]
DECONV_SOURCES = ["deconv_f32_wgmma.cu", "deconv_capi.cu"]
INTERP_SOURCES = ["interp_f32.cu", "interp_capi.cu"]
GATHER_SOURCES = ["gather.cu", "gather_capi.cu"]
SCATTER_SOURCES = ["scatter.cu", "scatter_capi.cu"]
RNN_SOURCES = ["rnn.cu", "rnn_capi.cu"]
GRID_SAMPLE_SOURCES = ["grid_sample_f32.cu", "grid_sample_capi.cu"]
# the shallow conv-group kernel, launched by libmnn_b200.so, which links against it
SHALLOW_SOURCES = ["conv_group_shallow_wgmma.cu"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + ["-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC,-ffp-contract=off,-fvisibility=hidden", "--expt-relaxed-constexpr"]
# every float operation in that file is an explicit intrinsic / PTX instruction: no implicit contraction wanted anywhere in it
PER_FILE_FLAGS = {"conv_group_wgmma.cu": ["--fmad=false"], "conv_group_shallow_wgmma.cu": ["--fmad=false"], "interp_f32.cu": ["--fmad=false"],
                  "grid_sample_f32.cu": ["--fmad=false"]}


def _compile(srcs, nvcc, verbose):
    objs, procs = [], []
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
    return objs


def build(force=False, verbose=False):
    """the nine libraries; returns the path of libmnn_b200.so"""
    srcs = [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    llm_srcs = [os.path.join(CSRC, s) for s in LLM_SOURCES]
    inc = os.path.join(HERE, "..", "include")
    deps = srcs + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))] + \
           [os.path.join(inc, "mnn_b200.h")]
    llm_deps = deps + llm_srcs + [os.path.join(inc, "mnn_b200_llm.h")]
    deconv_srcs = [os.path.join(CSRC, s) for s in DECONV_SOURCES]
    deconv_deps = deps + deconv_srcs + [os.path.join(inc, "mnn_b200_deconv.h")]
    interp_srcs = [os.path.join(CSRC, s) for s in INTERP_SOURCES]
    interp_deps = deps + interp_srcs + [os.path.join(inc, "mnn_b200_interp.h")]
    gather_srcs = [os.path.join(CSRC, s) for s in GATHER_SOURCES]
    gather_deps = deps + gather_srcs + [os.path.join(inc, "mnn_b200_gather.h")]
    scatter_srcs = [os.path.join(CSRC, s) for s in SCATTER_SOURCES]
    scatter_deps = deps + scatter_srcs + [os.path.join(inc, "mnn_b200_scatter.h")]
    rnn_srcs = [os.path.join(CSRC, s) for s in RNN_SOURCES]
    rnn_deps = deps + rnn_srcs + [os.path.join(inc, "mnn_b200_rnn.h")]
    gs_srcs = [os.path.join(CSRC, s) for s in GRID_SAMPLE_SOURCES]
    gs_deps = deps + gs_srcs + [os.path.join(inc, "mnn_b200_grid_sample.h")]
    fresh = lambda lib, ds: os.path.exists(lib) and all(os.path.getmtime(lib) > os.path.getmtime(d) for d in ds)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    shallow_srcs = [os.path.join(CSRC, s) for s in SHALLOW_SOURCES]
    shallow_deps = shallow_srcs + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    if force or not fresh(SHALLOW_LIB, shallow_deps):
        subprocess.check_call([nvcc, "-shared", "-o", SHALLOW_LIB] + _compile(shallow_srcs, nvcc, verbose) + ARCH + ["-lcudart"])
    if force or not fresh(LIB, deps + [SHALLOW_LIB]):
        subprocess.check_call([nvcc, "-shared", "-o", LIB] + _compile(srcs, nvcc, verbose) + ARCH +
                              ["-L" + HERE, "-lmnn_b200_shallow", "-Xlinker", "-rpath,$ORIGIN", "-lcudart"])
    if force or not fresh(LLM_LIB, llm_deps + [LIB]):
        subprocess.check_call([nvcc, "-shared", "-o", LLM_LIB] + _compile(llm_srcs, nvcc, verbose) + ARCH +
                              ["-L" + HERE, "-lmnn_b200", "-Xlinker", "-rpath,$ORIGIN", "-lcudart"])
    if force or not fresh(DECONV_LIB, deconv_deps + [LIB]):
        subprocess.check_call([nvcc, "-shared", "-o", DECONV_LIB] + _compile(deconv_srcs, nvcc, verbose) + ARCH +
                              ["-L" + HERE, "-lmnn_b200", "-Xlinker", "-rpath,$ORIGIN", "-lcudart"])
    if force or not fresh(INTERP_LIB, interp_deps + [LIB]):
        subprocess.check_call([nvcc, "-shared", "-o", INTERP_LIB] + _compile(interp_srcs, nvcc, verbose) + ARCH +
                              ["-L" + HERE, "-lmnn_b200", "-Xlinker", "-rpath,$ORIGIN", "-lcudart"])
    if force or not fresh(GATHER_LIB, gather_deps + [LIB]):
        subprocess.check_call([nvcc, "-shared", "-o", GATHER_LIB] + _compile(gather_srcs, nvcc, verbose) + ARCH +
                              ["-L" + HERE, "-lmnn_b200", "-Xlinker", "-rpath,$ORIGIN", "-lcudart"])
    if force or not fresh(SCATTER_LIB, scatter_deps + [LIB]):
        subprocess.check_call([nvcc, "-shared", "-o", SCATTER_LIB] + _compile(scatter_srcs, nvcc, verbose) + ARCH +
                              ["-L" + HERE, "-lmnn_b200", "-Xlinker", "-rpath,$ORIGIN", "-lcudart"])
    if force or not fresh(RNN_LIB, rnn_deps + [LIB]):
        subprocess.check_call([nvcc, "-shared", "-o", RNN_LIB] + _compile(rnn_srcs, nvcc, verbose) + ARCH +
                              ["-L" + HERE, "-lmnn_b200", "-Xlinker", "-rpath,$ORIGIN", "-lcudart"])
    if force or not fresh(GRID_SAMPLE_LIB, gs_deps + [LIB]):
        subprocess.check_call([nvcc, "-shared", "-o", GRID_SAMPLE_LIB] + _compile(gs_srcs, nvcc, verbose) + ARCH +
                              ["-L" + HERE, "-lmnn_b200", "-Xlinker", "-rpath,$ORIGIN", "-lcudart"])
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
