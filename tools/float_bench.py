#!/usr/bin/env python3
"""Float MobileNet-v2 at batch 32 (oracle/_ref/mbv2_f32.mnn, see oracle/float_models.py): one JSON line with
  conv_*        the 36 dense fp32 convolutions on the split-TF32 wgmma kernel, each on its own resident activation, all 36
                replayed as one CUDA graph and timed with CUDA events (device time per forward's conv set), with their
                algorithmic bytes (input + output + weights once, fp32) and FLOPs (2 x MACs; the split form issues 3x that on
                the tensor cores) computed from shapes, and the share of the HBM / TF32 bound reached;
  plugin_e2e    img/s of the WHOLE model through the unmodified Interpreter on libmnn_b200_plugin.so (refdump bench: input copy +
                runSession + output copy per iteration), with the plugin's created / declined command counts;
  cpu           img/s of MNN_FORWARD_CPU on the same model and batch;
  card          name and power limit, read in the same call.
With --model other than mbv2 (the other fp32 fixtures build() writes) the line has model, batch, card, plugin_e2e and cpu only.
Usage: python tools/float_bench.py [--model mbv2] [--batch 32] [--iters 50] [--cpu-threads 16]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BPS, TF32_FLOPS = 3.35e12, 495e12       # H100 SXM data sheet (700 W): the bounds, not reached figures
MODELS = {   # --model: (fixture under oracle/_ref, name in the JSON line)
    "mbv2": ("mbv2_f32.mnn", "MobileNet-v2 fp32 (seeded weights)"),
    "mbv3": ("mbv3_f32.mnn", "MobileNet-v3 fp32 (seeded weights)"),
    "nasnet": ("nasnet_f32.mnn", "NASNet fp32 (seeded weights)"),
    "inception_v3": ("inception_v3_f32.mnn", "Inception-v3 fp32 (seeded weights)"),
    "squeezenet_v10": ("squeezenet_v10_f32.mnn", "SqueezeNet v1.0 fp32 (seeded weights)"),
    "squeezenet_v11": ("squeezenet_v11_f32.mnn", "SqueezeNet v1.1 fp32 (seeded weights)"),
    "mbv1": ("mbv1_f32.mnn", "MobileNet-v1 fp32 (seeded weights)"),
    "resnext50": ("resnext50_f32.mnn", "ResNeXt-50 32x4d fp32 (seeded weights, oracle/refdump_gconv.cpp)"),
    "deeplab": ("deeplab_f32.mnn", "DeepLab-v3-style segmentation fp32, 128x128 (seeded weights, oracle/refdump_interp.cpp)"),
    "bert": ("bert_f32.mnn", "BERT-style encoder fp32, 4 layers, D 256, S 64, int32 ids and mask (seeded weights, oracle/refdump_gather.cpp)"),
    "vit": ("vit_f32.mnn", "ViT-style encoder fp32, 4 layers, D 192, 64x64 image (seeded weights, oracle/refdump_gather.cpp)"),
    "pillars": ("pillars_f32.mnn", "PointPillars-style BEV net fp32, 2,048 pillars into 64x48, batch 1 (seeded weights, oracle/refdump_scatter.cpp)"),
    "gnn": ("gnn_f32.mnn", "GraphSAGE-mean-style net fp32, 512 nodes, 4,096 skewed edges, batch 1 (seeded weights, oracle/refdump_scatter.cpp)"),
    "crnn": ("crnn_f32.mnn", "CRNN-style text recogniser fp32, 32x128 grey, 2 BiLSTM H 256 (seeded weights, oracle/refdump_rnn.cpp)"),
    "kws": ("kws_f32.mnn", "streaming keyword-spotter chunk fp32, 16 frames, LSTM H 128 + RNN H 64 with states (seeded weights, oracle/refdump_rnn.cpp)"),
    "flow": ("flow_f32.mnn", "two-frame flow-warp net fp32, 6x64x64, bilinear GridSample at 16x16 (seeded weights, oracle/refdump_grid_sample.cpp)"),
    "lut": ("lut_f32.mnn", "image-adaptive 3D-LUT enhancer fp32, 3x64x64, trilinear GridSample into 33^3 (seeded weights, oracle/refdump_grid_sample.cpp)"),
    "denoise": ("denoise_f32.mnn", "RNNoise-style streaming denoiser chunk fp32, 16 frames of 42 features, GRUs H 24 / 48 / 96 with states (seeded weights, oracle/refdump_gru.cpp)"),
    "tagger": ("tagger_f32.mnn", "BiGRU sequence tagger fp32, 64 int32 tokens, embedding 8000x128, 2 BiGRU H 256 (seeded weights, oracle/refdump_gru.cpp)"),
}
# models whose inputs refdump's bench does not fill (int32 token ids and masks): timed by oracle/refdump_gather's bench instead
GATHER_HARNESS = {"bert", "vit"}
# models with int32 pillar cells or edge lists, built for batch 1: timed at batch 1 by oracle/refdump_scatter's bench
SCATTER_HARNESS = {"pillars", "gnn"}
# models with sequence and state inputs (batch on dim 1): timed by oracle/refdump_rnn's bench
RNN_HARNESS = {"crnn", "kws"}
# GRU models with sequence, state or int32 token-id inputs (batch on dim 1): timed by oracle/refdump_gru's bench
GRU_HARNESS = {"denoise", "tagger"}


def shapes_from_cpu_run(model, refdump, env):
    """(conv op, input dims, output dims) of every dense Convolution, from a batch-1 CPU forward's command dump"""
    from mnn_b200 import mnn_file
    net = mnn_file.load(model)
    with tempfile.TemporaryDirectory() as d:
        subprocess.run([refdump, "run", model, "1", "3", d, "4"], env=env, check=True, capture_output=True, text=True)
        dims = {}
        for line in open(os.path.join(d, "index.txt")):
            _, name, _, dd = line.split("|")[:4]
            dims[name] = [int(v) for v in dd.split(",")]
    by_tensor = {}
    for op in net.ops:
        for t in op.outputs:
            by_tensor[t] = dims.get(op.name, op.attrs.get("dims"))
    out = []
    for op in net.ops:
        if op.type == "Convolution" and op.conv is not None and op.conv.group == 1:
            out.append((op.conv, by_tensor[op.inputs[0]], dims[op.name]))
    return out


def time_convs(layers, batch, iters):
    import numpy as np
    import torch
    from mnn_b200 import _capi
    from mnn_b200._capi import ConvDesc
    from mnn_b200.backend import Runtime
    L = _capi.lib()
    torch.cuda.set_stream(torch.cuda.Stream())
    rt = Runtime(0)
    rng = np.random.default_rng(0)
    hs, bufs, bytes_, macs = [], [], 0.0, 0.0
    for cv, din, dout in layers:
        ic, ih, iw = din[1], din[2], din[3]
        oc, oh0, ow0 = dout[1], dout[2], dout[3]
        kh, kw = cv.kernel
        w = (rng.uniform(-1, 1, (oc, ic, kh, kw)) / np.sqrt(ic * kh * kw)).astype(np.float32)
        d = ConvDesc(ic, oc, kh, kw, cv.stride[0], cv.stride[1], cv.pad[0], cv.pad[1], cv.dilate[0], cv.dilate[1], 1, 0)
        h = C.c_void_p()
        _capi.check(L.mnnb200_conv_f32_create(rt._h, C.byref(d), w.ctypes.data_as(C.c_void_p), None, int(cv.relu6), C.byref(h)))
        oh, ow = C.c_int(oh0), C.c_int(ow0)
        _capi.check(L.mnnb200_conv_f32_resize(h, batch, ih, iw, C.byref(oh), C.byref(ow)))
        b, m = C.c_double(), C.c_double()
        L.mnnb200_exec_cost(h, C.byref(b), C.byref(m))
        bytes_ += b.value
        macs += m.value
        x = torch.randn(batch, ic, ih, iw, device="cuda")
        y = torch.empty(batch, oc, oh.value, ow.value, device="cuda")
        hs.append(h)
        bufs.append((x, y))

    def step():
        for h, (x, y) in zip(hs, bufs):
            _capi.check(L.mnnb200_conv_f32_execute(h, C.c_void_p(x.data_ptr()), C.c_void_p(y.data_ptr())))

    step()
    _capi.check(L.mnnb200_runtime_sync(rt._h))
    g = C.c_void_p()
    _capi.check(L.mnnb200_graph_begin_capture(rt._h))
    step()
    _capi.check(L.mnnb200_graph_end_capture(rt._h, C.byref(g)))
    for _ in range(5):
        L.mnnb200_graph_launch(rt._h, g)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    windows = []
    for _ in range(5):
        e0.record()
        for _ in range(iters):
            L.mnnb200_graph_launch(rt._h, g)
        e1.record()
        torch.cuda.synchronize()
        windows.append(e0.elapsed_time(e1) / iters)
    L.mnnb200_graph_destroy(g)
    for h in hs:
        L.mnnb200_exec_destroy(h)
    ms = sorted(windows)[len(windows) // 2]
    bound_ms = max(bytes_ / HBM_BPS, 3 * 2 * macs / TF32_FLOPS) * 1e3
    return dict(conv_layers=len(hs), conv_device_ms=round(ms, 4), conv_img_per_s=round(batch / ms * 1e3, 1),
                conv_algorithmic_bytes=bytes_, conv_flops=2 * macs, conv_tensor_flops_split=3 * 2 * macs,
                conv_GBps=round(bytes_ / ms / 1e6, 1), conv_bound="hbm" if bytes_ / HBM_BPS > 6 * macs / TF32_FLOPS else "tf32",
                conv_bound_ms=round(bound_ms, 4), conv_share_of_bound=round(bound_ms / ms, 3),
                conv_ms_windows=[round(v, 4) for v in windows])


def refdump_bench(refdump, model, batch, threads, env, iters):
    r = subprocess.run([refdump, "bench", model, str(batch), str(threads), "2", str(iters)], env=env, check=True,
                       capture_output=True, text=True, timeout=1800)
    line = [l for l in r.stdout.splitlines() if l.startswith("{")][-1]
    j = json.loads(line)
    j["img_per_s"] = round(batch / j["ms_median_window"] * 1e3, 1)
    return j


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", choices=sorted(MODELS), default="mbv2")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--cpu-threads", type=int, default=os.cpu_count() or 4)
    a = ap.parse_args()
    from oracle import oracle as O
    fixture, title = MODELS[a.model]
    model = os.path.join(O.REF_DIR, fixture)
    if not O.have_reference() or not os.path.exists(model):
        sys.exit(f"float_bench: needs oracle/_ref (refdump, libMNN.so, {fixture}) as build() leaves it")
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = O.REF_DIR + ":" + os.path.join(ROOT, "mnn_b200") + ":" + env.get("LD_LIBRARY_PATH", "")
    env.pop("REFDUMP_PLUGIN", None)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True, check=True).stdout.strip().splitlines()[0]
    if a.model in SCATTER_HARNESS:
        a.batch = 1
    res = dict(model=title, batch=a.batch, card=card)
    if a.model == "mbv2":
        res.update(time_convs(shapes_from_cpu_run(model, O.REFDUMP, env), a.batch, a.iters))
    harness = O.REFDUMP
    if a.model in GATHER_HARNESS:
        from oracle import gather_oracle
        harness = gather_oracle.REFDUMP_GATHER
    if a.model in SCATTER_HARNESS:
        from oracle import scatter_oracle
        harness = scatter_oracle.REFDUMP_SCATTER
    if a.model in RNN_HARNESS:
        from oracle import rnn_oracle
        harness = rnn_oracle.REFDUMP_RNN
    if a.model in GRU_HARNESS:
        from oracle import gru_oracle
        harness = gru_oracle.REFDUMP_GRU
    penv = dict(env, REFDUMP_BENCH_WINDOWS="5", REFDUMP_PLUGIN=os.path.join(ROOT, "mnn_b200", "libmnn_b200_plugin.so"))
    p = refdump_bench(harness, model, a.batch, 4, penv, 20)
    res.update(plugin_e2e_img_per_s=p["img_per_s"], plugin_e2e_ms=p["ms_median_window"], plugin_created=p["plugin_created"],
               plugin_declined=p["plugin_declined"])
    c = refdump_bench(harness, model, a.batch, a.cpu_threads, dict(env, REFDUMP_BENCH_WINDOWS="1"), 2)
    res.update(cpu_img_per_s=c["img_per_s"], cpu_threads=a.cpu_threads)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
