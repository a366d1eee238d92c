"""Secondary bench lines (BASELINE.json configs[2] and configs[3]); same JSON contract as bench.py, selected with
`python bench.py --workload resnet_wino|qwen`.  The driver's default line stays MobileNet-v2 (configs[1]).

  resnet_wino  ResNet-50 int8, batch 64, the 13 3x3/s1 convs on the int8 Winograd path F(m,3) (m = --wino-unit)
               (C,HW) in {(64,56)x2,(128,28)x3,(256,14)x5,(512,7)x3}                      SURVEY 8d C3
  qwen         Qwen-1.8B int8 linear layers, seq 512 x batch 8 = 4096 tokens, 24 x {2048->6144(+bias), 2048->2048,
               2048->5504 x2, 5504->2048} + lm_head on the 8 last tokens                  SURVEY 8d C4
"""
import ctypes as C
import json
import os
import struct
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
INT8_DENSE_PEAK_TOPS = 1979.0   # H100 SXM data sheet, dense int8 (a card at a lower power limit reaches less)


def _peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        return float(json.load(open(p))["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
    return 3350.0, "H100 SXM data sheet (3.35 TB/s HBM3)"


def _timeit(torch, stream, fn, K, W):
    for _ in range(W):
        fn()
    stream.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(stream):
        e0.record()
    for _ in range(K):
        fn()
    with torch.cuda.stream(stream):
        e1.record()
    stream.synchronize()
    return e0.elapsed_time(e1) / K


RESNET_LAYERS = [(64, 56)] * 2 + [(128, 28)] * 3 + [(256, 14)] * 5 + [(512, 7)] * 3


def run_resnet_wino(args, sampler_cls, rank=0, world=1, local_rank=0):
    import torch
    from mnn_b200 import _capi
    from mnn_b200.backend import Op, QuantAttr, Runtime, Tensor, encode_winograd_attr
    unit, B = args.wino_unit, 64
    a2 = (unit + 2) ** 2
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        rt = Runtime(local_rank)
    be = rt.onCreate()
    rng = np.random.default_rng(0)
    g = torch.Generator(device="cpu").manual_seed(0)
    layers, bytes_alg, macs = [], 0.0, 0.0
    t_bytes = {"in": 0.0, "out": 0.0}
    gemm_ops = 0.0
    mag = {2: 4.0, 4: 40.0, 6: 400.0}[unit]
    with torch.cuda.stream(stream):
        for (Cn, HW) in RESNET_LAYERS:
            w = rng.integers(-127, 128, (Cn, Cn, 3, 3)).astype(np.int8)
            ws = (rng.uniform(0.003, 0.012, Cn) / np.sqrt(Cn * 9)).astype(np.float32)
            bias = rng.uniform(-0.5, 0.5, Cn).astype(np.float32)
            s_in = 0.05
            ins = np.full(a2, s_in * mag, np.float32)
            inz = np.zeros(a2, np.int32)
            wsc = np.broadcast_to((ws * 127 * 2.0 / 120)[None, :], (a2, Cn)).astype(np.float32)
            attr = encode_winograd_attr([(0, 0, 3, 3, unit, unit, ins, inz, wsc)])
            op = Op(type="ConvInt8", conv=dict(ic=Cn, oc=Cn, kernel=(3, 3), stride=(1, 1), pad=(1, 1), group=1, relu=True),
                    weight=w, wscale=ws, bias=bias, extra=dict(winograd_attr=attr))
            x = be.onAcquire(Tensor((B, Cn, HW, HW), "int8", QuantAttr(s_in, 0, -128, 127)))
            x.data.copy_(torch.randint(-127, 128, tuple(x.data.shape), generator=g, dtype=torch.int8))
            y = Tensor((B, Cn, 1, 1), "int8", QuantAttr(0.1, 0, -127, 127))
            ex = be.onCreate([x], [y], op)
            assert ex.onResize([x], [y]) == 0, _capi.lib().mnnb200_last_error()
            be.onAcquire(y)
            b_, m_ = ex.cost()
            bytes_alg += b_
            macs += m_
            tiles = B * (-(-HW // unit)) ** 2
            t_bytes["in"] += B * HW * HW * Cn + a2 * tiles * Cn              # int8 input read + int8 V write
            t_bytes["out"] += a2 * tiles * Cn * 4 + B * HW * HW * Cn          # fp32 M read + int8 output write
            gemm_ops += 2.0 * a2 * tiles * Cn * Cn
            layers.append((ex, x, y))
    stream.synchronize()
    L = _capi.lib()

    def enqueue(ph):
        for ex, x, y in layers:
            st = L.mnnb200_conv_int8_wino_execute_phases(ex._h, x.ptr(), y.ptr(), ph)
            assert st == 0, L.mnnb200_last_error()

    def graph_of(ph):
        with torch.cuda.stream(stream):
            enqueue(ph)
        stream.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=stream):
            enqueue(ph)
        return gr

    W, K = max(args.warmup, 3), args.steps
    graphs = {ph: graph_of(ph) for ph in (7, 1, 2, 4, 6)}
    sampler = sampler_cls(0)
    sampler.start()

    def replay(ph):
        def f():
            with torch.cuda.stream(stream):
                graphs[ph].replay()
        return f
    ms = {ph: _timeit(torch, stream, replay(ph), K, W) for ph in (7, 1, 2, 4, 6)}
    sampler.stop_flag = True
    sampler.join()
    # e2e: the first layer's int8 NCHW input from pinned host memory in, last layer's output out, every step
    ex0, x0, _ = layers[0]
    _, _, yl = layers[-1]
    n, c, h, w = x0.shape
    hx = torch.randint(-127, 128, (n, c, h, w), dtype=torch.int8).pin_memory()
    dstage = torch.empty((n, c, h, w), dtype=torch.int8, device="cuda")
    hy = torch.empty(tuple(yl.data.shape), dtype=torch.int8).pin_memory()

    def e2e():
        with torch.cuda.stream(stream):
            dstage.copy_(hx, non_blocking=True)
            assert L.mnnb200_pack_nchw_int8(rt._h, C.c_void_p(dstage.data_ptr()), n, c, h, w, x0.ptr()) == 0
            graphs[7].replay()
            hy.copy_(yl.data, non_blocking=True)
        stream.synchronize()
    e2e_ms = _timeit(torch, stream, e2e, K, W)
    peak, src = _peaks()
    dom = max((1, 4), key=lambda ph: ms[ph])
    tb = t_bytes["in"] if dom == 1 else t_bytes["out"]
    achieved = tb / (ms[dom] / 1e3) / 1e9
    line = {
        "metric": "inferences/sec (ResNet-50-int8 224x224, 13 3x3/s1 convs on the int8 Winograd path, device-timed)",
        "value": B / (ms[7] / 1e3), "unit": "img/s", "n_gpus": 1, "steps": K, "warmup": W, "ms_per_step": ms[7],
        "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "s8 (fp32 transforms)", "data": "synthetic",
        "config": {"workload": f"ResNet-50 int8 3x3/s1 layer set, batch 64, int8 Winograd F({unit},3) (synthetic winogradAttr), "
                               "CUDA-graph replay", "batch_per_gpu": B, "wino_unit": unit,
                   "l2": "scratch V/M operands (>= 0.25 GB per layer at C=64) exceed L2"},
        "roofline": {"bound": "hbm", "kernel": "wino_input_kernel" if dom == 1 else "wino_output_kernel",
                     "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak, "traffic": None,
                     "peak_source": src, "algorithmic_bytes_per_launch_set": tb,
                     "phases_ms": {"input_transform": ms[1], "position_gemms_unfused": ms[2], "output_transform_unfused": ms[4],
                                   "gemms_plus_output_as_executed": ms[6], "all": ms[7],
                                   "note": "F(2,3) executes the position GEMMs and the output transform as ONE kernel (accumulators of all "
                                           "16 positions resident in registers); the unfused kernels are timed for comparison"},
                     "gemm": {"bound": "tensor", "achieved": gemm_ops / (ms[2] / 1e3) / 1e12, "peak": INT8_DENSE_PEAK_TOPS,
                              "unit": "TOP/s", "frac": gemm_ops / (ms[2] / 1e3) / 1e12 / INT8_DENSE_PEAK_TOPS,
                              "peak_source": "nominal dense int8 (4.5 POPS)"},
                     "direct_equivalent": {"gop_per_batch": 2 * macs / 1e9, "algorithmic_mb": bytes_alg / 1e6}},
        "e2e": {"value": B / (e2e_ms / 1e3), "unit": "img/s", "h2d_bytes_per_step": int(hx.numel()), "d2h_bytes_per_step": int(hy.numel())},
        "gpu_launches": 3 * len(layers) * K, "clocks": sampler.result(),
    }
    return line


def run_resnet_direct(args, sampler_cls, rank=0, world=1, local_rank=0):
    """The same 13 ResNet-50 3x3/s1 layers at batch 64 WITHOUT a winogradAttr (what a Revert-quantised r50 .mnn carries): the direct
    int8 convolution.  Three device-timed variants: the round-1 mma.sync implicit GEMM (variant 1), the wgmma implicit GEMM one
    launch per layer (variant 2), and all 13 layers in one conv-group launch.  Tensor-bound: 192.4 GOP per batch (SURVEY 8d C3)."""
    import torch
    from mnn_b200 import _capi
    from mnn_b200.backend import ConvGroupExecution, Op, QuantAttr, Runtime, Tensor
    B = 64
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        rt = Runtime(local_rank)
    be = rt.onCreate()
    rng = np.random.default_rng(0)
    g = torch.Generator(device="cpu").manual_seed(0)
    layers, macs, bytes_alg = [], 0.0, 0.0
    with torch.cuda.stream(stream):
        for (Cn, HW) in RESNET_LAYERS:
            w = rng.integers(-127, 128, (Cn, Cn, 3, 3)).astype(np.int8)
            ws = (rng.uniform(0.003, 0.012, Cn) / np.sqrt(Cn * 9)).astype(np.float32)
            bias = rng.uniform(-0.5, 0.5, Cn).astype(np.float32)
            op = Op(type="ConvInt8", conv=dict(ic=Cn, oc=Cn, kernel=(3, 3), stride=(1, 1), pad=(1, 1), group=1, relu=True),
                    weight=w, wscale=ws, bias=bias)
            x = be.onAcquire(Tensor((B, Cn, HW, HW), "int8", QuantAttr(0.05, 0, -128, 127)))
            x.data.copy_(torch.randint(-127, 128, tuple(x.data.shape), generator=g, dtype=torch.int8))
            y = Tensor((B, Cn, 1, 1), "int8", QuantAttr(0.1, 0, -127, 127))
            ex = be.onCreate([x], [y], op)
            assert ex.onResize([x], [y]) == 0, _capi.lib().mnnb200_last_error()
            be.onAcquire(y)
            b_, m_ = ex.cost()
            bytes_alg += b_
            macs += m_
            layers.append((ex, x, y))
    stream.synchronize()
    grp = ConvGroupExecution(be, [l[0] for l in layers])
    assert grp.bind([l[1] for l in layers], [l[2] for l in layers]) == 0, _capi.lib().mnnb200_last_error()

    def graph_of(fn):
        with torch.cuda.stream(stream):
            fn()
        stream.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=stream):
            fn()
        return gr

    def per_layer(variant):
        def f():
            for ex, x, y in layers:
                ex.set_variant(variant)
                assert ex.onExecute([x], [y]) == 0, _capi.lib().mnnb200_last_error()
        return f
    W, K = max(args.warmup, 3), args.steps
    ms = {}
    sampler = sampler_cls(local_rank)
    sampler.start()
    for name, fn in (("mma_sync_per_layer", per_layer(1)), ("wgmma_per_layer", per_layer(2)), ("wgmma_conv_group", lambda: grp.onExecute())):
        gr = graph_of(fn)

        def replay(gr=gr):
            with torch.cuda.stream(stream):
                gr.replay()
        ms[name] = _timeit(torch, stream, replay, K, W)
    sampler.stop_flag = True
    sampler.join()
    best = min(ms, key=ms.get)
    tops = 2 * macs / (ms[best] / 1e3) / 1e12
    return {
        "metric": "inferences/sec (ResNet-50-int8 224x224, 13 3x3/s1 convs, direct int8 convolution, device-timed)",
        "value": B / (ms[best] / 1e3), "unit": "img/s", "n_gpus": 1, "steps": K, "warmup": W, "ms_per_step": ms[best],
        "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "s8", "data": "synthetic",
        "config": {"workload": "ResNet-50 int8 3x3/s1 layer set, batch 64, direct convolution (no winogradAttr)", "batch_per_gpu": B,
                   "best_variant": best},
        "variants_ms": ms,
        "roofline": {"bound": "tensor", "kernel": "conv_group_wgmma_kernel (implicit GEMM, wgmma s8)", "achieved": tops,
                     "peak": INT8_DENSE_PEAK_TOPS, "unit": "TOP/s", "frac": tops / INT8_DENSE_PEAK_TOPS, "traffic": None,
                     "peak_source": "H100 SXM data sheet, dense int8",
                     "gop_per_batch": 2 * macs / 1e9, "algorithmic_mb": bytes_alg / 1e6},
        "gpu_launches": K, "clocks": sampler.result(),
    }


QWEN = dict(hidden=2048, layers=24, ffn=5504, vocab=151936, tokens=4096, batch=8)


def qwen_shapes():
    h, f = QWEN["hidden"], QWEN["ffn"]
    return [(h, 3 * h, True), (h, h, False), (h, f, False), (h, f, False), (f, h, False)]


def run_qwen_decode(args, sampler_cls, rank=0, world=1, local_rank=0):
    """The decode step of the same model (SURVEY 8f rank 3): ONE token through the 24 x 5 linear layers + lm_head; every int8 weight
    is read exactly once per token, so the bound is HBM bandwidth (1.52 GB per token)."""
    return run_qwen(args, sampler_cls, rank=rank, world=world, local_rank=local_rank, decode=True)


def run_qwen(args, sampler_cls, rank=0, world=1, local_rank=0, decode=False):
    """BASELINE configs[3] (and north_star's Qwen at 1/2/4/8 GPUs): every rank runs one replica on its own batch of 8 x 512
    tokens (weak scaling, no steady-state collective); rank 0 builds the int8 weights and ONE NCCL broadcast ships them."""
    import torch
    import torch.distributed as dist
    from mnn_b200 import _capi
    from mnn_b200.backend import Op, Runtime, Tensor
    dev = torch.device("cuda", local_rank)
    stream = torch.cuda.Stream(device=dev)
    with torch.cuda.stream(stream):
        rt = Runtime(local_rank)
    be = rt.onCreate()
    rng = np.random.default_rng(0)
    T = 1 if decode else QWEN["tokens"]
    LMB = 1 if decode else QWEN["batch"]            # tokens that reach lm_head
    nl = QWEN["layers"] if decode else args.qwen_layers
    execs, macs, wbytes = [], 0.0, 0.0
    # ---- weights: rank 0 generates the whole int8 arena (+ fp32 scales / offsets / biases), one broadcast, peers unpack
    specs = []
    for li in range(nl):
        for (ic, oc, hb) in qwen_shapes():
            specs.append((ic, oc, hb, True))
    specs.append((QWEN["hidden"], QWEN["vocab"], False, False))          # lm_head (symmetric)
    from mnn_b200.dist_util import broadcast_linear_arena, linear_arena_layout, unpack_linear
    shapes = [(ic, oc) for ic, oc, _, _ in specs]
    wtot, ftot, _ = linear_arena_layout(shapes)
    t_build0 = time.time()
    w_arena = f_arena = None
    if rank == 0:
        w_arena = rng.integers(-128, 128, wtot, dtype=np.int8)
        f_arena = np.empty(ftot, np.float32)
        o = 0
        for (ic, oc, hb, asym) in specs:
            alpha = rng.uniform(0.001, 0.01, oc).astype(np.float32)
            f_arena[o:o + oc] = alpha
            f_arena[o + oc:o + 2 * oc] = (alpha * rng.uniform(-8, 8, oc)).astype(np.float32)   # asymmetric {offset, scale} like the LLM export
            f_arena[o + 2 * oc:o + 3 * oc] = rng.uniform(-1, 1, oc).astype(np.float32)
            o += 3 * oc
    # ONE collective per arena over NCCL (mnn_b200/dist_util.py; the same function runs over gloo in tests/test_multi_rank.py)
    w_arena, f_arena = broadcast_linear_arena(w_arena, f_arena, shapes, rank, world, device=dev)
    with torch.cuda.stream(stream):
        xs = {ic: torch.empty((T, ic), dtype=torch.float32, device=dev).uniform_(-1, 1) for ic in (QWEN["hidden"], QWEN["ffn"])}
        ys = {}
        for li, (ic, oc, hb, asym) in enumerate(specs[:-1]):
            wq, alpha, wz, bias = unpack_linear(w_arena, f_arena, shapes, li)
            op = Op(type="LinearW8", conv=dict(ic=ic, oc=oc), weight=wq, wscale=alpha, wzero=wz, bias=bias if hb else None)
            x = Tensor((T, ic), "float", None, xs[ic])
            if oc not in ys:
                ys[oc] = torch.empty((T, oc), dtype=torch.float32, device=dev)
            y = Tensor((T, oc), "float", None, ys[oc])
            ex = be.onCreate([x], [y], op)
            assert ex.onResize([x], [y]) == 0
            execs.append((ex, x, y))
            macs += float(T) * ic * oc
            wbytes += float(ic) * oc
        # lm_head on the last token of each of the 8 sequences
        ic, oc = QWEN["hidden"], QWEN["vocab"]
        wq_l, alpha_l, _, _ = unpack_linear(w_arena, f_arena, shapes, len(specs) - 1)
        op = Op(type="LinearW8", conv=dict(ic=ic, oc=oc), weight=wq_l, wscale=alpha_l)
        xl = Tensor((LMB, ic), "float", None, torch.empty((LMB, ic), dtype=torch.float32, device=dev).uniform_(-1, 1))
        yl = Tensor((LMB, oc), "float", None, torch.empty((LMB, oc), dtype=torch.float32, device=dev))
        exl = be.onCreate([xl], [yl], op)
        assert exl.onResize([xl], [yl]) == 0
        scale_layers = QWEN["layers"] / nl
    stream.synchronize()
    del w_arena
    build_s = time.time() - t_build0

    def enqueue():
        for ex, x, y in execs:
            assert ex.onExecute([x], [y]) == 0
        assert exl.onExecute([xl], [yl]) == 0
    with torch.cuda.stream(stream):
        enqueue()
    stream.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr, stream=stream):
        enqueue()

    def replay():
        with torch.cuda.stream(stream):
            gr.replay()

    def sync_all():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def maxr(v):
        t = torch.tensor([v], device=dev)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())
    W, K = max(args.warmup, 3), args.steps
    sampler = sampler_cls(local_rank)
    sampler.start()
    sync_all()
    ms = maxr(_timeit(torch, stream, replay, K, W))
    sampler.stop_flag = True
    sampler.join()
    # e2e: the prefill's hidden states [4096, 2048] fp32 from pinned host memory, logits [8, vocab] back to the host
    hx = torch.empty((T, QWEN["hidden"]), dtype=torch.float32).uniform_(-1, 1).pin_memory()
    hy = torch.empty((LMB, QWEN["vocab"]), dtype=torch.float32).pin_memory()

    def e2e():
        with torch.cuda.stream(stream):
            xs[QWEN["hidden"]].copy_(hx, non_blocking=True)
            gr.replay()
            hy.copy_(yl.data, non_blocking=True)
        stream.synchronize()
    sync_all()
    e2e_ms = maxr(_timeit(torch, stream, e2e, K, W))
    lm_macs = float(LMB) * QWEN["hidden"] * QWEN["vocab"]
    ops = 2.0 * (macs + lm_macs)
    if decode:
        hbm, hbm_src = _peaks()
        # algorithmic bytes of one token: every int8 weight once (+ fp32 scales / offsets / biases / activations: < 0.5 %)
        tok_bytes = wbytes + float(QWEN["hidden"]) * QWEN["vocab"]
        ach = tok_bytes / (ms / 1e3) / 1e9
        return {
            "metric": "tokens/sec (Qwen-1.8B-int8 decode step, batch 1 per GPU, quantized MatMul (W8A8 dynamic) layers, device-timed)",
            "value": world * 1e3 / ms, "unit": "tok/s", "n_gpus": world, "steps": K, "warmup": W, "ms_per_step": ms,
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "s8 x s8 -> s32, fp32 out", "data": "synthetic",
            "config": {"workload": "Qwen-1.8B linear layers, 1 token per GPU (decode), 24 transformer layers x 5 linears + lm_head, "
                                   "CUDA-graph replay", "parallelism": f"dp{world} replicas", "build_seconds": build_s,
                       "l2": f"{tok_bytes / 1e9:.2f} GB of distinct int8 weights per token exceed L2"},
            "roofline": {"bound": "hbm", "kernel": "linear_w8_gemv_kernel", "achieved": ach, "peak": hbm, "unit": "GB/s", "frac": ach / hbm,
                         "traffic": None, "peak_source": hbm_src, "bytes_per_step": tok_bytes},
            "e2e": {"value": world * 1e3 / e2e_ms, "unit": "tok/s", "h2d_bytes_per_step": int(hx.numel() * 4),
                    "d2h_bytes_per_step": int(hy.numel() * 4)},
            "gpu_launches": (len(execs) + 1) * K, "clocks": sampler.result(),     # one fused quantise + GEMV kernel per linear layer
        }
    full_ms = (ms * scale_layers) if nl != QWEN["layers"] else ms
    achieved = ops / (ms / 1e3) / 1e12
    line = {
        "metric": "inferences/sec (Qwen-1.8B-int8 prefill 8x512 per GPU, quantized MatMul (W8A8 dynamic) layers, device-timed)",
        "value": world * 1e3 / full_ms, "unit": "fwd/s", "n_gpus": world, "steps": K, "warmup": W, "ms_per_step": full_ms,
        "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "s8 x s8 -> s32, fp32 out", "data": "synthetic",
        "config": {"workload": f"Qwen-1.8B linear layers, 4096 tokens per GPU, {nl} of 24 transformer layers instantiated"
                               + ("" if nl == 24 else " (time scaled to 24)") + " + lm_head(8 tokens), CUDA-graph replay",
                   "tokens_per_gpu": T, "layers_instantiated": nl,
                   "parallelism": f"dp{world} replicas (sequences sharded), one NCCL broadcast of the int8 weight arena at build",
                   "build_seconds": build_s,
                   "l2": f"distinct int8 weights per layer ({wbytes / 1e6:.0f} MB + 311 MB lm_head) exceed L2"},
        "roofline": {"bound": "tensor", "kernel": "gemm_i8_wgmma_kernel (2-CTA cluster)", "achieved": achieved, "peak": INT8_DENSE_PEAK_TOPS,
                     "unit": "TOP/s", "frac": achieved / INT8_DENSE_PEAK_TOPS, "traffic": None,
                     "peak_source": "H100 SXM data sheet, dense int8", "ops_per_step_per_gpu": ops},
        "e2e": {"value": world * 1e3 / (e2e_ms * (scale_layers if nl != 24 else 1.0)), "unit": "fwd/s",
                "h2d_bytes_per_step": int(hx.numel() * 4), "d2h_bytes_per_step": int(hy.numel() * 4)},
        "gpu_launches": 2 * (len(execs) + 1) * K, "clocks": sampler.result(),
    }
    if not args.no_cpu_baseline and rank == 0:
        try:
            line["cpu_baseline"] = qwen_cpu_baseline()
        except Exception as e:
            line["cpu_baseline"] = {"value": None, "kind": "unavailable", "sample": repr(e)[:200]}
    return line


def qwen_cpu_baseline():
    """reference MNN_FORWARD_CPU (Memory_Low => W8A8 dynamic quant) on ONE layer shape at 256 tokens, scaled by MACs."""
    from oracle import oracle as O
    assert O.have_reference(), "oracle/_ref not present"
    tokens, ic, oc = 256, 2048, 2048
    rng = np.random.default_rng(0)
    x = rng.uniform(-1, 1, (tokens, ic)).astype(np.float32)
    wq = rng.integers(-128, 128, (oc, ic)).astype(np.int8)
    alpha = rng.uniform(0.001, 0.01, oc).astype(np.float32)
    threads = min(os.cpu_count() or 1, 32)
    os.environ["REFDUMP_TIMING_ITERS"] = "5"
    try:
        with tempfile.TemporaryDirectory() as d:
            req, out = os.path.join(d, "req.bin"), os.path.join(d, "out.bin")
            open(req, "wb").write(struct.pack("<8i", tokens, ic, oc, 0, 0, 0, 0, 0) + x.tobytes() + wq.tobytes() + alpha.tobytes())
            r = O._run_refdump(["linear", req, out, threads])
    finally:
        os.environ.pop("REFDUMP_TIMING_ITERS", None)
    j = json.loads([l for l in r.stdout.splitlines() if l.startswith("{")][-1])
    macs_s = tokens * ic * oc / (j["ms_per_iter"] / 1e3)
    total = sum(QWEN["tokens"] * ic_ * oc_ for ic_, oc_, _ in qwen_shapes()) * QWEN["layers"] + QWEN["batch"] * QWEN["hidden"] * QWEN["vocab"]
    return {"value": macs_s / total, "unit": "fwd/s", "cores": threads, "kind": "reference",
            "sample": f"refdump linear {tokens}x{ic}->{oc}, 5 timed runs, scaled by MACs to the full forward ({total / 1e12:.2f} TMAC)"}
