"""Sessions over a parsed .mnn model: the role of Session/Pipeline (source/core/Session.cpp, Pipeline.cpp) for the
hot path -- create executions (weights -> HBM once), resize (shapes + quant fold), run (enqueue; CUDA-graph replay).

ConvPathSession runs ONLY the dense int8 convolutions of a model, each on its own resident synthetic activation
(BASELINE.json configs[1]: "ConvInt8 im2col+IMMA path only").  WholeNetSession (added later) chains every op.
"""
import ctypes as C
from typing import List, Optional

import numpy as np
import torch

from . import _capi, graph, mnn_file
from .backend import Backend, ConvGroupExecution, Op, QuantAttr, Runtime, Tensor, up16


def _qattr(q: Optional[mnn_file.QuantInfo]) -> QuantAttr:
    return QuantAttr(q.scale, q.zero, q.min, q.max) if q is not None else QuantAttr()


def conv_op_from_node(node: mnn_file.OpNode) -> Op:
    c = node.conv
    ph, pw = node.attrs.get("resolved_pad", c.pad)
    depthwise = node.type in ("ConvolutionDepthwise", "DepthwiseConvInt8")
    taps = c.kernel[0] * c.kernel[1]
    if not depthwise:
        # a grouped (group > 1, not depthwise) convolution carries oc * (ic / group) * taps weights: the dense-conv C ABI
        # would index it as oc * ic * taps.  The plugin declines those (b200_plugin.cpp: cm->group() != 1); so does this host.
        if c.group != 1:
            raise NotImplementedError(f"{node.name}: grouped convolution (group={c.group}) is outside the dense int8 conv path")
        ic = c.ic if c.ic > 0 else (c.weight.size // (c.oc * taps) if c.weight is not None else 0)   # inputCount may be 0 (derived from the weight)
        if c.weight is not None and c.weight.size != c.oc * ic * taps:
            raise ValueError(f"{node.name}: weight has {c.weight.size} elements, expected oc*ic*kh*kw = {c.oc * ic * taps}")
    else:
        ic = c.oc
    return Op(type="DepthwiseConvInt8" if depthwise else "ConvInt8", name=node.name,
              conv=dict(ic=ic, oc=c.oc, kernel=c.kernel, stride=c.stride, pad=(ph, pw),
                        dilate=c.dilate, group=c.group if depthwise else 1,
                        relu=c.relu or c.relu6),   # relu6 is treated as relu on the int8 path (ConvInt8TiledExecutor.cpp:81)
              weight=c.weight, wscale=c.alpha, bias=c.bias,
              # ConvInt8Winograd::mustUse (CPUConvolution.cpp:336-339): a conv that carries a winogradAttr runs as Winograd
              extra=dict(shape_known=True, **({"winograd_attr": c.winograd_attr} if (c.winograd_attr is not None and not depthwise) else {})))


class ConvPathSession:
    def __init__(self, model, batch: int, device_id: int = 0, input_hw=(224, 224), seed: int = 0):
        self.stream = torch.cuda.Stream(device=device_id)
        with torch.cuda.stream(self.stream):
            self.runtime = Runtime(device_id)            # adopts self.stream
        self.backend: Backend = self.runtime.onCreate()
        self.net = model if isinstance(model, mnn_file.Net) else mnn_file.load(model)
        self.batch = batch
        ic0 = next(op for op in self.net.ops if op.type == "Input").attrs["dims"][1]
        self.shapes = graph.infer_shapes(self.net, (batch, ic0) + tuple(input_hw))
        self.layers = []
        g = torch.Generator(device="cpu").manual_seed(seed)
        self.bytes = 0.0
        self.macs = 0.0
        with torch.cuda.stream(self.stream):
            for node in graph.dense_convs(self.net):
                op = conv_op_from_node(node)
                n, c, h, w = node.attrs["in_shape"]
                x = self.backend.onAcquire(Tensor((n, c, h, w), "int8", _qattr(self.net.quant.get(node.inputs[0]))))
                # synthetic activations, resident in HBM; channel padding stays zero
                x.data[..., :c] = torch.randint(-127, 128, (n, h, w, c), generator=g, dtype=torch.int8).to(x.data.device)
                y = Tensor(self.shapes[node.outputs[0]], "int8", _qattr(self.net.quant.get(node.outputs[0])))
                ex = self.backend.onCreate([x], [y], op)
                if ex is None:
                    raise RuntimeError(f"no CUDA execution for {node.name}: there is no CPU fallback")
                st = ex.onResize([x], [y])
                if st != 0:
                    raise RuntimeError(f"onResize({node.name}) -> {st}: {_capi.lib().mnnb200_last_error().decode()}")
                self.backend.onAcquire(y)
                b, m = ex.cost()
                self.bytes += b
                self.macs += m
                self.layers.append((node, ex, x, y))
            # every layer here reads its own resident activation, so all GEMM-shaped layers (1x1, stride 1) go into ONE
            # persistent launch (conv group); the rest (3x3 stem, strided convs) keep their own kernels
            self.group = None
            self.singles = list(self.layers)
            members = [l for l in self.layers if ConvGroupExecution.groupable(l[1])]
            if len(members) >= 2:
                self.group = ConvGroupExecution(self.backend, [l[1] for l in members])
                st = self.group.bind([l[2] for l in members], [l[3] for l in members])
                if st != 0:
                    raise RuntimeError(f"conv_group_bind -> {st}: {_capi.lib().mnnb200_last_error().decode()}")
                ids = {id(l[1]) for l in members}
                self.singles = [l for l in self.layers if id(l[1]) not in ids]
        self.stream.synchronize()
        self.graph: Optional[torch.cuda.CUDAGraph] = None
        self.launches_per_step = len(self.singles) + (self.group.launches() if self.group is not None else 0)

    def enqueue(self):
        for node, ex, x, y in self.singles:
            st = ex.onExecute([x], [y])
            if st != 0:
                raise RuntimeError(f"onExecute({node.name}) -> {st}: {_capi.lib().mnnb200_last_error().decode()}")
        if self.group is not None:
            st = self.group.onExecute()
            if st != 0:
                raise RuntimeError(f"conv_group_execute -> {st}: {_capi.lib().mnnb200_last_error().decode()}")

    def capture(self):
        with torch.cuda.stream(self.stream):
            self.enqueue()                      # warm (module load, attribute set) outside capture
        self.stream.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph, stream=self.stream):
            self.enqueue()
        return self.graph

    def run(self):
        """One step: all dense convs of the model over one batch (enqueue only)."""
        with torch.cuda.stream(self.stream):
            if self.graph is not None:
                self.graph.replay()
            else:
                self.enqueue()

    # ---- e2e: host buffers in, host buffers out, through the same C ABI
    def make_host_io(self):
        node0, _, x0, _ = self.layers[0]
        n, c, h, w = x0.shape
        self.h_in = torch.empty((n, c, h, w), dtype=torch.float32).uniform_(-1, 1).pin_memory()
        self.d_in = torch.empty((n, c, h, w), dtype=torch.float32, device=self.runtime.device)
        nodeL, _, _, yL = self.layers[-1]
        self.d_out = torch.empty(yL.shape, dtype=torch.float32, device=self.runtime.device)
        self.h_out = torch.empty(yL.shape, dtype=torch.float32).pin_memory()
        return self.h_in.numel() * 4, self.h_out.numel() * 4

    def run_e2e(self):
        L, rt = _capi.lib(), self.runtime._h
        _, _, x0, _ = self.layers[0]
        _, _, _, yL = self.layers[-1]
        with torch.cuda.stream(self.stream):
            self.d_in.copy_(self.h_in, non_blocking=True)                       # H2D from pinned memory
            n, c, h, w = x0.shape
            q = x0.quant
            _capi.check(L.mnnb200_float_to_int8(rt, C.c_void_p(self.d_in.data_ptr()), n, c, h, w, q.scale, q.zero,
                                                int(q.min), int(q.max), x0.ptr()))
            if self.graph is not None:
                self.graph.replay()
            else:
                self.enqueue()
            n, c, h, w = yL.shape
            q = yL.quant
            _capi.check(L.mnnb200_int8_to_float(rt, yL.ptr(), n, c, h, w, q.scale, q.zero,
                                                C.c_void_p(self.d_out.data_ptr())))
            self.h_out.copy_(self.d_out, non_blocking=True)                     # D2H of the result


    def run_e2e_pipelined(self, steps: int):
        """`steps` end-to-end steps with the host<->device copies of step k+1 overlapped with the kernels of step k -- what a
        serving loop does with two pinned input buffers.  Every step still copies ITS OWN input from pinned host memory and its
        own result back to the host; ordering is enforced with events (copy stream <-> compute stream), nothing is skipped."""
        L, rt = _capi.lib(), self.runtime._h
        _, _, x0, _ = self.layers[0]
        _, _, _, yL = self.layers[-1]
        if not hasattr(self, "_pipe"):
            self._pipe = dict(copy=torch.cuda.Stream(device=self.runtime.device),
                              d_in=[torch.empty_like(self.d_in) for _ in range(2)],
                              h_out=[torch.empty_like(self.h_out).pin_memory() for _ in range(2)],
                              in_ready=[torch.cuda.Event() for _ in range(2)], in_free=[torch.cuda.Event() for _ in range(2)])
        P = self._pipe
        n, c, h, w = x0.shape
        qi, qo = x0.quant, yL.quant
        on, oc, oh, ow = yL.shape
        for k in range(steps):
            b = k & 1
            with torch.cuda.stream(P["copy"]):
                if k >= 2:
                    P["copy"].wait_event(P["in_free"][b])            # the cast of step k-2 has consumed this buffer
                P["d_in"][b].copy_(self.h_in, non_blocking=True)       # H2D of step k's input
                P["in_ready"][b].record(P["copy"])
            with torch.cuda.stream(self.stream):
                self.stream.wait_event(P["in_ready"][b])
                _capi.check(L.mnnb200_float_to_int8(rt, C.c_void_p(P["d_in"][b].data_ptr()), n, c, h, w, qi.scale, qi.zero,
                                                    int(qi.min), int(qi.max), x0.ptr()))
                P["in_free"][b].record(self.stream)
                if self.graph is not None:
                    self.graph.replay()
                else:
                    self.enqueue()
                _capi.check(L.mnnb200_int8_to_float(rt, yL.ptr(), on, oc, oh, ow, qo.scale, qo.zero,
                                                    C.c_void_p(self.d_out.data_ptr())))
                P["h_out"][b].copy_(self.d_out, non_blocking=True)     # D2H of step k's result
        self.stream.synchronize()
        P["copy"].synchronize()


class WholeNetSession:
    """Runs EVERY op of an int8 CNN .mnn on the GPU (no CPU fallback), following the reference pipeline's
    quantisation decisions (source/core/Pipeline.cpp:241-400 with the rules of CPUBackend.cpp:898-980):
      Convolution / ConvolutionDepthwise (IDST int8 weights), BinaryOp, Softmax  -> int8
      Pooling                         -> int8 only when in/out quant attrs are equal, else float bracketed by casts
                                         (here: one fused kernel with the same arithmetic)
      Reshape / Squeeze / ConvertTensor (geometry "Raster")  -> int8 only when in/out quant attrs are equal, else float
      casts (FloatToInt8 / Int8ToFloat) are inserted where producer and consumer disagree.
    The network input is fp32 NCHW (FloatToInt8 inside the copy), the output fp32 (dequantised)."""

    def __init__(self, model, batch: int, device_id: int = 0, input_hw=(224, 224)):
        self.stream = torch.cuda.Stream(device=device_id)
        with torch.cuda.stream(self.stream):
            self.runtime = Runtime(device_id)
        self.backend: Backend = self.runtime.onCreate()
        self.net = model if isinstance(model, mnn_file.Net) else mnn_file.load(model)
        net = self.net
        self.batch = batch
        in_node = next(op for op in net.ops if op.type == "Input")
        ic0 = in_node.attrs["dims"][1]
        self.shapes = graph.infer_shapes(net, (batch, ic0) + tuple(input_hw))
        self.T = {}          # tensor index -> Tensor (current materialisation)
        self.steps = []      # (name, execution, inputs, outputs)
        self.bytes = 0.0     # algorithmic bytes of the dense convs only (the roofline figure of BASELINE configs[1])
        self.checkpoints = {}
        dev = self.runtime.device
        with torch.cuda.stream(self.stream):
            self._build(net, in_node, dev)
        self.stream.synchronize()
        self.graph = None
        self.launches_per_step = len(self.steps)

    # -- helpers
    def _q(self, idx):
        return _qattr(self.net.quant.get(idx))

    def _shape4(self, idx):
        s = self.shapes[idx]
        return s if len(s) == 4 else (s[0], s[1], 1, 1)

    def _add(self, name, ex, ins, outs):
        st = ex.onResize(ins, outs)
        if st != 0:
            raise RuntimeError(f"onResize({name}) -> {st}: {_capi.lib().mnnb200_last_error().decode()}")
        for o in outs:
            if o.data is None:
                self.backend.onAcquire(o)
        self.steps.append((name, ex, ins, outs))

    def _as_int8(self, idx, name):
        t = self.T[idx]
        if t.dtype == "int8":
            return t
        q = Tensor(self._shape4(idx), "int8", self._q(idx))
        self._add(name + "_FloatToInt8", self.backend.onCreate([t], [q], Op(type="FloatToInt8")), [t], [q])
        return q

    def _as_float(self, idx, name):
        t = self.T[idx]
        if t.dtype == "float":
            return t
        f = Tensor(self._shape4(idx), "float")
        self._add(name + "_Int8ToFloat", self.backend.onCreate([t], [f], Op(type="Int8ToFloat")), [t], [f])
        return f

    def _build(self, net, in_node, dev):
        n, c, h, w = self.shapes[in_node.outputs[0]]
        self.input = self.backend.onAcquire(Tensor((n, c, h, w), "float"))
        self.T[in_node.outputs[0]] = self.input
        same_q = lambda a, b: (self._q(a).scale == self._q(b).scale and self._q(a).zero == self._q(b).zero and self._q(a).scale != 0)
        for node in net.ops:
            t = node.type
            if t == "Input":
                continue
            if t in ("Convolution", "ConvolutionDepthwise"):
                x = self._as_int8(node.inputs[0], node.name)
                y = Tensor(self._shape4(node.outputs[0]), "int8", self._q(node.outputs[0]))
                op = conv_op_from_node(node)
                ex = self.backend.onCreate([x], [y], op)
                if ex is None:
                    raise RuntimeError(f"no CUDA execution for {node.name}: there is no CPU fallback")
                self._add(node.name, ex, [x], [y])
                if t == "Convolution":
                    self.bytes += ex.cost()[0]
                self.T[node.outputs[0]] = y
            elif t == "BinaryOp":
                if node.attrs.get("op_type", 0) != 0:
                    raise NotImplementedError("BinaryOp other than ADD")
                a = self._as_int8(node.inputs[0], node.name)
                b = self._as_int8(node.inputs[1], node.name)
                y = Tensor(self._shape4(node.outputs[0]), "int8", self._q(node.outputs[0]))
                self._add(node.name, self.backend.onCreate([a, b], [y], Op(type="BinaryAddInt8")), [a, b], [y])
                self.T[node.outputs[0]] = y
            elif t == "Pooling":
                if node.attrs.get("pool_type", 0) != 1:
                    raise NotImplementedError("max pooling")
                # float pooling between casts == the fused kernel; with equal quant attrs the reference would take its
                # int8 pooling ((sum*factor)>>24, CPUPoolInt8.cpp), which is not implemented here
                if same_q(node.inputs[0], node.outputs[0]):
                    raise NotImplementedError("int8 pooling with identical quant attrs (CPUPoolInt8 fixed-point path)")
                x = self._as_int8(node.inputs[0], node.name)
                y = Tensor(self._shape4(node.outputs[0]), "int8", self._q(node.outputs[0]))
                self._add(node.name, self.backend.onCreate([x], [y], Op(type="AvgPoolInt8", extra=node.attrs)), [x], [y])
                self.T[node.outputs[0]] = y
            elif t in ("ConvertTensor", "Squeeze", "Reshape"):
                src = node.inputs[0]
                s4 = self._shape4(src)
                assert s4[2] == 1 and s4[3] == 1, "layout-changing Raster on a spatial tensor is outside the path"
                if same_q(src, node.outputs[0]) and self.T[src].dtype == "int8":
                    v = self.T[src]
                    self.T[node.outputs[0]] = Tensor(self._shape4(node.outputs[0]), "int8", self._q(node.outputs[0]), v.data)
                else:
                    v = self._as_float(src, node.name)
                    self.T[node.outputs[0]] = Tensor(self._shape4(node.outputs[0]), "float", None, v.data)
            elif t == "Shape":
                self.T[node.outputs[0]] = None
            elif t == "Softmax":
                x = self._as_int8(node.inputs[0], node.name)
                y = Tensor(self._shape4(node.outputs[0]), "int8", self._q(node.outputs[0]))
                self._add(node.name, self.backend.onCreate([x], [y], Op(type="SoftmaxInt8")), [x], [y])
                self.T[node.outputs[0]] = y
            else:
                raise NotImplementedError(f"op {t} ({node.name}) is outside the int8 CNN path: no CPU fallback")
            if node.outputs and self.T.get(node.outputs[0]) is not None:
                self.checkpoints[node.name] = self.T[node.outputs[0]]
        last = [op for op in net.ops if op.outputs][-1].outputs[0]
        self.output = self._as_float(last, "output")

    def enqueue(self):
        for name, ex, ins, outs in self.steps:
            st = ex.onExecute(ins, outs)
            if st != 0:
                raise RuntimeError(f"onExecute({name}) -> {st}: {_capi.lib().mnnb200_last_error().decode()}")

    def capture(self):
        with torch.cuda.stream(self.stream):
            self.enqueue()
        self.stream.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph, stream=self.stream):
            self.enqueue()
        return self.graph

    def run(self):
        with torch.cuda.stream(self.stream):
            if self.graph is not None:
                self.graph.replay()
            else:
                self.enqueue()

    def set_input(self, x_nchw: np.ndarray):
        with torch.cuda.stream(self.stream):
            self.input.data.copy_(torch.from_numpy(np.ascontiguousarray(x_nchw, np.float32)))

    def get_output(self) -> np.ndarray:
        self.stream.synchronize()
        return self.output.data.cpu().numpy().reshape(self.shapes[[op for op in self.net.ops if op.outputs][-1].outputs[0]])

    def read_int8(self, name) -> np.ndarray:
        """a checkpoint tensor as logical NCHW int8 (or fp32 for float tensors)"""
        self.stream.synchronize()
        t = self.checkpoints[name]
        with torch.cuda.stream(self.stream):
            out = self.backend.onCopyBuffer(t, "same")
        return out

    # ---- e2e with host buffers
    def make_host_io(self):
        self.h_in = torch.empty(self.input.shape, dtype=torch.float32).uniform_(-1, 1).pin_memory()
        self.h_out = torch.empty(tuple(self.output.data.shape), dtype=torch.float32).pin_memory()
        return self.h_in.numel() * 4, self.h_out.numel() * 4

    def run_e2e(self):
        with torch.cuda.stream(self.stream):
            self.input.data.copy_(self.h_in, non_blocking=True)
            if self.graph is not None:
                self.graph.replay()
            else:
                self.enqueue()
            self.h_out.copy_(self.output.data, non_blocking=True)
