"""The conv-group kernel's clamp (conv_group_wgmma.cu, -m gpu): the epilogue clamps the rounded integers on s16 pairs, and clears
the pad channels' bytes only in the chunk that holds channels >= OC of a layer whose clamp excludes 0.  Layers with narrowed,
full-range, all-negative and empty (min > max) clamps and ReLU with a non-zero output zero point, in both layer modes, with
many outputs at both bounds, equal the C oracle bit for bit; NHWC16 channel padding must come back zero."""
import numpy as np
import pytest

from oracle import oracle as O
from tests.test_gpu_conv_group import Layer, Pending, acc_u, case, pool, run_group

pytestmark = pytest.mark.gpu


class ClampLayer(Layer):
    """A Layer whose output quantisation carries the clamp c["clamp"] = (min, max) instead of [-127, 127]."""

    def resize(self):
        from mnn_b200.backend import QuantAttr, Tensor
        c, be = self.c, self.backend
        n, ic, ih, iw = c["x"].shape
        lo, hi = c["clamp"]
        qi, qo = QuantAttr(c["s_in"], c["z_in"], -128, 127), QuantAttr(c["s_out"], c["z_out"], lo, hi)
        self.xin = be.onAcquire(Tensor((n, ic, ih, iw), "int8", qi))
        be.onCopyBuffer(c["x"], self.xin)
        self.yout = Tensor((n, self.oc, 1, 1), "int8", qo)
        if self.ex is None:
            self.ex = be.onCreate([self.xin], [self.yout], self.op)
        assert self.ex.onResize([self.xin], [self.yout]) == 0
        be.onAcquire(self.yout)

    def bounds(self):
        lo, hi = self.c["clamp"]
        return (self.c["z_out"] if self.c["relu"] else lo), hi

    def submit(self, images=None):
        c = self.c
        bf, sx = O.fold_modern(c["w"], c["ws"], c["bias"], c["s_in"], c["z_in"], c["s_out"], c["z_out"])
        lo, hi = self.bounds()
        x = c["x"] if images is None else c["x"][list(images)]
        parts = np.array_split(np.arange(x.shape[0]), x.shape[0])
        run = lambda idx: O.conv_int8(x[idx], c["w"], c["ws"], sx, bf, stride=c["stride"], pad=c["pad"], dilate=c["dilate"],
                                      z_in=c["z_in"], min_v=lo, max_v=hi)
        return Pending([pool().submit(run, p) for p in parts if p.size])


def spread(c, width):
    """Scale the weight scales so that the requantised values spread over about +-width around the output zero point."""
    oc = c["w"].shape[0]
    real = acc_u(c) - (c["z_in"] + 128) * c["w"].astype(np.int64).reshape(oc, -1).sum(1)[None, :, None, None]
    c["ws"] = np.full(oc, width / (real.std() * np.float32(c["s_in"]) / np.float32(c["s_out"])), np.float32)
    c["bias"] = np.zeros(oc, np.float32)
    return c


def test_conv_group_clamps(backend):
    rng = np.random.default_rng(77)
    specs = [
        # name, (ic, oc, k, n, hw, pad), relu, z_in, z_out, clamp, spread, masked (the chunk with pad channels clears them)
        ("relu_zp6", (64, 40, (1, 1), 2, (9, 13), (0, 0)), 1, 0, 6, (-127, 127), 120, True),
        ("narrow", (48, 72, (1, 1), 2, (10, 11), (0, 0)), 0, 2, -3, (-60, 45), 200, False),
        ("negative", (32, 37, (3, 3), 2, (10, 12), (1, 1)), 0, 4, -5, (-100, -20), 200, True),
        ("full_range", (200, 130, (1, 1), 2, (9, 10), (0, 0)), 0, -3, 1, (-128, 127), 400, False),
        ("empty", (40, 24, (3, 3), 1, (8, 9), (1, 1)), 1, -2, 5, (-127, 3), 100, True),
    ]
    layers = []
    for name, (ic, oc, k, n, hw, pad), relu, z_in, z_out, clamp, width, _ in specs:
        c = spread(case(rng, ic, oc, k, n, hw, pad=pad, relu=relu, z_in=z_in), width)
        c["z_out"], c["clamp"] = z_out, clamp
        layers.append(ClampLayer(backend, c))
    refs = [L.submit() for L in layers]
    for L, (name, (_, oc, k, *_), _, _, _, _, _, masked) in zip(layers, specs):
        p = L.plan()
        assert p["mode"] == (0 if k == (1, 1) else 1), (name, p)
        lo, hi = L.bounds()
        assert (oc % 16 != 0 and (lo > 0 or hi < 0)) == masked, name
    run_group(backend, layers)
    for L, (name, *_), r in zip(layers, specs, refs):
        y = L.check(r.result()).astype(int)
        lo, hi = L.bounds()
        if lo > hi:
            assert (y == lo).all(), name
        else:
            assert y.min() >= lo and y.max() <= hi, name
            assert 0.05 <= (y == lo).mean() and 0.05 <= (y == hi).mean(), (name, (y == lo).mean(), (y == hi).mean())


def test_clamp_outside_s16_is_not_grouped(backend):
    # the kernel packs to s16 before it clamps: bounds outside that range are left to the mma.sync kernel
    from mnn_b200.backend import ConvGroupExecution
    rng = np.random.default_rng(3)
    c = case(rng, 32, 16, (1, 1), 1, (4, 4))
    c["clamp"] = (-127, 40000)
    assert not ConvGroupExecution.groupable(ClampLayer(backend, c).ex)
    c = case(rng, 32, 16, (1, 1), 1, (4, 4))
    c["clamp"] = (-127, 127)
    assert ConvGroupExecution.groupable(ClampLayer(backend, c).ex)
