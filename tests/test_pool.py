"""Float Pooling (CPUPool): the oracle's restatement (O.pool_f32 / O.pool_resolve) against the reference CPU backend and the
committed fixture, and the session path's parameter resolution against the oracle's.  POOL_CONFIGS is shared with the GPU
tests (tests/test_gpu_neighbours.py) and with tests/golden/make_golden.py."""
import os

import numpy as np
import pytest

from oracle import oracle as O

GOLD = os.path.join(os.path.dirname(__file__), "golden", "pool_golden.npz")
needs_ref = pytest.mark.skipif(not O.have_reference(), reason="oracle/_ref not built")
CAFFE, VALID, SAME = O.POOL_CAFFE, O.POOL_VALID, O.POOL_SAME
DEFAULT, INCLUDE, EXCLUDE = 0, 1, 2


def pc(ih, iw, k, s, pad=(0, 0), pads=None, pt=CAFFE, ct=DEFAULT, ceil=True, glob=False):
    return dict(ih=ih, iw=iw, kernel=k, stride=s, pad=pad, pads=pads, pad_type=pt, count_type=ct, ceil_model=ceil,
                is_global=glob)


# pad types x count types, `pads` of 2 and 4 values, kernels larger than the padded input, strides larger than the kernel,
# ceil mode (windows that start past the input), windows wholly in the padding, global pooling
POOL_CONFIGS = [
    pc(7, 9, (3, 3), (2, 2), (1, 1)),                                   # CAFFE DEFAULT: border windows count the padding
    pc(8, 8, (3, 3), (2, 2), (1, 1), ct=INCLUDE, ceil=False),
    pc(8, 7, (3, 3), (2, 2), (1, 1), ct=EXCLUDE),
    pc(5, 5, (2, 2), (3, 3), (1, 1)),                                   # stride > kernel, ceil: the last window starts past the input
    pc(6, 9, (1, 2), (2, 3), (0, 1), ct=EXCLUDE),
    pc(7, 6, (3, 3), (2, 2), pads=[1, 0, 2, 1]),                        # 4 pads: begin pads from pads, runs as VALID
    pc(7, 6, (3, 3), (2, 2), pads=[1, 2, 0, 1], ct=INCLUDE),
    pc(6, 6, (3, 3), (1, 1), (0, 1), pads=[1, 1]),                      # 2 pads: height grows, begin pads stay padY / padX
    pc(7, 5, (2, 2), (2, 2), (1, 0), pads=[0, 2], ct=INCLUDE),
    pc(9, 8, (3, 3), (2, 2), pt=VALID),
    pc(5, 6, (3, 2), (1, 2), pt=VALID, ct=INCLUDE),
    pc(7, 8, (3, 3), (2, 2), pt=SAME),
    pc(7, 8, (3, 3), (2, 2), pt=SAME, ct=INCLUDE),
    pc(10, 11, (4, 4), (3, 3), pt=SAME, ct=EXCLUDE),
    pc(4, 5, (7, 7), (1, 1), (1, 1)),                                   # kernel larger than the padded input
    pc(3, 3, (5, 5), (1, 1), pt=SAME),                                  # ... and its SAME pad uses the unclamped kernel
    pc(4, 5, (6, 6), (2, 2), pt=VALID, ct=INCLUDE),
    pc(8, 8, (3, 3), (2, 2)),                                           # ceil mode without padding: partial last windows
    pc(5, 6, (3, 3), (2, 2), (3, 3), ceil=False),                       # windows wholly in the padding
    pc(7, 7, (1, 1), (1, 1), glob=True),                                # MobileNet's global pool
    pc(5, 3, (2, 2), (2, 2), (1, 1), pt=SAME, ct=INCLUDE, glob=True),
]
POOL_ATTRS = ("kernel", "stride", "pad", "pads", "pad_type", "count_type", "ceil_model", "is_global")


def pool_kwargs(cfg):
    return {k: cfg[k] for k in POOL_ATTRS}


def pool_input(rng, n, c, cfg):
    return rng.uniform(-4, 4, (n, c, cfg["ih"], cfg["iw"])).astype(np.float32)


def session_attrs(cfg):
    """the Pooling node attrs mnn_file.py produces for this config"""
    a = dict(kernel=cfg["kernel"], stride=cfg["stride"], pad=cfg["pad"], pad_type=cfg["pad_type"],
             count_type=cfg["count_type"], ceil_model=cfg["ceil_model"], is_global=cfg["is_global"], pool_type=1)
    if cfg["pads"] is not None:
        a["pads"] = list(cfg["pads"])
    return a


def test_pool_oracle_vs_golden():
    """tests/golden/pool_golden.npz: float Pooling outputs of the reference CPU backend (make_golden.py pool)."""
    g = np.load(GOLD)
    assert int(g["ncase"]) >= 12
    for i in range(int(g["ncase"])):
        cfg = POOL_CONFIGS[int(g[f"p{i}_cfg"])]
        y = O.pool_f32(g[f"p{i}_x"], bool(g[f"p{i}_avg"]), **pool_kwargs(cfg))
        ref = g[f"p{i}_y"]
        assert y.shape == ref.shape and np.array_equal(y.view(np.uint32), ref.view(np.uint32)), (i, cfg)


@needs_ref
@pytest.mark.reference
@pytest.mark.parametrize("is_avg", [True, False], ids=["ave", "max"])
@pytest.mark.parametrize("ci", range(len(POOL_CONFIGS)))
def test_pool_oracle_vs_live_reference(ci, is_avg):
    cfg = POOL_CONFIGS[ci]
    x = pool_input(np.random.default_rng(100 + ci), 2, 5, cfg)
    ref = O.ref_pool_f32(x, is_avg, **pool_kwargs(cfg))
    y = O.pool_f32(x, is_avg, **pool_kwargs(cfg))
    assert y.shape == ref.shape
    assert np.array_equal(y.view(np.uint32), ref.view(np.uint32)), np.argwhere(y != ref)[:5]


@pytest.mark.parametrize("ci", range(len(POOL_CONFIGS)))
def test_session_pool_params_vs_oracle(ci):
    """The session path (AvgPoolInt8Execution) resolves output size, kernel, stride, begin pads and pad type as CPUPool does."""
    from mnn_b200.graph import float_pool_params
    cfg = POOL_CONFIGS[ci]
    oh, ow, k, s, p, pt = O.pool_resolve(cfg["ih"], cfg["iw"], cfg["kernel"], cfg["stride"], cfg["pad"], cfg["pads"],
                                         cfg["pad_type"], cfg["ceil_model"], cfg["is_global"])
    got = float_pool_params(cfg["ih"], cfg["iw"], session_attrs(cfg))
    assert (got[0], got[1], tuple(got[2]), tuple(got[3]), tuple(got[4]), got[5]) == (oh, ow, k, s, p, pt)
