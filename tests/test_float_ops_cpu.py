"""The float64 restatements and bounds of oracle/ops_oracle.py against the live reference CPU (oracle/_ref/refdump_ops, -m reference,
no GPU): the Softmax and SUM / MEAN / PROD Reduction cases that tests/test_gpu_plugin_float_ops.py holds to bounds lie within
them on the CPU too, the CPU's own error on the transcendental UnaryOps is what that module adds to the GPU's bound, and the CPU
behaviours the fp32 kernels restate (MIN / MAX and max-pool selection, the fused ReLU, ABS / NEG, the Reduction's first element,
Scale's single rounding) are what the CPU computes."""
import numpy as np
import pytest

from oracle import ops_oracle as O

pytestmark = pytest.mark.reference
CASES = O.all_cases()
# the CPU's worst error against float64 in ulps, measured over each op's case (x86 with AVX512).  Its polynomial EXP, SIGMOID,
# GELU, GELU_STANDARD and SILU clamp their argument, so in the saturated tails it returns 0, a clamped value or FLT_MAX-range
# numbers where float64 has tiny or overflowing ones: the large maxima below are those tails, not noise
CPU_ULPS = {"EXP": 1.91e7, "LOG": 0.69, "SIGMOID": 1.18e7, "TANH": 758, "GELU": 1.68e7, "GELU_STANDARD": 1.68e7, "SILU": 1.30e9}


@pytest.fixture(scope="module")
def cpu():
    if not O.have_refdump():
        pytest.skip("oracle/_ref/refdump_ops is built by build() where the reference sources are")
    return dict(zip(CASES, O.run(list(CASES.values()))))


def _one(case):
    r = O.run([case])[0]
    assert r["ok"]
    return r["ys"][0]


@pytest.mark.parametrize("name", [n for n in CASES if CASES[n]["kind"] == "softmax" and not n.startswith("declined")
                                  and "special" not in n])
def test_softmax_within_bound(cpu, name):
    c = CASES[name]
    for xs, y in zip(c["runs"], cpu[name]["ys"]):
        axis = c["ip"][0]
        assert (np.abs(y - O.softmax64(xs[0], axis)) <= O.softmax_bound(xs[0], axis)).all()


@pytest.mark.parametrize("name", [n for n in CASES if CASES[n]["kind"] == "reduce" and "special" not in n and
                                  CASES[n]["ip"][0] in (O.REDUCE["SUM"], O.REDUCE["MEAN"], O.REDUCE["PROD"])])
def test_sum_mean_prod_within_bound(cpu, name):
    c = CASES[name]
    op = [k for k, v in O.REDUCE.items() if v == c["ip"][0]][0]
    x, y = c["runs"][0][0], cpu[name]["ys"][0]
    y64 = O.reduce64(x, op, c["ip"][2:], c["ip"][1])
    assert (np.abs(y - y64) <= O.sum_bound(x, c["ip"][2:], op).reshape(y64.shape)).all()


@pytest.mark.parametrize("op", O.UNARY_TRANSCENDENTAL)
def test_unary_cpu_error_is_the_measured_one(cpu, op):
    x, y = CASES[f"unary_{op}"]["runs"][0][0], cpu[f"unary_{op}"]["ys"][0]
    e = O.ulp_error(y, O.unary64(op, x))
    print(f"{op}: CPU max {e.max():.3g} ulp vs float64")
    assert e.max() <= CPU_ULPS[op]


def test_min_max_take_the_second_operand_unless_the_first_wins(cpu):
    """VecBinaryMin / VecBinaryMax are minps / maxps in the vector body and in the tail alike"""
    a = np.array([-0.0, 0.0, np.nan, 1, 2, 0.0, -0.0], np.float32)
    b = np.array([0.0, -0.0, 1, np.nan, 3, -0.0, 0.0], np.float32)
    for op, pick in (("MAXIMUM", a > b), ("MINIMUM", a < b)):
        for n in (7, 4 * 7):   # tail only, vector body
            aa, bb = np.tile(a, n // 7), np.tile(b, n // 7)
            y = _one(O.case("binary", [[aa, bb]], ip=[O.BINARY[op], 0]))
            assert O.same_bits(y, np.where(np.tile(pick, n // 7), aa, bb))


def test_fused_relu_and_relu_keep_the_sign_of_zero_and_nan(cpu):
    """CPURelu(0): x < 0 ? x * 0 : x, so -3 -> -0, -inf -> NaN, NaN -> NaN"""
    v = np.array([-3, -0.0, 0, np.nan, -np.inf, np.inf, 2, -1e-40, 5], np.float32)
    def relu(v):
        with np.errstate(invalid="ignore"):
            return np.where(v < 0, v * np.float32(0), v)
    assert O.same_bits(_one(O.case("relu", [[v]], fp=[0.0])), relu(v))
    assert O.same_bits(_one(O.case("binary", [[v, np.zeros_like(v)]], ip=[O.BINARY["ADD"], 1])), relu(v + np.float32(0)))


def test_abs_and_neg_forms(cpu):
    """ABS is MNNReluWithSlope(x, -1): |-0| = +0, |NaN| = +0; NEG is x * -1 + 0: -(+0) = +0"""
    v = np.array([-3, -0.0, 0, np.nan, -np.inf, 2, -1e-40], np.float32)
    assert O.same_bits(_one(O.case("unary", [[v]], ip=[O.UNARY["ABS"]])),
                       np.array([3, 0, 0, 0, np.inf, 2, 1e-40], np.float32))
    assert O.same_bits(_one(O.case("unary", [[v]], ip=[O.UNARY["NEG"]])),
                       np.array([3, 0, 0, np.nan, np.inf, -2, 1e-40], np.float32))


def test_reduction_max_starts_from_the_first_element(cpu):
    """a row of -inf reduces to -inf, a NaN is kept only when it comes first, of -0 and +0 the first stays"""
    x = np.array([[-np.inf] * 3, [np.nan, 1, 2], [1, np.nan, 2], [-0.0, 0.0, 1e-45 * 0], [0.0, -0.0, -1]], np.float32)
    y = _one(O.case("reduce", [[x]], ip=[O.REDUCE["MAXIMUM"], 0, 1]))
    assert O.same_bits(y, np.array([-np.inf, np.nan, 2, -0.0, 0.0], np.float32))


def test_max_pool_takes_the_tap_unless_the_running_max_is_greater(cpu):
    """VEC::max(max, tap) in tap order: a NaN tap is replaced by the next tap, a NaN last tap stays"""
    x = np.array([[[[np.nan, 1], [2, 3]], [[1, 2], [3, np.nan]]]], np.float32)
    y = _one(O.case("pool", [[x]], ip=[O.POOL_MAX, 2, 2, 1, 1, O.PAD_VALID, 0, 0, 0, 0, 0, 0]))
    assert O.same_bits(y.reshape(-1), np.array([3, np.nan], np.float32))


def test_scale_rounds_once(cpu):
    """MNNScaleAndAddBias on AVX512 is one fused multiply-add per element"""
    c = CASES["scale_bias1"]
    x, s, b = c["runs"][0][0], np.array(c["fp"][:5], np.float32), np.array(c["fp"][5:], np.float32)
    once = (x.astype(np.float64) * s[None, :, None, None] + b[None, :, None, None]).astype(np.float32)
    assert O.same_bits(cpu["scale_bias1"]["ys"][0], once)
