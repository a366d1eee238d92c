"""The LLM linear layer's decode GEMV (linear_w8_gemv.cu, <= 8 tokens) in every launch cell, for every weight form, bit for bit.

The launcher picks the tokens template T (1, 2, 4, 8; 4-bit layers run one token on T = 2), the rows per warp R (1, 2, 4; four
only for <= 2 tokens and 8-bit weights), a grid capped at 8 blocks per SM and so the passes each warp makes over the output rows
(ceil(oc / (grid * 8 * R)): two or more exactly when oc > 64 * R * SMs), from the shape and the SM count.  mnnb200_linear_w8_plan
reports that launch (gemv_t, gemv_r, gemv_grid, gemv_passes, gemv_smem, gemv_w4); every case asserts it equals launch() below,
the launcher restated, and derives its shape from the SM count, so a case that moves off its cell fails.  The census test fails
if the cases, at a given SM count, miss a reachable cell (on the CPU for 114 and 132 SMs, on the GPU at its own count).

What every case checks (-m gpu):
  * every output is written and the guard rows behind it keep their NaN (test_gpu_linear_cells.Layer);
  * sampled output columns equal the C oracle bit for bit.  A column depends only on its own weight row, its constants and x,
    so the oracle runs on a row subset: the first and last R-row group of every pass, the ragged tail, oc - 1 and a seeded
    sample.  The 4-bit oracle picks its weightKernelSum rounding from oc % 64 == 0 (and ic % 4) of the layer it is given, so
    a 4-bit subset keeps the layer's class (sample_rows);
  * for 2..8 tokens, the whole output equals the same execution forced onto the tensor-core GEMM (variant 2)."""
import ctypes as C

import numpy as np
import pytest

from tests.test_gpu_dispatch import create_linear, linear_oracle
from tests.test_gpu_linear_cells import FORMS, GEMM, GEMV, NOT_SUPPORT, PLAN_FIELDS, REFUSED, Layer, lib, sm_count, up

GEMV_FIELDS = ("gemv_t", "gemv_r", "gemv_grid", "gemv_passes", "gemv_smem", "gemv_w4")
SMEM_DEFAULT = 40 * 1024        # above it the launcher raises the kernel's dynamic shared-memory limit
SMEM_LIMIT = 200 * 1024         # linear_w8_gemv_supported
ROUND = 2048                    # bytes of a weight row one warp streams per K round (32 lanes x 16 bytes x 4 chunks)
WINDOW = 512                    # bytes of a weight row in one block window of the K-blocked branch


# ---- the launcher, restated (linear_w8_gemv.cu: linear_w8_gemv_launch, linear_w8_gemv_supported) ----------------------------
def padded_ic(ic, w4):
    return up(ic, 32 if w4 else 16)


def supported(tokens, icp, bs, w4):
    extra = (8 * (icp // bs) + 8 * 18 * (16 << w4)) * 4 if bs else 0
    return 1 <= tokens <= 8 and 8 * icp + extra <= SMEM_LIMIT


def launch(tokens, ic, oc, bs, w4, sms):
    """the plan's six GEMV fields"""
    icp = padded_ic(ic, w4)
    t = 1 if tokens <= 1 and not w4 else 2 if tokens <= 2 else 4 if tokens <= 4 else 8
    r = 4 if t <= 2 and not w4 and oc >= 64 * sms else 2 if oc >= 32 * sms else 1
    grid = min(-(-oc // (8 * r)), 8 * sms)
    passes = -(-oc // (grid * 8 * r))
    smem = t * icp + ((t * (ic // bs) + 8 * (t * r + r) * (16 << w4)) * 4 if bs else 0)
    return dict(gemv_t=t, gemv_r=r, gemv_grid=grid, gemv_passes=passes, gemv_smem=smem, gemv_w4=int(bool(w4) and t > 1 and r < 4))


def x_path(ic, tokens, aligned=True):
    """how the kernel reads x: in registers (ic <= 8192), through the float4 loop (ic > 8192, more than one token) or scalar
    (one token outside registers, ic % 4 != 0 or x not 16-byte aligned)"""
    vec = ic % 4 == 0 and aligned
    if vec and ic <= 8192:
        return "registers"
    return "vector" if vec and tokens > 1 else "scalar"


# ---- the layer ----------------------------------------------------------------------------------------------------------
class GemvLayer(Layer):
    """test_gpu_linear_cells.Layer with random weight bytes (every byte is a valid int8 weight or a pair of 4-bit ones, and
    bytes are cheap to draw for a 151,936-row layer), the fused relu / relu6, and the whole plan"""

    def __init__(self, backend, form, ic, oc, bs=0, seed=0, relu=0, relu6=0):
        self.backend, self.form, self.ic, self.oc = backend, form, ic, oc
        self.bs = bs if form.endswith("blocked") else 0
        self.blocks = ic // self.bs if self.bs else 1
        assert ic % self.blocks == 0
        self.relu, self.relu6 = int(relu), int(relu6)
        rng = np.random.default_rng(seed)
        w4 = form.startswith("w4")
        self.bits = 4 if w4 else 8
        self.alpha = rng.uniform(0.001, 0.01, (oc, self.blocks)).astype(np.float32)
        self.wzero = (rng.uniform(-0.01, 0.09, (oc, self.blocks)) if w4 else rng.uniform(-0.05, 0.05, (oc, self.blocks))).astype(np.float32)
        self.bias = rng.uniform(-1, 1, oc).astype(np.float32)
        raw = np.frombuffer(rng.bytes(oc * ic // 2 if w4 else oc * ic), np.uint8)
        self.w = raw if w4 else raw.view(np.int8).reshape(oc, ic)
        if form == "w8":
            self.alpha, self.wzero = self.alpha[:, 0].copy(), self.wzero[:, 0].copy()
        self.h = self.create()
        self.tokens = 0

    def create(self):
        st, h = create_linear(self.backend, self.ic, self.oc, self.w, self.alpha, self.wzero, self.bias, self.bits,
                              relu=self.relu, relu6=self.relu6)
        assert st == 0, lib().mnnb200_last_error()
        return h

    def fresh(self):
        """a new execution of the same layer"""
        f = type(self).__new__(type(self))
        f.__dict__.update(self.__dict__)
        f.h = self.create()
        f.tokens = 0
        return f

    def plan(self):
        fields = PLAN_FIELDS + GEMV_FIELDS
        f = (C.c_int * len(fields))()
        assert lib().mnnb200_linear_w8_plan(self.h, f, len(f)) == 0, lib().mnnb200_last_error()
        return dict(zip(fields, f))

    def launch(self, tokens, sms):
        return launch(tokens, self.ic, self.oc, self.bs, self.bits == 4, sms)

    def x(self, tokens, seed, zero_row=None):
        x = np.random.default_rng(seed).uniform(-1, 1, (tokens, self.ic)).astype(np.float32)
        if zero_row is not None:
            x[zero_row] = 0
        return x

    def oracle_rows(self, x, rows):
        """the oracle of the layer restricted to output rows `rows`"""
        rows = np.asarray(rows)
        w = self.w.reshape(self.oc, self.ic // 2)[rows] if self.bits == 4 else self.w[rows]
        wz = None if self.wzero is None else self.wzero[rows]
        return linear_oracle(x, w, self.alpha[rows], wz, self.bias[rows], self.bits, relu=bool(self.relu), relu6=bool(self.relu6))

    def check_rows(self, x, y, rows, what):
        ref = self.oracle_rows(x, rows)
        got = y[:, rows]
        bad = got != ref
        if bad.any():
            t, c = np.argwhere(bad)[0]
            raise AssertionError(f"{what}: {int(bad.sum())} of {bad.size} sampled outputs differ; first at token {t} row "
                                 f"{rows[c]}: {got[t, c]!r} against {ref[t, c]!r}")


def device_x(x, misalign=False):
    """x on the device, 16-byte aligned or 4 bytes past it"""
    import torch
    if not misalign:
        return torch.from_numpy(x).cuda()
    buf = torch.zeros(x.size + 8, dtype=torch.float32, device="cuda")
    xd = buf[1:1 + x.size].view(x.shape)
    xd.copy_(torch.from_numpy(x))
    assert xd.data_ptr() % 16 == 4
    return xd


def sample_rows(oc, stride, r, bits, seed, n_random=48):
    """output rows for the oracle: the first and last R-row group of every pass (`stride` rows apart), the ragged tail, oc - 1
    and a seeded sample.  4-bit: as many rows as keep the layer's weightKernelSum class (oc % 64 == 0 or not)"""
    rows = set()
    for p0 in range(0, oc, stride):
        end = min(oc, p0 + stride)
        rows |= set(range(p0, min(p0 + r, oc))) | set(range((end - 1) // r * r, end))
    rows |= set(range(oc // r * r, oc)) | {oc - 1}
    rng = np.random.default_rng(seed)
    rows |= set(rng.choice(oc, min(oc, n_random), replace=False).tolist())
    if bits == 4 and len(rows) < oc:
        spare = (i for i in rng.permutation(oc).tolist() if i not in rows)
        if oc % 64 == 0:
            while len(rows) % 64:
                rows.add(next(spare))
        elif len(rows) % 64 == 0:
            rows.add(next(spare))
    rows = sorted(rows)
    assert bits == 8 or (len(rows) % 64 == 0) == (oc % 64 == 0)
    return rows


def run_gemv(layer, tokens, x, sms, what, misalign=False, gemm=True):
    """resize to `tokens` on auto, assert the GEMV and its restated launch, execute, check the sampled rows against the
    oracle and (2..8 tokens) the whole output against the forced GEMM; returns (plan, output on the host)"""
    pl = layer.resize(tokens, 0)
    want = layer.launch(tokens, sms)
    assert pl["path"] == GEMV and all(pl[k] == 0 for k in PLAN_FIELDS[1:]), pl
    got = {k: pl[k] for k in GEMV_FIELDS}
    assert got == want, f"{what}: plan {got}, the launcher restated {want}"
    xd = device_x(x, misalign)
    y = layer.execute(xd).cpu().numpy()
    rows = sample_rows(layer.oc, pl["gemv_grid"] * 8 * pl["gemv_r"], pl["gemv_r"], layer.bits, tokens * 7 + layer.oc)
    layer.check_rows(x, y, rows, what)
    if gemm and tokens >= 2:
        pg = layer.resize(tokens, 2)
        assert pg["path"] == GEMM and all(pg[k] == 0 for k in GEMV_FIELDS), pg
        yg = layer.execute(xd).cpu().numpy()
        if not np.array_equal(y, yg):
            t, c = np.argwhere(y != yg)[0]
            raise AssertionError(f"{what}: {int((y != yg).sum())} outputs differ from the forced GEMM; first at token {t} row "
                                 f"{c}: {y[t, c]!r} against {yg[t, c]!r}")
        layer.resize(tokens, 0)
    return pl, y


# ---- the cell matrix ----------------------------------------------------------------------------------------------------
# (T, R, more than one pass) each form reaches
REACHABLE_W8 = {(1, 1, 0), (1, 2, 0), (1, 4, 0), (2, 1, 0), (2, 2, 0), (2, 4, 0), (4, 1, 0), (4, 2, 0), (8, 1, 0), (8, 2, 0),
                (1, 4, 1), (2, 4, 1), (4, 2, 1), (8, 2, 1)}
REACHABLE_W4 = {(2, 1, 0), (2, 2, 0), (4, 1, 0), (4, 2, 0), (8, 1, 0), (8, 2, 0), (2, 2, 1), (4, 2, 1), (8, 2, 1)}
REACHABLE = {"w8": REACHABLE_W8, "w8_blocked": REACHABLE_W8, "w4": REACHABLE_W4, "w4_blocked": REACHABLE_W4}

# (form, tokens, rows per warp, passes, ic, bs (0 per channel), oc a multiple of 64, activation); oc comes from cell_oc
CELL_CASES = [
    ("w8", 1, 1, 1, 1040, 0, False, ""), ("w8", 1, 2, 1, 2100, 0, False, ""), ("w8", 1, 4, 1, 4100, 0, False, "relu"),
    ("w8", 2, 1, 1, 3000, 0, False, ""), ("w8", 2, 2, 1, 1040, 0, False, ""), ("w8", 2, 4, 1, 2100, 0, False, ""),
    ("w8", 3, 1, 1, 2100, 0, False, ""), ("w8", 4, 2, 1, 1040, 0, False, "relu6"), ("w8", 5, 1, 1, 2100, 0, False, ""),
    ("w8", 7, 2, 1, 3000, 0, False, ""),
    ("w8", 1, 4, 2, 2100, 0, False, ""), ("w8", 2, 4, 2, 2100, 0, False, ""), ("w8", 3, 2, 2, 2100, 0, False, ""),
    ("w8", 8, 2, 2, 2100, 0, False, ""),
    ("w8_blocked", 1, 1, 1, 2112, 64, False, ""), ("w8_blocked", 1, 2, 1, 1056, 32, False, ""),
    ("w8_blocked", 1, 4, 1, 2304, 256, False, ""), ("w8_blocked", 2, 1, 1, 1024, 512, False, ""),
    ("w8_blocked", 2, 2, 1, 2176, 128, False, ""), ("w8_blocked", 2, 4, 1, 3136, 64, False, "relu"),
    ("w8_blocked", 3, 1, 1, 2560, 512, False, ""), ("w8_blocked", 4, 2, 1, 512, 256, False, ""),
    ("w8_blocked", 5, 1, 1, 1120, 32, False, ""), ("w8_blocked", 7, 2, 1, 2112, 64, False, "relu6"),
    ("w8_blocked", 1, 4, 2, 2112, 64, False, ""), ("w8_blocked", 2, 4, 2, 1152, 128, False, ""),
    ("w8_blocked", 4, 2, 2, 2080, 32, False, ""), ("w8_blocked", 8, 2, 2, 2304, 256, False, ""),
    ("w4", 1, 1, 1, 2048, 0, True, ""), ("w4", 2, 1, 1, 1000, 0, False, ""), ("w4", 1, 2, 1, 4160, 0, True, "relu"),
    ("w4", 2, 2, 1, 5504, 0, False, ""), ("w4", 3, 1, 1, 1000, 0, False, ""), ("w4", 4, 2, 1, 6144, 0, True, ""),
    ("w4", 8, 1, 1, 2080, 0, False, "relu6"), ("w4", 7, 2, 1, 4672, 0, True, ""),
    ("w4", 1, 2, 2, 4160, 0, False, ""), ("w4", 2, 2, 2, 2080, 0, True, ""), ("w4", 3, 2, 2, 2496, 0, False, ""),
    ("w4", 5, 2, 2, 4160, 0, True, ""),
    ("w4_blocked", 1, 1, 1, 2112, 64, True, ""), ("w4_blocked", 2, 1, 1, 1024, 512, False, ""),
    ("w4_blocked", 2, 2, 1, 4608, 512, False, ""), ("w4_blocked", 1, 2, 1, 3264, 32, False, "relu"),
    ("w4_blocked", 3, 1, 1, 5248, 128, True, ""), ("w4_blocked", 4, 2, 1, 2560, 256, False, ""),
    ("w4_blocked", 5, 1, 1, 1088, 64, False, "relu6"), ("w4_blocked", 8, 2, 1, 4352, 256, True, ""),
    ("w4_blocked", 1, 2, 2, 2112, 64, True, ""), ("w4_blocked", 2, 2, 2, 1088, 32, False, ""),
    ("w4_blocked", 3, 2, 2, 4608, 512, False, ""), ("w4_blocked", 7, 2, 2, 2176, 128, True, ""),
]


def case_id(c):
    form, tokens, r, passes, ic, bs, oc64, act = c
    return f"{form}-{tokens}tok-r{r}-{'multipass' if passes > 1 else 'onepass'}-ic{ic}" + (f"-bs{bs}" if bs else "") + \
           ("-oc64" if oc64 else "") + (f"-{act}" if act else "")


def cell_oc(r, passes, oc64, sms):
    """an oc in the cell at this SM count: R = 1 below 32 * SMs rows, R = 2 from there (below 64 * SMs for 8-bit <= 2 tokens),
    R = 4 from 64 * SMs; two passes over stride = 64 * R * SMs rows with a ragged second one that leaves the later half of the
    warps idle"""
    if passes > 1:
        stride = 64 * r * sms
        oc = stride + stride // 2 + 3
    else:
        oc = {1: 16 * sms + 5, 2: 48 * sms + 3, 4: 64 * sms + 13}[r]
    return up(oc - 2, 64) if oc64 else oc


def case_shape(c, sms):
    """(form, tokens, ic, oc, bs, relu, relu6) of a cell case"""
    form, tokens, r, passes, ic, bs, oc64, act = c
    return form, tokens, ic, cell_oc(r, passes, oc64, sms), bs, act == "relu", act == "relu6"


def census(sms):
    """{form: {(T, R, passes > 1)}} the cell cases reach at this SM count, by the restated launcher"""
    out = {f: set() for f in FORMS}
    for c in CELL_CASES:
        form, tokens, ic, oc, bs, _, _ = case_shape(c, sms)
        lc = launch(tokens, ic, oc, bs, form.startswith("w4"), sms)
        out[form].add((lc["gemv_t"], lc["gemv_r"], int(lc["gemv_passes"] > 1)))
    return out


def check_census(sms):
    cells = census(sms)
    for form in FORMS:
        missing = REACHABLE[form] - cells[form]
        assert not missing, f"{form} at {sms} SMs: no case in cells {sorted(missing)}"
        assert cells[form] <= REACHABLE[form], f"{form} at {sms} SMs: cells outside the table {sorted(cells[form] - REACHABLE[form])}"
    for c in CELL_CASES:
        form, tokens, r, passes, ic, bs, oc64, act = c
        _, _, _, oc, _, _, _ = case_shape(c, sms)
        w4 = form.startswith("w4")
        lc = launch(tokens, ic, oc, bs, w4, sms)
        assert (lc["gemv_r"], lc["gemv_passes"] > 1) == (r, passes > 1), (case_id(c), sms, lc)
        assert supported(tokens, padded_ic(ic, w4), bs, w4)
        row = padded_ic(ic, w4) >> w4
        assert row % ROUND, f"{case_id(c)}: K ends in a whole {ROUND}-byte round"
        if lc["gemv_passes"] > 1:
            stride = lc["gemv_grid"] * 8 * r
            assert oc % stride and oc % stride <= stride - 8 * r, f"{case_id(c)}: the last pass leaves no warp idle"
        if bs and 2 * bs != ic and not (bs == 512 and not w4):
            assert row % WINDOW, f"{case_id(c)}: the last block window is whole"
        assert (oc % 64 == 0) == oc64
    multi = [c for c in CELL_CASES if c[3] > 1]
    assert any(cell_oc(c[2], c[3], c[6], sms) % c[2] for c in multi), "no multi-pass case with oc % R != 0"
    for form in ("w8_blocked", "w4_blocked"):
        bss = {c[5] for c in CELL_CASES if c[0] == form}
        assert bss == {32, 64, 128, 256, 512} and any(2 * c[5] == c[4] for c in CELL_CASES if c[0] == form), (form, bss)
    for form in ("w4", "w4_blocked"):
        assert {c[6] for c in CELL_CASES if c[0] == form} == {True, False}, f"{form}: oc % 64 == 0 on one side only"
        assert {c[1] for c in CELL_CASES if c[0] == form and c[1] <= 2} == {1, 2}, f"{form}: T = 2 not at 1 and 2 tokens"
    tokens = {c[1] for c in CELL_CASES}
    assert {3, 5, 7} <= tokens and {"relu", "relu6"} <= {c[7] for c in CELL_CASES}


@pytest.mark.parametrize("sms", [114, 132])
def test_gemv_cell_census_on_cpu(sms):
    """the cases reach every cell of the table at the H100 PCIe's and the H100 SXM's SM counts, with the shape rules each
    cell case was written for (ragged passes, partial K rounds and block windows, both 4-bit weightKernelSum classes)"""
    check_census(sms)


@pytest.mark.gpu
def test_gemv_cell_census():
    check_census(sm_count())


@pytest.mark.gpu
@pytest.mark.parametrize("case", CELL_CASES, ids=case_id)
def test_gemv_cell(backend, case):
    sms = sm_count()
    form, tokens, ic, oc, bs, relu, relu6 = case_shape(case, sms)
    layer = GemvLayer(backend, form, ic, oc, bs, seed=ic + oc + tokens, relu=relu, relu6=relu6)
    try:
        x = layer.x(tokens, oc + tokens, zero_row=tokens // 2 if tokens > 1 else None)
        pl, y = run_gemv(layer, tokens, x, sms, case_id(case))
        print(f"{case_id(case)}: oc {oc} on {sms} SMs, plan {({k: pl[k] for k in GEMV_FIELDS})}")
        if relu or relu6:
            assert (y == 0).any() and (y > 0).any(), "the activation never bites"
    finally:
        layer.destroy()


# ---- edges of the three later forms -------------------------------------------------------------------------------------
LATER = ("w8_blocked", "w4", "w4_blocked")
# name: (tokens, ic, bs of the blocked forms, x 4 bytes past alignment, the x path it must take)
X_EDGES = {
    "x_registers_1tok": (1, 4096, 128, False, "registers"), "x_registers_4tok": (4, 4096, 64, False, "registers"),
    "x_ic11008_1tok": (1, 11008, 256, False, "scalar"), "x_ic11008_6tok": (6, 11008, 128, False, "vector"),
    "x_ic11008_2tok": (2, 11008, 64, False, "vector"),
    "x_misaligned_1tok": (1, 2048, 64, True, "scalar"), "x_misaligned_3tok": (3, 2048, 32, True, "scalar"),
    "smem_over_40k_8tok": (8, 5504, 128, False, "registers"),
}


@pytest.mark.gpu
@pytest.mark.parametrize("form", LATER)
@pytest.mark.parametrize("edge", list(X_EDGES))
def test_gemv_x_paths_and_shared_memory(backend, form, edge):
    """x in registers, through the float4 loop (ic 11,008 as in a 7B-class FFN down projection; one token outside registers
    reads scalars) and 4 bytes past 16-byte alignment, each at one token and more; dynamic shared memory above 40 KB"""
    sms = sm_count()
    tokens, ic, bs, mis, path = X_EDGES[edge]
    oc = 40 * sms + 17 if tokens > 1 else 20 * sms + 1
    w4 = form.startswith("w4")
    assert x_path(ic, tokens, not mis) == path
    layer = GemvLayer(backend, form, ic, oc, bs, seed=ic + tokens + len(edge))
    try:
        if edge.startswith("smem"):
            assert layer.launch(tokens, sms)["gemv_smem"] > SMEM_DEFAULT
        x = layer.x(tokens, ic + tokens, zero_row=tokens - 1 if tokens > 1 else None)
        run_gemv(layer, tokens, x, sms, f"{form} {edge}", misalign=mis)
    finally:
        layer.destroy()


BOUNDARY_BS = {"w8": 0, "w8_blocked": 32, "w4": 0, "w4_blocked": 512}


def largest_ic(form):
    """the largest ic linear_w8_gemv_supported accepts for the form (at BOUNDARY_BS), and one block past it (per channel: one
    padding unit)"""
    w4, bs = form.startswith("w4"), BOUNDARY_BS[form]
    unit = bs or (32 if w4 else 16)
    ic = unit
    while supported(8, padded_ic(ic + unit, w4), bs, w4):
        ic += unit
    assert not supported(1, padded_ic(ic + unit, w4), bs, w4)
    return ic, ic + unit


@pytest.mark.gpu
@pytest.mark.parametrize("form", FORMS)
def test_gemv_largest_ic_and_one_block_past(backend, form):
    """at the largest ic the GEMV takes (dynamic shared memory near 200 KB at 8 tokens) the GEMV runs, bit for bit; one block
    past it the plan is the GEMM for 2..8 tokens and a refusal for one token and under variant 4, and execute agrees"""
    import torch
    sms = sm_count()
    ic, past = largest_ic(form)
    oc = 300
    layer = GemvLayer(backend, form, ic, oc, BOUNDARY_BS[form], seed=ic)
    try:
        for tokens in (1, 8):
            x = layer.x(tokens, ic + tokens, zero_row=3 if tokens > 1 else None)
            pl, _ = run_gemv(layer, tokens, x, sms, f"{form} ic {ic}")
            if tokens == 8:
                assert pl["gemv_smem"] > SMEM_LIMIT - 10 * 1024, pl
    finally:
        layer.destroy()
    layer = GemvLayer(backend, form, past, oc, BOUNDARY_BS[form], seed=past)
    try:
        y = torch.zeros((8, oc), dtype=torch.float32, device="cuda")
        for tokens in range(1, 9):
            x = layer.x(tokens, past + tokens)
            xd = device_x(x)
            for variant in (0, 4):
                pl = layer.resize(tokens, variant)
                want = REFUSED if tokens == 1 or variant == 4 else GEMM
                assert pl["path"] == want and all(pl[k] == 0 for k in GEMV_FIELDS), (form, past, tokens, variant, pl)
                if want == REFUSED:
                    st = lib().mnnb200_linear_w8_execute(layer.h, C.c_void_p(xd.data_ptr()), C.c_void_p(y.data_ptr()))
                    assert st == NOT_SUPPORT, (tokens, variant, st)
                else:
                    yg = layer.execute(xd).cpu().numpy()
                    layer.check_rows(x, yg, sample_rows(oc, oc, 1, layer.bits, tokens), f"{form} ic {past} on the GEMM")
    finally:
        layer.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["w8_blocked", "w4_blocked"])
@pytest.mark.parametrize("tokens", [1, 8])
def test_gemv_lm_head(backend, form, tokens):
    """a 151,936 x 2,048 Qwen lm_head exported K-blocked (bs 64): several passes over the output rows on every decode step"""
    sms = sm_count()
    layer = GemvLayer(backend, form, 2048, 151936, 64, seed=151936 + tokens)
    try:
        assert layer.launch(tokens, sms)["gemv_passes"] > 1
        x = layer.x(tokens, tokens, zero_row=5 if tokens > 1 else None)
        run_gemv(layer, tokens, x, sms, f"{form} lm_head")
    finally:
        layer.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("form", FORMS)
def test_gemv_one_execution_resized(backend, form):
    """one execution resized 8 -> 1 -> 3 -> 2 -> 8 tokens gives, at each step, the plan and the output of a fresh execution,
    and its sampled rows equal the oracle; the layer's cell changes along the way"""
    sms = sm_count()
    layer = GemvLayer(backend, form, 2080, 70 * sms + 5, 32, seed=55)
    cells = set()
    try:
        for tokens in (8, 1, 3, 2, 8):
            x = layer.x(tokens, tokens * 11, zero_row=1 if tokens > 1 else None)
            pl, y = run_gemv(layer, tokens, x, sms, f"{form} resized to {tokens}", gemm=False)
            f = layer.fresh()
            try:
                fpl = f.resize(tokens, 0)
                fy = f.execute(device_x(x)).cpu().numpy()
            finally:
                f.destroy()
            assert pl == fpl, (pl, fpl)
            assert np.array_equal(y, fy), f"{form} at {tokens} tokens: the re-resized execution differs from a fresh one"
            cells.add((pl["gemv_t"], pl["gemv_r"]))
    finally:
        layer.destroy()
    assert len(cells) >= 3, cells


def chain_layers(backend, sms):
    """a decode-shaped chain, each layer reading the previous one's output: 8-bit, 4-bit K-blocked with > 40 KB of shared
    memory, 8-bit K-blocked over two passes, 4-bit per channel reading a 25k-wide input"""
    oc3 = 192 * sms + 4
    specs = [("w8", 2048, 5504, 0), ("w4_blocked", 5504, 2048, 128), ("w8_blocked", 2048, oc3, 64), ("w4", oc3, 1000, 0)]
    return [GemvLayer(backend, f, ic, oc, bs, seed=i + 1) for i, (f, ic, oc, bs) in enumerate(specs)]


@pytest.mark.gpu
def test_gemv_dependent_chain_eager_and_graph(backend):
    """four GEMVs back to back on one stream, each reading x that the launch before it writes (programmatic dependent launch:
    each one's weights are requested before it waits for its producer), eagerly and as a replayed CUDA graph; both equal the
    same layers run one at a time with a sync between them, and each layer's sampled rows equal the oracle.  The intermediate
    buffers are NaN-filled before every run, so an x read that did not wait for its producer shows"""
    import torch
    sms = sm_count()
    tokens = 5
    layers = chain_layers(backend, sms)
    g = C.c_void_p()
    try:
        plans = []
        for i, layer in enumerate(layers):
            pl = layer.resize(tokens, 0)
            assert pl["path"] == GEMV and {k: pl[k] for k in GEMV_FIELDS} == layer.launch(tokens, sms), pl
            plans.append(pl)
        assert plans[1]["gemv_smem"] > SMEM_DEFAULT and plans[2]["gemv_passes"] > 1, plans
        x = layers[0].x(tokens, 99, zero_row=2)
        xd = device_x(x)
        bufs = [torch.empty((tokens, l.oc), dtype=torch.float32, device="cuda") for l in layers]
        rt = backend.runtime._h

        def run(sync):
            for b in bufs:
                b.fill_(float("nan"))
            src = xd
            for layer, b in zip(layers, bufs):
                assert lib().mnnb200_linear_w8_execute(layer.h, C.c_void_p(src.data_ptr()), C.c_void_p(b.data_ptr())) == 0
                if sync:
                    backend.onSync()
                src = b

        def outputs():
            backend.onSync()
            return [b.cpu().numpy() for b in bufs]

        run(True)
        ref = outputs()
        src = x
        for layer, y in zip(layers, ref):
            assert not np.isnan(y).any()
            layer.check_rows(src, y, sample_rows(layer.oc, layer.oc, 1, layer.bits, 3, n_random=64), f"chain {layer.form}")
            src = y
        run(False)
        eager = outputs()
        for i, (a, b) in enumerate(zip(eager, ref)):
            assert np.array_equal(a, b), f"eager chain, layer {i}: {int((a != b).sum())} outputs differ from the synced run"
        for b in bufs:
            b.fill_(float("nan"))
        backend.onSync()
        assert lib().mnnb200_graph_begin_capture(rt) == 0
        src = xd
        for layer, b in zip(layers, bufs):
            assert lib().mnnb200_linear_w8_execute(layer.h, C.c_void_p(src.data_ptr()), C.c_void_p(b.data_ptr())) == 0
            src = b
        assert lib().mnnb200_graph_end_capture(rt, C.byref(g)) == 0, lib().mnnb200_last_error()
        for b in bufs:
            b.fill_(float("nan"))
        assert lib().mnnb200_graph_launch(rt, g) == 0
        replay = outputs()
        for i, (a, b) in enumerate(zip(replay, ref)):
            assert np.array_equal(a, b), f"graph replay, layer {i}: {int((a != b).sum())} outputs differ from the synced run"
    finally:
        if g.value:
            lib().mnnb200_graph_destroy(g)
        for layer in layers:
            layer.destroy()
