"""nm_gemm exactly, at every dispatch boundary of its wgmma engine, and the dense fp16 products exactly.

Operands, bias and the C that beta = 1 adds to are small integers times powers of two.  Every product and every
partial sum is then exact in TF32, fp16 and fp32 whatever the order of summation, and whether the hardware rounds or
truncates to TF32: the tensor-core engine (operands by TMA or by its producer threads, split-K slices meeting in
atomic adds in any order), the CUDA-core engine and an fp64 product on the device must agree exactly.  With tanh and
sigmoid the result is within a few fp32 ulps of the fp64 activation of the exact pre-activation (tanhf and expf are
not correctly rounded).  The random-data tests of test_gpu_gemm.py stay: a wrong TF32 rounding only shows there.

Every output is a window of a sentinel-filled buffer, with rows above and below it and columns on both sides, and
every operand a window of a NaN-filled one: a read beyond M, N or K poisons the result, and nothing outside the
output window may change.

The wgmma cases are the named branches of tests/gemm_plan_cases.py, found for this device's SM count.  Each runs
through nm_gemm in all four transpose combinations, through ops.gemm (K-major TF32 copies) and on the CUDA cores;
the six runs take the six epilogue variants below in an order that rotates from case to case."""
import math

import pytest
import torch

from tests import gemm_plan_cases as G
from tests.test_gpu_gemm16_persistent import F16_SHAPES, F16_TN_SHAPES

pytestmark = pytest.mark.gpu

NM_E_UNSUPPORTED = -2
SENTINEL = -1234.5678          # finite, with low mantissa bits set: a stray store or add changes its bits
GUARD_ROWS = (2, 3)            # above and below every output window
TRANSPOSES = [(False, False), (False, True), (True, False), (True, True)]
# (beta, bias, first column of the output window, ragged dimensions).  Column 0 of a pitch of 4k floats allows the
# coalesced and vector stores / reductions; columns 1 and 3 and a bias offset by one float force the per-row stores
# and the scalar atomics.
VARIANTS = [
    (0.0, None, 0, ""),
    (1.0, "aligned", 1, "mnk"),
    (0.0, "offset", 3, "mn"),
    (1.0, None, 0, "k"),
    (0.0, "aligned", 0, "mnk"),
    (1.0, "offset", 0, ""),
]


def _lib():
    from neuralmonkey_b200 import lib
    return lib


@pytest.fixture(scope="module")
def sms():
    return _lib().device_info()["sm_count"]


def _ints(shape, log2_unit, g, dtype=torch.float32):
    """Integers in [-3, 3] times 2^-log2_unit, on the device."""
    x = torch.randint(-3, 4, shape, device="cuda", generator=g, dtype=torch.int32).float() * 2.0 ** -log2_unit
    return x.to(dtype)


def _stored(x, align=4):
    """x [r, c] as a window of a NaN buffer: a NaN row above and below, NaN columns after it up to a row pitch of
    at least 4 more elements, rounded up to `align` elements.  The window starts on a 16-byte boundary."""
    r, c = x.shape
    pitch = (c + 4 + align - 1) // align * align
    buf = torch.full((r + 2, pitch), float("nan"), device="cuda", dtype=x.dtype)
    buf[1:1 + r, :c] = x
    return buf[1:1 + r, :c]


class Guarded:
    """An output window [m, n] at column c0 of a sentinel buffer; row pitch a multiple of 4 floats with at least 4
    guard columns right of the window."""

    def __init__(self, m, n, c0, fill):
        self.r0, self.c0, self.m, self.n = GUARD_ROWS[0], c0, m, n
        ldc = (c0 + n + 4 + 3) // 4 * 4
        self.big = torch.full((self.r0 + m + GUARD_ROWS[1], ldc), SENTINEL, device="cuda")
        self.win[...] = fill
        self.before = self.big.clone()

    @property
    def win(self):
        return self.big[self.r0:self.r0 + self.m, self.c0:self.c0 + self.n]

    def outside_unchanged(self):
        a, b = self.big.clone(), self.before.clone()
        for t in (a, b):
            t[self.r0:self.r0 + self.m, self.c0:self.c0 + self.n] = 0.0
        return torch.equal(a.view(torch.int32), b.view(torch.int32))

    def untouched(self):
        return torch.equal(self.big.view(torch.int32), self.before.view(torch.int32))


def _bias(values, offset):
    """values in a NaN buffer, starting 16 bytes in (or 20 with `offset`)."""
    n = values.numel()
    buf = torch.full(((n + 12) // 4 * 4,), float("nan"), device="cuda")
    buf[4 + offset:4 + offset + n] = values
    return buf[4 + offset:4 + offset + n]


def _ulp(x):
    a = x.float().abs()
    return (torch.nextafter(a, torch.full_like(a, float("inf"))) - a).double()


def _check(out, want, act_part, act, what):
    """out (fp32) against the exact fp64 result `want`; act_part is the fp64 activation output inside it."""
    assert torch.isfinite(out).all(), "{}: {} non-finite outputs".format(what, int((~torch.isfinite(out)).sum()))
    if act in ("none", "relu"):
        assert torch.equal(want.float().double(), want), "{}: the test data is not exact in fp32".format(what)
        bad = out != want.float()
    else:
        bad = (out.double() - want).abs() > 4 * (_ulp(act_part) + _ulp(want))
    if bad.any():
        r, c = [int(i) for i in bad.nonzero()[0]]
        pytest.fail("{}: {} of {} outputs differ, first at ({}, {}): {!r} instead of {!r}".format(
            what, int(bad.sum()), bad.numel(), r, c, float(out[r, c]), float(want[r, c])))


def _act64(x, act):
    return {"none": lambda t: t, "relu": torch.relu, "tanh": torch.tanh, "sigmoid": torch.sigmoid}[act](x)


def _addr(t):
    """Device address of a view, also of an empty one (whose data_ptr() is 0)."""
    return None if t is None else t.untyped_storage().data_ptr() + t.storage_offset() * t.element_size()


def _nm_gemm(backend, ta, tb, a, b, out, bias, act, beta):
    """nm_gemm on the operands as stored; returns the status instead of raising."""
    lib = _lib()
    k = a.size(0) if ta else a.size(1)
    return lib.load().nm_gemm(int(ta), int(tb), out.size(0), out.size(1), k, _addr(a), a.stride(0), _addr(b),
                              b.stride(0), _addr(out), out.stride(0), _addr(bias), lib.NM_ACT[act], float(beta),
                              backend, lib.stream())


def _runs(idx):
    """(engine, trans_a, trans_b) of the six runs of case idx."""
    return ([("tc",) + t for t in TRANSPOSES]
            + [("ops.gemm",) + TRANSPOSES[idx % 4], ("simt",) + TRANSPOSES[(idx + 2) % 4]])


@pytest.mark.parametrize("case", G.CASES, ids=lambda c: c.name)
def test_nm_gemm_exact(case, sms):
    from neuralmonkey_b200 import lib, ops
    shape = G.find_shape(case, sms)
    if shape is None:
        pytest.skip("{}: no candidate shape lands on this branch at {} SMs".format(case.name, sms))
    plan = G.plan(*shape, case.act, sms)
    assert G.plan(*shape, case.act) == plan, "nm_gemm_tc_plan(sms=0) does not use this device's SM count"
    idx = G.CASES.index(case)
    M, N, K = shape
    Mr, Nr, Kr = G.ragged(shape)
    g = torch.Generator(device="cuda").manual_seed(1000 + idx)
    s = max(1, round(math.log2(4 * math.sqrt(K)) / 2))   # operands 2^-s: pre-activations of order one
    unit = 2 * s                                           # every product, bias and C entry: integer * 2^-unit
    a, b = _ints((M, K), s, g), _ints((K, N), s, g)
    bias_in, c_in = _ints((N,), unit, g), _ints((M, N), unit, g)
    prod_kr = a[:, :Kr].double() @ b[:Kr].double()
    prod_k = prod_kr + a[:, Kr:].double() @ b[Kr:].double()

    for j, (engine, ta, tb) in enumerate(_runs(idx)):
        beta, bias_kind, c0, rag = VARIANTS[(idx + j) % len(VARIANTS)]
        m, n, k = (Mr if "m" in rag else M), (Nr if "n" in rag else N), (Kr if "k" in rag else K)
        what = "{} {} trans_a={} trans_b={} {}x{}x{} beta={} bias={} c0={} plan={}".format(
            case.name, engine, int(ta), int(tb), m, n, k, beta, bias_kind, c0, tuple(plan))
        bias = None if bias_kind is None else _bias(bias_in[:n], 1 if bias_kind == "offset" else 0)
        pre = (prod_k if k == K else prod_kr)[:m, :n]
        if bias is not None:
            pre = pre + bias.double()
        act_part = _act64(pre, case.act)
        want = act_part + beta * c_in[:m, :n].double()
        out = Guarded(m, n, c0, c_in[:m, :n] if beta else float("nan"))
        a_st = _stored(a[:m, :k].t().contiguous() if ta else a[:m, :k])
        b_st = _stored(b[:k, :n].t().contiguous() if tb else b[:k, :n])
        if engine == "ops.gemm":
            ops.gemm(a_st, b_st, out.win, trans_a=ta, trans_b=tb, bias=bias, act=case.act, beta=beta,
                     backend=lib.GEMM_TC)
        else:
            rc = _nm_gemm(lib.GEMM_TC if engine == "tc" else lib.GEMM_SIMT, ta, tb, a_st, b_st, out.win, bias,
                          case.act, beta)
            assert rc == 0, "{}: status {}: {}".format(what, rc, lib.load().nm_last_error())
        torch.cuda.synchronize()
        _check(out.win, want, act_part, case.act, what)
        assert out.outside_unchanged(), "{}: wrote outside the output window".format(what)


def _small_product(m, n, k, g):
    a, b = _stored(_ints((m, k), 2, g)), _stored(_ints((k, n), 2, g))
    bias = _stored(_ints((1, n), 4, g))[0]
    return a, b, bias


@pytest.mark.parametrize("act", ["none", "relu"])
@pytest.mark.parametrize("beta", [0.0, 1.0])
def test_k_zero(act, beta):
    """K = 0: AUTO gives act(bias) + beta * C on the CUDA cores; the wgmma backend refuses and writes nothing."""
    lib = _lib()
    m, n = 70, 45
    g = torch.Generator(device="cuda").manual_seed(7)
    a, b, bias = _small_product(m, n, 0, g)
    c_in = _ints((m, n), 4, g)
    want = _act64(bias.double().expand(m, n), act) + beta * c_in.double()
    out = Guarded(m, n, 1, c_in if beta else float("nan"))
    assert _nm_gemm(lib.GEMM_AUTO, False, False, a, b, out.win, bias, act, beta) == 0
    torch.cuda.synchronize()
    _check(out.win, want, want, act, "K = 0")
    assert out.outside_unchanged()
    out = Guarded(m, n, 0, c_in)
    assert _nm_gemm(lib.GEMM_TC, False, False, a, b, out.win, bias, act, beta) == NM_E_UNSUPPORTED
    torch.cuda.synchronize()
    assert out.untouched()


@pytest.mark.parametrize("m,n", [(0, 96), (96, 0), (0, 0)])
def test_empty_output_writes_nothing(m, n):
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(8)
    a, b, bias = _small_product(m, n, 64, g)
    for backend in (lib.GEMM_AUTO, lib.GEMM_SIMT, lib.GEMM_TC):
        for beta in (0.0, 1.0):
            out = Guarded(m, n, 0, 0.0)
            assert _nm_gemm(backend, False, False, a, b, out.win, bias, "none", beta) == 0
            torch.cuda.synchronize()
            assert out.untouched(), (backend, beta)


@pytest.mark.parametrize("beta", [0.5, 2.0, -1.0])
def test_beta_other_than_zero_or_one_is_refused(beta):
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(9)
    a, b, bias = _small_product(64, 96, 64, g)
    for backend in (lib.GEMM_AUTO, lib.GEMM_SIMT, lib.GEMM_TC):
        out = Guarded(64, 96, 0, _ints((64, 96), 4, g))
        assert _nm_gemm(backend, False, False, a, b, out.win, bias, "none", beta) == NM_E_UNSUPPORTED
        torch.cuda.synchronize()
        assert out.untouched(), backend


# ---- the dense fp16 products (csrc/gemm16.cu): stream-K ranges that cut tiles between CTAs ----
# Operands integers * 2^-2 in fp16, alpha and the row scales powers of two: every sum and every scaled piece is
# exact in fp32, so the pieces of a cut tile add up exactly in any order.

def _f16_operands(rows_a, rows_b, k, g, a_major_k=True):
    """A [rows_a, k] and B [rows_b, k] (K-major) or A [k, rows_a] and B [k, rows_b] (MN-major), fp16 windows of NaN
    buffers with row pitches of multiples of 8 elements."""
    a, b = _ints((rows_a, k), 2, g), _ints((rows_b, k), 2, g)
    if a_major_k:
        return a, b, _stored(a.half(), 8), _stored(b.half(), 8)
    return a, b, _stored(a.t().contiguous().half(), 8), _stored(b.t().contiguous().half(), 8)


@pytest.mark.parametrize("m,n,k", F16_SHAPES)
def test_gemm_f16_exact(m, n, k):
    """nm_gemm_f16: C = alpha * row_scale[m] * A . B^T (+ C), stored as C or C^T."""
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(m + n + k)
    a, b, a16, b16 = _f16_operands(m, n, k, g)
    prod = a.double() @ b.double().t()
    alpha = torch.tensor([0.5], device="cuda")
    row_scale = 2.0 ** torch.randint(-1, 2, (m,), device="cuda", generator=g).float()
    for i, (transposed, beta) in enumerate([(0, 0.0), (0, 1.0), (1, 0.0), (1, 1.0)]):
        rs = row_scale if i != 1 else None
        want = prod * 0.5 * (rs.double()[:, None] if rs is not None else 1.0)
        if transposed:
            want = want.t()
        c_in = _ints(tuple(want.shape), 6, g)
        want = want + beta * c_in.double()
        out = Guarded(want.size(0), want.size(1), i % 2, c_in if beta else float("nan"))
        lib.call("nm_gemm_f16", m, n, k, lib.ptr(a16), a16.stride(0), lib.ptr(b16), b16.stride(0), lib.ptr(out.win),
                 out.win.stride(0), lib.ptr(alpha), lib.ptr(rs), beta, transposed, lib.stream())
        torch.cuda.synchronize()
        what = "nm_gemm_f16 {}x{}x{} transposed={} beta={} row_scale={}".format(m, n, k, transposed, beta,
                                                                                 rs is not None)
        _check(out.win, want, want, "none", what)
        assert out.outside_unchanged(), what


@pytest.mark.parametrize("m,n,k,c_offset", F16_TN_SHAPES)
def test_gemm_f16_tn_exact(m, n, k, c_offset, sms):
    """nm_gemm_f16_tn_ctas: C = alpha * A^T . B (+ C) with both operands stored [K, *], on budgets of 1, 7 and every
    SM (the products too long for one SM on the last only)."""
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(m + n + k + 1)
    a, b, a16, b16 = _f16_operands(m, n, k, g, a_major_k=False)
    prod = a.double() @ b.double().t()
    alpha = torch.tensor([0.25], device="cuda")
    budgets = (1, 7, sms) if m * n * k <= 10 ** 9 else (sms,)
    for budget in budgets:
        for beta in (0.0, 1.0):
            c_in = _ints((m, n), 6, g)
            want = prod * 0.25 + beta * c_in.double()
            out = Guarded(m, n, c_offset % 4, c_in if beta else float("nan"))
            lib.call("nm_gemm_f16_tn_ctas", m, n, k, lib.ptr(a16), a16.stride(0), lib.ptr(b16), b16.stride(0),
                     lib.ptr(out.win), out.win.stride(0), lib.ptr(alpha), beta, budget, lib.stream())
            torch.cuda.synchronize()
            what = "nm_gemm_f16_tn {}x{}x{} beta={} max_ctas={}".format(m, n, k, beta, budget)
            _check(out.win, want, want, "none", what)
            assert out.outside_unchanged(), what
