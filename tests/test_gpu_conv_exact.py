"""The convolution kernels exactly, at every dispatch boundary: conv2d forward, data and weight gradients
(csrc/cnn.cu), the GLU conv1d (csrc/glu_conv.cu) and the VGG primitives (csrc/conv.cu), on both engines.

Operands and biases are small integers times powers of two, and where a sum runs over many pixels one operand is in
{-1, 0, 1}: every product and every partial sum stays below 2^24 units and is exact in TF32 and fp32 whatever the
order of summation.  So the wgmma engine, the CUDA-core engine and an fp64 convolution agree exactly, for every
split plan and workspace size.  Only the GLU's sigmoid is inexact: y and dz are held within a few fp32 ulps of the
fp64 expression evaluated on the exact z.  The random-data tests of test_gpu_cnn.py and test_gpu_convs2s.py stay:
a wrong TF32 rounding only shows there.

Every output is a window of a sentinel-filled buffer with guard elements before and after it, and every input a
window of a NaN-filled one: a read outside x, w, dy or dz poisons the result, and nothing outside the output may
change.  Each case also runs with the gathered input (and the GLU filter) one float off a 16-byte boundary, which
keeps C % 4 == 0 but forces the scalar gathers."""
import math

import pytest
import torch
import torch.nn.functional as F

from tests import conv_plan_cases as P

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")]

SENTINEL = -1234.5678          # finite, with low mantissa bits set: a stray store or add changes its bits
GUARD = 8                      # sentinel / NaN floats before and after every window
NM_E_INVALID = -1
ENGINES = ("tc", "simt")


def _lib():
    from neuralmonkey_b200 import lib
    return lib


def _backend(engine):
    lib = _lib()
    return lib.GEMM_TC if engine == "tc" else lib.GEMM_SIMT


@pytest.fixture(scope="module")
def sms():
    return _lib().device_info()["sm_count"]


def _ints(shape, g, lo=-3, hi=3, log2_unit=0):
    """Integers in [lo, hi] times 2^-log2_unit, fp32 on the device."""
    return torch.randint(lo, hi + 1, shape, device="cuda", generator=g).float() * 2.0 ** -log2_unit


def _unit(terms):
    """log2 of the operand unit that keeps a sum of `terms` products of two [-3, 3] operands of order one."""
    return max(0, round(math.log2(2 * math.sqrt(terms)) / 2))


def _stored(t, shift=0):
    """t as a window of a NaN buffer, starting 16 bytes in (plus `shift` floats)."""
    n = t.numel()
    buf = torch.full((n + 2 * GUARD + 4,), float("nan"), device="cuda")
    s = GUARD + shift
    buf[s:s + n] = t.reshape(-1)
    return buf[s:s + n].view(t.shape)


class Guarded:
    """An output window of `shape` inside a sentinel buffer, GUARD floats on either side; starts 16-byte aligned."""

    def __init__(self, shape, fill=float("nan")):
        n = math.prod(shape)
        self.big = torch.full((n + 2 * GUARD,), SENTINEL, device="cuda")
        self.win = self.big[GUARD:GUARD + n].view(shape)
        self.win[...] = fill
        self.n = n
        self.before = self.big.clone()

    def outside_unchanged(self):
        a, b = self.big.view(torch.int32), self.before.view(torch.int32)
        return torch.equal(a[:GUARD], b[:GUARD]) and torch.equal(a[GUARD + self.n:], b[GUARD + self.n:])

    def untouched(self):
        return torch.equal(self.big.view(torch.int32), self.before.view(torch.int32))


def _exact(out, want, what):
    """out (fp32) equals the exact fp64 `want` in every element."""
    assert torch.equal(want.float().double(), want), "{}: the test data is not exact in fp32".format(what)
    bad = out.double() != want
    if bad.any():
        i = [int(v) for v in bad.nonzero()[0]]
        pytest.fail("{}: {} of {} outputs differ, first at {}: {!r} instead of {!r}".format(
            what, int(bad.sum()), bad.numel(), i, float(out[tuple(i)]), float(want[tuple(i)])))


def _ulp(x):
    a = x.float().abs()
    return (torch.nextafter(a, torch.full_like(a, float("inf"))) - a).double()


def _near(out, want, tol, what):
    assert torch.isfinite(out).all(), "{}: non-finite outputs".format(what)
    bad = (out.double() - want).abs() > tol
    if bad.any():
        i = [int(v) for v in bad.nonzero()[0]]
        pytest.fail("{}: {} of {} outputs off by more than a few ulps, first at {}: {!r} instead of {!r}".format(
            what, int(bad.sum()), bad.numel(), i, float(out[tuple(i)]), float(want[tuple(i)])))


def _addr(t):
    return None if t is None else t.data_ptr()


# ---------------------------------------------------------------------------------------------------------------
# conv2d forward and data gradient: nm_conv2d_fwd with flip = 0 and 1
# ---------------------------------------------------------------------------------------------------------------

def _same(k):
    return P._same(k)


VALID = (0, 0, 0, 0)

# (name, (N, H, W, Cin, Cout, k, (pt, pb, pl, pr)), act, bias).  The data gradient of each runs from dY [N,Ho,Wo,Cout]
# with pads k-1-p, as ops._Conv2d does, so its gathered channels are Cout.
FWD_CASES = [
    ("m_128q_minus_1", (1, 15, 17, 4, 8, 3, _same(3)), "none", True),           # M = 255
    ("m_128q", (1, 16, 16, 3, 8, 3, _same(3)), "none", True),                    # M = 256
    ("m_128q_plus_1", (5, 7, 11, 4, 8, 3, _same(3)), "none", True),              # M = 385
    ("m_64q_minus_1", (1, 11, 29, 4, 8, 3, _same(3)), "relu", True),             # M = 319: the CUDA-core tile
    ("cout_1", (2, 9, 10, 4, 1, 3, _same(3)), "none", True),
    ("cout_63", (2, 9, 10, 4, 63, 3, _same(3)), "none", True),
    ("cout_64", (2, 9, 10, 4, 64, 3, _same(3)), "none", True),
    ("cout_65", (2, 9, 10, 4, 65, 3, _same(3)), "none", True),
    ("cout_129", (2, 9, 10, 4, 129, 3, _same(3)), "none", True),
    ("kdim_31", (2, 10, 12, 31, 12, 1, VALID), "none", True),                    # k*k*Cin = 31, one partial k-block
    ("kdim_32", (2, 10, 12, 8, 12, 2, _same(2)), "none", True),                  # 32: one full k-block
    ("kdim_33", (2, 10, 12, 33, 12, 1, VALID), "none", True),                    # 33: a k-block of one
    ("k1_cin4", (2, 10, 12, 4, 16, 1, VALID), "none", True),
    ("cin13_k5_taps_cross_kblocks", (2, 12, 10, 13, 17, 5, _same(5)), "none", True),
    ("cin_mult4_cout_not", (2, 9, 11, 8, 7, 3, _same(3)), "none", True),        # vector forward, scalar dgrad
    ("cin_not_mult4_cout_mult4", (2, 9, 11, 7, 8, 3, _same(3)), "none", True),
    ("valid_k3", (2, 9, 11, 4, 8, 3, VALID), "none", True),
    ("same_odd_k5", (2, 9, 11, 4, 8, 5, _same(5)), "none", True),
    ("same_even_k2", (2, 9, 11, 4, 8, 2, _same(2)), "none", True),               # pt = 0 < pb = 1
    ("same_even_k4", (2, 9, 11, 4, 8, 4, _same(4)), "none", True),               # pt = 1 < pb = 2
    ("pads_0202", (2, 9, 11, 4, 8, 3, (0, 2, 2, 0)), "none", True),              # H and W pads differ
    ("pads_2011", (2, 9, 11, 4, 8, 3, (2, 0, 1, 1)), "relu", True),
    ("window_fills_padded_height", (3, 3, 9, 4, 8, 3, VALID), "none", True),    # Ho = 1
    ("window_fills_padded_width", (3, 9, 2, 4, 8, 3, (1, 0, 0, 1)), "none", True),   # Wo = 1 with pads
    ("h_1", (3, 1, 37, 4, 8, 3, _same(3)), "none", True),
    ("w_1", (3, 37, 1, 4, 8, 3, _same(3)), "none", True),
    ("relu", (2, 9, 11, 4, 8, 3, _same(3)), "relu", True),
    ("no_bias", (2, 9, 11, 4, 8, 3, _same(3)), "none", False),
    ("no_bias_relu", (2, 9, 11, 5, 8, 3, _same(3)), "relu", False),
]


def _conv_ref(x, w, bias, pads, act):
    """fp64 conv2d: NHWC x, HWIO w, pads (pt, pb, pl, pr)."""
    pt, pb, pl, pr = pads
    xn = F.pad(x.double().permute(0, 3, 1, 2), (pl, pr, pt, pb))
    y = F.conv2d(xn, w.double().permute(3, 2, 0, 1)).permute(0, 2, 3, 1)
    if bias is not None:
        y = y + bias.double()
    return torch.relu(y) if act == "relu" else y


def _conv_fwd(engine, x, w_stored, bias, y, k, pads, flip, act):
    n, h, wd, c = x.shape
    lib = _lib()
    return lib.load().nm_conv2d_fwd(_addr(x), _addr(w_stored), _addr(bias), _addr(y), n, h, wd, c, y.shape[-1], k,
                                    *pads, flip, lib.NM_ACT[act], _backend(engine), lib.stream())


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("case", FWD_CASES, ids=lambda c: c[0])
def test_conv2d_fwd_and_dgrad_exact(case, engine):
    """y = act(conv(x, w) + b) and dX = conv(dY, w turned, pads k-1-p) through the C ABI, each aligned and with
    the gathered tensor one float off."""
    name, shape, act, has_bias = case
    n, h, wd, cin, cout, k, pads = shape
    ho, wo = P.conv_out(shape)
    g = torch.Generator(device="cuda").manual_seed(sum(shape[:6]) + len(name))
    w = _ints((k, k, cin, cout), g, log2_unit=_unit(k * k * max(cin, cout)))
    bias = _ints((max(cin, cout),), g, log2_unit=4) if has_bias else None
    dpads = tuple(k - 1 - p for p in pads)
    runs = [
        # flip = 0: x [N,H,W,Cin] -> y [N,Ho,Wo,Cout] with w as stored
        ("fwd", 0, _ints((n, h, wd, cin), g, log2_unit=1), w, w, pads),
        # flip = 1: dY [N,Ho,Wo,Cout] -> dX [N,H,W,Cin]; the kernel turns the stored forward filter, so the
        # reference convolves with w turned by 180 degrees and its channel axes swapped
        ("dgrad", 1, _ints((n, ho, wo, cout), g, log2_unit=1), w, w.flip(0, 1).transpose(2, 3), dpads),
    ]
    for what, flip, src, w_stored, w_eff, pp in runs:
        oc = w_eff.shape[-1]
        b = None if bias is None else bias[:oc]
        want = _conv_ref(src, w_eff, b, pp, act)
        for shift in (0, 1):
            tag = "{} {} {} shift={} x{} pads={}".format(name, engine, what, shift, tuple(src.shape), pp)
            x_st, w_st = _stored(src, shift), _stored(w_stored)
            b_st = None if b is None else _stored(b)
            out = Guarded(tuple(want.shape))
            rc = _conv_fwd(engine, x_st, w_st, b_st, out.win, k, pp, flip, act)
            assert rc == 0, "{}: status {}: {}".format(tag, rc, _lib().load().nm_last_error())
            torch.cuda.synchronize()
            _exact(out.win, want, tag)
            assert out.outside_unchanged(), "{}: wrote outside the output".format(tag)


def test_conv2d_fwd_int64_addressing():
    """An output of more than 2^31 elements on the wgmma engine: the first and the last 128-row tiles."""
    n, h, wd, cin, cout = 1, 1024, 1024, 4, 2064
    numel = n * h * wd * cout
    assert numel > 2 ** 31
    need = (numel + n * h * wd * cin) * 4 + (1 << 30)
    if torch.cuda.mem_get_info()[0] < need:
        pytest.skip("needs {:.1f} GB of free device memory".format(need / 2 ** 30))
    g = torch.Generator(device="cuda").manual_seed(31)
    x = _ints((n, h, wd, cin), g, log2_unit=1)
    w = _ints((1, 1, cin, cout), g, log2_unit=2)
    bias = _ints((cout,), g, log2_unit=4)
    out = torch.full((numel + GUARD,), SENTINEL, device="cuda")
    try:
        y = out[:numel].view(n * h * wd, cout)
        rc = _conv_fwd("tc", x, w, bias, y, 1, VALID, 0, "none")
        assert rc == 0, _lib().load().nm_last_error()
        torch.cuda.synchronize()
        xs = x.view(-1, cin).double()
        for rows in (slice(0, 128), slice(n * h * wd - 128, n * h * wd)):
            want = xs[rows] @ w.view(cin, cout).double() + bias.double()
            _exact(y[rows], want, "int64 addressing rows {}".format(rows))
        assert torch.equal(out[numel:], torch.full((GUARD,), SENTINEL, device="cuda"))
    finally:
        del out
        torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------
# weight gradients: nm_conv2d_wgrad and nm_glu_conv1d_wgrad at the plans of tests/conv_plan_cases.py
# ---------------------------------------------------------------------------------------------------------------

def _wgrad_params():
    return [pytest.param(c, kind, id="{}-{}".format(kind, c.name)) for c in P.WGRAD_CASES for kind in c.kinds]


def test_wgrad_plan_restatement_matches_the_device(sms):
    """nm_conv2d_wgrad_workspace / nm_glu_conv1d_wgrad_workspace = splits x slice of the restated plan, for every
    case's candidates on both engines."""
    lib = _lib().load()
    for case in P.WGRAD_CASES:
        for kind in case.kinds:
            for engine in ENGINES:
                for shape in (case.conv if kind == "conv2d" else case.glu):
                    p = P.plan_for(kind, engine, shape, sms)
                    if kind == "conv2d":
                        nn, h, wd, cin, cout, k, pads = shape
                        got = lib.nm_conv2d_wgrad_workspace(nn, h, wd, cin, cout, k, *pads, _backend(engine))
                    else:
                        got = lib.nm_glu_conv1d_wgrad_workspace(*shape, _backend(engine))
                    assert got == p.splits * p.part, (case.name, kind, engine, shape, p)


def _glu_patches(x, k):
    """fp64 patch matrix of the GLU convolution: [B*T, k*F], TF's `same` padding, zeros outside each sequence."""
    b, t, f = x.shape
    pb = (k - 1) // 2
    xp = F.pad(x.double(), (0, 0, pb, k - 1 - pb))
    return torch.cat([xp[:, j:j + t] for j in range(k)], dim=2).reshape(b * t, k * f)


def _conv_patches(x, k, pads):
    """fp64 patch matrix of conv2d: [N*Ho*Wo, k*k*Cin], columns (ky, kx, c)."""
    pt, pb, pl, pr = pads
    n, h, wd, c = x.shape
    xp = F.pad(x.double(), (0, 0, pl, pr, pt, pb))
    ho, wo = h + pt + pb - k + 1, wd + pl + pr - k + 1
    return torch.cat([xp[:, ky:ky + ho, kx:kx + wo] for ky in range(k) for kx in range(k)],
                     dim=3).reshape(n * ho * wo, k * k * c)


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("case,kind", _wgrad_params())
def test_wgrad_exact(case, kind, engine, sms):
    """dw = start + patches^T dy and db = start + sum dy exactly, at the case's plan; the workspace starts NaN, so a
    slice the reduction reads but no CTA wrote shows."""
    lib = _lib()
    shape = P.find_shape(case, kind, engine, sms)
    assert shape is not None, "{}: no candidate shape lands on this branch at {} SMs".format(case.name, sms)
    ws_floats = P.workspace(case, kind, engine, shape, sms)
    plan = P.plan_for(kind, engine, shape, sms, ws_floats)
    rows, cols, m = P.gemm_dims(kind, shape)
    g = torch.Generator(device="cuda").manual_seed(2 * P.WGRAD_CASES.index(case) + (kind == "glu"))
    if kind == "conv2d":
        nn, h, wd, cin, cout, k, pads = shape
        ho, wo = P.conv_out(shape)
        x = _ints((nn, h, wd, cin), g, -1, 1, log2_unit=1)
        dy = _ints((nn, ho, wo, cout), g, log2_unit=2)
        patches = _conv_patches(x, k, pads)
        wshape = (k, k, cin, cout)
    else:
        b, t, f, k = shape
        x = _ints((b, t, f), g, -1, 1, log2_unit=1)
        dy = _ints((b, t, 2 * f), g, log2_unit=2)
        patches = _glu_patches(x, k)
        wshape = (k, f, 2 * f)
    dy2 = dy.reshape(m, cols).double()
    assert 3 * m < 2 ** 23
    dw0 = _ints(wshape, g, log2_unit=3)
    db0 = _ints((cols,), g, log2_unit=3)
    want_dw = dw0.double() + (patches.t() @ dy2).reshape(wshape)
    want_db = db0.double() + dy2.sum(0)
    for shift in (0, 1):
        tag = "{} {} {} shift={} shape={} plan={}".format(case.name, kind, engine, shift, shape, tuple(plan))
        x_st, dy_st = _stored(x, shift), _stored(dy)
        dw, db = Guarded(wshape, dw0), (Guarded((cols,), db0) if case.db else None)
        ws = torch.full((ws_floats,), float("nan"), device="cuda")
        if kind == "conv2d":
            rc = lib.load().nm_conv2d_wgrad(_addr(x_st), _addr(dy_st), _addr(dw.win), _addr(db and db.win),
                                            _addr(ws), ws_floats, nn, h, wd, cin, cout, k, *pads, _backend(engine),
                                            lib.stream())
        else:
            rc = lib.load().nm_glu_conv1d_wgrad(_addr(x_st), _addr(dy_st), _addr(dw.win), _addr(db.win), _addr(ws),
                                                ws_floats, b, t, f, k, _backend(engine), lib.stream())
        assert rc == 0, "{}: status {}: {}".format(tag, rc, lib.load().nm_last_error())
        torch.cuda.synchronize()
        _exact(dw.win, want_dw, tag + " dw")
        assert dw.outside_unchanged(), tag + " dw: wrote outside"
        if db is not None:
            _exact(db.win, want_db, tag + " db")
            assert db.outside_unchanged(), tag + " db: wrote outside"
        # the kernels wrote exactly plan.splits slices: the rest of a capped workspace keeps its NaNs
        assert torch.isnan(ws[plan.splits * plan.part:]).all(), tag + ": wrote past the plan's slices"
        assert not torch.isnan(ws[:plan.splits * plan.part]).any(), tag + ": a slice of the plan was not written"


# ---------------------------------------------------------------------------------------------------------------
# GLU conv1d: forward, dz, data gradient
# ---------------------------------------------------------------------------------------------------------------

# (name, (B, T, F, k))
GLU_CASES = [
    ("f63", (3, 23, 63, 3)),        # the forward's 64-feature tile, each with its gate
    ("f64", (3, 23, 64, 3)),
    ("f65", (3, 23, 65, 3)),
    ("f127", (2, 37, 127, 3)),      # the data gradient's 128-column tile
    ("f128", (2, 37, 128, 3)),
    ("f129", (2, 37, 129, 3)),
    ("f_odd_k2", (4, 19, 9, 2)),    # odd F: scalar gathers
    ("f_even_k4", (4, 19, 12, 4)),
    ("t1", (37, 1, 8, 3)),
    ("t_below_k", (29, 2, 8, 5)),
    ("t5_many_sequences_per_tile", (61, 5, 8, 3)),
    ("t5_k4", (61, 5, 7, 4)),
]


def _glu_refs(x, w, bias, k):
    """fp64 z = conv1d_same(x, w) + b [B*T, 2F]."""
    b, t, f = x.shape
    return _glu_patches(x, k) @ w.double().reshape(k * f, 2 * f) + bias.double()


def _glu_y_check(y, z, x, what):
    """y = z_lin * sigmoid(z_gate) + x within a few ulps of the fp64 expression on the exact z."""
    f = x.shape[-1]
    zl, zg = z[:, :f], z[:, f:]
    part = zl * torch.sigmoid(zg)
    want = part + x.reshape(-1, f).double()
    _near(y.reshape(-1, f), want, 4 * (_ulp(part) + _ulp(want)), what)


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("case", GLU_CASES, ids=lambda c: c[0])
def test_glu_conv1d_fwd_and_dgrad_exact(case, engine):
    """nm_glu_conv1d_fwd (z exact, y to a few ulps, z = NULL gives the same y bits) and nm_glu_conv1d_dgrad (exact),
    each aligned and with x and w one float off."""
    lib = _lib()
    name, (b, t, f, k) = case
    g = torch.Generator(device="cuda").manual_seed(b * 1000 + t * 10 + f + k)
    x = _ints((b, t, f), g, -1, 1)
    w = _ints((k, f, 2 * f), g, log2_unit=_unit(k * f))
    bias = _ints((2 * f,), g, log2_unit=4)
    z_want = _glu_refs(x, w, bias, k)
    dz = _ints((b, t, 2 * f), g, log2_unit=1)
    dy = _ints((b, t, f), g, log2_unit=3)
    pb = (k - 1) // 2
    # dX = conv1d(dZ, w with taps reversed and channel axes swapped, pads k-1-pb before) + dY
    w_turned = w.double().flip(0).transpose(1, 2).reshape(k * 2 * f, f)
    dzp = F.pad(dz.double(), (0, 0, k - 1 - pb, pb))
    dx_want = (torch.cat([dzp[:, j:j + t] for j in range(k)], dim=2).reshape(b * t, k * 2 * f) @ w_turned
               + dy.reshape(b * t, f).double()).reshape(b, t, f)
    for shift in (0, 1):
        tag = "{} {} shift={} B={} T={} F={} k={}".format(name, engine, shift, b, t, f, k)
        x_st, w_st, b_st = _stored(x, shift), _stored(w, shift), _stored(bias)
        y, z = Guarded((b, t, f)), Guarded((b, t, 2 * f))
        rc = lib.load().nm_glu_conv1d_fwd(_addr(x_st), _addr(w_st), _addr(b_st), _addr(y.win), _addr(z.win), b, t, f,
                                          k, _backend(engine), lib.stream())
        assert rc == 0, "{}: status {}: {}".format(tag, rc, lib.load().nm_last_error())
        y2 = Guarded((b, t, f))
        rc = lib.load().nm_glu_conv1d_fwd(_addr(x_st), _addr(w_st), _addr(b_st), _addr(y2.win), None, b, t, f, k,
                                          _backend(engine), lib.stream())
        assert rc == 0, "{}: status {}".format(tag, rc)
        torch.cuda.synchronize()
        _exact(z.win.reshape(b * t, 2 * f), z_want, tag + " z")
        _glu_y_check(y.win, z_want, x, tag + " y")
        assert torch.equal(y.win.view(torch.int32), y2.win.view(torch.int32)), tag + ": z = NULL changes y"
        assert y.outside_unchanged() and z.outside_unchanged() and y2.outside_unchanged(), tag + ": wrote outside"

        dz_st, dy_st = _stored(dz, shift), _stored(dy)
        dx = Guarded((b, t, f))
        rc = lib.load().nm_glu_conv1d_dgrad(_addr(dz_st), _addr(w_st), _addr(dy_st), _addr(dx.win), b, t, f, k,
                                            _backend(engine), lib.stream())
        assert rc == 0, "{}: status {}: {}".format(tag, rc, lib.load().nm_last_error())
        torch.cuda.synchronize()
        _exact(dx.win, dx_want, tag + " dx")
        assert dx.outside_unchanged(), tag + " dx: wrote outside"


@pytest.mark.parametrize("m,f", [(1, 1), (37, 63), (129, 64), (300, 129)])
def test_glu_dz_within_ulps(m, f):
    """dZ = [dY s, dY a s (1 - s)], s = sigmoid(gate), a = the linear half, against fp64 on the same z: the error
    of s (a few ulps of s) enters the gate half scaled by |dY a (1 - 2s)| <= |dY a|."""
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(m + f)
    z = _ints((m, 2 * f), g, log2_unit=0)          # |gate| <= 3: s stays clear of 0 and 1
    dy = _ints((m, f), g, log2_unit=2)
    dz = Guarded((m, 2 * f))
    dy_st, z_st = _stored(dy, 1), _stored(z, 1)       # held until the kernel has run: a freed buffer is reused
    rc = lib.load().nm_glu_conv1d_dz(_addr(dy_st), _addr(z_st), _addr(dz.win), m, f, lib.stream())
    assert rc == 0
    torch.cuda.synchronize()
    a, gate, d = z[:, :f].double(), z[:, f:].double(), dy.double()
    s = torch.sigmoid(gate)
    s_ulp = _ulp(s)
    want_lin, want_gate = d * s, d * a * s * (1 - s)
    _near(dz.win[:, :f], want_lin, 4 * (_ulp(want_lin) + d.abs() * s_ulp), "dz linear half")
    _near(dz.win[:, f:], want_gate, 4 * (_ulp(want_gate) + (d * a).abs() * s_ulp), "dz gate half")
    assert dz.outside_unchanged()


# ---------------------------------------------------------------------------------------------------------------
# VGG primitives: nm_im2col3x3, nm_conv3x3_bias_relu_fwd, ops.conv3x3_bias_relu, nm_maxpool2x2_fwd
# ---------------------------------------------------------------------------------------------------------------

def _vgg_ref(x, w, bias):
    return _conv_ref(x, w, bias, (1, 1, 1, 1), "relu")


@pytest.mark.parametrize("cin,ldc", [(3, 27), (3, 29), (4, 36), (4, 39), (4, 44), (13, 120), (64, 580)])
def test_im2col3x3_exact(cin, ldc):
    """Every patch entry is the input pixel or zero; columns [9*Cin, ldc) and the rows past M keep the sentinel.
    A pitch that is not a multiple of 4 floats, or an input one float off, takes the scalar copy."""
    lib = _lib()
    n, h, wd = 3, 7, 5
    m = n * h * wd
    g = torch.Generator(device="cuda").manual_seed(cin * 100 + ldc)
    x = _ints((n, h, wd, cin), g)
    want = _conv_patches(x, 3, (1, 1, 1, 1))
    for shift in (0, 1):
        cols = Guarded((m + 3, ldc), SENTINEL)
        x_st = _stored(x, shift)
        rc = lib.load().nm_im2col3x3(_addr(x_st), _addr(cols.win), n, h, wd, cin, ldc, lib.stream())
        assert rc == 0, lib.load().nm_last_error()
        torch.cuda.synchronize()
        tag = "im2col Cin={} ldc={} shift={}".format(cin, ldc, shift)
        _exact(cols.win[:m, :9 * cin], want, tag)
        rest = torch.cat([cols.win[:m, 9 * cin:].reshape(-1), cols.win[m:].reshape(-1)])
        assert torch.equal(rest.view(torch.int32), torch.full_like(rest, SENTINEL).view(torch.int32)), \
            tag + ": wrote past 9*Cin or M"
        assert cols.outside_unchanged(), tag


@pytest.mark.parametrize("m_shape", [(1, 9, 7), (1, 8, 8), (1, 5, 13), (3, 7, 7)], ids=lambda s: "m{}".format(
    s[0] * s[1] * s[2]))
@pytest.mark.parametrize("cout", [3, 63, 64, 65])
def test_conv3x3_bias_relu_fwd_exact(m_shape, cout):
    """The CUDA-core VGG convolution at M = 63, 64, 65 and 147 pixels (64-row tiles) and Cout around the 64-column
    tile."""
    lib = _lib()
    n, h, wd = m_shape
    cin = 5
    g = torch.Generator(device="cuda").manual_seed(n * h * wd + cout)
    x = _ints((n, h, wd, cin), g, log2_unit=1)
    w = _ints((3, 3, cin, cout), g, log2_unit=2)
    bias = _ints((cout,), g, log2_unit=3)
    want = _vgg_ref(x, w, bias)
    for shift in (0, 1):
        y = Guarded((n, h, wd, cout))
        x_st, w_st, b_st = _stored(x, shift), _stored(w), _stored(bias)
        rc = lib.load().nm_conv3x3_bias_relu_fwd(_addr(x_st), _addr(w_st), _addr(b_st), _addr(y.win), n, h, wd, cin,
                                                 cout, lib.stream())
        assert rc == 0, lib.load().nm_last_error()
        torch.cuda.synchronize()
        _exact(y.win, want, "conv3x3 {} Cout={} shift={}".format(m_shape, cout, shift))
        assert y.outside_unchanged()


def test_conv3x3_batch_split():
    """ceil(N*H*W / 64) > 65535 pixel tiles: the batch is launched in parts of 63 images; the images on each side
    of the seam are exact."""
    lib = _lib()
    n, h, wd, c = 65, 256, 256, 4
    assert -(-n * h * wd // 64) > 65535
    per = 65535 * 64 // (h * wd)
    g = torch.Generator(device="cuda").manual_seed(65)
    x = _ints((n, h, wd, c), g, log2_unit=1)
    w = _ints((3, 3, c, c), g, log2_unit=2)
    bias = _ints((c,), g, log2_unit=3)
    y = Guarded((n, h, wd, c))
    rc = lib.load().nm_conv3x3_bias_relu_fwd(_addr(x), _addr(w), _addr(bias), _addr(y.win), n, h, wd, c, c,
                                             lib.stream())
    assert rc == 0, lib.load().nm_last_error()
    torch.cuda.synchronize()
    for i in (0, per - 1, per, n - 1):
        _exact(y.win[i:i + 1], _vgg_ref(x[i:i + 1], w, bias), "batch split image {}".format(i))
    assert y.outside_unchanged()


@pytest.fixture
def auto_backend():
    from neuralmonkey_b200 import ops
    ops.set_gemm_backend("auto")
    yield
    ops.set_gemm_backend("auto")


def _entry_points(fn):
    lib = _lib()
    lib.profile_start()
    try:
        out = fn()
    finally:
        calls = lib.profile_stop()
    return out, {k.split("[")[0]: v["calls"] for k, v in calls.items()}


def test_conv3x3_bias_relu_im2col_chunks(auto_backend):
    """ops.conv3x3_bias_relu under `auto` with a patch matrix of more than 768 MB: two im2col chunks (85 images
    and 2) through the wgmma GEMM; the images at the chunk seam are exact."""
    from neuralmonkey_b200 import ops
    n, h, wd, cin, cout = 87, 64, 64, 64, 4
    per_image = h * wd * ((9 * cin + 3) // 4 * 4) * 4     # bytes of one image's patch rows, pitch a multiple of 4
    chunk = (768 << 20) // per_image
    assert 1 < chunk < n
    g = torch.Generator(device="cuda").manual_seed(83)
    x = _ints((n, h, wd, cin), g, -1, 1)
    w = _ints((3, 3, cin, cout), g, log2_unit=2)
    bias = _ints((cout,), g, log2_unit=3)
    y, calls = _entry_points(lambda: ops.conv3x3_bias_relu(x, w, bias))
    torch.cuda.synchronize()
    assert calls.get("nm_im2col3x3") == -(-n // chunk) and "nm_conv3x3_bias_relu_fwd" not in calls, calls
    for i in (0, chunk - 1, chunk, n - 1):
        _exact(y[i:i + 1], _vgg_ref(x[i:i + 1], w, bias), "im2col chunk seam image {}".format(i))


@pytest.mark.parametrize("cout", [3, 5])
def test_conv3x3_bias_relu_auto_fallback(auto_backend, cout):
    """Cout % 4 != 0 under `auto`: the CUDA-core kernel, exact."""
    from neuralmonkey_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(cout)
    x = _ints((2, 9, 11, 6), g, log2_unit=1)
    w = _ints((3, 3, 6, cout), g, log2_unit=2)
    bias = _ints((cout,), g, log2_unit=3)
    y, calls = _entry_points(lambda: ops.conv3x3_bias_relu(x, w, bias))
    torch.cuda.synchronize()
    assert calls.get("nm_conv3x3_bias_relu_fwd") == 1 and "nm_im2col3x3" not in calls, calls
    _exact(y, _vgg_ref(x, w, bias), "conv3x3 auto fallback Cout={}".format(cout))


@pytest.mark.parametrize("shape", [(2, 6, 8, 1), (3, 4, 10, 5), (1, 2, 2, 64)])
def test_maxpool2x2_exact_with_ties(shape):
    """Values from {-1, 0, 1}, so most windows tie; C = 1 included."""
    lib = _lib()
    n, h, wd, c = shape
    g = torch.Generator(device="cuda").manual_seed(sum(shape))
    x = _ints(shape, g, -1, 1)
    want = F.max_pool2d(x.double().permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1)
    for shift in (0, 1):
        y = Guarded((n, h // 2, wd // 2, c))
        x_st = _stored(x, shift)
        rc = lib.load().nm_maxpool2x2_fwd(_addr(x_st), _addr(y.win), n, h, wd, c, lib.stream())
        assert rc == 0
        torch.cuda.synchronize()
        _exact(y.win, want, "maxpool {} shift={}".format(shape, shift))
        assert y.outside_unchanged()


@pytest.mark.parametrize("h,w", [(5, 4), (4, 7), (1, 2)])
def test_maxpool2x2_refuses_odd_sizes(h, w):
    lib = _lib()
    x = _stored(torch.zeros(2, h, w, 3, device="cuda"))
    y = Guarded((2, max(h // 2, 1), max(w // 2, 1), 3))
    assert lib.load().nm_maxpool2x2_fwd(_addr(x), _addr(y.win), 2, h, w, 3, lib.stream()) == NM_E_INVALID
    torch.cuda.synchronize()
    assert y.untouched()
