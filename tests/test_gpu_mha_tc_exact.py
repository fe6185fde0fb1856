"""The tensor-core attention (csrc/mha_tc.cu) stage by stage, through `nm_mha_tc_fwd` / `nm_mha_tc_bwd`, at every
tile and padding boundary of its batched wgmma products.

Q, K, V and dO are integers in [-3, 3] times 2^-s, with s = 1, 0, 2 for sentences 0, 1, 2, 3, ...  Every partial sum
of Q.K^T and dO.V^T is then exact in fp32 and their operands exact in TF32, so the energies and dP are known exactly
whatever the order of summation and whether the hardware rounds or truncates to TF32.  Each stage is compared with
fp64 computed from the kernel's own stored inputs to that stage, against a bound derived per element:

  probs       fp64 softmax of the exact energies times the fp32 1/sqrtf(dh), masked as the reference masks them
              (causal entries replaced by -1e9, padded keys x*m + (1-m)*(-1e9)); a few fp32 ulps of the energy in
              log2 units plus ex2.approx's relative error
  probs_drop  probs * drop in fp32, bit for bit
  ds_work     P * (dP*drop - sum(P * dP*drop)) / sqrt(dh) from the stored P and the exact dP, zero where masked
  out, dq,    (P*drop).V, dS.K, dS^T.Q and (P*drop)^T.dO from the stored [Tq, Tk] matrices: the stored operand is
  dk, dv      rounded or truncated to TF32, the other is exact, so the bound per element is
              sum ulp_tf32(a)*|b| plus an fp32 accumulation term

The [B, heads, Tq, Tk] storage is padded to multiples of 32 in both time extents, and the products reduce over
whole 32-element blocks of it while the other operand's rows run on into the next sentence: the padding must be
exactly zero.  Every output lives in a NaN-filled buffer whose margins must stay NaN, and every operand is a window
of one, so a read past the last sentence shows.  The end-to-end fp64 check of test_gpu_mha_tc.py runs as well."""
import math

import numpy as np
import pytest
import torch

from tests.helpers import max_abs, rel_err
from tests.test_gpu_mha_tc import _reference

pytestmark = pytest.mark.gpu

NM_E_UNSUPPORTED = -2
U = 2.0 ** -24              # fp32 unit roundoff
EX2_REL = 2.0 ** -21        # relative error of ex2.approx.ftz.f32 (about 2^-22), with a factor 2 of margin
TINY = 2.0 ** -120          # ex2.approx.ftz flushes results below 2^-126 to zero
LOG2E = 1.4426950408889634
GUARD = 32                  # NaN floats on either side of every buffer (keeps 16-byte alignment)
SCALES = (1, 0, 2)          # sentence b's operands are integers times 2^-SCALES[b % 3]
KEEP = 0.7

# name: ((B, Tq, Tk, heads, dh), key mask, causal, dropout).  Key masks: "ragged" = lengths Tk, 1, Tk/2, ...;
# "empty" = Tk/2, 0, Tk, ... (sentence 1 has no keys: uniform rows).  The dropout-mask rows load as 16-byte vectors
# for the 32-key chunks that are complete when Tk % 4 == 0, element by element otherwise.
CASES = {
    # both edges of every count of 32-key chunks; heads = 1 and >= 3 for every head size
    "tk1": ((3, 8, 1, 2, 32), None, False, False),
    "tk31_dh64_h3_drop_scalar": ((3, 40, 31, 3, 64), "ragged", False, True),
    "tk32_dh96_h1_causal_mask_drop_vector": ((3, 32, 32, 1, 96), "ragged", True, True),
    "tk33_tq129_dh32_h4_empty": ((3, 129, 33, 4, 32), "empty", False, False),
    "tk64_dh128_h1_causal_drop_vector": ((2, 64, 64, 1, 128), None, True, True),
    "tk65_tq33": ((3, 33, 65, 2, 64), "ragged", False, False),
    "tk96_tq257_dh96_h3": ((2, 257, 96, 3, 96), "ragged", False, False),
    "tk97_dh32_h1_causal_mask_drop_scalar": ((3, 97, 97, 1, 32), "ragged", True, True),
    "tk127_tq8_dh128_h4_empty_drop": ((2, 8, 127, 4, 128), "empty", False, True),
    "tk128_dh64_h1_causal_empty_drop_vector": ((2, 128, 128, 1, 64), "empty", True, True),
    # dropout: vector chunks, then a scalar one
    "drop_tk36": ((3, 20, 36, 2, 64), None, False, True),
    "drop_tk100_dh32_h3": ((2, 50, 100, 3, 32), "ragged", False, True),
    "drop_tk37_dh96_h3_causal_scalar": ((2, 37, 37, 3, 96), None, True, True),
    # fewer than 8 queries: the C ABI takes them, ops.mha_core sends them to the exact kernels
    "tq1_abi": ((4, 1, 50, 2, 32), "ragged", False, False),
    "tq7_abi_causal_drop": ((3, 7, 7, 2, 64), None, True, True),
    # 2048 (sentence, head) problems: many more work items than SMs
    "items2048_mask_drop": ((256, 40, 40, 8, 32), "ragged", False, True),
}


def _lib():
    from neuralmonkey_b200 import lib
    return lib


def _pad32(x):
    return (x + 31) // 32 * 32


class Guarded:
    """A tensor of `shape` inside a NaN-filled buffer with GUARD floats on either side, 16-byte aligned."""

    def __init__(self, shape, device, values=None):
        n = math.prod(shape)
        self.big = torch.full((n + 2 * GUARD,), float("nan"), device=device)
        self.t = self.big[GUARD:GUARD + n].view(shape)
        if values is not None:
            self.t.copy_(values)

    def margins_nan(self):
        return bool(torch.isnan(self.big[:GUARD]).all() and torch.isnan(self.big[-GUARD:]).all())

    def bits(self):
        return self.big.view(torch.int32)


def _inputs(shape, mask_kind, use_drop, seed):
    bsz, tq, tk, heads, dh = shape
    g = torch.Generator(device="cuda").manual_seed(seed)
    unit = torch.tensor([2.0 ** -SCALES[b % 3] for b in range(bsz)], device="cuda").view(bsz, 1, 1)

    def ints(t):
        return torch.randint(-3, 4, (bsz, t, heads * dh), device="cuda", generator=g).float() * unit
    inp = {"q": ints(tq), "k": ints(tk), "v": ints(tk), "dout": ints(tq), "mask": None, "drop": None}
    if mask_kind is not None:
        lens = {"ragged": (tk, 1, (tk + 1) // 2), "empty": ((tk + 1) // 2, 0, tk)}[mask_kind]
        lens = torch.tensor([lens[b % 3] for b in range(bsz)], device="cuda")
        inp["mask"] = (torch.arange(tk, device="cuda")[None, :] < lens[:, None]).float()
    if use_drop:
        inp["drop"] = (torch.rand(bsz, heads, tq, tk, device="cuda", generator=g) < KEEP).float() / KEEP
    return inp


def _call(inp, shape, causal):
    """nm_mha_tc_fwd, then nm_mha_tc_bwd, on operands and into outputs that are windows of NaN buffers."""
    lib = _lib()
    bsz, tq, tk, heads, dh = shape
    dev = inp["q"].device
    src = {n: None if t is None else Guarded(t.shape, dev, t) for n, t in inp.items()}
    wshape = (bsz, heads, _pad32(tq), _pad32(tk))
    o = {"out": Guarded((bsz, tq, heads * dh), dev), "probs": Guarded(wshape, dev),
         "probs_drop": Guarded(wshape, dev) if inp["drop"] is not None else None,
         "dq": Guarded((bsz, tq, heads * dh), dev), "dk": Guarded((bsz, tk, heads * dh), dev),
         "dv": Guarded((bsz, tk, heads * dh), dev), "ds_work": Guarded(wshape, dev)}

    def p(d, n):
        return lib.ptr(d[n].t) if d[n] is not None else None
    lib.call("nm_mha_tc_fwd", p(src, "q"), p(src, "k"), p(src, "v"), p(src, "mask"), int(causal), p(src, "drop"),
             p(o, "out"), p(o, "probs"), p(o, "probs_drop"), bsz, tq, tk, heads, dh, lib.stream())
    lib.call("nm_mha_tc_bwd", p(src, "q"), p(src, "k"), p(src, "v"), p(src, "mask"), int(causal), p(src, "drop"),
             p(o, "probs"), p(o, "probs_drop"), p(src, "dout"), p(o, "dq"), p(o, "dk"), p(o, "dv"), p(o, "ds_work"),
             bsz, tq, tk, heads, dh, lib.stream())
    torch.cuda.synchronize()
    return {n: b for n, b in o.items() if b is not None}


def _heads(t, heads):
    """[B, T, heads * dh] -> [B, heads, T, dh] in fp64."""
    bsz, t_len, d = t.shape
    return t.double().view(bsz, t_len, heads, d // heads).transpose(1, 2)


def _replaced(shape, mask, causal, device):
    """[B, 1, Tq, Tk]: True where the reference puts -1e9 (a future key, or a padded one)."""
    bsz, tq, tk = shape[0], shape[1], shape[2]
    out = torch.zeros(bsz, 1, tq, tk, dtype=torch.bool, device=device)
    if causal:
        out |= torch.ones(tq, tk, dtype=torch.bool, device=device).triu(1)
    if mask is not None:
        out |= (mask == 0).view(bsz, 1, 1, tk)
    return out


def _tf32_ulp(a):
    """One TF32 ulp of each fp32 value in a (fp64): what rounding or truncating it to TF32 can change.  Values that
    may flush to zero can lose themselves."""
    _, e = torch.frexp(a)
    ulp = torch.where(a == 0, torch.zeros_like(a), torch.ldexp(torch.ones_like(a), e - 11))
    return torch.maximum(ulp, torch.where(a.abs() < 2.0 ** -126, a.abs(), torch.zeros_like(a)))


def _product(a, b, k_len):
    """a @ b in fp64 and the bound on the kernel's product: a (stored fp32) goes to TF32 either way, b is exact,
    accumulation in fp32 over k_len terms (two ulps per term: truncating tensor-core additions included)."""
    want = a @ b
    bound = _tf32_ulp(a) @ b.abs() + k_len * 2.0 ** -22 * (a.abs() @ b.abs()) + TINY
    return want, bound


def _within(got, want, bound, what):
    bad = ~((got.double() - want).abs() <= bound)        # NaN counts as outside
    if bad.any():
        idx = tuple(int(i) for i in bad.nonzero()[0])
        pytest.fail("{}: {} of {} elements outside the bound, first at {}: {!r} instead of {!r} (bound {:.3g})".format(
            what, int(bad.sum()), bad.numel(), idx, float(got[idx]), float(want[idx]), float(bound[idx])))


def _check(inp, o, shape, causal, what):
    """Every stage of one forward + backward against fp64 from its own stored inputs."""
    bsz, tq, tk, heads, dh = shape
    tqp, tkp = _pad32(tq), _pad32(tk)
    mask, drop = inp["mask"], inp["drop"]
    for name, b in o.items():
        assert b.margins_nan(), "{}: {} written outside its buffer".format(what, name)
    for name in ("probs", "probs_drop", "ds_work"):
        if name in o:
            w = o[name].t
            assert bool((w[:, :, tq:, :] == 0).all()), "{}: {} padding rows not zero".format(what, name)
            assert bool((w[:, :, :, tk:] == 0).all()), "{}: {} padding columns not zero".format(what, name)
    probs = o["probs"].t[:, :, :tq, :tk]
    replaced = _replaced(shape, mask, causal, probs.device)

    # probs: softmax of the exact energies, scaled by the fp32 1/sqrtf(dh)
    scale = float(np.float32(1.0) / np.sqrt(np.float32(dh)))
    y = _heads(inp["q"], heads) @ _heads(inp["k"], heads).transpose(-1, -2) * scale
    p64 = torch.softmax(y.masked_fill(replaced, -1e9), -1)
    y2 = y * LOG2E                                       # the kernel works in log2 units
    y2max = y2.masked_fill(replaced, -math.inf).amax(-1, keepdim=True)
    y2max = torch.where(torch.isinf(y2max), torch.zeros_like(y2max), y2max)
    # error of the exponent: 4 ulps of the energy and of the row max (scale * LOG2E, acc * it), one of the difference
    delta = (4 * U * (y2.abs() + y2max.abs()) + U * (y2 - y2max).abs()).masked_fill(replaced, 0.0)
    eta = math.log(2.0) * delta + EX2_REL
    bound = 2 * p64 * (eta + eta.amax(-1, keepdim=True) + (tk + 2) * U) + TINY
    _within(probs, p64, bound, what + ": probs")

    weights = o["probs"].t
    if drop is not None:
        pd = o["probs_drop"].t
        assert torch.equal(pd[:, :, :tq, :tk], probs * drop), what + ": probs_drop != probs * drop in fp32"
        weights = pd
    w = weights[:, :, :tq, :tk].double()

    # out = (P * drop) V from the stored weights
    want, bound = _product(w, _heads(inp["v"], heads), tkp)
    _within(_heads(o["out"].t, heads), want, bound, what + ": out")

    # ds_work from the stored P and the exact dP
    dp = _heads(inp["dout"], heads) @ _heads(inp["v"], heads).transpose(-1, -2)
    pr = probs.double()
    t = dp * (drop.double() if drop is not None else 1.0)
    dot = (pr * t).sum(-1, keepdim=True)
    dot_abs = (pr * t).abs().sum(-1, keepdim=True)
    want = (pr * (t - dot) * scale).masked_fill(replaced, 0.0)
    err = pr * scale * (t.abs() * U + dot_abs * (tkp + 1) * U + (t - dot).abs() * U) + 2 * U * want.abs()
    ds = o["ds_work"].t[:, :, :tq, :tk]
    _within(ds, want, (2 * err + TINY).masked_fill(replaced, 0.0), what + ": ds_work")

    # dq = dS K, dk = dS^T Q, dv = (P * drop)^T dO from the stored matrices
    ds = ds.double()
    for name, a, b, k_len in (("dq", ds, inp["k"], tkp), ("dk", ds.transpose(-1, -2), inp["q"], tqp),
                              ("dv", w.transpose(-1, -2), inp["dout"], tqp)):
        want, bound = _product(a, _heads(b, heads), k_len)
        _within(_heads(o[name].t, heads), want, bound, "{}: {}".format(what, name))


@pytest.mark.parametrize("name", list(CASES))
def test_stages_against_fp64(name):
    shape, mask_kind, causal, use_drop = CASES[name]
    bsz, tq, tk, heads, dh = shape
    assert _lib().load().nm_mha_tc_supported(bsz, tq, tk, heads, dh) == 1
    inp = _inputs(shape, mask_kind, use_drop, seed=sum(shape) * 7 + len(name))
    o = _call(inp, shape, causal)
    _check(inp, o, shape, causal, name)

    again = _call(inp, shape, causal)
    for n in o:
        assert torch.equal(o[n].bits(), again[n].bits()), "{}: {} differs between two calls".format(name, n)

    # end to end against fp64 autograd of the reference, with test_gpu_mha_tc.py's TF32 bar
    cpu = {n: None if t is None else t.cpu() for n, t in inp.items()}
    q64, k64, v64 = (cpu[n].double().requires_grad_(True) for n in ("q", "k", "v"))
    ref, p = _reference(q64, k64, v64, cpu["mask"], causal, heads, cpu["drop"])
    (ref * cpu["dout"].double()).sum().backward()
    assert max_abs(o["probs"].t[:, :, :tq, :tk], p) < 2e-3, "probabilities"
    assert rel_err(o["out"].t, ref) < 3e-3, "context"
    for n, want in (("dq", q64.grad), ("dk", k64.grad), ("dv", v64.grad)):
        if bool(want.any()):       # a single key: dq = dk = 0, held to the stage bounds above
            assert rel_err(o[n].t, want) < 5e-3, n


@pytest.mark.parametrize("tk,dh", [(40, 16), (40, 48), (40, 160), (129, 32)],
                         ids=["dh16", "dh48", "dh160", "tk129"])
def test_refused_shapes_launch_nothing(tk, dh):
    """Head sizes that are not a multiple of 32 (or above 128) and more than 128 keys: NM_E_UNSUPPORTED from both
    entry points, no launch, no output written."""
    lib = _lib()
    bsz, tq, heads = 2, 40, 2
    h = lib.load()
    assert h.nm_mha_tc_supported(bsz, tq, tk, heads, dh) == 0
    inp = _inputs((bsz, tq, tk, heads, dh), "ragged", True, seed=tk + dh)
    wshape = (bsz, heads, _pad32(tq), _pad32(tk))
    outs = [Guarded(s, "cuda") for s in ((bsz, tq, heads * dh), wshape, wshape, (bsz, tq, heads * dh),
                                         (bsz, tk, heads * dh), (bsz, tk, heads * dh), wshape)]
    out, probs, probs_drop, dq, dk, dv, ds = (lib.ptr(b.t) for b in outs)
    before = [b.bits().clone() for b in outs]
    q, k, v, dout, mask, drop = (lib.ptr(inp[n]) for n in ("q", "k", "v", "dout", "mask", "drop"))
    torch.cuda.synchronize()
    launches = lib.launch_count()
    rc = h.nm_mha_tc_fwd(q, k, v, mask, 0, drop, out, probs, probs_drop, bsz, tq, tk, heads, dh, lib.stream())
    assert rc == NM_E_UNSUPPORTED, rc
    rc = h.nm_mha_tc_bwd(q, k, v, mask, 0, drop, probs, probs_drop, dout, dq, dk, dv, ds, bsz, tq, tk, heads, dh,
                         lib.stream())
    assert rc == NM_E_UNSUPPORTED, rc
    torch.cuda.synchronize()
    assert lib.launch_count() == launches
    for b, bits in zip(outs, before):
        assert torch.equal(b.bits(), bits)


def _offset_copy(t, offset):
    """t as a contiguous view that starts `offset` bytes past a 16-byte boundary."""
    buf = torch.empty(t.numel() + 4, device=t.device)
    view = buf[offset // 4:offset // 4 + t.numel()].view(t.shape)
    view.copy_(t)
    assert view.is_contiguous() and view.data_ptr() % 16 == offset
    return view


@pytest.mark.parametrize("use_drop", [False, True])
@pytest.mark.parametrize("offset", [4, 8])
def test_misaligned_inputs_through_mha_core(offset, use_drop):
    """q, k, v and the upstream gradient as contiguous views off the 16-byte boundary the tensor maps need: the same
    bits as the aligned call."""
    from neuralmonkey_b200 import ops
    shape = (2, 40, 37, 2, 64)
    bsz, tq, tk, heads, dh = shape
    assert ops._mha_on_tensor_cores(bsz, tq, tk, heads, dh)
    inp = _inputs(shape, "ragged", use_drop, seed=offset)
    results = []
    for place in (lambda t: t.clone(), lambda t: _offset_copy(t, offset)):
        q, k, v = (place(inp[n]).requires_grad_(True) for n in ("q", "k", "v"))
        out, weights = ops.mha_core(q, k, v, inp["mask"], False, heads, inp["drop"])
        out.backward(place(inp["dout"]))
        torch.cuda.synchronize()
        results.append((out.detach(), weights, q.grad, k.grad, v.grad))
    for n, a, b in zip(("context", "weights", "dq", "dk", "dv"), *results):
        assert torch.equal(a, b), n
