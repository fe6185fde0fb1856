"""nm_bahdanau_fwd / nm_bahdanau_bwd (through ops.bahdanau_attention) against fp64 autograd on the device, at the
tolerances of test_gpu_ops.test_bahdanau_fwd_bwd: weights 1e-5 and contexts 5e-5 absolute, gradients 1e-4
relative.  Covers the en-de training shape, query counts around the chunk and register-chunk boundaries, long
and single-key sentences, odd attention and value widths, and the two-SFU tanh the kernels fall back to when a
sentence's keys or queries leave the range of the factorised form."""
import pytest
import torch

from tests.helpers import max_abs, rel_err

pytestmark = pytest.mark.gpu

# (B, Tx, NQ, A, C)
SHAPES = ([(256, 50, 50, 600, 600)]                                          # en-de training step
          + [(40, 33, nq, 14, 10) for nq in (1, 7, 8, 50, 51, 65)]
          + [(264, 9, 5, 10, 14), (264, 9, 13, 14, 10)]                     # one and two query chunks per sentence
          + [(3, tx, 9, 601, 600) for tx in (1, 33, 196)]
          + [(5, 20, 13, a, c) for a, c in ((10, 601), (14, 14), (600, 10), (601, 601))])


def _inputs(dims, use_mask, seed):
    bsz, tx, nq, a, c = dims
    g = torch.Generator().manual_seed(seed)
    keys, values = torch.randn(bsz, tx, a, generator=g), torch.randn(bsz, tx, c, generator=g)
    q = torch.randn(bsz, nq, a, generator=g)
    v, bias = torch.randn(a, generator=g) * 0.3, torch.randn(1, generator=g)
    mask = None
    if use_mask:
        lens = torch.randint(1, tx + 1, (bsz,), generator=g)
        lens[0] = tx
        mask = (torch.arange(tx).unsqueeze(0) < lens.unsqueeze(1)).float()
    dctx = torch.randn(bsz, nq, c, generator=g)
    return keys, values, mask, q, v, bias, dctx


def _reference(keys, values, mask, q, v, bias, dctx, chunk=16):
    """fp64 on the device, a few sentences at a time (the en-de tanh tensor alone is 3 GB in fp64)."""
    v64 = v.cuda().double().requires_grad_(True)
    b64 = bias.cuda().double().requires_grad_(True)
    out = {n: [] for n in ("w", "ctx", "keys", "values", "q")}
    for s in range(0, keys.shape[0], chunk):
        k64, val64, q64 = (t[s:s + chunk].cuda().double().requires_grad_(True) for t in (keys, values, q))
        e = (v64 * torch.tanh(k64.unsqueeze(1) + q64.unsqueeze(2))).sum(-1) + b64
        w = torch.softmax(e, -1)
        if mask is not None:
            w = w * mask[s:s + chunk].cuda().double().unsqueeze(1)
            w = w / (w.sum(-1, keepdim=True) + 1e-8)
        ctx = w @ val64
        (ctx * dctx[s:s + chunk].cuda().double()).sum().backward()
        for n, t in (("w", w.detach()), ("ctx", ctx.detach()), ("keys", k64.grad), ("values", val64.grad),
                     ("q", q64.grad)):
            out[n].append(t)
    out = {n: torch.cat(t) for n, t in out.items()}
    out["v"], out["bias"] = v64.grad, b64.grad
    return out


def _run(keys, values, mask, q, v, bias, dctx):
    from neuralmonkey_b200 import ops
    leaves = [t.clone().cuda().requires_grad_(True) for t in (keys, values, q, v, bias)]
    ctx, w = ops.bahdanau_attention(leaves[0], leaves[1], mask.cuda() if mask is not None else None,
                                    leaves[2], leaves[3], leaves[4])
    (ctx * dctx.cuda()).sum().backward()
    got = {"w": w.detach(), "ctx": ctx.detach()}
    got.update({n: t.grad for n, t in zip(("keys", "values", "q", "v", "bias"), leaves)})
    return got


def _check(got, ref):
    assert torch.isfinite(got["w"]).all() and torch.isfinite(got["ctx"]).all()
    assert max_abs(got["w"], ref["w"]) < 1e-5
    assert max_abs(got["ctx"], ref["ctx"]) < 5e-5
    for name in ("keys", "values", "q", "v"):
        assert torch.isfinite(got[name]).all(), name
        assert rel_err(got[name], ref[name]) < 1e-4, name
    # softmax is shift invariant: the scalar bias has (mathematically) zero gradient.  It is a sum of B*NQ rows
    # that each vanish, so its fp32 rounding grows like the square root of the row count.
    rows = got["w"].shape[0] * got["w"].shape[1]
    assert abs(float(got["bias"]) - float(ref["bias"])) < 1e-4 * max(1.0, (rows / 16) ** 0.5)


@pytest.mark.parametrize("use_mask", [True, False])
@pytest.mark.parametrize("dims", SHAPES)
def test_bahdanau_against_fp64(dims, use_mask):
    args = _inputs(dims, use_mask, seed=11)
    _check(_run(*args), _reference(*args))


@pytest.mark.parametrize("use_mask", [True, False])
def test_bahdanau_out_of_range_sentences(use_mask):
    """Keys and queries beyond +-40 in single sentences: there e^{2k} e^{2q} would be inf * 0, so those sentences
    take the two-SFU tanh; their neighbours keep the factorised form.  Sentence 1 has k = 50 meeting
    q = -49.5 (tanh(0.5), not saturated), sentence 4 a query of -45, sentence 6 a key of -41."""
    keys, values, mask, q, v, bias, dctx = _inputs((8, 33, 12, 600, 64), use_mask, seed=12)
    keys[1, 3, 5], q[1, 2, 5] = 50.0, -49.5
    q[4, 7, 100] = -45.0
    keys[6, 0, 599] = -41.0
    got, ref = _run(keys, values, mask, q, v, bias, dctx), _reference(keys, values, mask, q, v, bias, dctx)
    _check(got, ref)
    for b in range(8):              # every sentence on its own, the fast-form neighbours included
        assert max_abs(got["w"][b], ref["w"][b]) < 1e-5, b
        assert max_abs(got["ctx"][b], ref["ctx"][b]) < 5e-5, b
        for name in ("keys", "q"):
            assert rel_err(got[name][b], ref[name][b]) < 1e-4, (name, b)


def test_bahdanau_repeat_calls():
    """Every output is bit-identical across calls except dv and dbias, which are summed over sentences with
    atomic adds in whatever order the CTAs finish: they agree to 1e-6 relative."""
    args = _inputs((64, 50, 50, 600, 600), True, seed=13)
    first, second = _run(*args), _run(*args)
    for name in ("w", "ctx", "keys", "values", "q"):
        assert torch.equal(first[name], second[name]), name
    assert rel_err(first["v"], second["v"]) < 1e-6
    assert abs(float(first["bias"]) - float(second["bias"])) < 1e-6
