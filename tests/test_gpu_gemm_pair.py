"""CTA-pair tiles of the wgmma products (a cluster of two CTAs per 256 x BN tile, the B tile multicast to both).

A pair computes exactly the products and sums of the one-CTA instance (same operands, same K order), so
every family is run with `nm_gemm_set_pair_mode(0)` and `(1)` on the same inputs and compared bit for bit,
and the pair result is checked against fp64 on its own."""
import pytest
import torch

from tests.helpers import rel_err

pytestmark = pytest.mark.gpu


@pytest.fixture
def pair_switch():
    from neuralmonkey_b200 import lib

    def switch(mode):
        lib.call("nm_gemm_set_pair_mode", mode)
    yield switch
    lib.call("nm_gemm_set_pair_mode", -1)


def _operands(m, n, k, ta, tb, seed=0):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(k, m, generator=g) if ta else torch.randn(m, k, generator=g)
    b = torch.randn(n, k, generator=g) if tb else torch.randn(k, n, generator=g)
    return a, b


@pytest.mark.parametrize("ta", [False, True])
@pytest.mark.parametrize("tb", [False, True])
@pytest.mark.parametrize("shape", [(256, 128, 32), (512, 384, 96), (1000, 600, 300), (300, 1000, 1024),
                                   (257, 260, 36), (4096, 512, 512), (640, 2048, 200),
                                   (300, 600, 12800)])          # the last one: split-K inside pair tiles
def test_pair_gemm_equals_single_cta(pair_switch, ta, tb, shape):
    from neuralmonkey_b200 import lib, ops
    m, n, k = shape
    if (m % 4 and ta) or (n % 4 and not tb) or (k % 4 and (not ta or tb)):
        pytest.skip("operand rows not 16-byte multiples: not TMA-addressable")
    a, b = _operands(m, n, k, ta, tb)
    ad, bd = a.cuda(), b.cuda()
    outs = []
    for mode in (0, 1):
        pair_switch(mode)
        out = torch.full((m, n), float("nan"), device="cuda")
        ops.gemm(ad, bd, out, trans_a=ta, trans_b=tb, backend=lib.GEMM_TC)
        torch.cuda.synchronize()
        outs.append(out)
    ref = (a.double().t() if ta else a.double()) @ (b.double().t() if tb else b.double())
    assert torch.isfinite(outs[1]).all()
    assert rel_err(outs[1], ref) < 2e-3
    if k <= 512:                       # longer reductions may be cut (split-K: partial tiles meet in atomics,
        assert torch.equal(outs[0], outs[1]), float((outs[0] - outs[1]).abs().max())   # order-dependent rounding)
    else:
        assert rel_err(outs[1], outs[0].double()) < 1e-6


@pytest.mark.parametrize("act", [None, "tanh", "relu"])
def test_pair_gemm_epilogue(pair_switch, act):
    from neuralmonkey_b200 import lib, ops
    g = torch.Generator().manual_seed(5)
    m, n, k = 700, 520, 300
    a, b = torch.randn(m, k, generator=g).cuda(), (torch.randn(k, n, generator=g) * 0.1).cuda()
    bias = torch.randn(n, generator=g).cuda()
    c0 = torch.randn(m, n, generator=g).cuda()
    outs = []
    for mode in (0, 1):
        pair_switch(mode)
        out = c0.clone()
        ops.gemm(a, b, out, bias=bias, act=act, beta=1.0, backend=lib.GEMM_TC)
        torch.cuda.synchronize()
        outs.append(out)
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("m,n,k", [(300, 301, 1000), (1100, 300, 8200), (4100, 512, 520)])
@pytest.mark.parametrize("transposed", [0, 1])
def test_pair_gemm_f16(pair_switch, m, n, k, transposed):
    from neuralmonkey_b200 import lib
    g = torch.Generator().manual_seed(1)
    kp = (k + 7) // 8 * 8
    a = torch.full((m, kp), 9.0, dtype=torch.float16)
    b = torch.full((n, kp), 9.0, dtype=torch.float16)
    a[:, :k] = (torch.randn(m, k, generator=g) * 0.5).half()
    b[:, :k] = (torch.randn(n, k, generator=g) * 0.5).half()
    alpha_d = torch.tensor([0.37]).cuda()
    scale_d = (torch.rand(m, generator=g) + 0.5).cuda()
    ad, bd = a.cuda(), b.cuda()
    want = (a[:, :k].double() @ b[:, :k].double().t()) * 0.37 * scale_d.double().cpu()[:, None]
    want = want.t() if transposed else want
    outs = []
    for mode in (0, 1):
        pair_switch(mode)
        c = torch.zeros((n, m) if transposed else (m, n), device="cuda")
        lib.call("nm_gemm_f16", m, n, k, lib.ptr(ad), kp, lib.ptr(bd), kp, lib.ptr(c), c.stride(0),
                 lib.ptr(alpha_d), lib.ptr(scale_d), 0.0, transposed, lib.stream())
        torch.cuda.synchronize()
        outs.append(c)
    assert rel_err(outs[1], want) < 1e-5
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("m,n,k", [(301, 1000, 1100), (301, 4100, 12800), (512, 260, 72)])
def test_pair_gemm_f16_tn(pair_switch, m, n, k):
    from neuralmonkey_b200 import lib
    g = torch.Generator().manual_seed(3)
    mp, np_ = (m + 7) // 8 * 8, (n + 7) // 8 * 8
    a = torch.full((k, mp), 9.0, dtype=torch.float16)
    b = torch.full((k, np_), 9.0, dtype=torch.float16)
    a[:, :m] = (torch.randn(k, m, generator=g) * 0.5).half()
    b[:, :n] = (torch.randn(k, n, generator=g) * 0.5).half()
    want = 0.37 * (a[:, :m].double().t() @ b[:, :n].double())
    ad, bd, alpha_d = a.cuda(), b.cuda(), torch.tensor([0.37]).cuda()
    outs = []
    for mode in (0, 1):
        pair_switch(mode)
        c = torch.zeros(m, n, device="cuda")
        lib.call("nm_gemm_f16_tn", m, n, k, lib.ptr(ad), mp, lib.ptr(bd), np_, lib.ptr(c), c.stride(0),
                 lib.ptr(alpha_d), 0.0, lib.stream())
        torch.cuda.synchronize()
        outs.append(c)
    assert rel_err(outs[1], want) < 5e-5
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("xent16", ["0", "1"])
@pytest.mark.parametrize("m,k,v,unk", [(1100, 300, 4100, 3), (512, 64, 1000, -1)])
def test_pair_logits_xent(pair_switch, monkeypatch, xent16, m, k, v, unk):
    """Fused vocabulary projection + cross-entropy, forward and backward, TF32 and fp16 instances."""
    from neuralmonkey_b200 import ops
    monkeypatch.setenv("NMB200_XENT16", xent16)
    g = torch.Generator().manual_seed(2)
    x0 = (torch.randn(m, k, generator=g) * 0.7).cuda()
    flat = torch.zeros(k * v + v, device="cuda")
    grads = torch.zeros_like(flat)
    w, b = flat[:k * v].view(k, v), flat[k * v:]
    w.copy_((torch.randn(k, v, generator=g) * 0.1).cuda())
    b.copy_((torch.randn(v, generator=g) * 0.1).cuda())
    targets = torch.randint(4, v, (m,), generator=g).cuda()
    weights = (torch.rand(m, generator=g) > 0.2).float().cuda()
    results = []
    for mode in (0, 1):
        pair_switch(mode)
        grads.zero_()
        x = x0.clone().requires_grad_(True)
        wv, bv = w.detach().requires_grad_(True), b.detach().requires_grad_(True)
        wv.nm_grad, bv.nm_grad = grads[:k * v].view(k, v), grads[k * v:]
        xent, lse, argmax, logits = ops.logits_xent(x, wv, bv, targets, weights, unk, False, keep_logits=True)
        (xent.sum() / weights.sum()).backward()
        torch.cuda.synchronize()
        results.append((xent.detach().clone(), lse.clone(), argmax.clone(), logits.clone(), x.grad.clone(),
                        grads.clone()))
    one, two = results
    assert torch.isfinite(two[0]).all() and torch.isfinite(two[5]).all()
    assert torch.equal(one[2], two[2])                         # argmax
    assert torch.equal(one[3], two[3])                         # logits
    assert float((one[0] - two[0]).abs().max()) < 1e-5         # the per-tile partials are split differently
    assert float((one[1] - two[1]).abs().max()) < 1e-5
    assert rel_err(two[4], one[4].double()) < 1e-5
    assert rel_err(two[5], one[5].double()) < 1e-5
