"""The fp16-operand vocabulary projection (csrc/xent16.cu, ops._LogitsXent16: the default on the
tensor-core engine) against fp64 references and against the TF32 path (ops._LogitsXent)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _lib():
    from neuralmonkey_b200 import lib
    return lib


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


@pytest.mark.parametrize("rows,cols", [(5, 7), (130, 300), (257, 96)])
def test_cast_f16(rows, cols):
    lib = _lib()
    g = torch.Generator().manual_seed(0)
    src = torch.randn(rows, cols + 3, generator=g).cuda()[:, :cols]
    scale = (torch.rand(rows, generator=g) + 0.5).cuda()
    ld = (cols + 7) // 8 * 8
    dst = torch.full((rows, ld), 7.0, device="cuda", dtype=torch.float16)
    lib.call("nm_cast_f16", lib.ptr(src), src.stride(0), lib.ptr(dst), ld, rows, cols, lib.ptr(scale), 0, 0,
             lib.stream())
    want = (src * scale[:, None]).half()
    assert torch.equal(dst[:, :cols], want) and float(dst[:, cols:].abs().max() if ld > cols else 0) == 0.0
    ld1 = (cols + 1 + 7) // 8 * 8                     # with the scaled column of ones behind the data
    dst1 = torch.full((rows, ld1), 7.0, device="cuda", dtype=torch.float16)
    lib.call("nm_cast_f16", lib.ptr(src), src.stride(0), lib.ptr(dst1), ld1, rows, cols, lib.ptr(scale), 0, 1,
             lib.stream())
    assert torch.equal(dst1[:, :cols], want) and torch.equal(dst1[:, cols], scale.half())
    assert ld1 == cols + 1 or float(dst1[:, cols + 1:].abs().max()) == 0.0
    ldt = (rows + 7) // 8 * 8
    dst_t = torch.full((cols + 1, ldt), 7.0, device="cuda", dtype=torch.float16)
    lib.call("nm_cast_f16", lib.ptr(src), src.stride(0), lib.ptr(dst_t), ldt, rows, cols, lib.ptr(scale), 1, 1,
             lib.stream())
    assert torch.equal(dst_t[:cols, :rows], want.t())
    assert torch.equal(dst_t[cols, :rows], scale.half())
    if ldt > rows:
        assert float(dst_t[:, rows:].abs().max()) == 0.0


@pytest.mark.parametrize("m,n,k", [(128, 64, 64), (300, 301, 1000), (1100, 300, 8200), (4100, 160, 520)])
@pytest.mark.parametrize("transposed,beta", [(0, 0.0), (0, 1.0), (1, 0.0), (1, 1.0)])
def test_gemm_f16(m, n, k, transposed, beta):
    lib = _lib()
    g = torch.Generator().manual_seed(1)
    kp = (k + 7) // 8 * 8
    a = torch.zeros(m, kp, dtype=torch.float16)
    b = torch.zeros(n, kp, dtype=torch.float16)
    a[:, :k] = (torch.randn(m, k, generator=g) * 0.5).half()
    b[:, :k] = (torch.randn(n, k, generator=g) * 0.5).half()
    a[:, k:], b[:, k:] = 9.0, 9.0                      # padding must never be read (TMA bounds = K)
    alpha = torch.tensor([0.37])
    row_scale = torch.rand(m, generator=g) + 0.5
    c0 = torch.randn(n, m, generator=g) if transposed else torch.randn(m, n, generator=g)
    want = (a[:, :k].double() @ b[:, :k].double().t()) * 0.37 * row_scale.double()[:, None]
    want = (want.t() if transposed else want) + beta * c0.double()
    c = c0.clone().cuda()
    ad, bd = a.cuda(), b.cuda()
    alpha_d, scale_d = alpha.cuda(), row_scale.cuda()      # kept alive: the call only sees raw pointers
    lib.call("nm_gemm_f16", m, n, k, lib.ptr(ad), kp, lib.ptr(bd), kp, lib.ptr(c), c.stride(0),
             lib.ptr(alpha_d), lib.ptr(scale_d), beta, transposed, lib.stream())
    torch.cuda.synchronize()
    assert _rel(c, want) < 1e-5


@pytest.mark.parametrize("m,n,k", [(64, 64, 64), (301, 1000, 1100), (301, 4100, 12800), (130, 96, 72), (40, 260, 8200)])
@pytest.mark.parametrize("beta", [0.0, 1.0])
def test_gemm_f16_tn(m, n, k, beta):
    """C[M,N] = alpha * A^T . B with A [K,M], B [K,N] stored reduction-major (MN-major operands)."""
    lib = _lib()
    g = torch.Generator().manual_seed(3)
    mp, np_ = (m + 7) // 8 * 8, (n + 7) // 8 * 8
    a = torch.full((k, mp), 9.0, dtype=torch.float16)       # padding columns must never be read
    b = torch.full((k, np_), 9.0, dtype=torch.float16)
    a[:, :m] = (torch.randn(k, m, generator=g) * 0.5).half()
    b[:, :n] = (torch.randn(k, n, generator=g) * 0.5).half()
    c0 = torch.randn(m, n, generator=g)
    want = 0.37 * (a[:, :m].double().t() @ b[:, :n].double()) + beta * c0.double()
    c = c0.clone().cuda()
    ad, bd, alpha_d = a.cuda(), b.cuda(), torch.tensor([0.37]).cuda()
    lib.call("nm_gemm_f16_tn", m, n, k, lib.ptr(ad), mp, lib.ptr(bd), np_, lib.ptr(c), c.stride(0),
             lib.ptr(alpha_d), beta, lib.stream())
    torch.cuda.synchronize()
    assert _rel(c, want) < 5e-5       # fp32 accumulation over up to 12800 products


@pytest.mark.parametrize("m,k,v,unk", [(96, 24, 200, 3), (1100, 300, 4100, -1)])
def test_logits_xent16_matches_the_tf32_path(m, k, v, unk):
    from neuralmonkey_b200 import ops
    g = torch.Generator().manual_seed(2)
    x0 = (torch.randn(m, k, generator=g) * 0.7).cuda()
    flat = torch.zeros(k * v + v, device="cuda")           # weight segment, then the bias segment
    grads = torch.zeros_like(flat)
    w = flat[:k * v].view(k, v)
    b = flat[k * v:]
    w.copy_((torch.randn(k, v, generator=g) * 0.1).cuda())
    b.copy_((torch.randn(v, generator=g) * 0.1).cuda())
    targets = torch.randint(4, v, (m,), generator=g).cuda()
    weights = (torch.rand(m, generator=g) > 0.2).float().cuda()
    results = {}
    for mode in ("0", "1"):
        grads.zero_()
        x = x0.clone().requires_grad_(True)
        wv, bv = w.detach().requires_grad_(True), b.detach().requires_grad_(True)
        wv.nm_grad, bv.nm_grad = grads[:k * v].view(k, v), grads[k * v:]
        if mode == "0":     # every product in TF32
            xent, lse, argmax, logits = ops._LogitsXent.apply(x, wv, bv, targets, weights, unk, False, True)
        else:               # ops.logits_xent's choice for these inputs: fp16 operands
            xent, lse, argmax, logits = ops.logits_xent(x, wv, bv, targets, weights, unk, False, keep_logits=True)
        (xent.sum() / weights.sum()).backward()
        results[mode] = (xent.detach().clone(), lse.clone(), argmax.clone(), logits.clone(), x.grad.clone(),
                         grads.clone())
    base, new = results["0"], results["1"]
    assert float((new[0] - base[0]).abs().max()) < 2e-2
    assert float((new[1] - base[1]).abs().max()) < 2e-2
    assert float((new[2] == base[2]).float().mean()) > 0.99          # argmax flips only on near-ties
    assert _rel(new[4], base[4]) < 5e-3                              # dX
    assert _rel(new[5][:k * v], base[5][:k * v]) < 5e-3              # dW
    assert _rel(new[5][k * v:], base[5][k * v:]) < 5e-3              # db
    # and both against fp64
    xd, wd, bd = x0.double().cpu().requires_grad_(True), w.double().cpu().requires_grad_(True), b.double().cpu().requires_grad_(True)
    lg = xd @ wd + bd
    if unk >= 0:
        pen = torch.zeros(v, dtype=torch.float64)
        pen[unk] = -1e9
        lg = lg + pen
    loss = ((torch.logsumexp(lg, -1) - lg.gather(1, targets.cpu()[:, None])[:, 0]) * weights.double().cpu()).sum() / weights.double().cpu().sum()
    loss.backward()
    assert _rel(new[4], xd.grad) < 3e-3 and _rel(new[5][:k * v].view(k, v), wd.grad) < 3e-3
    assert _rel(new[5][k * v:], bd.grad) < 3e-3
