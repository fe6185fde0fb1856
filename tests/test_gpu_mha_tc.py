"""K8 on the tensor cores (csrc/mha_tc.cu): attention as batched wgmma products with the softmax and its
backward in the GEMM epilogues, against an fp64 restatement of attention/scaled_dot_product.py:160-214 (masking
order, -1e9 replacement, dropout on the weights) and against the exact fp32 kernels.  TF32 operands: 10-bit
mantissas, so the bar is relative 3e-3 / 5e-3 on outputs / gradients and 2e-3 absolute on the probabilities."""
import pytest
import torch

from tests.helpers import max_abs, rel_err

pytestmark = pytest.mark.gpu

# (bsz, tq, tk, heads, dh): ragged times (padding rows / columns of the [Tq, Tk] matrices), cross-attention,
# two query tiles, the bench shape, the widest head
SHAPES = [(3, 50, 37, 4, 32), (2, 64, 64, 8, 64), (2, 8, 128, 2, 64), (3, 130, 96, 2, 32), (2, 33, 40, 1, 128)]


def _reference(q, k, v, mask, causal, heads, drop):
    bsz, tq, d = q.shape
    tk, dh = k.shape[1], d // heads

    def split(t):
        return t.view(bsz, -1, heads, dh).transpose(1, 2)
    e = split(q) @ split(k).transpose(-1, -2) / (dh ** 0.5)
    if causal:
        tri = torch.tril(torch.ones(tq, tk, dtype=torch.bool))
        e = torch.where(tri, e, torch.full_like(e, -1e9))
    if mask is not None:
        m4 = mask.double().view(bsz, 1, 1, tk)
        e = e * m4 + (1 - m4) * -1e9
    p = torch.softmax(e, -1)
    pd = p if drop is None else p * drop.double()
    return (pd @ split(v)).transpose(1, 2).reshape(bsz, tq, d), p


@pytest.mark.parametrize("use_drop", [False, True])
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("use_mask", [False, True])
@pytest.mark.parametrize("shape", SHAPES)
def test_tensor_core_attention(monkeypatch, shape, use_mask, causal, use_drop):
    from neuralmonkey_b200 import lib, ops
    monkeypatch.setenv("NMB200_MHA_TC", "1")
    bsz, tq, tk, heads, dh = shape
    if causal:
        tk = tq
        if tk > 128:
            pytest.skip("more than 128 keys: served by the CUDA-core kernels")
    assert lib.load().nm_mha_tc_supported(bsz, tq, tk, heads, dh) == 1
    g = torch.Generator().manual_seed(8)
    q, k, v = (torch.randn(bsz, t, heads * dh, generator=g) for t in (tq, tk, tk))
    mask = None
    if use_mask:
        lens = torch.tensor([tk, 3, 1][:bsz])
        mask = (torch.arange(tk).unsqueeze(0) < lens.unsqueeze(1)).float()
    drop = None
    if use_drop:
        drop = (torch.rand(bsz, heads, tq, tk, generator=g) < 0.7).float() / 0.7
    do = torch.randn(bsz, tq, heads * dh, generator=g)
    results = {}
    for engine in ("auto", "simt"):
        ops.set_gemm_backend(engine)
        try:
            qd, kd, vd = (t.clone().cuda().requires_grad_(True) for t in (q, k, v))
            out, probs = ops.mha_core(qd, kd, vd, mask.cuda() if use_mask else None, causal, heads,
                                      drop.cuda() if use_drop else None)
            (out * do.cuda()).sum().backward()
            torch.cuda.synchronize()
            results[engine] = (out.detach().cpu(), probs.detach().cpu().clone(), qd.grad.cpu(), kd.grad.cpu(),
                               vd.grad.cpu())
        finally:
            ops.set_gemm_backend("auto")
    q64, k64, v64 = (t.double().requires_grad_(True) for t in (q, k, v))
    ref, p = _reference(q64, k64, v64, mask, causal, heads, drop)
    (ref * do.double()).sum().backward()
    tc, exact = results["auto"], results["simt"]
    assert tc[1].shape == (bsz, heads, tq, tk)
    assert all(torch.isfinite(t).all() for t in tc)
    assert max_abs(tc[1], p) < 2e-3, "probabilities"
    assert max_abs(exact[1], p) < 1e-5
    assert rel_err(tc[0], ref) < 3e-3, "context"
    for name, got, want in (("dq", tc[2], q64.grad), ("dk", tc[3], k64.grad), ("dv", tc[4], v64.grad)):
        assert rel_err(got, want) < 5e-3, name
    # rows whose keys are all masked (softmax over -1e9 everywhere) stay uniform, as in the reference
    assert abs(float(tc[1].sum(-1).mean()) - 1.0) < 1e-4


def test_padding_of_the_weight_matrices_is_zero(monkeypatch):
    """The [Tq32, Tk32] storage behind the returned weights: the padding must be zeros (the backward products
    reduce over whole 32-element blocks of it)."""
    from neuralmonkey_b200 import ops
    monkeypatch.setenv("NMB200_MHA_TC", "1")
    g = torch.Generator().manual_seed(1)
    q, k, v = (torch.randn(2, t, 64, generator=g).cuda() for t in (37, 50, 50))
    _out, weights = ops.mha_core(q, k, v, None, False, 2)
    base = weights._base if weights._base is not None else weights
    assert base.shape == (2, 2, 64, 64)
    assert float(base[:, :, 37:, :].abs().max()) == 0.0 and float(base[:, :, :, 50:].abs().max()) == 0.0
    assert abs(float(base[:, :, :37, :50].sum(-1).mean()) - 1.0) < 1e-5
