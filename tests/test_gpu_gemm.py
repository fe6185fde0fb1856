"""nm_gemm on the GPU: wgmma/TMA path and CUDA-core path against an fp64 product."""
import pytest
import torch

from tests.helpers import max_abs, rel_err

pytestmark = pytest.mark.gpu

# tf32 operands (10-bit mantissa, rounded), fp32 accumulate: |err| <= ~2^-10 * sum|a||b|
TC_REL = 2e-3
SIMT_REL = 2e-6


def _operands(m, n, k, ta, tb, seed=0):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(k, m, generator=g) if ta else torch.randn(m, k, generator=g)
    b = torch.randn(n, k, generator=g) if tb else torch.randn(k, n, generator=g)
    return a, b


def _ref(a, b, ta, tb):
    a64, b64 = a.double(), b.double()
    return (a64.t() if ta else a64) @ (b64.t() if tb else b64)


@pytest.mark.parametrize("ta", [False, True])
@pytest.mark.parametrize("tb", [False, True])
@pytest.mark.parametrize("shape", [(128, 128, 32), (256, 384, 96), (200, 300, 300), (1000, 600, 300),
                                   (12, 900, 1200), (300, 1000, 1024), (129, 257, 36),
                                   (256, 128, 32), (512, 384, 96), (257, 260, 36), (4096, 512, 512),
                                   (640, 2048, 200), (300, 600, 12800),
                                   (8192, 1024, 64),     # enough tiles for 256-wide ones
                                   (1100, 300, 8192)])   # skinny N, long K: 160-wide tiles (+ split-K)
def test_tc_gemm_matches_fp64(ta, tb, shape):
    from neuralmonkey_b200 import lib, ops
    m, n, k = shape
    if (m % 4 and ta) or (n % 4 and not tb) or (k % 4 and (not ta or tb)):
        pytest.skip("operand rows not 16-byte multiples: not TMA-addressable")
    a, b = _operands(m, n, k, ta, tb)
    ad, bd = a.cuda(), b.cuda()
    out = torch.full((m, n), float("nan"), device="cuda")
    ops.gemm(ad, bd, out, trans_a=ta, trans_b=tb, backend=lib.GEMM_TC)
    ref = _ref(a, b, ta, tb)
    assert torch.isfinite(out).all()
    assert rel_err(out, ref) < TC_REL, (rel_err(out, ref), max_abs(out, ref))


@pytest.mark.parametrize("ta", [False, True])
@pytest.mark.parametrize("tb", [False, True])
@pytest.mark.parametrize("shape", [(5, 7, 3), (16, 70, 9), (33, 65, 130), (200, 300, 300)])
def test_simt_gemm_matches_fp64(ta, tb, shape):
    from neuralmonkey_b200 import lib, ops
    m, n, k = shape
    a, b = _operands(m, n, k, ta, tb, seed=1)
    out = torch.empty(m, n, device="cuda")
    ops.gemm(a.cuda(), b.cuda(), out, trans_a=ta, trans_b=tb, backend=lib.GEMM_SIMT)
    assert rel_err(out, _ref(a, b, ta, tb)) < SIMT_REL


@pytest.mark.parametrize("backend_name", ["simt", "tc"])
@pytest.mark.parametrize("act", [None, "tanh", "relu"])
def test_gemm_epilogue_bias_act_beta(backend_name, act):
    from neuralmonkey_b200 import lib, ops
    backend = {"simt": lib.GEMM_SIMT, "tc": lib.GEMM_TC}[backend_name]
    m, n, k = 260, 132, 64
    a, b = _operands(m, n, k, False, False, seed=2)
    bias = torch.randn(n)
    c0 = torch.randn(m, n)
    out = c0.clone().cuda()
    ops.gemm(a.cuda(), b.cuda(), out, bias=bias.cuda(), act=act, beta=1.0, backend=backend)
    pre = a.double() @ b.double() + bias.double()
    if act == "tanh":
        pre = torch.tanh(pre)
    elif act == "relu":
        pre = torch.relu(pre)
    ref = pre + c0.double()
    tol = 5e-3 if backend_name == "tc" else 1e-5
    assert max_abs(out, ref) < tol * max(1.0, float(ref.abs().max()))


def test_gemm_strided_views():
    """Column slices of wider buffers (ld > cols) as the GRU input projection uses them."""
    from neuralmonkey_b200 import lib, ops
    m, k, h = 96, 64, 32
    x = torch.randn(m, k)
    w = torch.randn(k + h, 2 * h)
    buf = torch.zeros(m, 3 * h, device="cuda")
    for backend in (lib.GEMM_SIMT, lib.GEMM_TC):
        buf.zero_()
        ops.gemm(x.cuda(), w.cuda()[:k], buf[:, :2 * h], backend=backend)
        ref = x.double() @ w[:k].double()
        assert rel_err(buf[:, :2 * h], ref) < TC_REL
        assert float(buf[:, 2 * h:].abs().max()) == 0.0


def test_tc_rounding_mode_report(capsys):
    """Not an assertion about the hardware: records whether TMA/MMA rounds or truncates fp32
    to tf32 (a truncating path biases products low by ~2^-11 and would show as a mean
    signed error)."""
    from neuralmonkey_b200 import lib, ops
    m, n, k = 512, 512, 512
    g = torch.Generator().manual_seed(3)
    a = torch.rand(m, k, generator=g) + 0.5
    b = torch.rand(k, n, generator=g) + 0.5
    out = torch.empty(m, n, device="cuda")
    ops.gemm(a.cuda(), b.cuda(), out, backend=lib.GEMM_TC)
    ref = a.double() @ b.double()
    signed = float(((out.double().cpu() - ref) / ref).mean())
    with capsys.disabled():
        print("\n[tf32 path] mean signed relative error = {:.3e} (|.| << 2.4e-4 means rounding)"
              .format(signed))
    assert abs(signed) < 1e-3


@pytest.mark.parametrize("beta", [0.0, 1.0])
def test_tc_gemm_split_k_weight_gradient_shape(beta):
    """Tiny output, long reduction: the kernel splits K over the SMs and adds partial tiles."""
    from neuralmonkey_b200 import lib, ops
    m, n, k = 300, 600, 12800
    a, b = _operands(m, n, k, True, False, seed=5)
    bias = torch.randn(n)
    c0 = torch.randn(m, n)
    out = c0.clone().cuda()
    ops.gemm(a.cuda(), b.cuda(), out, trans_a=True, bias=bias.cuda(), beta=beta, backend=lib.GEMM_TC)
    ref = a.double().t() @ b.double() + bias.double() + beta * c0.double()
    assert rel_err(out, ref) < TC_REL
