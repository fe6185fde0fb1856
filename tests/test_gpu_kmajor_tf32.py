"""K-major TF32 copies of MN-major GEMM operands (nm_transpose_tf32, ops.kmajor_tf32, and ops.gemm handing them to
the wgmma kernel): the copy is the transpose rounded exactly as cvt.rna.tf32 rounds, the products through the copies
equal the products that read the MN-major operands as stored, and the exact engine never sees a rounded operand."""
import pytest
import torch

from tests.helpers import rel_err

pytestmark = pytest.mark.gpu

SIMT_REL = 2e-6


def _tf32_rna_bits(x: torch.Tensor) -> torch.Tensor:
    """cvt.rna.tf32.f32 on the bit pattern: round half away from zero at mantissa bit 13, clear the low 13 bits."""
    bits = x.contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    return (bits + 0x1000) & 0xFFFFE000


def _bits(x: torch.Tensor) -> torch.Tensor:
    return x.contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF


# (rows, cols, source pitch, first column of the slice, destination pitch or None = rows rounded up to 4)
TRANSPOSE_CASES = [
    (5, 7, 7, 0, None), (67, 33, 41, 3, None), (130, 300, 300, 0, 136), (257, 96, 97, 1, None),
    (1000, 600, 900, 0, None), (1000, 300, 900, 600, None), (64, 64, 64, 0, None), (63, 65, 72, 4, 72),
]


@pytest.mark.parametrize("rows,cols,ld_src,col0,ld_dst", TRANSPOSE_CASES)
def test_transpose_tf32_is_rounded_transpose(rows, cols, ld_src, col0, ld_dst):
    from neuralmonkey_b200 import lib
    g = torch.Generator().manual_seed(rows * 7 + cols)
    base = torch.randn(rows, ld_src, generator=g) * 3.0
    # exact ties of the rounding (bit 12 set, bits 0-11 clear), both signs, and zeros
    base[0, :min(4, ld_src)] = torch.tensor([1.0 + 2.0 ** -11, -(1.0 + 2.0 ** -11), 0.0, -0.0])[:min(4, ld_src)]
    src = base.cuda()[:, col0:col0 + cols]
    ld_dst = ld_dst or (rows + 3) // 4 * 4
    dst = torch.full((cols, ld_dst), float("nan"), device="cuda")
    lib.call("nm_transpose_tf32", lib.ptr(src), src.stride(0), lib.ptr(dst), ld_dst, rows, cols, lib.stream())
    torch.cuda.synchronize()
    want = _tf32_rna_bits(base[:, col0:col0 + cols].t())
    assert torch.equal(_bits(dst[:, :rows].cpu()), want)
    if ld_dst > rows:
        assert torch.isnan(dst[:, rows:]).all(), "the padding columns are not written"


def test_kmajor_tf32_view():
    from neuralmonkey_b200 import ops
    x = torch.randn(301, 70, device="cuda")
    xt = ops.kmajor_tf32(x[:, 3:53])
    assert xt.shape == (50, 301) and xt.stride() == (304, 1) and xt.data_ptr() % 16 == 0
    assert torch.equal(_bits(xt.cpu()), _tf32_rna_bits(x[:, 3:53].t().cpu()))


def _direct(a, b, out, ta, tb, bias=None, act=None, beta=0.0):
    """nm_gemm on the operands exactly as stored: MN-major operands are read and transposed by the kernel's
    producer threads."""
    from neuralmonkey_b200 import lib
    m, n = out.shape
    k = a.size(0) if ta else a.size(1)
    lib.call("nm_gemm", int(ta), int(tb), m, n, k, lib.ptr(a), a.stride(0), lib.ptr(b), b.stride(0), lib.ptr(out),
             out.stride(0), lib.ptr(bias), lib.NM_ACT[act], float(beta), lib.GEMM_AUTO, lib.stream())
    return out


def _operands(m, n, k, ta, tb, seed):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(k, m, generator=g) if ta else torch.randn(m, k, generator=g)
    b = torch.randn(n, k, generator=g) if tb else torch.randn(k, n, generator=g)
    return a.cuda(), b.cuda()


# products that are not cut into split-K slices: one CTA sums a whole reduction in a fixed order
@pytest.mark.parametrize("ta,tb,m,n,k", [
    (True, False, 300, 600, 480), (True, False, 1000, 1200, 2000), (True, True, 600, 300, 448),
    (False, False, 12800, 600, 300), (False, False, 4096, 2048, 512), (False, False, 200, 900, 1200),
])
@pytest.mark.parametrize("beta", [0.0, 1.0])
def test_gemm_through_kmajor_copies_is_bit_identical(ta, tb, m, n, k, beta):
    from neuralmonkey_b200 import ops
    a, b = _operands(m, n, k, ta, tb, seed=m + n + k)
    bias = torch.randn(n, device="cuda")
    c0 = torch.randn(m, n, device="cuda") if beta else torch.full((m, n), float("nan"), device="cuda")
    act = None if ta else "tanh"
    got = ops.gemm(a, b, c0.clone(), ta, tb, bias=bias, act=act, beta=beta)
    want = _direct(a, b, c0.clone(), ta, tb, bias=bias, act=act, beta=beta)
    torch.cuda.synchronize()
    assert torch.isfinite(got).all()
    assert torch.equal(got, want), float((got - want).abs().max())


def test_gemm_column_slices_bit_identical():
    """The GRU's operands: a row range of a kernel as B of the input projection, column slices of dxproj (pitch 3H)
    as B of the weight-gradient products."""
    from neuralmonkey_b200 import ops
    g = torch.Generator().manual_seed(9)
    bt, e, h = 448, 300, 300          # a reduction of 14 k-blocks: not cut into split-K slices
    x = torch.randn(bt, e, generator=g).cuda()
    w = torch.randn(e + h, 2 * h, generator=g).cuda()
    got = torch.zeros(bt, 3 * h, device="cuda")
    want = torch.zeros(bt, 3 * h, device="cuda")
    ops.gemm(x, w[:e], got[:, :2 * h])
    _direct(x, w[:e], want[:, :2 * h], False, False)
    torch.cuda.synchronize()
    assert torch.equal(got, want)
    dxp = torch.randn(bt, 3 * h, generator=g).cuda()
    for dz, cols in ((dxp[:, :2 * h], 2 * h), (dxp[:, 2 * h:], h)):
        got = ops.gemm(x, dz, torch.empty(e, cols, device="cuda"), trans_a=True)
        want = _direct(x, dz, torch.empty(e, cols, device="cuda"), True, False)
        torch.cuda.synchronize()
        assert torch.equal(got, want)


@pytest.mark.parametrize("beta", [0.0, 1.0])
def test_gemm_split_k_weight_gradient_within_reorder_noise(beta):
    """300 x 600 x 12800 (a weight gradient of the en-de GRU): the reduction is cut into slices that meet in
    atomic adds, whose order varies from run to run."""
    from neuralmonkey_b200 import ops
    m, n, k = 300, 600, 12800
    a, b = _operands(m, n, k, True, False, seed=5)
    c0 = torch.randn(m, n, device="cuda") * beta
    got = ops.gemm(a, b, c0.clone(), trans_a=True, beta=beta)
    want = _direct(a, b, c0.clone(), True, False, beta=beta)
    ref = a.double().t() @ b.double() + c0.double()
    torch.cuda.synchronize()
    assert rel_err(got, want.double()) < 1e-6
    assert rel_err(got, ref) < 2e-3


@pytest.mark.parametrize("ta,tb", [(True, False), (False, False), (True, True)])
def test_simt_backend_reads_operands_as_given(ta, tb):
    """The exact engine: no rounded copy is made (one launch per product) and the result meets the fp32 bar."""
    from neuralmonkey_b200 import lib, ops
    m, n, k = 200, 300, 320
    a, b = _operands(m, n, k, ta, tb, seed=4)
    ref = (a.double().t() if ta else a.double()) @ (b.double().t() if tb else b.double())
    ops.set_gemm_backend("simt")
    try:
        launches = lib.launch_count()
        out = ops.gemm(a, b, torch.empty(m, n, device="cuda"), ta, tb)
        torch.cuda.synchronize()
        assert lib.launch_count() - launches == 1
    finally:
        ops.set_gemm_backend("auto")
    assert rel_err(out, ref) < SIMT_REL


def test_misaligned_operand_keeps_the_cuda_core_path():
    """An MN-major operand that TMA cannot address (a base that is not 16-byte aligned) sends the product to the
    CUDA cores, which read it as stored: no copy is made."""
    from neuralmonkey_b200 import lib, ops
    m, n, k = 64, 96, 128
    g = torch.Generator().manual_seed(6)
    a = torch.randn(k, m + 4, generator=g).cuda()[:, 1:m + 1]      # pitch 68 floats, base 4 bytes past 16
    b = torch.randn(k, n, generator=g).cuda()
    launches = lib.launch_count()
    out = ops.gemm(a, b, torch.empty(m, n, device="cuda"), trans_a=True)
    torch.cuda.synchronize()
    assert lib.launch_count() - launches == 1
    assert rel_err(out, a.double().t() @ b.double()) < SIMT_REL
