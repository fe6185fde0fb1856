"""The persistent stream-K fp16 GEMM behind nm_gemm_f16 and nm_gemm_f16_tn (csrc/gemm16.cu) against fp64 products
of the fp16-rounded operands: the vocabulary-gradient shapes of the en-de bench, accumulation into a strided view of
a flat buffer, transposed stores with a row scale, ragged edges, tiles cut between CTAs and CTAs spanning tiles."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _lib():
    from neuralmonkey_b200 import lib
    return lib


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _pad8(n):
    return (n + 7) // 8 * 8


def _operand(rows, cols, ld, scale, g):
    """fp16 [rows, ld] on the GPU; the padding columns hold 9.0 so that reading them shows in the result."""
    t = torch.full((rows, ld), 9.0, device="cuda", dtype=torch.float16)
    t[:, :cols] = (torch.randn(rows, cols, device="cuda", generator=g) * scale).half()
    return t


def _gemm_f16(m, n, k, transposed, beta, row_scale=True, seed=1, a_scale=0.5):
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(seed)
    kp = _pad8(k)
    a, b = _operand(m, k, kp, a_scale, g), _operand(n, k, kp, 0.5, g)
    alpha = torch.tensor([0.37], device="cuda")
    scale = torch.rand(m, device="cuda", generator=g) + 0.5 if row_scale else None
    c0 = torch.randn(n, m, device="cuda", generator=g) if transposed else torch.randn(m, n, device="cuda", generator=g)
    want = (a[:, :k].double() @ b[:, :k].double().t()) * 0.37
    if scale is not None:
        want = want * scale.double()[:, None]
    want = (want.t() if transposed else want) + beta * c0.double()
    c = c0.clone()
    lib.call("nm_gemm_f16", m, n, k, lib.ptr(a), kp, lib.ptr(b), kp, lib.ptr(c), c.stride(0), lib.ptr(alpha),
             lib.ptr(scale) if scale is not None else None, beta, transposed, lib.stream())
    torch.cuda.synchronize()
    return _rel(c, want)


F16_SHAPES = [
    (12800, 300, 32000),     # dX of the bench step: 100 tiles of 500 k-blocks, every tile cut between CTAs
    (2048, 300, 32000),
    (1000, 300, 640),        # 80 k-blocks in all: one per CTA, every tile summed from ten pieces
    (38400, 300, 100),       # 600 k-blocks: a CTA's range spans two or three tiles, whole ones stored directly
    (333, 320, 517),         # a full 320-column tile, ragged rows and K
    (333, 321, 517),         # one column into a second column tile
    (40, 77, 1030),          # fewer rows than one warpgroup's 64
    (200, 600, 90),
]


@pytest.mark.parametrize("m,n,k", F16_SHAPES)
@pytest.mark.parametrize("transposed,beta", [(0, 0.0), (0, 1.0), (1, 0.0), (1, 1.0)])
def test_gemm_f16_persistent(m, n, k, transposed, beta):
    # fp32 accumulation: over 32000 products about 2e-5 here (4e-5 on the one-CTA-per-tile kernel this replaced)
    assert _gemm_f16(m, n, k, transposed, beta) < (1e-5 if k <= 8200 else 5e-5)


def test_gemm_f16_without_row_scale():
    assert _gemm_f16(700, 300, 3000, 0, 0.0, row_scale=False) < 1e-5


def _gemm_f16_tn(m, n, k, beta, seed=3, c_offset=0, b_scale=0.5):
    """C[M,N] (a strided view of a flat buffer from element c_offset) = 0.37 * A^T . B (+ C), A [K,M], B [K,N]."""
    lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(seed)
    a, b = _operand(k, m, _pad8(m), 0.5, g), _operand(k, n, _pad8(n), b_scale, g)
    flat = torch.randn(c_offset + m * n + 5, device="cuda", generator=g)
    c = torch.as_strided(flat, (m, n), (n, 1), c_offset)
    want = 0.37 * (a[:, :m].double().t() @ b[:, :n].double()) + beta * c.double()
    before, after = flat[:c_offset].clone(), flat[c_offset + m * n:].clone()
    alpha = torch.tensor([0.37], device="cuda")
    lib.call("nm_gemm_f16_tn", m, n, k, lib.ptr(a), a.stride(0), lib.ptr(b), b.stride(0), lib.ptr(c), n,
             lib.ptr(alpha), beta, lib.stream())
    torch.cuda.synchronize()
    assert torch.equal(flat[:c_offset], before) and torch.equal(flat[c_offset + m * n:], after)
    return _rel(c, want)


F16_TN_SHAPES = [
    (301, 32000, 12800, 3),    # [dW; db] of the bench step into the gradient buffer: C^T = B^T A, 250 x 200 k-blocks
    (301, 32000, 2048, 90000),
    (301, 4100, 640, 1),       # tiles cut between CTAs
    (64, 38400, 100, 0),       # CTAs spanning tiles
    (320, 1000, 517, 2),
    (321, 1000, 517, 0),
    (40, 260, 1030, 0),        # fewer than 64 of the smaller dimension
    (1000, 333, 300, 1),       # M > N: M down the rows, no transposed store
]


@pytest.mark.parametrize("m,n,k,c_offset", F16_TN_SHAPES)
@pytest.mark.parametrize("beta", [0.0, 1.0])
def test_gemm_f16_tn_persistent(m, n, k, c_offset, beta):
    assert _gemm_f16_tn(m, n, k, beta, c_offset=c_offset) < 5e-5


@pytest.mark.parametrize("ctas", [1, 5, 48])
def test_gemm_f16_tn_on_an_sm_budget(ctas):
    """nm_gemm_f16_tn_ctas: the same product on fewer persistent CTAs (longer ranges, other cuts)."""
    lib = _lib()
    m, n, k = 301, 4100, 1500
    g = torch.Generator(device="cuda").manual_seed(5)
    a, b = _operand(k, m, _pad8(m), 0.5, g), _operand(k, n, _pad8(n), 0.5, g)
    for beta in (0.0, 1.0):
        c0 = torch.randn(m, n, device="cuda", generator=g)
        want = 0.37 * (a[:, :m].double().t() @ b[:, :n].double()) + beta * c0.double()
        c, alpha = c0.clone(), torch.tensor([0.37], device="cuda")
        lib.call("nm_gemm_f16_tn_ctas", m, n, k, lib.ptr(a), a.stride(0), lib.ptr(b), b.stride(0), lib.ptr(c), n,
                 lib.ptr(alpha), beta, ctas, lib.stream())
        torch.cuda.synchronize()
        assert _rel(c, want) < 5e-5
