"""nm_logits_xent_fwd16 / nm_logits_xent_bwd16 called directly, against fp64 computed from the fp16-rounded operands:
ragged M and V, the persistent kernel (K <= 320) and the generic-GEMM instances (longer K), exact argmax ties, targets in the last
partial column tile, masked rows, and run-to-run bit identity."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _lib():
    from neuralmonkey_b200 import lib
    return lib


class Problem:
    def __init__(self, m, v, k, unk, seed=0, wt=None, x=None):
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.m, self.v, self.k, self.unk = m, v, k, unk
        self.kpad, self.vpad = (k + 7) // 8 * 8, (v + 7) // 8 * 8
        self.x16 = torch.full((m, self.kpad), 9.0, device="cuda", dtype=torch.float16)   # padding never read
        self.wt16 = torch.full((v, self.kpad), 9.0, device="cuda", dtype=torch.float16)
        self.x16[:, :k] = (torch.randn(m, k, device="cuda", generator=g) * 0.7).half() if x is None else x
        self.wt16[:, :k] = (torch.randn(v, k, device="cuda", generator=g) * 0.2).half() if wt is None else wt
        self.b = torch.randn(v, device="cuda", generator=g) * 0.1
        self.targets = torch.randint(4, v, (m,), device="cuda", generator=g)   # never <unk> (3)
        self.targets[-1] = v - 1                                  # a target in the last, partial column tile
        self.mask = (torch.rand(m, device="cuda", generator=g) > 0.25).float()

    def reference(self):
        lg = self.x16[:, :self.k].double() @ self.wt16[:, :self.k].double().t() + self.b.double()
        if self.unk >= 0:
            lg[:, self.unk] += -1e9
        return lg

    def fwd(self, keep_logits=True):
        lib = _lib()
        m, v = self.m, self.v
        lse, xent = torch.empty(m, device="cuda"), torch.empty(m, device="cuda")
        argmax = torch.empty(m, device="cuda", dtype=torch.int64)
        part = torch.empty(lib.load().nm_logits_xent_scratch(m, v), device="cuda")
        logits = torch.empty(m, v, device="cuda") if keep_logits else None
        lib.call("nm_logits_xent_fwd16", lib.ptr(self.x16), self.kpad, lib.ptr(self.wt16), self.kpad, lib.ptr(self.b),
                 self.unk, lib.ptr(self.targets), lib.ptr(self.mask), lib.ptr(lse), lib.ptr(xent), lib.ptr(argmax),
                 lib.ptr(part), lib.ptr(logits), v, m, v, self.k, lib.stream())
        torch.cuda.synchronize()
        return lse, xent, argmax, logits, part

    def bwd(self, lse):
        lib = _lib()
        dl16 = torch.full((self.m, self.vpad), 7.0, device="cuda", dtype=torch.float16)
        lib.call("nm_logits_xent_bwd16", lib.ptr(self.x16), self.kpad, lib.ptr(self.wt16), self.kpad,
                 lib.ptr(self.b), self.unk, lib.ptr(self.targets), lib.ptr(self.mask), lib.ptr(lse),
                 lib.ptr(dl16), self.vpad, self.m, self.v, self.k, lib.stream())
        torch.cuda.synchronize()
        return dl16


def _check_fwd(pb, lse, xent, argmax, logits):
    ref = pb.reference()
    lse_ref = torch.logsumexp(ref, 1)
    tgt = ref.gather(1, pb.targets[:, None])[:, 0]
    assert float((lse.double() - lse_ref).abs().max()) < 1e-4
    assert float((xent.double() - (lse_ref - tgt) * pb.mask.double()).abs().max()) < 1e-4
    assert bool(((logits.double() - ref).abs() <= 1e-4 + 1e-7 * ref.abs()).all())   # fp32 ulp at the -1e9 of <unk>
    # argmax: a column whose exact logit is the row maximum up to fp32 accumulation error
    best = ref.max(1).values
    assert bool((ref.gather(1, argmax[:, None])[:, 0] >= best - 1e-5).all())
    return ref, lse_ref


@pytest.mark.parametrize("m", [1, 63, 129, 12801])
@pytest.mark.parametrize("v", [200, 4100, 32001])
def test_fwd_bwd_ragged(m, v):
    unk = 3 if (m + v) % 2 else -1
    pb = Problem(m, v, 300, unk, seed=m + v)
    lse, xent, argmax, logits, _ = pb.fwd()
    ref, lse_ref = _check_fwd(pb, lse, xent, argmax, logits)
    dl16 = pb.bwd(lse)
    p_ref = torch.softmax(ref, 1)
    p_ref[torch.arange(m, device="cuda"), pb.targets] -= 1.0
    p_ref *= pb.mask.double()[:, None]
    got = dl16[:, :v].double()
    assert float((got - p_ref).abs().max()) < 1e-3                   # fp16 rounding of values in [-1, 1]
    assert float(got[pb.mask == 0].abs().max() if bool((pb.mask == 0).any()) else 0.0) == 0.0
    if pb.vpad > v:
        assert bool((dl16[:, v:] == 7.0).all())                      # the padding columns are not written


@pytest.mark.parametrize("m,v,k", [(12800, 32000, 300), (700, 4100, 24), (700, 4100, 512), (129, 32001, 520)])
def test_shapes_and_k(m, v, k):
    pb = Problem(m, v, k, 1, seed=k)
    lse, xent, argmax, logits, _ = pb.fwd()
    _check_fwd(pb, lse, xent, argmax, logits)
    lse2, _, _, _, _ = pb.fwd(keep_logits=False)
    assert torch.equal(lse, lse2)


@pytest.mark.parametrize("lo,hi", [(8, 16), (10, 200), (300, 4000), (4099, 4100), (0, 4100)])
def test_argmax_ties_lowest_column(lo, hi):
    """Duplicated W columns give bit-identical logits: the lowest column wins, whether the copies sit in the same
    thread's columns, in the same 256-column tile or in different tiles."""
    m, v, k = 130, 4101, 300
    g = torch.Generator().manual_seed(5)
    wt = (torch.randn(v, k, generator=g) * 0.05).half()
    wt[lo] = (torch.rand(k, generator=g) + 0.5).half()
    wt[hi] = wt[lo]
    x = (torch.rand(m, k, generator=g) + 0.2).half()               # x . wt[lo] dominates every row
    pb = Problem(m, v, k, -1, x=x.cuda(), wt=wt.cuda())
    pb.b.zero_()
    lse, xent, argmax, logits, _ = pb.fwd()
    assert torch.equal(logits[:, lo], logits[:, hi])
    assert bool((argmax == lo).all())


def test_repeat_calls_are_bit_identical():
    pb = Problem(2051, 32000, 300, 1, seed=9)
    lse_a, _, _, _, part_a = pb.fwd(keep_logits=False)
    lse_b, _, _, _, part_b = pb.fwd(keep_logits=False)
    assert torch.equal(part_a, part_b) and torch.equal(lse_a, lse_b)
    assert torch.equal(pb.bwd(lse_a), pb.bwd(lse_a))
