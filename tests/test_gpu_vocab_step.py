"""The vocabulary softmax of one decoding step (csrc/xent.cu) and the beam kernels (csrc/beam.cu), called through
the C ABI on both engines and compared with plain references.

Exact operands: with X in {-3..3}, W in {-3..3}/16, the bias in {-8..8}/16 and K <= 520, every product and every
partial sum is an exact fp32 number, and TF32 holds every operand exactly.  The logits are then exact on the
tensor cores and on the CUDA cores, in any summation order.  So argmax (with its ties), symbols, finished flags,
masks and the unfinished counter are compared bit for bit on both engines; lse and xent, whose exponentials are
rounded (ex2.approx on the tensor cores), are compared with fp64 within LSE_TOL.

Also here: the row kernel at its three block sizes with duplicated maxima in one thread's columns, in one warp
and in different warps; the backward and the log-softmax past 65,535 rows; the beam step for beams above 8 on
log-probs and on logits with their logsumexp, bit-exact against the fp32 oracle; and the backtrack against
re-gathering the whole history at every step."""
import functools

import pytest
import torch

from oracle import nm_oracle as O

pytestmark = pytest.mark.gpu

UNK = 3            # <unk>
END = 2            # </s>
SENTINEL = 12345.0
# |lse - fp64| and |xent - fp64|: below 200 in magnitude, both are sums of at most 32,000 rounded exponentials
# (expf, or ex2.approx on the tensor cores) and one fp32 logf; 5e-5 is about 6 fp32 ulps at 200.
LSE_TOL = 5e-5


def _lib():
    from neuralmonkey_b200 import lib
    return lib


def _first_argmax(x: torch.Tensor) -> torch.Tensor:
    """First column of the row maximum (tf.argmax order), spelled out rather than left to a library's tie rule."""
    cols = torch.arange(x.shape[1], device=x.device).expand_as(x)
    return torch.where(x == x.max(1, keepdim=True).values, cols, x.shape[1]).min(1).values


def _mask_unk(logits32: torch.Tensor, unk: int) -> torch.Tensor:
    """The kernels' <unk> mask: the fp32 sum logit + (-1e9f), in place on a CPU fp32 tensor."""
    if unk >= 0:
        logits32[:, unk] += torch.tensor(-1e9, dtype=torch.float32)
    return logits32


def _close(got: torch.Tensor, want64: torch.Tensor, tol: float) -> None:
    err = float((got.detach().cpu().double() - want64.cpu()).abs().max()) if got.numel() else 0.0
    assert err <= tol, (err, tol)


# ---------------------------------------------------------------------------------------------------------------
# a. nm_xent_fwd: one CTA per row of materialised logits
# ---------------------------------------------------------------------------------------------------------------
def _row_threads(v: int) -> int:
    return 32 if v < 256 else (128 if v < 4096 else 512)     # the row kernel's block size for V columns


def _tie_pairs(v: int):
    """Column pairs (lo, hi) holding the row maximum twice.  Thread t of the row kernel reads columns t, t+T, ..."""
    t = _row_threads(v)
    pairs = [(3, 3 + t), (v - 1 - t, v - 1),      # one thread's columns
             (5, 6), (0, 31)]                      # one warp
    if t > 32:
        pairs += [(7, 7 + 32), (t - 1, t), (40, t - 2)]   # different warps; (t-1, t): the lower column in the last warp
    else:
        pairs += [(31, 32)]                        # thread 31, and thread 0's second column
    return pairs


@pytest.mark.parametrize("v", [70, 255, 256, 4095, 4096, 32000])
@pytest.mark.parametrize("mode", ["weighted", "unweighted", "no_targets", "unk_at_tie"])
def test_xent_rows_kernel(v, mode):
    lib = _lib()
    pairs = _tie_pairs(v)
    m, ldl = 3 * len(pairs) + 2, v + 5
    g = torch.Generator().manual_seed(v)
    logits = (torch.randn(m, ldl, generator=g) * 2).clamp(-7, 7)
    logits[:, v:] = 100.0                                   # padding: would win every row if it were read
    for r in range(m - 2):
        lo, hi = pairs[r % len(pairs)]
        logits[r, lo] = logits[r, hi] = 8.0 + 0.25 * (r % 4)
    logits[m - 2, v - 1] = 9.0                               # the maximum in the last column
    logits[m - 1, :v] = -1.5                                 # a constant row: column 0
    unk = pairs[0][0] if mode == "unk_at_tie" else -1
    targets = torch.randint(0, v, (m,), generator=g)
    targets[targets == pairs[0][0]] += 1                     # no <unk> target: its xent of ~1e9 is checked elsewhere
    targets[0], targets[-1] = pairs[0][1], v - 1
    weights = torch.rand(m, generator=g) if mode != "unweighted" else None
    with_targets = mode != "no_targets"

    d_logits = logits.cuda()
    lse = torch.full((m,), SENTINEL, device="cuda")
    xent = torch.full((m,), SENTINEL, device="cuda")
    argmax = torch.full((m,), -7, device="cuda", dtype=torch.int64)
    d_t = targets.cuda() if with_targets else None
    d_w = weights.cuda() if weights is not None else None
    lib.call("nm_xent_fwd", lib.ptr(d_logits), unk, lib.ptr(d_t), lib.ptr(d_w), lib.ptr(lse), lib.ptr(xent),
             lib.ptr(argmax), m, v, ldl, lib.stream())
    torch.cuda.synchronize()

    ref = _mask_unk(logits.clone(), unk)
    assert torch.equal(d_logits.cpu(), ref)                 # the mask written back, nothing else touched
    ref = ref[:, :v]
    want_arg = _first_argmax(ref)
    for r in range(m - 2):                                   # the pairs really are the maxima
        lo, hi = pairs[r % len(pairs)]
        assert int(want_arg[r]) == (hi if lo == unk else lo)
    assert int(want_arg[m - 2]) == v - 1 and int(want_arg[m - 1]) == 0
    assert torch.equal(argmax.cpu(), want_arg)
    lse64 = torch.logsumexp(ref.double(), 1)
    _close(lse, lse64, LSE_TOL)
    if with_targets:
        xent64 = lse64 - ref.double().gather(1, targets[:, None])[:, 0]
        if weights is not None:
            xent64 = xent64 * weights.double()
        _close(xent, xent64, LSE_TOL)
    else:
        assert bool((xent == SENTINEL).all())               # no targets: xent is not written


def test_xent_rows_from_column_one():
    """ops.xent_rows(first_col=1), as `decoded` calls it: the window starts one float past an aligned base, and a
    tie at the window's first column (relative index 0) must win over copies in the same thread, warp and others."""
    from neuralmonkey_b200 import ops
    m, v = 10, 4097                                          # 4096 columns in the window: 512 threads
    g = torch.Generator().manual_seed(3)
    logits = (torch.randn(m, v, generator=g) * 2).clamp(-7, 7)
    logits[:, 0] = 50.0                                      # outside the window
    partners = [513, 2, 97, 4096, 33]                        # same thread, same warp, warp 3, last warp, warp 1
    for r in range(m):
        logits[r, 1] = logits[r, partners[r % len(partners)]] = 8.0
    targets = torch.randint(0, v - 1, (m,), generator=g)
    targets[0] = 0
    weights = torch.rand(m, generator=g)
    lse, xent, arg = ops.xent_rows(logits.cuda(), targets.cuda(), weights.cuda(), want_argmax=True, first_col=1)
    torch.cuda.synchronize()
    win = logits[:, 1:].double()
    assert bool((arg.cpu() == 0).all())
    lse64 = torch.logsumexp(win, 1)
    _close(lse, lse64, LSE_TOL)
    _close(xent, (lse64 - win.gather(1, targets[:, None])[:, 0]) * weights.double(), LSE_TOL)


# ---------------------------------------------------------------------------------------------------------------
# b. nm_log_softmax and nm_xent_bwd, including more rows than grid.y holds
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m,v,pad", [(37, 70, 3), (37, 4097, 7), (19, 32000, 4), (70001, 33, 2)])
def test_log_softmax_and_xent_bwd(m, v, pad):
    lib = _lib()
    ldl = v + pad
    g = torch.Generator().manual_seed(m + v)
    logits = torch.randn(m, ldl, generator=g) * 3
    logits[:, v:] = 777.0
    lse64 = torch.logsumexp(logits[:, :v].double(), 1)
    lse = lse64.float()
    targets = torch.randint(0, v, (m,), generator=g)
    targets[-1] = v - 1
    weights = torch.rand(m, generator=g)
    scale = torch.tensor([0.5])
    d_logits, d_lse, d_t, d_w, d_s = (t.cuda() for t in (logits, lse, targets, weights, scale))

    out = torch.full((m, v), SENTINEL, device="cuda")
    lib.call("nm_log_softmax", lib.ptr(d_logits), lib.ptr(d_lse), lib.ptr(out), m, v, ldl, lib.stream())
    torch.cuda.synchronize()
    assert torch.equal(out.cpu(), logits[:, :v] - lse[:, None])   # one fp32 subtraction per element
    _close(out, logits[:, :v].double() - lse64[:, None], 1e-5)

    dl = torch.full((m, ldl), 777.0, device="cuda")
    lib.call("nm_xent_bwd", lib.ptr(d_logits), lib.ptr(d_t), lib.ptr(d_w), lib.ptr(d_lse), lib.ptr(d_s), lib.ptr(dl),
             m, v, ldl, lib.stream())
    torch.cuda.synchronize()
    want = torch.softmax(logits[:, :v].double(), 1)
    want[torch.arange(m), targets] -= 1.0
    want *= weights.double()[:, None] * 0.5
    # p = expf(logit - lse) carries the rounding of lse to fp32 and of expf: a few 1e-7 at most, for |p| <= 1
    _close(dl[:, :v], want, 2e-6)
    assert bool((dl[:, v:] == 777.0).all())
    inplace = d_logits.clone()                               # the exact engine's loss backward runs it in place
    lib.call("nm_xent_bwd", lib.ptr(inplace), lib.ptr(d_t), lib.ptr(d_w), lib.ptr(d_lse), lib.ptr(d_s),
             lib.ptr(inplace), m, v, ldl, lib.stream())
    torch.cuda.synchronize()
    assert torch.equal(inplace[:, :v], dl[:, :v]) and bool((inplace[:, v:] == 777.0).all())


def test_logits_xent_exact_engine_past_65535_rows():
    """ops.logits_xent on the exact engine at M = 70,001 tokens: forward and backward against fp64 autograd."""
    from neuralmonkey_b200 import ops
    m, k, v = 70001, 16, 33
    g = torch.Generator().manual_seed(7)
    x = torch.randn(m, k, generator=g)
    w = torch.randn(k, v, generator=g) * 0.3
    b = torch.randn(v, generator=g) * 0.1
    targets = torch.randint(UNK + 1, v, (m,), generator=g)
    weights = (torch.rand(m, generator=g) > 0.2).float()
    ops.set_gemm_backend("simt")
    try:
        xd, wd, bd = (t.cuda().requires_grad_() for t in (x, w, b))
        xent, lse, arg, _ = ops.logits_xent(xd, wd, bd, targets.cuda(), weights.cuda(), unk_index=UNK)
        xent.sum().backward()
        torch.cuda.synchronize()
    finally:
        ops.set_gemm_backend("auto")
    x64, w64, b64 = (t.double().requires_grad_() for t in (x, w, b))
    unk_mask = torch.zeros(v, dtype=torch.float64)
    unk_mask[UNK] = -1e9
    lg = x64 @ w64 + b64 + unk_mask
    lse64 = torch.logsumexp(lg, 1)
    xent64 = (lse64 - lg.gather(1, targets[:, None])[:, 0]) * weights.double()
    xent64.sum().backward()
    _close(xent, xent64.detach(), 1e-4)
    _close(lse, lse64.detach(), 1e-4)
    top2 = lg.detach().topk(2, 1).values
    clear = (top2[:, 0] - top2[:, 1]) > 1e-4                 # rows without a near-tie at fp32 resolution
    assert torch.equal(arg.cpu()[clear], lg.detach().argmax(1)[clear])
    dl64 = (torch.softmax(lg.detach(), 1) - torch.nn.functional.one_hot(targets, v)) * weights.double()[:, None]
    _close(xd.grad, x64.grad, 1e-5)
    # weight and bias gradients sum 70,001 rows in fp32: bound by the sum of the terms' magnitudes
    wbound = float((x.double().abs().t() @ dl64.abs()).max())
    _close(wd.grad, w64.grad, 1e-5 * wbound)
    _close(bd.grad, b64.grad, 1e-5 * float(dl64.abs().sum(0).max()))


# ---------------------------------------------------------------------------------------------------------------
# c. nm_decode_logits_step on exact operands, both engines
# ---------------------------------------------------------------------------------------------------------------
class Step:
    """One decoding step on exact operands.  X [M,K] is a column slice of a wider buffer (ldx > K); W is [K,V] with a
    row pitch that is a multiple of 4 floats, or [V,K] (trans_w); padding holds 100.0, which would show if read.
    Without `edit`, rows with r % 4 == 1 put their maximum on column 2 (</s>); `edit(x, w, b)` replaces that with
    its own changes to the operands."""

    def __init__(self, m, v, k, trans_w, seed, unk=UNK, edit=None):
        g = torch.Generator().manual_seed(seed)
        self.m, self.v, self.k, self.trans_w, self.unk = m, v, k, trans_w, unk
        x = torch.randint(-3, 4, (m, k), generator=g).float()
        w = torch.randint(-3, 4, (k, v), generator=g).float() / 16           # logical [K, V]
        b = torch.randint(-8, 9, (v,), generator=g).float() / 16
        if edit is not None:
            edit(x, w, b)
        else:                                  # rows 1, 5, 9, ...: X = 3 and W, b at their largest on column 2
            w[:, END] = 3 / 16
            b[END] = 0.5
            x[1::4] = 3.0
        xb = torch.full((m, k + 8), 100.0)
        xb[:, 4:4 + k] = x
        self.xbuf = xb.cuda()
        self.xd, self.ldx = self.xbuf[:, 4:4 + k], k + 8
        if trans_w:
            wb = torch.full((v, k + 4), 100.0)
            wb[:, :k] = w.t()
            self.ldw = k + 4
        else:
            # a multiple of 4 floats, so the tensor cores can load W; above V also when V is one (small V only)
            self.ldw = (v + 3) // 4 * 4 + (4 if v % 4 == 0 and v < 1000 else 0)
            wb = torch.full((k, self.ldw), 100.0)
            wb[:, :v] = w
        self.wd, self.bd = wb.cuda(), b.cuda()
        self.fin = torch.rand(m, generator=g) < 0.3
        self.fin[1] = False                                                  # an </s> row that finishes now
        self.targets = torch.randint(0, v, (m,), generator=g)
        self.targets[self.targets == unk] += 1
        self.targets[0], self.targets[-1] = unk if unk >= 0 else 0, v - 1    # <unk>, and the last partial tile
        self.weights = torch.rand(m, generator=g)
        self.fin_d, self.t_d, self.w_d = (t.cuda() for t in (self.fin.to(torch.uint8), self.targets, self.weights))

        exact = x.double() @ w.double() + b.double()
        self.logits = exact.float()
        assert torch.equal(self.logits.double(), exact)                      # the operands keep every sum exact
        _mask_unk(self.logits, unk)
        self.argmax = _first_argmax(self.logits)
        self.lse64 = torch.logsumexp(self.logits.double(), 1)
        self.xent64 = (self.lse64 - self.logits.double().gather(1, self.targets[:, None])[:, 0]) * self.weights.double()
        self.sym = torch.where(self.fin, 0, self.argmax)
        self.fin_out = self.fin | (self.sym == END)

    def run(self, backend, targets=True, stats=True, alias=False, logits_out=True, preset=7):
        lib = _lib()
        m, v = self.m, self.v
        out = dict(lse=torch.full((m,), SENTINEL, device="cuda"), xent=torch.full((m,), SENTINEL, device="cuda"),
                   argmax=torch.full((m,), -7, device="cuda", dtype=torch.int64),
                   sym=torch.full((m,), -7, device="cuda", dtype=torch.int64),
                   mask=torch.full((m,), 9, device="cuda", dtype=torch.uint8),
                   count=torch.full((1,), preset, device="cuda", dtype=torch.int32))
        fin_in = self.fin_d.clone()
        out["fin"] = fin_in if alias else torch.full((m,), 9, device="cuda", dtype=torch.uint8)
        out["logits"] = torch.full((m, v + 5), 777.0, device="cuda") if logits_out else None
        part = torch.empty(lib.load().nm_logits_xent_scratch(m, v), device="cuda")
        lib.call("nm_decode_logits_step", lib.ptr(self.xd), self.ldx, lib.ptr(self.wd), self.ldw, int(self.trans_w),
                 lib.ptr(self.bd), self.unk, lib.ptr(fin_in), lib.ptr(self.t_d) if targets else None,
                 lib.ptr(self.w_d) if targets else None, lib.ptr(out["lse"]) if stats else None,
                 lib.ptr(out["argmax"]) if stats else None, lib.ptr(out["xent"]) if stats else None,
                 lib.ptr(out["sym"]), lib.ptr(out["fin"]), lib.ptr(out["mask"]), lib.ptr(out["count"]), lib.ptr(part),
                 lib.ptr(out["logits"]), v + 5, m, v, self.k, backend, lib.stream())
        torch.cuda.synchronize()
        return {key: (t.cpu() if t is not None else None) for key, t in out.items()}

    def check(self, out, targets=True, stats=True, preset=7):
        v = self.v
        if out["logits"] is not None:
            assert torch.equal(out["logits"][:, :v], self.logits)            # exact, <unk> mask included
            assert bool((out["logits"][:, v:] == 777.0).all())
        assert torch.equal(out["sym"], self.sym)
        assert torch.equal(out["fin"], self.fin_out.to(torch.uint8))
        assert torch.equal(out["mask"], (~self.fin_out).to(torch.uint8))
        assert int(out["count"][0]) == preset + int((~self.fin_out).sum())
        if stats:
            assert torch.equal(out["argmax"], self.argmax)
            _close(out["lse"], self.lse64, LSE_TOL)
            if targets:
                _close(out["xent"], self.xent64, LSE_TOL * 2e7)               # the <unk> target's xent is ~1e9
                _close(out["xent"][1:], self.xent64[1:], LSE_TOL)
            else:
                assert bool((out["xent"] == SENTINEL).all())
        else:
            assert bool((out["lse"] == SENTINEL).all()) and bool((out["argmax"] == -7).all())
            assert bool((out["xent"] == SENTINEL).all())


STEP_SHAPES = [(37, 256, 32, False), (64, 4097, 300, False), (256, 32000, 300, False), (130, 511, 64, True)]


@functools.lru_cache(maxsize=None)
def _step(m, v, k, trans_w):
    return Step(m, v, k, trans_w, seed=m + v + k)


@pytest.mark.parametrize("shape", STEP_SHAPES, ids=lambda s: "{}x{}x{}{}".format(*s[:3], "T" if s[3] else ""))
@pytest.mark.parametrize("backend", ["simt", "tc"])
@pytest.mark.parametrize("variant", ["full", "no_targets", "aliased_no_stats"])
def test_decode_step_exact_operands(shape, backend, variant):
    lib = _lib()
    pb = _step(*shape)
    assert bool((pb.sym == END).any()) and bool(pb.fin.any()) and bool((~pb.fin_out).any())
    kw = dict(targets=variant != "no_targets", stats=variant != "aliased_no_stats")
    out = pb.run({"simt": lib.GEMM_SIMT, "tc": lib.GEMM_TC}[backend], alias=variant == "aliased_no_stats", **kw)
    pb.check(out, **kw)


@pytest.mark.parametrize("shape", STEP_SHAPES, ids=lambda s: "{}x{}x{}{}".format(*s[:3], "T" if s[3] else ""))
def test_decode_step_engines_agree(shape):
    """Both engines give the same logits and integer outputs; the tensor-core step's lse and xent are
    nm_logits_xent_fwd's, bit for bit."""
    lib = _lib()
    pb = _step(*shape)
    simt, tc = pb.run(lib.GEMM_SIMT), pb.run(lib.GEMM_TC)
    for key in ("logits", "argmax", "sym", "fin", "mask", "count"):
        assert torch.equal(simt[key], tc[key]), key
    m, v = pb.m, pb.v
    lse, xent = torch.empty(m, device="cuda"), torch.empty(m, device="cuda")
    argmax = torch.empty(m, device="cuda", dtype=torch.int64)
    part = torch.empty(lib.load().nm_logits_xent_scratch(m, v), device="cuda")
    lib.call("nm_logits_xent_fwd", lib.ptr(pb.xd), pb.ldx, lib.ptr(pb.wd), pb.ldw, int(pb.trans_w), lib.ptr(pb.bd),
             pb.unk, lib.ptr(pb.t_d), lib.ptr(pb.w_d), lib.ptr(lse), lib.ptr(xent), lib.ptr(argmax), lib.ptr(part),
             None, v, m, v, pb.k, lib.stream())
    torch.cuda.synchronize()
    assert torch.equal(tc["lse"], lse.cpu()) and torch.equal(tc["xent"], xent.cpu())
    assert torch.equal(tc["argmax"], argmax.cpu())


def test_decode_step_operands_not_tma_addressable():
    """K = 9 (row pitch 17 floats): the tensor-core engine refuses, AUTO needs logits_out and then runs the exact
    engine."""
    lib = _lib()
    pb = Step(40, 300, 9, False, seed=9)
    with pytest.raises(ValueError):
        pb.run(lib.GEMM_TC)
    with pytest.raises(ValueError):
        pb.run(lib.GEMM_AUTO, logits_out=False)
    pb.check(pb.run(lib.GEMM_AUTO))


# ---------------------------------------------------------------------------------------------------------------
# d. TF32 tie placement: a duplicated maximum across chunks, epilogue halves and tiles of the xent epilogue
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lo,hi", [(8, 16), (10, 42), (10, 74), (300, 4000), (4099, 4100), (0, 4100)],
                         ids=["same_chunk", "two_halves", "same_half", "two_tiles", "last_tile", "first_last"])
@pytest.mark.parametrize("unk_at_lo", [False, True])
def test_tf32_argmax_ties(lo, hi, unk_at_lo):
    lib = _lib()
    m, v, k = 130, 4101, 300

    def edit(x, w, b):          # every row's maximum sits twice, on columns lo and hi: X > 0, W and b largest there
        x.abs_().clamp_(min=1.0)
        w[:, lo] = w[:, hi] = 3 / 16
        b[lo] = b[hi] = 0.5

    pb = Step(m, v, k, False, seed=lo + hi, unk=lo if unk_at_lo else -1, edit=edit)
    want = hi if unk_at_lo else lo
    assert bool((pb.argmax == want).all())
    for backend in (lib.GEMM_TC, lib.GEMM_SIMT):
        out = pb.run(backend)
        assert bool((out["argmax"] == want).all()), backend
        pb.check(out)
    lse = torch.empty(m, device="cuda")
    argmax = torch.empty(m, device="cuda", dtype=torch.int64)
    part = torch.empty(lib.load().nm_logits_xent_scratch(m, v), device="cuda")
    lib.call("nm_logits_xent_fwd", lib.ptr(pb.xd), pb.ldx, lib.ptr(pb.wd), pb.ldw, 0, lib.ptr(pb.bd), pb.unk, None,
             None, lib.ptr(lse), None, lib.ptr(argmax), lib.ptr(part), None, v, m, v, k, lib.stream())
    torch.cuda.synchronize()
    assert bool((argmax.cpu() == want).all())


# ---------------------------------------------------------------------------------------------------------------
# e. nm_beam_step and nm_beam_step_logits against the fp32 oracle
# ---------------------------------------------------------------------------------------------------------------
BEAM_SHAPES = [(3, 9, 1000), (2, 16, 32000), (2, 17, 32000), (1, 64, 32000), (4, 64, 5), (2, 12, 4096),
               (2, 12, 4097), (5, 33, 4095), (2, 8, 4096), (3, 4, 1000)]
BEAM_OUTPUTS = ("scores", "word_ids", "beam_ids", "logprob_sum", "lengths", "finished")


def _beam_state(bsz, k, v, state, seed):
    """(logits, their fp32 logsumexp, logprob_sum, lengths, finished) of one search step."""
    g = torch.Generator().manual_seed(seed)
    logits = torch.randn(bsz, k, v, generator=g) * 3
    lsum = -torch.rand(bsz, k, generator=g) * 10
    lens = torch.randint(0, 20, (bsz, k), generator=g, dtype=torch.int32)
    fin = torch.rand(bsz, k, generator=g) < 0.3
    if state == "sentence_finished":          # every beam of sentence 0 finished: all its candidates but <pad> at -1e9
        fin[0] = True
    elif state == "initial":                  # logprob_sum = [0, -1e9, ...] (beam_search_decoder.py:283-295)
        lsum.fill_(-O.INF)
        lsum[:, 0] = 0.0
        lens.zero_()
        fin.zero_()
    elif state == "constant":                 # constant rows: thousands of equal scores in a phase-1 chunk
        logits[:, ::2] = 1.25
        if k > 1:                             # beams 0 and 1 identical: every candidate ties across the two
            logits[:, 1], lsum[:, 1], lens[:, 1] = logits[:, 0], lsum[:, 0], lens[:, 0]
            fin[:, :2] = False
    return logits, torch.logsumexp(logits, -1), lsum, lens, fin


def _beam_call(name, first, lse, lsum, lens, fin, alpha, count=None):
    lib = _lib()
    bsz, k, v = first.shape
    out = dict(scores=torch.empty(bsz, k, device="cuda"),
               word_ids=torch.empty(bsz, k, device="cuda", dtype=torch.int64),
               beam_ids=torch.empty(bsz, k, device="cuda", dtype=torch.int32),
               logprob_sum=torch.empty(bsz, k, device="cuda"),
               lengths=torch.empty(bsz, k, device="cuda", dtype=torch.int32),
               finished=torch.empty(bsz, k, device="cuda", dtype=torch.uint8))
    scratch = torch.empty(lib.load().nm_beam_scratch(bsz, k, v), device="cuda", dtype=torch.int32)
    state = [lib.ptr(lsum), lib.ptr(lens), lib.ptr(fin), float(alpha)] + [lib.ptr(out[n]) for n in BEAM_OUTPUTS]
    if name == "nm_beam_step":
        lib.call(name, lib.ptr(first), *state, lib.ptr(scratch), bsz, k, v, lib.stream())
    else:
        lib.call(name, lib.ptr(first), lib.ptr(lse), *state, lib.ptr(count), lib.ptr(scratch), bsz, k, v, lib.stream())
    torch.cuda.synchronize()
    return {n: t.cpu() for n, t in out.items()}


def _assert_beam_equal(got, want):
    for name, w in zip(BEAM_OUTPUTS, want):
        g = got[name].bool() if name == "finished" else got[name]
        assert g.dtype == w.dtype and torch.equal(g, w), name


@pytest.mark.parametrize("shape", BEAM_SHAPES, ids=lambda s: "B{}k{}V{}".format(*s))
@pytest.mark.parametrize("alpha", [0.0, 0.6, 1.0])
@pytest.mark.parametrize("state", ["random", "sentence_finished", "initial", "constant"])
def test_beam_step_kernels_bit_exact(shape, alpha, state):
    """Both entry points against O.beam_step on fp32(logits - lse) from the CPU; the log-probs the first one reads
    are nm_log_softmax's, which must be that same fp32 subtraction."""
    lib = _lib()
    bsz, k, v = shape
    logits, lse, lsum, lens, fin = _beam_state(bsz, k, v, state, seed=bsz * 1000 + k * 7 + v)
    logprobs = logits - lse[..., None]
    want = O.beam_step(logprobs, lsum, lens, fin, alpha)
    d_logits, d_lse, d_lsum, d_lens = logits.cuda(), lse.cuda(), lsum.cuda(), lens.cuda()
    d_fin = fin.to(torch.uint8).cuda()
    d_lp = torch.empty(bsz, k, v, device="cuda")
    lib.call("nm_log_softmax", lib.ptr(d_logits), lib.ptr(d_lse), lib.ptr(d_lp), bsz * k, v, v, lib.stream())
    torch.cuda.synchronize()
    assert torch.equal(d_lp.cpu(), logprobs)
    _assert_beam_equal(_beam_call("nm_beam_step", d_lp, None, d_lsum, d_lens, d_fin, alpha), want)
    count = torch.full((1,), 5, device="cuda", dtype=torch.int32)
    got = _beam_call("nm_beam_step_logits", d_logits, d_lse, d_lsum, d_lens, d_fin, alpha, count)
    _assert_beam_equal(got, want)
    assert int(count[0]) == 5 + int((~want[5]).sum())         # += hypotheses unfinished after the step


def test_beam_step_refuses_beams_above_64():
    from neuralmonkey_b200 import ops
    bsz, k, v = 1, 65, 100
    lp = torch.log_softmax(torch.randn(bsz, k, v), -1).cuda()
    with pytest.raises(ValueError):
        ops.beam_step(lp, torch.zeros(bsz, k, device="cuda"), torch.zeros(bsz, k, device="cuda", dtype=torch.int32),
                      torch.zeros(bsz, k, device="cuda", dtype=torch.uint8), 0.6)


# ---------------------------------------------------------------------------------------------------------------
# f. nm_beam_backtrack against re-gathering the whole history at every step
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bsz", [1, 5])
@pytest.mark.parametrize("k", [1, 3, 64])
@pytest.mark.parametrize("steps", [0, 1, 7, 50])
def test_beam_backtrack(bsz, k, steps):
    lib = _lib()
    g = torch.Generator().manual_seed(bsz * 100 + k * 10 + steps)
    first = torch.randint(0, 1000, (bsz, k), generator=g)
    words = torch.randint(0, 1000, (steps, bsz, k), generator=g)
    parents = torch.randint(0, k, (steps, bsz, k), generator=g, dtype=torch.int32)
    history = [first]                          # beam_search_decoder.py:546-551: gather every row, append the word
    for t in range(steps):
        history = [h.gather(1, parents[t].long()) for h in history] + [words[t]]
    want = torch.stack(history)
    out = torch.full((steps + 1, bsz, k), -1, device="cuda", dtype=torch.int64)
    d_words, d_parents = (words.cuda(), parents.cuda()) if steps else (None, None)
    d_first = first.cuda()
    lib.call("nm_beam_backtrack", lib.ptr(d_first), lib.ptr(d_words), lib.ptr(d_parents), lib.ptr(out), bsz, k,
             steps, lib.stream())
    torch.cuda.synchronize()
    assert torch.equal(out.cpu(), want)
