"""The element-wise and gate kernels of csrc/elementwise.cu called directly through the C ABI, against fp64
restatements of the formulas in include/nmb200.h: the embedding gather / scatter, activation backward, bias
column sums, maxout, the NematusGRUCell and LSTMCell gates, and the layer-norm entry points that ops.layer_norm
does not reach (the split backward calls and the argument checks).

Where a kernel only moves or selects fp32 values (gathers, maxout routing, relu) the comparison is exact.  Where
it sums, the inputs are multiples of 1/16 whose partial sums stay far below 2^20: fp32 represents every such
partial sum exactly, so the result is exact in any summation order and any lost, doubled or misrouted term
shows.  The remaining tolerances are derived next to each comparison.

Grid-stride kernels are capped at 8 blocks of 256 threads per SM (grid_for): 8 * 132 * 256 = 270,336 elements
on an H100 SXM.  The "large" shapes below exceed that, so every thread walks the loop more than once."""
import pytest
import torch

from tests.helpers import max_abs, rel_err

pytestmark = pytest.mark.gpu

U = 2.0 ** -24          # unit roundoff of fp32
ACTS = {"none": 0, "tanh": 1, "relu": 2, "sigmoid": 3}


def _lib():
    from neuralmonkey_b200 import lib
    return lib


def _dev(*tensors):
    """CUDA copies (None stays None).  The kernels get raw pointers, so the copies must be held in variables
    until the call has run: a temporary freed after lib.ptr() would hand its memory to the next allocation."""
    out = tuple(t.cuda() if t is not None else None for t in tensors)
    return out if len(out) > 1 else out[0]


def _dyadic(g, *shape, lim=64):
    """Values k / 16 with |k| <= lim: sums of up to 2^14 of them stay below 2^20 and are exact in fp32."""
    return torch.randint(-lim, lim + 1, shape, generator=g, dtype=torch.int16).float() / 16


def _offset_view(n, offset, fill=float("nan")):
    """A CUDA vector of n floats starting `offset` floats into its allocation (offset 1: 4-byte aligned only)."""
    buf = torch.full((n + offset,), fill, device="cuda")
    return buf[offset:]


# ---------------------------------------------------------------------------------------------------------------
# embedding
# ---------------------------------------------------------------------------------------------------------------
BAD_IDS = (-1, None, 2 ** 40)        # None stands for `vocab`


def _ids(g, n, vocab):
    ids = torch.randint(0, vocab, (n,), generator=g)
    pos = torch.randperm(n, generator=g)[:3 * len(BAD_IDS)]
    for k, p in enumerate(pos.tolist()):
        bad = BAD_IDS[k % len(BAD_IDS)]
        ids[p] = vocab if bad is None else bad
    return ids


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("emb,offset", [(7, 0), (12, 0), (300, 0), (8, 1)])
def test_embed_fwd_exact(emb, offset, masked):
    """out[i] = table[ids[i]] * mask[i], zero rows for ids outside [0, vocab).  emb % 4 != 0 or a table / output
    that is not 16-byte aligned (offset 1) takes the scalar variant.  A product of two fp32 values is correctly
    rounded on both sides, so the comparison is exact; the output starts as NaN so every element must be
    written."""
    lib = _lib()
    g = torch.Generator().manual_seed(emb + offset)
    vocab, n = 37, 501
    table = torch.randn(vocab, emb, generator=g)
    ids = _ids(g, n, vocab)
    mask = None
    if masked:
        mask = torch.rand(n, generator=g)
        mask[torch.rand(n, generator=g) < 0.2] = 0.0
    t_d = _offset_view(vocab * emb, offset)
    t_d.copy_(table.reshape(-1).cuda())
    out = _offset_view(n * emb, offset)
    ids_d, mask_d = _dev(ids, mask)
    lib.call("nm_embed_fwd", lib.ptr(ids_d), lib.ptr(t_d), lib.ptr(mask_d), lib.ptr(out), n, emb, vocab, lib.stream())
    valid = (ids >= 0) & (ids < vocab)
    want = torch.zeros(n, emb)
    want[valid] = table[ids[valid]]
    if masked:
        want = want * mask[:, None]
    got = out.reshape(n, emb).cpu()
    assert torch.equal(got, want)
    assert torch.equal(got[~valid], torch.zeros(int((~valid).sum()), emb))


@pytest.mark.parametrize("values", ["dyadic", "normal"])
@pytest.mark.parametrize("masked", [False, True])
def test_embed_bwd_colliding_atomics(values, masked):
    """~20,000 ids into a 7-row table: about 2,900 atomic additions land on every cell of dtable, which already
    holds a gradient.  Ids outside the table and rows with mask 0 add nothing."""
    lib = _lib()
    g = torch.Generator().manual_seed(3 + masked)
    vocab, emb, n = 7, 12, 20011
    ids = _ids(g, n, vocab)
    if values == "dyadic":
        dout, dtable0 = _dyadic(g, n, emb), _dyadic(g, vocab, emb)
        mask = (torch.randint(0, 3, (n,), generator=g).float() / 2) if masked else None   # 0, 1/2, 1
    else:
        dout, dtable0 = torch.randn(n, emb, generator=g), torch.randn(vocab, emb, generator=g)
        mask = torch.rand(n, generator=g) * (torch.rand(n, generator=g) > 0.2).float() if masked else None
    ids_d, dout_d, mask_d, dtable = _dev(ids, dout, mask, dtable0)
    lib.call("nm_embed_bwd", lib.ptr(ids_d), lib.ptr(dout_d), lib.ptr(mask_d), lib.ptr(dtable), n, emb, vocab,
             lib.stream())
    valid = (ids >= 0) & (ids < vocab)
    contrib = dout.double() * (mask.double()[:, None] if masked else 1.0)
    want = dtable0.double().index_add(0, ids[valid], contrib[valid])
    if values == "dyadic":
        # the products by 0, 1/2 or 1 are multiples of 1/32 and every partial sum stays below 2,900 * 4 + 4 < 2^14:
        # exact in fp32 in any order, so a lost, doubled or misrouted term shows
        assert torch.equal(dtable.cpu().double(), want)
    else:
        # general values: one rounded product and one rounded addition per term, so in any summation order
        # |error| <= (k + 1) u (|dtable0| + sum |term|) for a cell that receives k terms
        absum = torch.zeros(vocab, emb, dtype=torch.float64).index_add(0, ids[valid], contrib[valid].abs())
        count = torch.zeros(vocab, dtype=torch.float64).index_add(0, ids[valid], torch.ones(int(valid.sum()),
                                                                                           dtype=torch.float64))
        bound = (count[:, None] + 1) * U * (dtable0.double().abs() + absum)
        err = (dtable.cpu().double() - want).abs()
        assert bool((err <= bound).all()), float((err / bound).max())


# ---------------------------------------------------------------------------------------------------------------
# activation backward
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alias", [False, True])
@pytest.mark.parametrize("n", [1, 1027, 1_000_003])
@pytest.mark.parametrize("act", list(ACTS))
def test_act_bwd(act, n, alias):
    """dx = dy * act'(y) through the activation output y (tanh: 1 - y^2, relu: y > 0, sigmoid: y (1 - y)).
    none and relu only copy or zero dy: exact.  tanh and sigmoid are two products and one subtraction of
    fp32 values with |y| <= 1, each rounded to within u (a fused multiply-add rounds once less):
    |error| <= 3 u |dy| (1 + |y|)."""
    lib = _lib()
    g = torch.Generator().manual_seed(n + ACTS[act])
    pre = torch.randn(n, generator=g) * 2
    y = {"none": pre, "tanh": torch.tanh(pre), "relu": torch.relu(pre), "sigmoid": torch.sigmoid(pre)}[act]
    dy = torch.randn(n, generator=g)
    y_d, dy_d = y.cuda(), dy.cuda()
    dx = dy_d if alias else torch.full((n,), float("nan"), device="cuda")
    lib.call("nm_act_bwd", lib.ptr(y_d), lib.ptr(dy_d), lib.ptr(dx), n, ACTS[act], lib.stream())
    y64, dy64 = y.double(), dy.double()
    want = {"none": dy64, "tanh": dy64 * (1 - y64 * y64), "relu": torch.where(y64 > 0, dy64, 0 * dy64),
            "sigmoid": dy64 * y64 * (1 - y64)}[act]
    got = dx.cpu().double()
    if act in ("none", "relu"):
        assert torch.equal(got, want)
    else:
        bound = 3 * U * dy64.abs() * (1 + y64.abs())
        assert bool(((got - want).abs() <= bound).all())


# ---------------------------------------------------------------------------------------------------------------
# bias-gradient column sums
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pad", [0, 5])
@pytest.mark.parametrize("N", [1, 31, 33, 1000])
@pytest.mark.parametrize("M", [0, 1, 64, 65, 100_000])
def test_colsum(M, N, pad):
    """out[n] (+)= sum_m x[m, n] over a [M, N] slice of rows of pitch ldx = N + pad.  Row chunks of >= 64 rows
    meet by atomics (M = 65: two chunks; M = 100,000: up to 528).  Dyadic inputs keep every partial sum exact
    (|sum| <= 100,000 * 4 < 2^19), so both modes compare exactly.  accumulate = 0 writes over a NaN buffer,
    M = 0 included; accumulate = 1 adds to a nonzero buffer."""
    lib = _lib()
    g = torch.Generator().manual_seed(M + N + pad)
    ldx = N + pad
    x = _dyadic(g, max(M, 1), ldx)
    x_d = x.cuda()
    want = x[:M, :N].sum(0, dtype=torch.float64)
    out = torch.full((N,), float("nan"), device="cuda")
    lib.call("nm_colsum", lib.ptr(x_d), M, N, ldx, lib.ptr(out), 0, lib.stream())
    assert torch.equal(out.cpu().double(), want)
    base = _dyadic(g, N)
    out = base.cuda()
    lib.call("nm_colsum", lib.ptr(x_d), M, N, ldx, lib.ptr(out), 1, lib.stream())
    assert torch.equal(out.cpu().double(), base.double() + want)


# ---------------------------------------------------------------------------------------------------------------
# maxout
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,O", [(3, 5), (1100, 300)])
def test_maxout_ties_go_to_the_first_half(M, O):
    """y[m, j] = max(z[m, j], z[m, O + j]); the winner, and with it the whole gradient, is the second half only
    when it is strictly larger (tf.nn.max_pool's first maximal element).  A third of the pairs are exact ties.
    Selection and routing move values: exact.  M * O = 330,000 exceeds the grid cap."""
    lib = _lib()
    g = torch.Generator().manual_seed(M)
    a = torch.randn(M, O, generator=g)
    b = torch.randn(M, O, generator=g)
    tie = torch.rand(M, O, generator=g) < 1 / 3
    b[tie] = a[tie]
    if M > 1:
        a[1], b[1], tie[1] = 0.5, 0.5, True          # a whole row of ties
    z = torch.cat([a, b], 1)
    y = torch.full((M, O), float("nan"), device="cuda")
    which = torch.full((M, O), 7, dtype=torch.uint8, device="cuda")
    z_d = _dev(z)
    lib.call("nm_maxout_fwd", lib.ptr(z_d), lib.ptr(y), lib.ptr(which), M, O, lib.stream())
    second = b > a
    assert torch.equal(y.cpu(), torch.where(second, b, a))
    assert torch.equal(which.cpu(), second.to(torch.uint8))
    dy = torch.randn(M, O, generator=g)
    dz = torch.full((M, 2 * O), float("nan"), device="cuda")
    dy_d = _dev(dy)
    lib.call("nm_maxout_bwd", lib.ptr(dy_d), lib.ptr(which), lib.ptr(dz), M, O, lib.stream())
    zero = torch.zeros(M, O)
    assert torch.equal(dz.cpu(), torch.cat([torch.where(second, zero, dy), torch.where(second, dy, zero)], 1))
    assert torch.equal(dz.cpu()[:, :O][tie], dy[tie])


# ---------------------------------------------------------------------------------------------------------------
# gate kernels of the step-wise cell variants
# ---------------------------------------------------------------------------------------------------------------
# Operands are randn clamped to [-2, 2].  Each output is a chain of at most ~8 fp32 operations (expf and tanhf
# are within 2 ulp; the library is built without fast math) whose intermediate values stay below 4 in
# magnitude and whose sensitivity to each intermediate is at most ~2: the error is at most a few tens of ulp
# of 4, i.e. ~5e-6, and typically ~1e-7.  A wrong formula (say, a dropped forget bias) is off by ~0.1.
GATE_TOL = 5e-6
GATE_SHAPES = [(3, 5), (1000, 400)]         # B * H = 400,000 exceeds the grid cap


def _op(g, *shape):
    return torch.randn(*shape, generator=g).clamp(-2, 2)


@pytest.mark.parametrize("B,H", GATE_SHAPES)
def test_nematus_gate_fwd_bwd(B, H):
    """[r, u] = sigmoid(sg + gi);  cand = tanh(sc * r + ci);  out = u * state + (1 - u) * cand; backward:
    dgates (of sg and of gi), dcpre (of ci), dsc, dstate (the direct path)."""
    lib = _lib()
    g = torch.Generator().manual_seed(B * H)
    sg, gi, sc, ci, state = _op(g, B, 2 * H), _op(g, B, 2 * H), _op(g, B, H), _op(g, B, H), _op(g, B, H)
    dev = [t.cuda() for t in (sg, gi, sc, ci, state)]
    out = torch.full((B, H), float("nan"), device="cuda")
    saved = torch.full((B, 3 * H), float("nan"), device="cuda")
    lib.call("nm_nematus_gate_fwd", *[lib.ptr(t) for t in dev], lib.ptr(out), lib.ptr(saved), B, H, lib.stream())
    l64 = [t.double().requires_grad_(True) for t in (sg, gi, sc, ci, state)]
    sg64, gi64, sc64, ci64, st64 = l64
    gates = torch.sigmoid(sg64 + gi64)
    r, u = gates[:, :H], gates[:, H:]
    cand = torch.tanh(sc64 * r + ci64)
    ref = u * st64 + (1 - u) * cand
    assert max_abs(out, ref) < GATE_TOL
    assert max_abs(saved, torch.cat([r, u, cand], 1)) < GATE_TOL
    dout = _op(g, B, H)
    ref.backward(dout.double())
    grads = {n: torch.full(s, float("nan"), device="cuda")
             for n, s in (("dgates", (B, 2 * H)), ("dcpre", (B, H)), ("dsc", (B, H)), ("dstate", (B, H)))}
    dout_d = _dev(dout)
    lib.call("nm_nematus_gate_bwd", lib.ptr(dout_d), lib.ptr(saved), lib.ptr(dev[2]), lib.ptr(dev[4]),
             lib.ptr(grads["dgates"]), lib.ptr(grads["dcpre"]), lib.ptr(grads["dsc"]), lib.ptr(grads["dstate"]),
             B, H, lib.stream())
    # dstate is only the direct path u * dout: the projections' backward adds the rest
    direct = dout.double() * u.detach()
    assert max_abs(grads["dgates"], sg64.grad) < GATE_TOL
    assert max_abs(grads["dgates"], gi64.grad) < GATE_TOL
    assert max_abs(grads["dcpre"], ci64.grad) < GATE_TOL
    assert max_abs(grads["dsc"], sc64.grad) < GATE_TOL
    assert max_abs(grads["dstate"], direct) < GATE_TOL


@pytest.mark.parametrize("given", ["both", "no_dnew_c", "no_dnew_h"])
@pytest.mark.parametrize("B,H", GATE_SHAPES)
def test_lstm_gate_fwd_bwd(B, H, given):
    """z = (i, j, f, o);  c' = sigmoid(f + 1) c + sigmoid(i) tanh(j);  h' = sigmoid(o) tanh(c'), forget bias 1
    as tf.nn.rnn_cell.LSTMCell; the backward pass with either incoming gradient absent (NULL)."""
    lib = _lib()
    g = torch.Generator().manual_seed(B + H)
    z, c = _op(g, B, 4 * H), _op(g, B, H)
    z_d, c_d = z.cuda(), c.cuda()
    new_c, new_h = (torch.full((B, H), float("nan"), device="cuda") for _ in range(2))
    saved = torch.full((B, 5 * H), float("nan"), device="cuda")
    lib.call("nm_lstm_gate_fwd", lib.ptr(z_d), lib.ptr(c_d), lib.ptr(new_c), lib.ptr(new_h), lib.ptr(saved), B, H,
             lib.stream())
    z64, c64 = z.double().requires_grad_(True), c.double().requires_grad_(True)
    i, j, f, o = z64.chunk(4, dim=1)
    si, tj, sf, so = torch.sigmoid(i), torch.tanh(j), torch.sigmoid(f + 1.0), torch.sigmoid(o)
    nc = sf * c64 + si * tj
    tc = torch.tanh(nc)
    nh = so * tc
    assert max_abs(new_c, nc) < GATE_TOL
    assert max_abs(new_h, nh) < GATE_TOL
    assert max_abs(saved, torch.cat([si, tj, sf, so, tc], 1)) < GATE_TOL
    dnc = _op(g, B, H) if given != "no_dnew_c" else None
    dnh = _op(g, B, H) if given != "no_dnew_h" else None
    loss = sum((t * d.double()).sum() for t, d in ((nc, dnc), (nh, dnh)) if d is not None)
    loss.backward()
    dz = torch.full((B, 4 * H), float("nan"), device="cuda")
    dc = torch.full((B, H), float("nan"), device="cuda")
    dnc_d, dnh_d = _dev(dnc, dnh)
    lib.call("nm_lstm_gate_bwd", lib.ptr(dnc_d), lib.ptr(dnh_d), lib.ptr(saved), lib.ptr(c_d), lib.ptr(dz),
             lib.ptr(dc), B, H, lib.stream())
    assert max_abs(dz, z64.grad) < GATE_TOL
    assert max_abs(dc, c64.grad) < GATE_TOL


# ---------------------------------------------------------------------------------------------------------------
# layer norm: the split backward calls and the argument checks
# ---------------------------------------------------------------------------------------------------------------
def _ln_fwd(x, gamma, beta):
    lib = _lib()
    m, d = x.shape
    y = torch.empty_like(x)
    mean, rstd = torch.empty(m, device="cuda"), torch.empty(m, device="cuda")
    lib.call("nm_layernorm_fwd", lib.ptr(x), lib.ptr(gamma), lib.ptr(beta), lib.ptr(y), lib.ptr(mean), lib.ptr(rstd),
             m, d, 1e-6, lib.stream())
    return y, mean, rstd


@pytest.mark.parametrize("M,D", [(300, 33), (1000, 1025)])
def test_layernorm_bwd_split_calls_equal_the_joint_call(M, D):
    """dx alone (dgamma = dbeta = NULL) is the same kernel as in the joint call: bit-identical.  The parameter
    gradients alone (dx = NULL), added into nonzero buffers, agree with the joint call to the reordering of
    their atomic sums and with fp64 to the tolerance of the ops-level test."""
    lib = _lib()
    g = torch.Generator().manual_seed(M + D)
    x, gamma, beta = torch.randn(M, D, generator=g), torch.randn(D, generator=g), torch.randn(D, generator=g)
    dy, dg0, db0 = torch.randn(M, D, generator=g), torch.randn(D, generator=g), torch.randn(D, generator=g)
    x_d, g_d, dy_d = x.cuda(), gamma.cuda(), dy.cuda()
    _y, mean, rstd = _ln_fwd(x_d, g_d, beta.cuda())
    common = (lib.ptr(x_d), lib.ptr(g_d), lib.ptr(mean), lib.ptr(rstd), lib.ptr(dy_d))
    dx_j, dg_j, db_j = torch.empty(M, D, device="cuda"), dg0.cuda(), db0.cuda()
    lib.call("nm_layernorm_bwd", *common, lib.ptr(dx_j), lib.ptr(dg_j), lib.ptr(db_j), M, D, lib.stream())
    dx_s = torch.full((M, D), float("nan"), device="cuda")
    lib.call("nm_layernorm_bwd", *common, lib.ptr(dx_s), None, None, M, D, lib.stream())
    dg_s, db_s = dg0.cuda(), db0.cuda()
    lib.call("nm_layernorm_bwd", *common, None, lib.ptr(dg_s), lib.ptr(db_s), M, D, lib.stream())
    assert torch.equal(dx_s, dx_j)
    # the same fp32 terms summed in another order: sqrt(M)-scale rounding differences of O(1) terms
    assert rel_err(dg_s, dg_j) < 1e-6 and rel_err(db_s, db_j) < 1e-6
    x64 = x.double()
    mu = x64.mean(1, keepdim=True)
    xhat = (x64 - mu) / torch.sqrt(((x64 - mu) ** 2).mean(1, keepdim=True) + 1e-6)
    assert rel_err(dg_s, dg0.double() + (dy.double() * xhat).sum(0)) < 2e-5
    assert rel_err(db_s, db0.double() + dy.double().sum(0)) < 2e-5


def test_layernorm_rejects_what_it_cannot_do():
    lib = _lib()
    m, d = 4, 2049
    x, gamma = torch.randn(m, d, device="cuda"), torch.randn(d, device="cuda")
    y, dx = torch.empty_like(x), torch.empty_like(x)
    mean, rstd = torch.zeros(m, device="cuda"), torch.ones(m, device="cuda")
    dg, db = torch.zeros(d, device="cuda"), torch.zeros(d, device="cuda")
    p = lib.ptr
    with pytest.raises(ValueError, match=r"failed \(-2\)"):     # NM_E_UNSUPPORTED: D > 2048
        lib.call("nm_layernorm_fwd", p(x), p(gamma), p(gamma), p(y), p(mean), p(rstd), m, d, 1e-6, lib.stream())
    with pytest.raises(ValueError, match=r"failed \(-2\)"):
        lib.call("nm_layernorm_bwd", p(x), p(gamma), p(mean), p(rstd), p(x), p(dx), p(dg), p(db), m, d,
                 lib.stream())
    d = 2048
    x, dx = x[:, :d].contiguous(), dx[:, :d].contiguous()
    for dx_, dg_, db_ in ((dx, dg, None), (dx, None, db), (None, None, None)):    # NM_E_INVALID
        with pytest.raises(ValueError, match=r"failed \(-1\)"):
            lib.call("nm_layernorm_bwd", p(x), p(gamma), p(mean), p(rstd), p(x), p(dx_), p(dg_), p(db_), m, d,
                     lib.stream())
