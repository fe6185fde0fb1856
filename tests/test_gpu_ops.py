"""Every differentiable op of neuralmonkey_b200.ops against the CPU oracle (fp64 autograd)."""
import pytest
import torch

from oracle import nm_oracle as O
from tests.helpers import max_abs, rel_err

pytestmark = pytest.mark.gpu


def _leaf(t):
    return t.clone().cuda().requires_grad_(True)


def test_embed_fwd_bwd():
    from neuralmonkey_b200 import ops
    g = torch.Generator().manual_seed(0)
    table = torch.randn(50, 12, generator=g)
    ids = torch.randint(0, 50, (4, 7), generator=g)
    mask = (torch.rand(4, 7, generator=g) > 0.3).float()
    td = _leaf(table)
    out = ops.embed(ids.cuda(), td, mask.cuda())
    t64 = table.double().requires_grad_(True)
    ref = t64[ids] * mask.double().unsqueeze(-1)
    assert max_abs(out, ref) == 0.0
    dout = torch.randn(4, 7, 12, generator=g)
    out.backward(dout.cuda())
    ref.backward(dout.double())
    assert max_abs(td.grad, t64.grad) < 1e-5


@pytest.mark.parametrize("dims", [(6, 14), (33, 600), (5, 1000)])
def test_layer_norm_fwd_bwd(dims):
    from neuralmonkey_b200 import ops
    m, d = dims
    g = torch.Generator().manual_seed(1)
    x, gamma, beta = torch.randn(m, d, generator=g), torch.randn(d, generator=g), torch.randn(d, generator=g)
    xd, gd, bd = _leaf(x), _leaf(gamma), _leaf(beta)
    y = ops.layer_norm(xd, gd, bd)
    x64, g64, b64 = (t.double().requires_grad_(True) for t in (x, gamma, beta))
    ref = O.layer_norm(x64, g64, b64)
    assert max_abs(y, ref) < 2e-5
    dy = torch.randn(m, d, generator=g)
    y.backward(dy.cuda())
    ref.backward(dy.double())
    assert rel_err(xd.grad, x64.grad) < 2e-5
    assert rel_err(gd.grad, g64.grad) < 2e-5
    assert rel_err(bd.grad, b64.grad) < 2e-5


@pytest.mark.parametrize("reverse", [False, True])
@pytest.mark.parametrize("use_lengths", [False, True])
@pytest.mark.parametrize("dims", [(5, 6, 11, 7), (9, 4, 32, 32), (7, 6, 12, 300), (70, 3, 16, 64),
                                  (3, 5, 8, 100)])
@pytest.mark.parametrize("engine", ["exact", "tc"])
def test_gru_layer_fwd_bwd(reverse, use_lengths, dims, engine):
    """engine 'exact': every product in fp32 on the CUDA cores; 'tc': the default engine - the hoisted input
    projections on the TF32 tensor-core GEMM wherever the shape is TMA-addressable, the recurrence on the cluster
    kernels."""
    from neuralmonkey_b200 import ops
    ops.set_gemm_backend("simt" if engine == "exact" else "auto")
    tol, gtol = (2e-5, 5e-5) if engine == "exact" else (3e-3, 1e-2)
    try:
        bsz, steps, e, h = dims
        g = torch.Generator().manual_seed(2)
        x = torch.randn(bsz, steps, e, generator=g)
        # the reduced-precision engine is checked in the regime real models live in (recurrent
        # gain ~1, as with the orthogonal initialiser); randn*0.3 at H=300 has gain ~5, where the
        # recurrence amplifies ANY rounding difference by orders of magnitude within a few steps
        ws = 0.3 if engine == "exact" else min(0.3, 1.0 / h ** 0.5)
        wg, bg = torch.randn(e + h, 2 * h, generator=g) * ws, torch.randn(2 * h, generator=g) * 0.3
        wc, bc = torch.randn(e + h, h, generator=g) * ws, torch.randn(h, generator=g) * 0.3
        h0 = torch.randn(bsz, h, generator=g) * 0.5
        lengths = torch.randint(1, steps + 1, (bsz,), generator=g) if use_lengths else None
        if lengths is not None:
            lengths[0] = steps
            lengths[-1] = 1
        leaves = [_leaf(t) for t in (x, wg, bg, wc, bc, h0)]
        ld = lengths.to(torch.int32).cuda() if lengths is not None else None
        states, final, _raw = ops.gru_layer(*leaves, lengths=ld, reverse=reverse)
        l64 = [t.double().requires_grad_(True) for t in (x, wg, bg, wc, bc, h0)]
        x64 = l64[0]
        if reverse:
            lens = lengths if lengths is not None else torch.full((bsz,), steps)
            out_rev, fin = O.dynamic_gru(O.reverse_sequence(x64, lens), lengths, *l64[1:5], h0=l64[5])
            ref_states = O.reverse_sequence(out_rev, lens)
        else:
            ref_states, fin = O.dynamic_gru(x64, lengths, *l64[1:5], h0=l64[5])
        assert max_abs(states, ref_states) < tol
        assert max_abs(final, fin) < tol
        ds, df = torch.randn(bsz, steps, h, generator=g), torch.randn(bsz, h, generator=g)
        (states * ds.cuda()).sum().backward(retain_graph=True)
        (final * df.cuda()).sum().backward()
        ((ref_states * ds.double()).sum() + (fin * df.double()).sum()).backward()
        for got, want, name in zip(leaves, l64, ("x", "wg", "bg", "wc", "bc", "h0")):
            assert rel_err(got.grad, want.grad) < gtol, name
    finally:
        ops.set_gemm_backend("auto")


def test_gru_dropout_mask_recurrence():
    """The state fed back is the dropped-out output; the raw output is returned separately."""
    from neuralmonkey_b200 import ops
    ops.set_gemm_backend("simt")
    try:
        bsz, steps, e, h = 3, 5, 6, 4
        g = torch.Generator().manual_seed(5)
        x = torch.randn(bsz, steps, e, generator=g)
        wg, bg = torch.randn(e + h, 2 * h, generator=g) * 0.3, torch.zeros(2 * h)
        wc, bc = torch.randn(e + h, h, generator=g) * 0.3, torch.zeros(h)
        mask = (torch.rand(bsz, steps, h, generator=g) < 0.5).float() / 0.5
        leaves = [_leaf(t) for t in (x, wg, bg, wc, bc)]
        dropped, final, raw = ops.gru_layer(*leaves, drop_mask=mask.cuda())
        l64 = [t.double().requires_grad_(True) for t in (x, wg, bg, wc, bc)]
        hprev = torch.zeros(bsz, h, dtype=torch.float64)
        raws, drops = [], []
        for t in range(steps):
            r = O.gru_cell(l64[0][:, t], hprev, *l64[1:])
            hprev = r * mask[:, t].double()
            raws.append(r)
            drops.append(hprev)
        ref_raw, ref_drop = torch.stack(raws, 1), torch.stack(drops, 1)
        assert max_abs(raw, ref_raw) < 2e-5 and max_abs(dropped, ref_drop) < 2e-5
        d1, d2 = torch.randn(bsz, steps, h, generator=g), torch.randn(bsz, steps, h, generator=g)
        ((dropped * d1.cuda()).sum() + (raw * d2.cuda()).sum()).backward()
        ((ref_drop * d1.double()).sum() + (ref_raw * d2.double()).sum()).backward()
        for got, want in zip(leaves, l64):
            assert rel_err(got.grad, want.grad) < 5e-5
    finally:
        ops.set_gemm_backend("auto")


@pytest.mark.parametrize("use_mask", [True, False])
@pytest.mark.parametrize("dims", [(3, 6, 4, 14, 14), (4, 50, 9, 600, 600), (2, 196, 3, 10, 512)])
def test_bahdanau_fwd_bwd(use_mask, dims):
    from neuralmonkey_b200 import ops
    bsz, tx, nq, a, c = dims
    g = torch.Generator().manual_seed(3)
    keys, values = torch.randn(bsz, tx, a, generator=g), torch.randn(bsz, tx, c, generator=g)
    q = torch.randn(bsz, nq, a, generator=g)
    v, bias = torch.randn(a, generator=g) * 0.3, torch.randn(1, generator=g)
    mask = None
    if use_mask:
        lens = torch.randint(1, tx + 1, (bsz,), generator=g)
        lens[0] = tx
        mask = (torch.arange(tx).unsqueeze(0) < lens.unsqueeze(1)).float()
    leaves = [_leaf(t) for t in (keys, values, q, v, bias)]
    ctx, w = ops.bahdanau_attention(leaves[0], leaves[1], mask.cuda() if use_mask else None,
                                    leaves[2], leaves[3], leaves[4])
    k64, v64, q64, vv64, b64 = (t.double().requires_grad_(True) for t in (keys, values, q, v, bias))
    e = (vv64 * torch.tanh(k64.unsqueeze(1) + q64.unsqueeze(2))).sum(-1) + b64
    if use_mask:
        wa = torch.softmax(e, -1) * mask.double().unsqueeze(1)
        wref = wa / (wa.sum(-1, keepdim=True) + 1e-8)
    else:
        wref = torch.softmax(e, -1)
    cref = wref @ v64
    assert max_abs(w, wref) < 1e-5
    assert max_abs(ctx, cref) < 5e-5
    dctx = torch.randn(bsz, nq, c, generator=g)
    (ctx * dctx.cuda()).sum().backward()
    (cref * dctx.double()).sum().backward()
    for got, want, name in zip(leaves[:4], (k64, v64, q64, vv64), ("keys", "values", "q", "v")):
        assert rel_err(got.grad, want.grad) < 1e-4, name
    # softmax is shift invariant: the scalar bias has (mathematically) zero gradient
    assert abs(float(leaves[4].grad) - float(b64.grad)) < 1e-4


@pytest.mark.parametrize("cfg", [(37, 70, 9, "simt", False), (300, 1000, 64, "auto", False),
                                 (256, 4096, 300, "auto", False), (130, 520, 64, "auto", True)])
def test_logits_xent_fwd_bwd(cfg):
    from neuralmonkey_b200 import ops
    m, vocab, k, backend, trans_w = cfg
    ops.set_gemm_backend(backend)
    try:
        g = torch.Generator().manual_seed(4)
        x = torch.randn(m, k, generator=g)
        w = (torch.rand(vocab, k, generator=g) - 0.5) if trans_w else (torch.rand(k, vocab, generator=g) - 0.5)
        b = torch.randn(vocab, generator=g) * 0.1
        targets = torch.randint(0, vocab, (m,), generator=g)
        weights = (torch.rand(m, generator=g) > 0.2).float()
        xd, wd, bd = _leaf(x), _leaf(w), _leaf(b)
        xent, lse, argmax, logits = ops.logits_xent(xd, wd, bd, targets.cuda(), weights.cuda(),
                                                    unk_index=3, trans_w=trans_w, keep_logits=True)
        x64, w64, b64 = (t.double().requires_grad_(True) for t in (x, w, b))
        lg = x64 @ (w64.t() if trans_w else w64) + b64
        unk = torch.zeros(vocab, dtype=torch.float64)
        unk[3] = -1e9
        lg = lg + unk
        ref_lse = torch.logsumexp(lg, -1)
        ref_xent = (ref_lse - lg.gather(1, targets.unsqueeze(1)).squeeze(1)) * weights.double()
        # tf32 products: error grows with sum_k |x_k w_k| ~ 0.2 * K * 2^-11 for these operands
        tol = 1e-5 if backend == "simt" else max(5e-3, 4e-5 * k)
        keep = torch.ones(vocab, dtype=torch.bool)
        keep[3] = False  # the <unk> column holds -1e9 (+ O(1)): 64-ulp fp32 granularity
        assert max_abs(logits.cpu()[:, keep], lg[:, keep]) < tol * 10
        assert float(logits[:, 3].max()) < -9e8
        assert max_abs(lse, ref_lse) < tol
        assert max_abs(xent, ref_xent) < tol * 2
        # argmax: exact wherever the oracle's top-2 margin exceeds the kernel's error
        top2 = lg.topk(2, dim=-1).values
        clear = (top2[:, 0] - top2[:, 1]) > 4 * tol
        assert bool((argmax.cpu()[clear] == lg.argmax(-1)[clear]).all())
        scale = 1.0 / float(weights.sum())
        (xent.sum() * scale).backward()
        (ref_xent.sum() * scale).backward()
        gtol = 1e-4 if backend == "simt" else 3e-3
        assert rel_err(xd.grad, x64.grad) < gtol
        assert rel_err(wd.grad, w64.grad) < gtol
        assert rel_err(bd.grad, b64.grad) < gtol
    finally:
        ops.set_gemm_backend("auto")


def test_linear_and_maxout_grad():
    from neuralmonkey_b200 import ops
    ops.set_gemm_backend("simt")
    try:
        g = torch.Generator().manual_seed(6)
        x, w, b = torch.randn(5, 3, 10, generator=g), torch.randn(10, 8, generator=g), torch.randn(8, generator=g)
        xd, wd, bd = _leaf(x), _leaf(w), _leaf(b)
        y = ops.maxout(ops.linear(xd, wd, bd))
        x64, w64, b64 = (t.double().requires_grad_(True) for t in (x, w, b))
        z = x64 @ w64 + b64
        ref = torch.maximum(z[..., :4], z[..., 4:])
        assert max_abs(y, ref) < 1e-5
        dy = torch.randn(5, 3, 4, generator=g)
        (y * dy.cuda()).sum().backward()
        (ref * dy.double()).sum().backward()
        for got, want in ((xd, x64), (wd, w64), (bd, b64)):
            assert rel_err(got.grad, want.grad) < 1e-5
        xd2, wd2, bd2 = _leaf(x), _leaf(w), _leaf(b)
        y2 = ops.linear(xd2, wd2, bd2, act="tanh")
        x64b, w64b, b64b = (t.double().requires_grad_(True) for t in (x, w, b))
        ref2 = torch.tanh(x64b @ w64b + b64b)
        dy2 = torch.randn(5, 3, 8, generator=g)
        (y2 * dy2.cuda()).sum().backward()
        (ref2 * dy2.double()).sum().backward()
        assert max_abs(y2, ref2) < 1e-5
        for got, want in ((xd2, x64b), (wd2, w64b), (bd2, b64b)):
            assert rel_err(got.grad, want.grad) < 1e-5
    finally:
        ops.set_gemm_backend("auto")


# (bsz, tq, tk, heads, dh): row kernels (tq < 8 or dh % 8 != 0) and tiled kernels (one, two, three
# strips of 64 keys; ragged query blocks; cross-attention shapes)
MHA_SHAPES = [(3, 5, 7, 2, 8), (2, 9, 9, 3, 6), (3, 40, 40, 4, 16), (2, 70, 70, 2, 64),
              (2, 33, 130, 2, 32), (2, 1, 50, 4, 16), (1, 130, 64, 8, 64)]


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("use_mask", [False, True])
@pytest.mark.parametrize("shape", MHA_SHAPES)
def test_mha_core_fwd_bwd(causal, use_mask, shape):
    from neuralmonkey_b200 import ops
    bsz, tq, tk, heads, dh = shape
    if causal:
        tk = tq
    g = torch.Generator().manual_seed(8)
    q, k, v = (torch.randn(bsz, t, heads * dh, generator=g) for t in (tq, tk, tk))
    mask = None
    if use_mask:
        lens = torch.tensor([tk, 3, 1][:bsz])
        mask = (torch.arange(tk).unsqueeze(0) < lens.unsqueeze(1)).float()
    qd, kd, vd = _leaf(q), _leaf(k), _leaf(v)
    ops.set_gemm_backend("simt")          # the exact fp32 kernels (tensor-core attention: test_gpu_mha_tc.py)
    try:
        out, probs = ops.mha_core(qd, kd, vd, mask.cuda() if use_mask else None, causal, heads)
    finally:
        ops.set_gemm_backend("auto")
    q64, k64, v64 = (t.double().requires_grad_(True) for t in (q, k, v))

    def split(t):
        return t.view(bsz, -1, heads, dh).transpose(1, 2)

    e = split(q64 / (dh ** 0.5)) @ split(k64).transpose(-1, -2)
    if causal:
        tri = torch.tril(torch.ones(tq, tk, dtype=torch.bool))
        e = torch.where(tri, e, torch.full_like(e, -1e9))
    if use_mask:
        m4 = mask.double().view(bsz, 1, 1, tk)
        e = e * m4 + (1 - m4) * -1e9
    p = torch.softmax(e, -1)
    ref = (p @ split(v64)).transpose(1, 2).reshape(bsz, tq, heads * dh)
    assert max_abs(probs, p) < 1e-5
    assert max_abs(out, ref) < 1e-5
    do = torch.randn(bsz, tq, heads * dh, generator=g)
    (out * do.cuda()).sum().backward()
    (ref * do.double()).sum().backward()
    for got, want in ((qd, q64), (kd, k64), (vd, v64)):
        assert rel_err(got.grad, want.grad) < 2e-5
