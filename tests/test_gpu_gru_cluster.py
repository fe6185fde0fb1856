"""The persistent cluster GRU recurrence (nm_gru_seq_fwd / nm_gru_seq_bwd) against the fp64 oracle at the exact
tolerances, over batch sizes that leave a partial cluster, every slice length class of H and single-step
sequences; plus run-to-run determinism and the two-direction entry points."""
import pytest
import torch

from oracle import nm_oracle as O
from tests.helpers import max_abs, rel_err

pytestmark = pytest.mark.gpu

TOL, GTOL = 2e-5, 5e-5


def _leaf(t):
    return t.clone().cuda().requires_grad_(True)


def _weights(g, e, h, ws=0.3):
    wg, bg = torch.randn(e + h, 2 * h, generator=g) * ws, torch.randn(2 * h, generator=g) * 0.3
    wc, bc = torch.randn(e + h, h, generator=g) * ws, torch.randn(h, generator=g) * 0.3
    return wg, bg, wc, bc


def _reverse_sequence(x, lengths):
    """tf.reverse_sequence(x, lengths, seq_axis=1) as one gather: O.reverse_sequence walks the batch row by row,
    which autograd makes slow at a thousand rows."""
    t = torch.arange(x.shape[1])[None, :]
    n = lengths.long()[:, None]
    idx = torch.where(t < n, n - 1 - t, t)
    return x.gather(1, idx[:, :, None].expand(-1, -1, x.shape[2]))


def _lengths(g, bsz, steps):
    lengths = torch.randint(1, steps + 1, (bsz,), generator=g)
    lengths[0] = steps
    lengths[-1] = 1
    return lengths


# (B, T, H): partial clusters (B=17, 300), one row, every width class of the reduction slice
SHAPES = [(1, 1, 8), (17, 50, 8), (256, 1, 8), (300, 50, 100), (1, 50, 100), (17, 1, 300), (256, 50, 300),
          (300, 1, 320), (17, 50, 320),
          # H where ceil(H/8) units per CTA would leave the last CTAs of a cluster without units
          (17, 50, 9), (33, 20, 33), (5, 50, 49),
          # more clusters than are co-resident (15 on an H100): shared memory caps a cluster at 32 rows forward
          # and 22 backward for H = 320, 68 and 42 for H = 100, so these run in several waves
          (1024, 20, 320), (1100, 10, 100)]


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("variant", ["plain", "lengths_reverse_h0"])
def test_cluster_gru_vs_oracle(shape, variant):
    from neuralmonkey_b200 import ops
    bsz, steps, h = shape
    e = 16
    ops.set_gemm_backend("simt")
    try:
        g = torch.Generator().manual_seed(11 + bsz + steps + h)
        x = torch.randn(bsz, steps, e, generator=g)
        # gain ~1: at H=320 a gain-5 recurrence amplifies rounding past any fixed tolerance over 50 steps
        wg, bg, wc, bc = _weights(g, e, h, ws=min(0.3, 1.0 / h ** 0.5))
        use_extra = variant != "plain"
        h0 = torch.randn(bsz, h, generator=g) * 0.5 if use_extra else None
        lengths = _lengths(g, bsz, steps) if use_extra else None
        reverse = use_extra
        tensors = (x, wg, bg, wc, bc) + ((h0,) if h0 is not None else ())
        leaves = [_leaf(t) for t in tensors]
        ld = lengths.to(torch.int32).cuda() if lengths is not None else None
        states, final, _raw = ops.gru_layer(*leaves[:5], h0=leaves[5] if h0 is not None else None, lengths=ld,
                                            reverse=reverse)
        l64 = [t.double().requires_grad_(True) for t in tensors]
        h064 = l64[5] if h0 is not None else None
        if reverse:
            out_rev, fin = O.dynamic_gru(_reverse_sequence(l64[0], lengths), lengths, *l64[1:5], h0=h064)
            ref_states = _reverse_sequence(out_rev, lengths)
        else:
            ref_states, fin = O.dynamic_gru(l64[0], lengths, *l64[1:5], h0=h064)
        assert max_abs(states, ref_states) < TOL
        assert max_abs(final, fin) < TOL
        ds, df = torch.randn(bsz, steps, h, generator=g), torch.randn(bsz, h, generator=g)
        ((states * ds.cuda()).sum() + (final * df.cuda()).sum()).backward()
        ((ref_states * ds.double()).sum() + (fin * df.double()).sum()).backward()
        for got, want, name in zip(leaves, l64, ("x", "wg", "bg", "wc", "bc", "h0")):
            assert rel_err(got.grad, want.grad) < GTOL, name
    finally:
        ops.set_gemm_backend("auto")


@pytest.mark.parametrize("use_h0", [False, True])
@pytest.mark.parametrize("reverse", [False, True])
@pytest.mark.parametrize("shape", [(17, 12, 100), (9, 12, 300), (5, 8, 7), (6, 5, 330)])
def test_gru_zero_lengths(shape, reverse, use_h0):
    """Rows of length 0 among ragged ones, on the cluster kernels (H = 100, 300) and the per-step kernels (H = 7,
    330), as tf.nn.dynamic_rnn treats them: zero outputs, the final state is h0 (zeros without one), dh0 is
    dfinal and nothing flows into the inputs.  Those rows only carry values, so they compare exactly; the whole
    layer compares with the oracle at the exact tolerances."""
    from neuralmonkey_b200 import ops
    bsz, steps, h = shape
    e = 10
    ops.set_gemm_backend("simt")
    try:
        g = torch.Generator().manual_seed(bsz * steps + h)
        x = torch.randn(bsz, steps, e, generator=g)
        wg, bg, wc, bc = _weights(g, e, h, ws=min(0.3, 1.0 / h ** 0.5))
        lengths = torch.randint(1, steps + 1, (bsz,), generator=g)
        lengths[0] = steps
        zero = torch.arange(bsz) % 3 == 1
        lengths[zero] = 0
        h0 = torch.randn(bsz, h, generator=g) * 0.5 if use_h0 else None
        tensors = (x, wg, bg, wc, bc) + ((h0,) if use_h0 else ())
        leaves = [_leaf(t) for t in tensors]
        states, final, _raw = ops.gru_layer(*leaves[:5], h0=leaves[5] if use_h0 else None,
                                            lengths=lengths.to(torch.int32).cuda(), reverse=reverse)
        l64 = [t.double().requires_grad_(True) for t in tensors]
        h064 = l64[5] if use_h0 else None
        if reverse:
            out_rev, fin = O.dynamic_gru(_reverse_sequence(l64[0], lengths), lengths, *l64[1:5], h0=h064)
            ref_states = _reverse_sequence(out_rev, lengths)
        else:
            ref_states, fin = O.dynamic_gru(l64[0], lengths, *l64[1:5], h0=h064)
        assert torch.equal(states[zero.cuda()].cpu(), torch.zeros(int(zero.sum()), steps, h))
        assert torch.equal(final[zero.cuda()].cpu(), h0[zero] if use_h0 else torch.zeros(int(zero.sum()), h))
        assert max_abs(states, ref_states) < TOL
        assert max_abs(final, fin) < TOL
        ds, df = torch.randn(bsz, steps, h, generator=g), torch.randn(bsz, h, generator=g)
        ((states * ds.cuda()).sum() + (final * df.cuda()).sum()).backward()
        ((ref_states * ds.double()).sum() + (fin * df.double()).sum()).backward()
        assert torch.equal(leaves[0].grad[zero.cuda()].cpu(), torch.zeros(int(zero.sum()), steps, e))
        if use_h0:
            assert torch.equal(leaves[5].grad[zero.cuda()].cpu(), df[zero])
        for got, want, name in zip(leaves, l64, ("x", "wg", "bg", "wc", "bc", "h0")):
            assert rel_err(got.grad, want.grad) < GTOL, name
    finally:
        ops.set_gemm_backend("auto")


@pytest.mark.parametrize("shape", [(17, 50, 100), (300, 7, 320), (1, 1, 8)])
def test_cluster_gru_drop_mask_raw_outputs(shape):
    """The state fed back is the dropped-out output (dropout mask and raw outputs on the cluster path), with
    gradients arriving through the dropped outputs, the raw outputs and the final state."""
    from neuralmonkey_b200 import ops
    bsz, steps, h = shape
    e = 12
    ops.set_gemm_backend("simt")
    try:
        g = torch.Generator().manual_seed(7 + h)
        x = torch.randn(bsz, steps, e, generator=g)
        wg, bg, wc, bc = _weights(g, e, h, ws=min(0.3, 1.0 / h ** 0.5))
        mask = (torch.rand(bsz, steps, h, generator=g) < 0.7).float() / 0.7
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
        assert max_abs(raw, ref_raw) < TOL and max_abs(dropped, ref_drop) < TOL
        assert max_abs(final, hprev) < TOL
        d1, d2 = torch.randn(bsz, steps, h, generator=g), torch.randn(bsz, steps, h, generator=g)
        df = torch.randn(bsz, h, generator=g)
        ((dropped * d1.cuda()).sum() + (raw * d2.cuda()).sum() + (final * df.cuda()).sum()).backward()
        ((ref_drop * d1.double()).sum() + (ref_raw * d2.double()).sum() + (hprev * df.double()).sum()).backward()
        for got, want in zip(leaves, l64):
            assert rel_err(got.grad, want.grad) < GTOL
    finally:
        ops.set_gemm_backend("auto")


def _raw_fwd(xproj, wg, wc, h0, lengths, reverse, bsz, steps, h):
    from neuralmonkey_b200 import lib
    from neuralmonkey_b200.lib import call, ptr
    dev = xproj.device
    out = {n: torch.empty(bsz, steps, k * h, device=dev) for n, k in (("states", 1), ("gates", 3), ("hprev", 1),
                                                                      ("rh", 1))}
    out["final"] = torch.empty(bsz, h, device=dev)
    call("nm_gru_seq_fwd", ptr(xproj), ptr(wg), ptr(wc), ptr(h0), ptr(lengths), None, int(reverse),
         ptr(out["states"]), None, ptr(out["final"]), ptr(out["gates"]), ptr(out["hprev"]), ptr(out["rh"]),
         bsz, steps, h, 0, lib.stream())
    return out


def _raw_bwd(wg, wc, lengths, reverse, fwd, dstates, dfinal, bsz, steps, h):
    from neuralmonkey_b200 import lib
    from neuralmonkey_b200.lib import call, ptr
    dev = dstates.device
    dxproj = torch.empty(bsz, steps, 3 * h, device=dev)
    dh0 = torch.empty(bsz, h, device=dev)
    work = torch.empty(2 * bsz * h, device=dev)
    call("nm_gru_seq_bwd", ptr(wg), ptr(wc), ptr(lengths), None, int(reverse), ptr(fwd["gates"]),
         ptr(fwd["hprev"]), ptr(dstates), None, ptr(dfinal), ptr(dxproj), ptr(dh0), ptr(work), bsz, steps, h, 0,
         lib.stream())
    return dxproj, dh0


def _raw_inputs(bsz, steps, h, seed):
    g = torch.Generator().manual_seed(seed)
    xproj = (torch.randn(bsz, steps, 3 * h, generator=g) * 0.5).cuda()
    wg = (torch.randn(h, 2 * h, generator=g) / h ** 0.5).cuda()
    wc = (torch.randn(h, h, generator=g) / h ** 0.5).cuda()
    h0 = (torch.randn(bsz, h, generator=g) * 0.5).cuda()
    lengths = _lengths(g, bsz, steps).to(torch.int32).cuda()
    dstates = torch.randn(bsz, steps, h, generator=g).cuda()
    dfinal = torch.randn(bsz, h, generator=g).cuda()
    return xproj, wg, wc, h0, lengths, dstates, dfinal


def test_cluster_gru_bit_identical_repeats():
    bsz, steps, h = 256, 50, 300
    xproj, wg, wc, h0, lengths, dstates, dfinal = _raw_inputs(bsz, steps, h, 3)
    runs = []
    for _ in range(2):
        f = _raw_fwd(xproj, wg, wc, h0, lengths, True, bsz, steps, h)
        dx, dh0 = _raw_bwd(wg, wc, lengths, True, f, dstates, dfinal, bsz, steps, h)
        runs.append([f["states"], f["final"], f["gates"], f["hprev"], f["rh"], dx, dh0])
    torch.cuda.synchronize()
    for a, b in zip(*runs):
        assert torch.equal(a, b)


def test_cluster_gru_pair_equals_two_calls():
    from neuralmonkey_b200 import lib
    from neuralmonkey_b200.lib import call, ptr
    bsz, steps, h = 17, 50, 300
    xa, wga, wca, _h0, lengths, dsa, dfa = _raw_inputs(bsz, steps, h, 4)
    xb, wgb, wcb, _h0, _l, dsb, dfb = _raw_inputs(bsz, steps, h, 5)
    singles = [_raw_fwd(xa, wga, wca, None, lengths, False, bsz, steps, h),
               _raw_fwd(xb, wgb, wcb, None, lengths, True, bsz, steps, h)]
    pair = [{n: torch.empty_like(v) for n, v in s.items()} for s in singles]
    pa, pb = pair
    call("nm_gru_seq_fwd_pair",
         ptr(xa), ptr(wga), ptr(wca), 0, ptr(pa["states"]), ptr(pa["final"]), ptr(pa["gates"]), ptr(pa["hprev"]),
         ptr(pa["rh"]),
         ptr(xb), ptr(wgb), ptr(wcb), 1, ptr(pb["states"]), ptr(pb["final"]), ptr(pb["gates"]), ptr(pb["hprev"]),
         ptr(pb["rh"]),
         ptr(lengths), bsz, steps, h, lib.stream())
    for s, p in zip(singles, pair):
        for n in s:
            assert torch.equal(s[n], p[n]), n
    da, _ = _raw_bwd(wga, wca, lengths, False, singles[0], dsa, dfa, bsz, steps, h)
    db, _ = _raw_bwd(wgb, wcb, lengths, True, singles[1], dsb, dfb, bsz, steps, h)
    pda, pdb = torch.empty_like(da), torch.empty_like(db)
    work = torch.empty(2 * bsz * h, device=da.device)
    call("nm_gru_seq_bwd_pair",
         ptr(wga), ptr(wca), 0, ptr(pa["gates"]), ptr(pa["hprev"]), ptr(dsa), ptr(dfa), ptr(pda),
         ptr(wgb), ptr(wcb), 1, ptr(pb["gates"]), ptr(pb["hprev"]), ptr(dsb), ptr(dfb), ptr(pdb),
         ptr(lengths), ptr(work), bsz, steps, h, lib.stream())
    torch.cuda.synchronize()
    assert torch.equal(da, pda) and torch.equal(db, pdb)
