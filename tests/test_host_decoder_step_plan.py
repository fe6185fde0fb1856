"""The launch plan of the fused attention-decoder step (tests/decoder_step_plan.py) on the CPU, at the SM counts of the
H100 SXM (132) and PCIe (114): every named case finds a shape on its branch, the cases together reach every branch
and every refusal of the launcher, and the plan keeps the invariants the kernel relies on.
tests/test_gpu_decoder_step_exact.py checks the restatement against the library on the device."""
import itertools

import pytest

from tests import decoder_step_plan as P


@pytest.mark.parametrize("sms", P.SMS)
@pytest.mark.parametrize("case", P.CASES, ids=lambda c: c.name)
def test_named_case_lands_on_its_branch(case, sms):
    d = P.find_shape(case, sms)
    assert d is not None, "{}: no candidate at {} SMs".format(case.name, sms)
    p = P.plan(d, sms, case.aligned, case.cl)
    assert (p.refusal is None) == (case.near is None), (case.name, p)
    if case.near is not None:
        near = P.plan(case.near(d), sms, case.aligned, case.cl)
        assert near.refusal is None and near.vec == p.vec, (case.name, near)


def _plans(sms):
    out = {}
    for c in P.CASES:
        d = P.find_shape(c, sms)
        out[c.name] = (d, P.plan(d, sms, c.aligned, c.cl))
    return out


@pytest.mark.parametrize("sms", P.SMS)
def test_named_cases_cover_every_branch(sms):
    plans = _plans(sms)
    ok = {n: dp for n, dp in plans.items() if dp[1].refusal is None}
    # cluster size picked by the row count (no override), each with a ragged last cluster
    for cl in (1, 2, 4, 8):
        d, p = ok["cl{}".format(cl)]
        assert p.cl == cl and d.rows % P.DS_R and P.cluster(d.rows, sms) == cl
    assert P.find_shape(next(c for c in P.CASES if c.name == "ende_beam_cl1"), sms).rows == 1024
    # vector and scalar variants: one odd dimension at a time, aligned dimensions over a misaligned base
    assert any(p.vec for _, p in ok.values()) and any(not p.vec for _, p in ok.values())
    base = ok["cl8"][0]
    for dim in ("E", "H", "A", "C", "O"):
        d, p = ok["scalar_odd_" + dim]
        assert not p.vec and [k for k in d._fields if getattr(d, k) != getattr(base, k) and k != "rows"] == [dim]
    d, p = ok["scalar_misaligned"]
    assert not p.vec and P.plan(d, sms).vec
    # TMA ring: tiles of one time step, unequal key / value tiles, an encoder of exactly one key tile and of one
    # step more, many tiles wrapping the ring across several runs of one CTA
    assert ok["tck_1"][1].tck == 1 and ok["tcv_1"][1].tcv == 1
    assert ok["ende_beam_cl1_tiles_of_one_step"][1][4:6] == (1, 1)
    assert any(p.vec and p.tck != p.tcv for _, p in ok.values())
    d, p = ok["tx_is_tck"]
    assert d.Tx == p.tck and p.tcv < d.Tx
    d, p = ok["tx_is_tck_plus_1"]
    assert d.Tx == p.tck + 1
    d, p = ok["ring_wraps_over_runs"]
    assert P.ring_tiles(d, p) > P.DS_SLOTS and max(len(r) for r in P.runs(d, p)) >= 2
    d, p = ok["ende_beam_cl1"]
    assert p.cl == 1 and P.ring_tiles(d, p) >= 2 * P.DS_SLOTS
    # attention runs: one row per run on both variants, runs cut short by jt, a beam spanning two clusters, CTAs
    # with no attended row, CTAs with no columns of a product
    assert P.jt(*ok["jt1_vector"]) == 1 and ok["jt1_vector"][1].vec
    assert P.jt(*ok["jt1_scalar"]) == 1 and not ok["jt1_scalar"][1].vec
    assert ok["group16_spans_clusters"][0].group > P.DS_R
    assert P._has_idle_cta(*ok["idle_ctas"]) and P._cta_without_columns(*ok["cta_without_columns"])
    # ds_panel: every group width and K split the choice can make, on both variants
    seen = set()
    for d, p in ok.values():
        seen |= {(G, gw, min(ws, 2)) for G, gw, ws in P.panels(d, p)}
    reach = P.reachable_panels()
    assert seen >= reach
    assert {gw for G, gw, _ in reach if G == 1} == {2, 4, 8, 16} and {gw for G, gw, _ in reach if G == 4} == {2, 4, 8}
    assert {(G, ws) for G, _, ws in reach} == {(1, 1), (1, 2), (4, 1), (4, 2)}
    # every refusal
    refused = {(p.refusal, p.vec) for d, p in plans.values() if p.refusal}
    assert refused == {("context", False), ("context", True), ("tile", True), ("smem", False)}


@pytest.mark.parametrize("sms", P.SMS)
def test_plan_invariants(sms):
    """What the kernel takes for granted of an accepted plan: the layout fits, a ring slot holds one time step of
    keys and of values, a context column group per thread, the gate and result scratch hold a CTA's columns."""
    for rows, group, E, H, A, C, Tx, O, maxout, aligned, forced in itertools.product(
            (1, 7, 64, 533, 1024), (1, 8), (9, 32, 300), (8, 33, 300, 1024), (14, 64, 600, 4100), (14, 48, 600, 2048),
            (1, 50, 3000), (9, 300), (False, True), (False, True), (None, 1, 8)):
        d = P.Dims(rows, group, E, H, A, C, Tx, O, maxout)
        p = P.plan(d, sms, aligned, forced)
        where = (d, aligned, forced, p)
        if p.refusal is not None:
            continue
        G = 4 if p.vec else 1
        assert p.smem <= 4 * P.MAX_DYN_FLOATS and P.cdiv(C, G) <= P.DS_THREADS, where
        assert P.jt(d, p) >= 1, where
        if p.vec:
            assert p.slot % 32 == 0 and max(A, C) <= p.slot, where
            assert 1 <= p.tck <= Tx and 1 <= p.tcv <= Tx and p.tck * A <= p.slot and p.tcv * C <= p.slot, where
        res_ld = P.align4(P.cdiv(max(2 * H, A, (2 if maxout else 1) * O), p.cl) + 16)
        for rank in range(p.cl):
            un, an, on = (G * P._slice(P.cdiv(n, G), p.cl, rank) for n in (H, A, O))
            assert un <= P.cdiv(H, p.cl) + 8, where                                          # ug scratch
            assert max(2 * un, an, (2 if maxout else 1) * on) <= res_ld, where               # res scratch
