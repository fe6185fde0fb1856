"""nm_gemm_tc_plan on the CPU (the library loads without a GPU): the tile width and split-K plan of nm_gemm's wgmma
engine at the SM counts of the H100 SXM (132) and PCIe (114).  Every plan keeps the invariants the kernel relies
on, agrees with the restatement below over a grid of shapes, and each named case of tests/gemm_plan_cases.py
finds a shape on its branch."""
import itertools

import pytest

from tests import gemm_plan_cases as G

SMS = (132, 114)
ACTS = ("none", "tanh", "relu", "sigmoid")
GRID_M = (1, 37, 128, 129, 300, 1000, 2176, 4224, 8192, 12800, 22528)
GRID_N = (1, 31, 64, 65, 128, 129, 256, 300, 320, 321, 384, 512, 600, 1000, 1024, 1664, 2400, 2432, 4096, 32000)
GRID_K = (1, 31, 32, 480, 511, 512, 544, 1024, 8160, 8191, 8192, 8224, 10240, 12800, 32000)


def restated_plan(m, n, k, act, sms):
    """pick_bn and the two split-K rules of csrc/gemm_tc.cu (tc_dense_plan), restated: a change to the heuristics
    is a deliberate edit in both places."""
    cdiv = G.cdiv
    pad128, pad256, tiles256 = cdiv(n, 128) * 128, cdiv(n, 256) * 256, cdiv(m, 128) * cdiv(n, 256)
    if n <= 64:
        bn = 64
    elif n <= 128:
        bn = 128
    elif k >= 8192 and 256 < n <= 320:
        bn = 160
    elif (pad256 == pad128 and tiles256 >= sms) or (pad256 * 10 <= pad128 * 11 and tiles256 >= 2 * sms):
        bn = 256
    else:
        bn = 128
    tiles, num_kb, want = G.tiles(m, n, bn), cdiv(k, 32), 1
    if act == "none" and 2 * tiles <= sms and num_kb >= 16:
        want = min(cdiv(sms, tiles), num_kb // 8)
    elif act == "none" and num_kb >= 256 and tiles < 4 * sms:
        best_cost = float(cdiv(tiles, sms))
        for sp in range(2, 9):
            if num_kb // sp < 64:
                break
            cost = cdiv(tiles * sp, sms) / sp
            if cost < best_cost * 0.93:
                best_cost, want = cost, sp
    if want <= 1:
        return G.Plan(bn, 1, num_kb)
    kb_per = cdiv(num_kb, want)
    return G.Plan(bn, cdiv(num_kb, kb_per), kb_per)


@pytest.mark.parametrize("sms", SMS)
def test_plan_invariants_and_restatement(sms):
    for m, n, k, act in itertools.product(GRID_M, GRID_N, GRID_K, ACTS):
        p = G.plan(m, n, k, act, sms)
        where = (m, n, k, act, sms, p)
        num_kb, tiles = G.cdiv(k, 32), G.tiles(m, n, p.bn)
        assert p.bn in (64, 128, 160, 256), where
        assert act == "none" or p.splits == 1, where
        assert p.splits >= 1 and p.kb_per * p.splits >= num_kb > p.kb_per * (p.splits - 1), where   # no empty slice
        if p.splits > 1 and 2 * tiles <= sms:
            assert p.splits <= num_kb // 8, where                   # first rule: slices of at least 8 k-blocks
        elif p.splits > 1:
            assert p.splits <= 8 and p.kb_per >= 64 and tiles < 4 * sms, where
        assert p == restated_plan(m, n, k, act, sms), where


@pytest.mark.parametrize("sms", SMS)
@pytest.mark.parametrize("case", G.CASES, ids=lambda c: c.name)
def test_named_case_lands_on_its_branch(case, sms):
    shape = G.find_shape(case, sms)
    assert shape is not None, "{}: no candidate shape at {} SMs".format(case.name, sms)
    rag = G.ragged(shape)
    assert G.plan(*rag, case.act, sms) == G.plan(*shape, case.act, sms), (shape, rag)
    assert case.lands(*rag, sms), rag
    m, n, k = rag
    assert m % 128 and m % 32 and n % 32 and k % 32                   # ragged against every block size
    assert n % G.plan(*rag, case.act, sms).bn


def test_named_cases_cover_every_branch():
    """At either SM count the split cases see both rules and the slice counts 2 to 5 of the second."""
    for sms in SMS:
        plans = {c.name: G.plan(*G.find_shape(c, sms), c.act, sms) for c in G.CASES}
        assert {p.bn for p in plans.values()} == {64, 128, 160, 256}
        assert {plans["split2_sp{}".format(s)].splits for s in range(2, 6)} == {2, 3, 4, 5}
        assert all(p.splits == 1 for name, p in plans.items() if name.startswith(("outside_split", "bn")))
        assert plans["split1_kb17_clamped"] == (64, 2, 9)


@pytest.mark.parametrize("args", [
    (0, 64, 64, 0), (64, 0, 64, 0), (64, 64, 0, 0), (64, 64, 64, 4), (64, 64, 64, -1), (2 ** 31, 64, 64, 0),
])
def test_plan_rejects_bad_arguments(args):
    import ctypes
    from neuralmonkey_b200 import lib
    out = [ctypes.c_int() for _ in range(3)]
    assert lib.load().nm_gemm_tc_plan(*args, 132, *[ctypes.addressof(o) for o in out]) == -1
    assert lib.load().nm_gemm_tc_plan(64, 64, 64, 0, 132, None, None, None) == -1
