"""The convolution weight-gradient plans of tests/conv_plan_cases.py on the CPU, at the SM counts of the H100 SXM
(132) and PCIe (114): every named case finds a shape on its branch for both kernels and both engines, and the
restated plan keeps the invariants the kernels rely on.  tests/test_gpu_conv_exact.py checks the restatement
against the library on the device."""
import itertools

import pytest

from tests import conv_plan_cases as P


@pytest.mark.parametrize("sms", P.SMS)
@pytest.mark.parametrize("engine", ["tc", "simt"])
@pytest.mark.parametrize("case,kind", [(c, k) for c in P.WGRAD_CASES for k in c.kinds],
                         ids=lambda v: v.name if isinstance(v, P.WgradCase) else v)
def test_named_case_lands_on_its_branch(case, kind, engine, sms):
    shape = P.find_shape(case, kind, engine, sms)
    assert shape is not None, "{} {} {}: no candidate at {} SMs".format(case.name, kind, engine, sms)
    p = P.plan_for(kind, engine, shape, sms, P.workspace(case, kind, engine, shape, sms))
    if case.name == "ws_one_slice":
        assert p.splits == 1
    if case.name == "ws_between_slices":
        full = P.plan_for(kind, engine, shape, sms)
        assert 1 < p.splits < full.splits and P.workspace(case, kind, engine, shape, sms) % p.part


@pytest.mark.parametrize("sms", P.SMS)
def test_plan_invariants(sms):
    """No empty split, no split past the workspace or the launch limit, at least one split."""
    for rows, cols, m, (kind, engine), cap in itertools.product(
            (2, 28, 128, 129, 300, 4105), (1, 8, 63, 64, 65, 130, 1024), (1, 31, 32, 33, 800, 20000, 10 ** 6),
            P.TILES, (-1, 0, 1, 2, 7, 10 ** 9)):
        t = P.TILES[(kind, engine)]
        p = P.wgrad_plan(rows, cols, m, t, sms, cap * rows * cols if cap > 0 else cap)
        nkb = P.cdiv(m, t.bk)
        where = (rows, cols, m, kind, engine, cap, p)
        assert p.splits >= 1 and p.kb_per * p.splits >= nkb > p.kb_per * (p.splits - 1), where
        assert p.splits <= min(65535, nkb), where
        if cap > 0:
            assert p.splits <= cap, where


def test_cases_cover_the_plan_branches():
    """At either SM count the cases see one split, one k-block per split, uneven splits and both workspace caps."""
    for sms in P.SMS:
        for kind, engine in P.TILES:
            plans = {}
            for c in P.WGRAD_CASES:
                if kind in c.kinds:
                    s = P.find_shape(c, kind, engine, sms)
                    plans[c.name] = P.plan_for(kind, engine, s, sms, P.workspace(c, kind, engine, s, sms))
            assert plans["splits1_full_grid"].splits == 1
            assert plans["one_kblock_per_split"].kb_per == 1 < plans["one_kblock_per_split"].splits
            assert plans["uneven_last_split"].kb_per > 1
            assert plans["ws_one_slice"].splits == 1
            assert plans["rows_129"].rows == 129 and plans["rows_128"].rows == 128
