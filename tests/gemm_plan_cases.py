"""The launch-time choices of nm_gemm's wgmma engine (csrc/gemm_tc.cu, tc_dense_plan) as named cases.

Every tile width and each split-K rule gets a shape that lands on it, and each rule a shape just outside it.  The
shapes are not fixed: each case searches candidate shapes with nm_gemm_tc_plan at a given SM count, so a case
names the same branch on a 132-SM and a 114-SM H100.  A base shape has M a multiple of 128, N and K multiples of
32; `ragged` trims M by 37 rows, N by 5 columns and K by 7 elements, which keeps every tile and k-block count and
therefore the plan (tests/test_host_gemm_plan.py checks that)."""
import ctypes
from typing import Callable, NamedTuple, Optional, Sequence, Tuple

BM, BK = 128, 32
ACT = {"none": 0, "tanh": 1, "relu": 2, "sigmoid": 3}
RAGGED_M, RAGGED_N, RAGGED_K = 37, 5, 7


class Plan(NamedTuple):
    bn: int
    splits: int
    kb_per: int


def plan(m: int, n: int, k: int, act: str = "none", sms: int = 0) -> Plan:
    """nm_gemm_tc_plan: the plan nm_gemm's wgmma engine uses for this product on `sms` SMs (0: this device)."""
    from neuralmonkey_b200 import lib
    bn, splits, kb = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    lib.call("nm_gemm_tc_plan", m, n, k, ACT[act], sms, ctypes.addressof(bn), ctypes.addressof(splits),
             ctypes.addressof(kb))
    return Plan(bn.value, splits.value, kb.value)


def cdiv(a: int, b: int) -> int:
    return -(-a // b)


def tiles(m: int, n: int, bn: int) -> int:
    return cdiv(m, BM) * cdiv(n, bn)


def first_rule(m: int, n: int, k: int, sms: int) -> bool:
    """Split by the first rule: an output that fills at most half the SMs."""
    p = plan(m, n, k, "none", sms)
    return p.splits > 1 and 2 * tiles(m, n, p.bn) <= sms


def second_rule(m: int, n: int, k: int, sms: int) -> bool:
    """Split by the second rule: a few waves of very long tiles."""
    p = plan(m, n, k, "none", sms)
    return p.splits > 1 and 2 * tiles(m, n, p.bn) > sms


def equal_padding(n: int) -> bool:
    return cdiv(n, 256) * 256 == cdiv(n, 128) * 128


class Case(NamedTuple):
    name: str
    act: str
    ns: Sequence[int]
    ks: Sequence[int]
    lands: Callable[[int, int, int, int], bool]   # (m, n, k, sms) -> the shape is on this case's branch


def _unclamped_first(m, n, k, sms):
    p = plan(m, n, k, "none", sms)
    return first_rule(m, n, k, sms) and cdiv(sms, tiles(m, n, p.bn)) <= cdiv(k, BK) // 8 and p.splits >= 3


def _clamped_first(kb_per):
    def lands(m, n, k, sms):
        p = plan(m, n, k, "none", sms)
        return (first_rule(m, n, k, sms) and cdiv(sms, tiles(m, n, p.bn)) > cdiv(k, BK) // 8
                and (p.splits, p.kb_per) == (2, kb_per))
    return lands


def _second(sp):
    return lambda m, n, k, sms: second_rule(m, n, k, sms) and plan(m, n, k, "none", sms).splits == sp


_SECOND_NS = (256, 384, 512, 640, 768, 1024)

CASES = [
    Case("bn64", "relu", (64,), (96,), lambda m, n, k, sms: plan(m, n, k, "relu", sms).bn == 64),
    Case("bn128", "none", (128,), (64,), lambda m, n, k, sms: plan(m, n, k, "none", sms) == (128, 1, 2)),
    Case("bn160", "sigmoid", (320,), (8224,), lambda m, n, k, sms: plan(m, n, k, "sigmoid", sms).bn == 160),
    Case("bn256_equal_padding", "none", (1024,), (64,),
         lambda m, n, k, sms: plan(m, n, k, "none", sms).bn == 256 and equal_padding(n)),
    Case("bn256_within_10pct", "relu", (2432,), (64,),
         lambda m, n, k, sms: plan(m, n, k, "relu", sms).bn == 256 and not equal_padding(n)),
    Case("split1_kb16_clamped", "none", (64,), (512,), _clamped_first(8)),
    Case("split1_kb17_clamped", "none", (64,), (544,), _clamped_first(9)),     # slices of 9 and 8 k-blocks
    Case("split1_unclamped", "none", (600,), (12800,), _unclamped_first),
    Case("split2_sp2", "none", _SECOND_NS, (8192, 10240), _second(2)),
    Case("split2_sp3", "none", _SECOND_NS, (8192, 10240), _second(3)),
    Case("split2_sp4", "none", _SECOND_NS, (8192, 10240), _second(4)),
    Case("split2_sp5", "none", _SECOND_NS, (10240,), _second(5)),
    Case("split2_shape_with_tanh", "tanh", _SECOND_NS, (8192,),
         lambda m, n, k, sms: second_rule(m, n, k, sms) and plan(m, n, k, "tanh", sms).splits == 1),
    # just outside each rule: one k-block or one row of tiles short of it (or past it)
    Case("outside_split1_kb15", "none", (64,), (480,),
         lambda m, n, k, sms: plan(m, n, k, "none", sms).splits == 1 and first_rule(m, n, k + BK, sms)),
    Case("outside_split1_tiles", "none", (128, 256), (1024,),
         lambda m, n, k, sms: m > BM and plan(m, n, k, "none", sms).splits == 1 and first_rule(m - BM, n, k, sms)),
    Case("outside_split2_kb255", "none", _SECOND_NS, (8160,),
         lambda m, n, k, sms: plan(m, n, k, "none", sms).splits == 1 and second_rule(m, n, k + BK, sms)),
    Case("outside_split2_tiles", "none", (384, 640, 896, 1152, 128), (8192,),
         lambda m, n, k, sms: (plan(m, n, k, "none", sms).splits == 1
                               and tiles(m, n, 128) >= 4 * sms > tiles(m - BM, n, 128)
                               and plan(m, n, k, "none", sms).bn == 128)),
    Case("outside_bn256_equal_padding", "none", (256, 512, 768, 1024), (64,),
         lambda m, n, k, sms: (equal_padding(n) and plan(m, n, k, "none", sms).bn == 128
                               and plan(m + BM, n, k, "none", sms).bn == 256)),
    Case("outside_bn256_within_10pct", "none", (1664, 2432), (64,),
         lambda m, n, k, sms: (not equal_padding(n) and plan(m, n, k, "none", sms).bn == 128
                               and plan(m + BM, n, k, "none", sms).bn == 256)),
]

MAX_ROW_TILES = 320


def find_shape(case: Case, sms: int) -> Optional[Tuple[int, int, int]]:
    """The cheapest candidate (m, n, k) on the case's branch at `sms` SMs (fewest multiply-adds, then the smallest
    operands), or None."""
    cands = sorted(((BM * t, n, k) for t in range(1, MAX_ROW_TILES + 1) for n in case.ns for k in case.ks),
                   key=lambda s: (s[0] * s[1] * s[2], (s[0] + s[1]) * s[2]))
    for m, n, k in cands:
        if case.lands(m, n, k, sms):
            return m, n, k
    return None


def ragged(shape: Tuple[int, int, int]) -> Tuple[int, int, int]:
    m, n, k = shape
    return m - RAGGED_M, n - RAGGED_N, k - RAGGED_K
