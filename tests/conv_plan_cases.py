"""The weight-gradient plan of the convolution kernels (csrc/conv_igemm.cuh wgrad_plan, for conv2d's and the GLU
conv's tiles) restated in Python, and named cases that each land on one branch of it.

Both convolutions sum dW[r, o] = sum_m A'(r, m) dY(m, o) over the m = output pixels (positions) in k-blocks, split over
CTAs into a workspace of [rows, cols] slices, rows = (filter taps x input channels) + 1 for the bias row.  The
split count asks for about 4 CTAs per SM, at most one per k-block, at most what the workspace holds; the k-blocks
are then dealt out evenly, so the last split may be shorter.  The shapes of a case are not fixed: each case
searches its candidates at a given SM count, so it names the same branch on a 132-SM and a 114-SM H100."""
from typing import Callable, NamedTuple, Optional, Sequence, Tuple

SMS = (132, 114)          # H100 SXM and PCIe


class Tiles(NamedTuple):
    bm: int      # rows of A' per CTA
    bn: int      # output columns per CTA
    bk: int      # pixels per k-block


# (kind, engine) -> the weight-gradient tile: wgmma 128 x 64 (conv2d) or 128 x 128 (GLU) with k-blocks of 32,
# CUDA cores 64 x 64 with k-blocks of 16
TILES = {
    ("conv2d", "tc"): Tiles(128, 64, 32), ("conv2d", "simt"): Tiles(64, 64, 16),
    ("glu", "tc"): Tiles(128, 128, 32), ("glu", "simt"): Tiles(64, 64, 16),
}


class Plan(NamedTuple):
    rows: int
    part: int        # floats of one workspace slice
    tiles_r: int
    tiles_o: int
    splits: int
    kb_per: int


def cdiv(a: int, b: int) -> int:
    return -(-a // b)


def wgrad_plan(rows: int, cols: int, m: int, tiles: Tiles, sms: int, ws_cap: int = -1) -> Plan:
    """wgrad_plan: ws_cap < 0 is an unbounded workspace."""
    part = rows * cols
    tiles_r, tiles_o = cdiv(rows, tiles.bm), cdiv(cols, tiles.bn)
    total_kb = cdiv(m, tiles.bk)
    splits = min(cdiv(4 * sms, tiles_r * tiles_o), total_kb)
    if ws_cap >= 0:
        splits = min(splits, ws_cap // part)
    splits = max(1, min(splits, 65535))
    kb_per = cdiv(total_kb, splits)
    return Plan(rows, part, tiles_r, tiles_o, cdiv(total_kb, kb_per), kb_per)


# ---- geometry of a case's shape ----
# conv2d: (N, H, W, Cin, Cout, k, (pt, pb, pl, pr));  GLU conv1d: (B, T, F, k) with TF's `same` padding

def conv_out(shape) -> Tuple[int, int]:
    n, h, w, cin, cout, k, (pt, pb, pl, pr) = shape
    return h + pt + pb - k + 1, w + pl + pr - k + 1


def gemm_dims(kind: str, shape) -> Tuple[int, int, int]:
    """(rows of A' including the bias row, output columns, pixels) of the weight-gradient product."""
    if kind == "conv2d":
        n, h, w, cin, cout, k, pads = shape
        ho, wo = conv_out(shape)
        return k * k * cin + 1, cout, n * ho * wo
    b, t, f, k = shape
    return k * f + 1, 2 * f, b * t


def total_kb(kind: str, engine: str, shape) -> int:
    return cdiv(gemm_dims(kind, shape)[2], TILES[(kind, engine)].bk)


def plan_for(kind: str, engine: str, shape, sms: int, ws_cap: int = -1) -> Plan:
    rows, cols, m = gemm_dims(kind, shape)
    return wgrad_plan(rows, cols, m, TILES[(kind, engine)], sms, ws_cap)


class WgradCase(NamedTuple):
    name: str
    kinds: Sequence[str]                       # "conv2d", "glu"
    conv: Sequence                             # candidate conv2d shapes
    glu: Sequence                              # candidate GLU shapes
    lands: Callable                            # (kind, engine, shape, sms) -> on this case's branch
    ws: Callable = lambda full: -1             # workspace floats from the unbounded plan (-1: exactly that plan)
    db: bool = True                            # pass a bias gradient


def _same(k):
    return ((k - 1) // 2, k - 1 - (k - 1) // 2) * 2


def _valid():
    return (0, 0, 0, 0)


def _splits(kind, engine, shape, sms):
    return plan_for(kind, engine, shape, sms).splits


def _single_split(kind, engine, shape, sms):
    return _splits(kind, engine, shape, sms) == 1 and total_kb(kind, engine, shape) > 1


def _one_kb(kind, engine, shape, sms):
    p = plan_for(kind, engine, shape, sms)
    return p.kb_per == 1 and p.splits > 1


def _uneven(kind, engine, shape, sms):
    p = plan_for(kind, engine, shape, sms)
    return p.splits > 1 and p.kb_per > 1 and total_kb(kind, engine, shape) % p.kb_per != 0


def _ragged_m(kind, engine, shape, sms):
    return gemm_dims(kind, shape)[2] % 32 not in (0, 16) and _splits(kind, engine, shape, sms) > 1


def _several(kind, engine, shape, sms):
    return _splits(kind, engine, shape, sms) >= 2


def _between(kind, engine, shape, sms):
    full = plan_for(kind, engine, shape, sms)
    capped = plan_for(kind, engine, shape, sms, _ws_between(full))
    return full.splits >= 4 and 1 < capped.splits < full.splits and _ws_between(full) % full.part != 0


def _ws_between(full: Plan) -> int:
    return full.splits // 2 * full.part + full.part // 3


def _rows(r):
    return lambda kind, engine, shape, sms: gemm_dims(kind, shape)[0] == r and _splits(kind, engine, shape, sms) > 1


def _cols(c):
    return lambda kind, engine, shape, sms: gemm_dims(kind, shape)[1] == c and _splits(kind, engine, shape, sms) > 1


_BIG_FILTER_CONV = [(1, 6, 6, cin, 1024, 3, _same(3)) for cin in (456, 512)]
_BIG_FILTER_GLU = [(1, 40, f, 3) for f in (1200, 1400)]
_SMALL_CONV = [(2, 20, 20, 4, 8, 3, _same(3))]
_SMALL_GLU = [(4, 50, 8, 3)]
# k-blocks beyond 4 CTAs per SM: an odd number of pixels makes an odd k-block count
_LONG_CONV = [(n, 29, 29, 2, 4, 3, _same(3)) for n in range(20, 80)]
_LONG_GLU = [(b, 37, 4, 3) for b in range(440, 1400, 7)]

WGRAD_CASES = [
    WgradCase("splits1_full_grid", ("conv2d", "glu"), _BIG_FILTER_CONV, _BIG_FILTER_GLU, _single_split),
    WgradCase("one_kblock_per_split", ("conv2d", "glu"), _SMALL_CONV, _SMALL_GLU, _one_kb),
    WgradCase("uneven_last_split", ("conv2d", "glu"), _LONG_CONV, _LONG_GLU, _uneven),
    WgradCase("m_not_multiple_of_32", ("conv2d", "glu"), [(1, 13, 19, 3, 5, 3, _same(3))], [(3, 41, 5, 2)],
              _ragged_m),
    WgradCase("ws_one_slice", ("conv2d", "glu"), _SMALL_CONV, _SMALL_GLU, _several, ws=lambda full: full.part),
    WgradCase("ws_between_slices", ("conv2d", "glu"), _SMALL_CONV + _LONG_CONV, _SMALL_GLU + _LONG_GLU, _between,
              ws=_ws_between),
    WgradCase("rows_128", ("conv2d", "glu"), [(1, 9, 9, 127, 8, 1, _valid())], [(2, 30, 127, 1)], _rows(128)),
    WgradCase("rows_129", ("conv2d", "glu"), [(1, 9, 9, 8, 8, 4, _same(4))], [(2, 30, 64, 2)], _rows(129)),
    WgradCase("cout_63", ("conv2d",), [(1, 9, 11, 5, 63, 3, _same(3))], [], _cols(63)),
    WgradCase("cout_64", ("conv2d",), [(1, 9, 11, 5, 64, 3, _same(3))], [], _cols(64)),
    WgradCase("cout_65", ("conv2d",), [(1, 9, 11, 5, 65, 3, _same(3))], [], _cols(65)),
    WgradCase("db_null", ("conv2d",), [(2, 7, 9, 6, 12, 2, _same(2))], [], _several, db=False),
]


def find_shape(case: WgradCase, kind: str, engine: str, sms: int) -> Optional[tuple]:
    """The first candidate of the case that lands on its branch at `sms` SMs, or None."""
    for shape in (case.conv if kind == "conv2d" else case.glu):
        if case.lands(kind, engine, shape, sms):
            return shape
    return None


def workspace(case: WgradCase, kind: str, engine: str, shape, sms: int) -> int:
    """Workspace floats handed to the kernel: the unbounded plan's, or the case's cap."""
    full = plan_for(kind, engine, shape, sms)
    ws = case.ws(full)
    return full.splits * full.part if ws < 0 else ws
