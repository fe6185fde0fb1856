"""The launch plan of the fused attention-decoder step (csrc/decoder_step.cu: ds_plan, ds_layout, the attention run
schedule and ds_panel's warp grouping) restated in Python, and named cases that each land on one branch of it.

A cluster of `cl` CTAs owns 8 rows; each CTA attends for 8 / cl of them.  The vector variant (16-byte loads, key /
value tiles staged through a 4-slot TMA ring) needs E, H, A, C, O % 4 == 0 and 16-byte aligned weight, key and value
bases; everything else runs the scalar variant.  The shapes of a case are not fixed: each case searches its
candidates at a given SM count, so it names the same branch on a 132-SM and a 114-SM H100."""
from typing import Callable, List, NamedTuple, Optional, Sequence, Set, Tuple

SMS = (132, 114)          # H100 SXM and PCIe
DS_R, DS_THREADS, DS_WARPS, DS_SLOTS = 8, 512, 16, 4
DS_RED_FLOATS = 128 * 32
MAX_DYN_FLOATS = (227 * 1024 - 1024) // 4
SLOT_CAP = 8192


class Dims(NamedTuple):
    rows: int
    group: int
    E: int
    H: int
    A: int
    C: int
    Tx: int
    O: int
    maxout: bool


class Plan(NamedTuple):
    refusal: Optional[str]   # None, "context", "tile" or "smem"
    vec: bool
    cl: int
    slot: int                # floats per ring slot (vector variant)
    tck: int                 # time steps per staged key / value tile
    tcv: int
    smem: int                # bytes of dynamic shared memory


def cdiv(a: int, b: int) -> int:
    return -(-a // b)


def align4(x: int) -> int:
    return (x + 3) & ~3


def layout_total(d: Dims, cl: int, slot: int, tma: bool) -> int:
    """ds_layout(...).total in floats."""
    rpc = DS_R // cl
    maxn = max(2 * d.H, d.A, (2 if d.maxout else 1) * d.O)
    res_ld = align4(cdiv(maxn, cl) + 16)
    total = (align4(d.E * DS_R) + 3 * align4(d.H * DS_R) + align4(d.C * DS_R)
             + align4(DS_R * (cdiv(d.H, cl) + 8)) + DS_R * res_ld + DS_RED_FLOATS
             + align4(rpc * d.A) + align4(rpc * d.Tx) + align4(d.A))
    return total + (DS_SLOTS * slot if tma else 0) + 4 * DS_SLOTS


def cluster(rows: int, sms: int, forced: Optional[int] = None) -> int:
    """As many CTAs per cluster as fill the chip, at most 8; NMB200_DECSTEP_CLUSTER = 1, 2, 4 or 8 overrides."""
    if forced:
        return forced
    cl, clusters = 8, cdiv(rows, DS_R)
    while cl > 1 and clusters * cl > sms:
        cl //= 2
    return cl


def plan(d: Dims, sms: int, aligned: bool = True, forced_cl: Optional[int] = None) -> Plan:
    vec = aligned and all(x % 4 == 0 for x in (d.E, d.H, d.A, d.C, d.O))
    cl = cluster(d.rows, sms, forced_cl)
    if cdiv(d.C, 4 if vec else 1) > DS_THREADS:
        return Plan("context", vec, cl, 0, 0, 0, 0)
    if not vec:
        smem = 4 * layout_total(d, cl, 0, False)
        return Plan("smem" if smem > 4 * MAX_DYN_FLOATS else None, vec, cl, 0, d.Tx, d.Tx, smem)
    slot = (MAX_DYN_FLOATS - layout_total(d, cl, 0, True)) // DS_SLOTS
    slot -= slot % 32
    need = max(d.A, d.C)
    if slot < need:
        return Plan("tile", vec, cl, 0, 0, 0, 0)
    slot = min(slot, SLOT_CAP)
    if slot < need:
        slot = cdiv(need, 32) * 32
    smem = 4 * layout_total(d, cl, slot, True)
    assert smem <= 4 * MAX_DYN_FLOATS
    return Plan(None, vec, cl, slot, min(slot // d.A, d.Tx), min(slot // d.C, d.Tx), smem)


def jt(d: Dims, p: Plan) -> int:
    """Rows per attention run: a thread of the context pass owns one (row, column group) pair."""
    return min(DS_R, DS_THREADS // cdiv(d.C, 4 if p.vec else 1))


def ring_tiles(d: Dims, p: Plan) -> int:
    """Key tiles plus value tiles of one attention run (vector variant)."""
    return cdiv(d.Tx, p.tck) + cdiv(d.Tx, p.tcv)


def runs(d: Dims, p: Plan) -> List[List[Tuple[int, int]]]:
    """Per CTA: its attention runs as (encoder row, row count)."""
    rpc, out = DS_R // p.cl, []
    for cta in range(cdiv(d.rows, DS_R) * p.cl):
        my0 = (cta // p.cl) * DS_R + (cta % p.cl) * rpc
        mine: List[Tuple[int, int]] = []
        for r in range(my0, min(my0 + rpc, d.rows)):
            e = r // d.group
            if mine and mine[-1][0] == e and mine[-1][1] < jt(d, p):
                mine[-1] = (e, mine[-1][1] + 1)
            else:
                mine.append((e, 1))
        out.append(mine)
    return out


def panel_gw(ng: int, G: int) -> int:
    """ds_panel's warp group width: the one that keeps most of the 16 warps busy (ties: 4)."""
    gw, best = 4, 0
    cand = 2
    while cand <= 16:
        nqc = cdiv(ng, cand)
        busy = DS_WARPS if nqc >= DS_WARPS else nqc * (DS_WARPS // nqc)
        fits = nqc >= DS_WARPS or (DS_WARPS // nqc) * nqc * cand * DS_R * G <= DS_RED_FLOATS
        if fits and (busy > best or (busy == best and cand == 4)):
            best, gw = busy, cand
        cand *= 2
    return gw


def panel_passes(ng: int, G: int) -> List[Tuple[int, int]]:
    """(gw, wsplit) of every pass of ds_panel over `ng` column groups; wsplit > 1 joins K slices through `red`.
    A CTA that owns no column group of a product runs no pass."""
    if ng == 0:
        return []
    gw = panel_gw(ng, G)
    nquads = cdiv(ng, gw)
    out = []
    for qb in range(0, nquads, DS_WARPS):
        nq = min(DS_WARPS, nquads - qb)
        wsplit = DS_WARPS // nq
        assert wsplit == 1 or wsplit * nq * gw * DS_R * G <= DS_RED_FLOATS    # the K-split scratch holds it
        out.append((gw, wsplit))
    return out


def _slice(total: int, cl: int, rank: int) -> int:
    per = cdiv(total, cl)
    first = min(total, rank * per)
    return min(total, first + per) - first


def panels(d: Dims, p: Plan) -> Set[Tuple[int, int, int]]:
    """(G, gw, wsplit) of every ds_panel pass any CTA runs: gates, candidate, query and output products."""
    G = 4 if p.vec else 1
    out = set()
    for rank in range(p.cl):
        un = _slice(cdiv(d.H, G), p.cl, rank)
        an = _slice(cdiv(d.A, G), p.cl, rank)
        on = _slice(cdiv(d.O, G), p.cl, rank)
        for ng in (2 * un, un, an, (2 if d.maxout else 1) * on):
            out.update((G, gw, ws) for gw, ws in panel_passes(ng, G))
    return out


def reachable_panels() -> Set[Tuple[int, int, int]]:
    """Every (G, gw, wsplit > 1) the panel can choose, for column-group counts up to 1024."""
    out = set()
    for G in (1, 4):
        for ng in range(1, 1025):
            for gw, ws in panel_passes(ng, G):
                out.add((G, gw, min(ws, 2)))
    return out


class Case(NamedTuple):
    name: str
    cands: Sequence[Dims]                        # searched in order
    lands: Callable[[Dims, Plan], bool]
    aligned: bool = True                         # 16-byte aligned bases
    cl: Optional[int] = None                     # forced cluster size, None: the SM count decides
    near: Optional[Callable[[Dims], Dims]] = None   # refusal cases: the accepted shape next to it


def _d(rows=21, group=1, E=32, H=32, A=64, C=48, Tx=13, O=32, maxout=False) -> Dims:
    return Dims(rows, group, E, H, A, C, Tx, O, maxout)


def _rows(cands: Sequence[int], **kw) -> List[Dims]:
    return [_d(rows=r, **kw) for r in cands]


def _ok(p: Plan) -> bool:
    return p.refusal is None


def _has_idle_cta(d: Dims, p: Plan) -> bool:
    return any(not r for r in runs(d, p))


def _cta_without_columns(d: Dims, p: Plan) -> bool:
    G = 4 if p.vec else 1
    return any(_slice(cdiv(n, G), p.cl, rank) == 0 for n in (d.H, d.A, d.O) for rank in range(p.cl))


def _panel_lands(want: Tuple[int, int, int], p: Plan, d: Dims) -> bool:
    return any((G, gw, min(ws, 2)) == want for G, gw, ws in panels(d, p))


def _cl(n: int) -> Callable[[Dims, Plan], bool]:
    return lambda d, p: _ok(p) and p.cl == n and d.rows % DS_R != 0


ODD = dict(E=(33, "E"), H=(33, "H"), A=(65, "A"), C=(49, "C"), O=(33, "O"))
ENDE = dict(E=300, H=300, A=600, C=600, O=300)

CASES = [
    # cluster size from the row count, each with a ragged last cluster
    Case("cl8", _rows(range(13, 1100, 8)), _cl(8)),
    Case("cl4", _rows(range(5, 1100, 8)), _cl(4)),
    Case("cl2", _rows(range(5, 1100, 8)), _cl(2)),
    Case("cl1", _rows(range(5, 1100, 8)), _cl(1)),
    # the en-de beam batch: 128 sentences x beam 8 at cl = 1, a short and the longest encoder that fits
    Case("ende_beam_cl1", [_d(rows=1024, group=8, Tx=t, **ENDE) for t in (40, 50)],
         lambda d, p: _ok(p) and p.vec and p.cl == 1 and ring_tiles(d, p) >= 2 * DS_SLOTS),
    Case("ende_beam_cl1_tiles_of_one_step", [_d(rows=1024, group=8, Tx=t, **ENDE) for t in range(3000, 2000, -1)],
         lambda d, p: _ok(p) and p.cl == 1 and p.tck == 1 and p.tcv == 1),
    # scalar variant: one dimension not a multiple of 4 at a time, or a misaligned base
    *[Case("scalar_odd_" + k, [_d(**{k: v})], lambda d, p: _ok(p) and not p.vec) for k, (v, _n) in ODD.items()],
    Case("scalar_misaligned", [_d()], lambda d, p: _ok(p) and not p.vec, aligned=False),
    # TMA ring
    Case("tck_1", [_d(A=a) for a in range(4100, 8200, 4)], lambda d, p: _ok(p) and p.tck == 1 < p.tcv),
    Case("tcv_1", [_d(rows=5, C=2048, Tx=t) for t in range(1000, 6000, 4)],
         lambda d, p: _ok(p) and p.vec and p.tcv == 1 < p.tck, cl=1),
    Case("tx_is_tck", [_d(A=256, C=512, Tx=t) for t in range(8, 64)],
         lambda d, p: _ok(p) and p.vec and d.Tx == p.tck and p.tcv < d.Tx),
    Case("tx_is_tck_plus_1", [_d(A=a, Tx=t) for a in (256, 512) for t in range(8, 64)],
         lambda d, p: _ok(p) and p.vec and d.Tx == p.tck + 1),
    Case("ring_wraps_over_runs", [_d(rows=r, A=512, C=512, Tx=t) for t in (40, 60, 80) for r in range(5, 600, 8)],
         lambda d, p: (_ok(p) and p.vec and ring_tiles(d, p) > DS_SLOTS
                       and max(len(r) for r in runs(d, p)) >= 2)),
    # attention runs
    Case("jt1_vector", [_d(C=2048)], lambda d, p: _ok(p) and p.vec and jt(d, p) == 1, cl=1),
    Case("jt1_scalar", [_d(C=512, E=33)], lambda d, p: _ok(p) and not p.vec and jt(d, p) == 1, cl=1),
    Case("runs_cut_by_jt", [_d(rows=r, group=8, A=64, C=600) for r in (16, 24, 32)],
         lambda d, p: _ok(p) and any(len(r) > 1 and len({e for e, _ in r}) == 1 for r in runs(d, p)), cl=1),
    Case("group16_spans_clusters", [_d(rows=48, group=16)], lambda d, p: _ok(p) and d.group > DS_R),
    Case("cta_without_columns", [_d(E=33, H=h) for h in (9, 17, 25, 33)],
         lambda d, p: _ok(p) and p.cl == 8 and _cta_without_columns(d, p)),
    Case("idle_ctas", [_d(rows=r) for r in (3, 5)], lambda d, p: _ok(p) and _has_idle_cta(d, p)),
    # ds_panel: group widths and K splits through the scratch, both variants
    *[Case("panel_g{}_gw{}_{}".format(G, gw, "ksplit" if ws > 1 else "whole_k"),
           [_d(E=E, H=h, A=h, O=h) for h in range(4 // G, 2049, 4 // G)],
           lambda d, p, want=(G, gw, ws): _ok(p) and _panel_lands(want, p, d))
      for G, gw, ws, E in ((1, 2, 1, 33), (1, 2, 2, 33), (1, 4, 1, 33), (1, 4, 2, 33), (1, 8, 2, 33),
                           (1, 16, 2, 33), (4, 2, 1, 32), (4, 2, 2, 32), (4, 4, 1, 32), (4, 4, 2, 32),
                           (4, 8, 2, 32))],
    # refusals, each with the accepted shape next to it
    Case("refuse_context_scalar", [_d(E=33, C=513)], lambda d, p: p.refusal == "context",
         near=lambda d: d._replace(C=d.C - 1)),
    Case("refuse_context_vector", [_d(C=2052)], lambda d, p: p.refusal == "context",
         near=lambda d: d._replace(C=d.C - 4)),
    Case("refuse_tile_long_encoder", [_d(rows=5, C=2048, Tx=t) for t in range(2000, 4000)],
         lambda d, p: p.refusal == "tile", cl=1, near=lambda d: d._replace(Tx=d.Tx - 1)),
    # a 1024-unit decoder over a 2048-wide context with maxout 1024; H = 900 leaves a slot of exactly 2048 floats
    Case("refuse_tile_wide_decoder", [_d(H=h, A=2048, C=2048, O=1024, maxout=True) for h in range(900, 1025, 4)],
         lambda d, p: p.refusal == "tile", near=lambda d: d._replace(H=d.H - 4)),
    Case("refuse_smem_scalar", [_d(rows=5, E=33, A=14, C=14, Tx=t) for t in range(6000, 7000)],
         lambda d, p: p.refusal == "smem", cl=1, near=lambda d: d._replace(Tx=d.Tx - 1)),
]


def find_shape(case: Case, sms: int) -> Optional[Dims]:
    """The first candidate on the case's branch at `sms` SMs (for a refusal: whose neighbour is accepted)."""
    for d in case.cands:
        p = plan(d, sms, case.aligned, case.cl)
        if case.lands(d, p) and (case.near is None or _ok(plan(case.near(d), sms, case.aligned, case.cl))):
            return d
    return None
