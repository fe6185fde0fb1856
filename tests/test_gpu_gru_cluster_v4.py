"""The cluster GRU's exchanged vectors at the edges of their layout: every CTA of a cluster owns floor-divided
unit counts (H/8 rounded either way), its warps send their 4 units in a row as one 16-byte message, and the
lanes read their reduction slices in 16-, 8- or 4-byte pieces by slice length (the 16-byte pieces in swizzled
order at SL = 8).  Widths whose CTAs own unit counts that are not multiples of 4, down to a last warp with one
live unit, one width of every slice length, partial clusters, single steps, zero lengths, reverse with h0 and
dropout masks, against the fp64 oracle at the exact tolerances; and run-to-run bit identity at the en-de shape
with the decoder's dropout mask."""
import pytest
import torch

from tests import test_gpu_gru_cluster as cluster

pytestmark = pytest.mark.gpu

# H -> ceil(H/32) = slice length: 9, 12 -> 1; 33, 37 -> 2; 70 -> 3; 130 -> 5; 180 -> 6; 200 -> 7; 232, 250 -> 8;
# 270 -> 9; 299, 300, 317, 320 -> 10
WIDTHS = [9, 12, 33, 37, 70, 130, 180, 200, 232, 250, 270, 299, 300, 317, 320]


def _units(h):
    return [(r + 1) * h // 8 - r * h // 8 for r in range(8)]


def test_widths_cover_partial_quads():
    """The widths include CTAs whose last warp holds 1, 2 and 3 live units, and CTAs of one cluster that own
    different unit counts."""
    tails = {u % 4 for h in WIDTHS for u in _units(h)}
    assert tails == {0, 1, 2, 3}
    assert any(len(set(_units(h))) > 1 for h in WIDTHS)
    assert {h for h in WIDTHS if 1 in [u % 4 for u in _units(h)]} >= {33, 37, 232, 300}


@pytest.mark.parametrize("h", WIDTHS)
@pytest.mark.parametrize("variant", ["plain", "lengths_reverse_h0"])
def test_layout_widths_vs_oracle(h, variant):
    cluster.test_cluster_gru_vs_oracle((17, 12, h), variant)


@pytest.mark.parametrize("h", [12, 37, 250, 317])
def test_layout_single_step_partial_cluster(h):
    cluster.test_cluster_gru_vs_oracle((5, 1, h), "lengths_reverse_h0")


@pytest.mark.parametrize("h", [37, 232, 299])
@pytest.mark.parametrize("reverse", [False, True])
def test_layout_zero_lengths(h, reverse):
    cluster.test_gru_zero_lengths((9, 12, h), reverse, True)


@pytest.mark.parametrize("h", [33, 250, 317])
def test_layout_drop_mask_raw_outputs(h):
    cluster.test_cluster_gru_drop_mask_raw_outputs((17, 12, h))


def test_decoder_configuration_bit_identical_repeats():
    """B=256, T=50, H=300 forward with h0, a dropout mask and raw outputs, and its backward with dh0, twice."""
    from neuralmonkey_b200 import lib
    from neuralmonkey_b200.lib import call, ptr
    bsz, steps, h = 256, 50, 300
    xproj, wg, wc, h0, _lengths, dstates, dfinal = cluster._raw_inputs(bsz, steps, h, 6)
    g = torch.Generator().manual_seed(6)
    mask = ((torch.rand(bsz, steps, h, generator=g) < 0.7).float() / 0.7).cuda()
    runs = []
    for _ in range(2):
        out = {n: torch.empty(bsz, steps, k * h, device="cuda")
               for n, k in (("states", 1), ("raw", 1), ("gates", 3), ("hprev", 1), ("rh", 1), ("dx", 3))}
        out["final"], out["dh0"] = torch.empty(bsz, h, device="cuda"), torch.empty(bsz, h, device="cuda")
        work = torch.empty(2 * bsz * h, device="cuda")
        call("nm_gru_seq_fwd", ptr(xproj), ptr(wg), ptr(wc), ptr(h0), None, ptr(mask), 0, ptr(out["states"]),
             ptr(out["raw"]), ptr(out["final"]), ptr(out["gates"]), ptr(out["hprev"]), ptr(out["rh"]),
             bsz, steps, h, 0, lib.stream())
        call("nm_gru_seq_bwd", ptr(wg), ptr(wc), None, ptr(mask), 0, ptr(out["gates"]), ptr(out["hprev"]),
             ptr(dstates), None, ptr(dfinal), ptr(out["dx"]), ptr(out["dh0"]), ptr(work), bsz, steps, h, 0,
             lib.stream())
        runs.append(out)
    torch.cuda.synchronize()
    for n in runs[0]:
        assert torch.equal(runs[0][n], runs[1][n]), n
