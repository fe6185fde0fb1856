"""How the cluster GRU divides the batch: Bc, the rows per 8-CTA cluster, is a multiple of the two rows the
kernels walk at a time (not of 4), so every co-resident cluster takes part - at B=256 on an H100, 15 clusters
of 18 rows.  The plan is read back from the launched grid and shared-memory size; the partitions it creates
(one row pair per cluster, padding rows in the last cluster) are checked against the fp64 oracle."""
import json
import math
import os
import tempfile

import pytest
import torch

from tests import test_gpu_gru_cluster as cluster

pytestmark = pytest.mark.gpu

ROW_PAIR, CLUSTER, MAX_UNITS, XS = 2, 8, 40, 4


def _fwd_smem(bc, h):
    sl = math.ceil(h / 32)
    row = 32 * 4 * (((sl + 3) // 4) | 1)
    return 64 + 4 * bc * (3 * row + MAX_UNITS * (1 + 2 * XS) + 1)


def _expected_plan(bsz, resident):
    bc = -(-bsz // resident)
    bc = -(-bc // ROW_PAIR) * ROW_PAIR
    return bc, -(-bsz // bc)


def _launched(bsz, steps, h):
    """(grid x, dynamic shared memory) of the forward cluster kernel launched for one call."""
    from torch.profiler import ProfilerActivity, profile
    inp = cluster._raw_inputs(bsz, steps, h, 1)
    cluster._raw_fwd(inp[0], inp[1], inp[2], inp[3], inp[4], False, bsz, steps, h)  # load the module first
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        cluster._raw_fwd(inp[0], inp[1], inp[2], inp[3], inp[4], False, bsz, steps, h)
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]
    found = [e["args"] for e in events if "gru_seq_fwd_cluster_kernel" in e.get("name", "")]
    assert len(found) == 1, [e.get("name") for e in events if e.get("cat") == "kernel"]
    return found[0]["grid"][0], found[0]["shared memory"]


@pytest.mark.parametrize("bsz,h", [(256, 300), (30, 8), (250, 33), (17, 320)])
def test_cluster_plan_uses_every_resident_cluster(bsz, h):
    from neuralmonkey_b200 import lib
    resident = lib.load().nm_gru_resident_clusters(0)
    bc, clusters = _expected_plan(bsz, resident)
    grid, smem = _launched(bsz, 3, h)
    assert (grid, smem) == (CLUSTER * clusters, _fwd_smem(bc, h))
    if bsz == 256 and resident == 15:  # the en-de bench shape on an H100 SXM: 15 x 18, not 13 x 20
        assert (clusters, bc) == (15, 18)


# B = 30: one row pair per cluster; B = 250 and 256: the last cluster holds 16 and 4 real rows and padding;
# H = 8 .. 320 covers slice lengths 1, 2, 10
PLAN_SHAPES = [(30, 50, 8), (30, 20, 31), (250, 20, 32), (250, 20, 33), (256, 50, 300), (30, 50, 320)]


@pytest.mark.parametrize("shape", PLAN_SHAPES)
@pytest.mark.parametrize("variant", ["plain", "lengths_reverse_h0"])
def test_cluster_plan_shapes_vs_oracle(shape, variant):
    cluster.test_cluster_gru_vs_oracle(shape, variant)


@pytest.mark.parametrize("shape", [(30, 20, 33), (250, 7, 300)])
def test_cluster_plan_drop_mask_vs_oracle(shape):
    cluster.test_cluster_gru_drop_mask_raw_outputs(shape)
