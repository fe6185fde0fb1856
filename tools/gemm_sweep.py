"""Per-shape GPU time of nm_gemm for the products of the en-de and Transformer training steps.

Every shape is launched back to back REPS times between two CUDA events, operands rotating through enough
buffer sets to exceed the 50 MB L2 (so A and C come from / go to HBM as they do inside a step, while the
small weight operand stays L2-resident as it does inside a step).  Prints one line per shape:
time per launch, TFLOP/s, and the HBM floor (bytes of A, B and C once each at the measured copy rate).

    python tools/gemm_sweep.py [--reps 50] [--set ende|transformer|all]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from neuralmonkey_b200 import ops  # noqa: E402

# (label, transA, transB, M, N, K): op(A) [M,K] @ op(B) [K,N]
ENDE = [
    ("proj fwd  NN", 0, 0, 12800, 600, 300), ("proj fwd  NN", 0, 0, 12800, 300, 300),
    ("proj fwd  NN", 0, 0, 12800, 900, 300), ("proj fwd  NN", 0, 0, 12800, 600, 600),
    ("dgrad     NT", 0, 1, 12800, 300, 300), ("dgrad     NT", 0, 1, 12800, 300, 600),
    ("dgrad     NT", 0, 1, 12800, 600, 600), ("wgrad     TN", 1, 0, 300, 600, 12800),
    ("wgrad     TN", 1, 0, 300, 300, 12800), ("wgrad     TN", 1, 0, 600, 600, 12800),
]
TRANSFORMER = [
    ("qkv/out   NN", 0, 0, 4096, 512, 512), ("ffn in    NN", 0, 0, 4096, 2048, 512),
    ("ffn out   NN", 0, 0, 4096, 512, 2048), ("dgrad     NT", 0, 1, 4096, 512, 512),
    ("dgrad     NT", 0, 1, 4096, 512, 2048), ("dgrad     NT", 0, 1, 4096, 2048, 512),
    ("wgrad     TN", 1, 0, 512, 512, 4096), ("wgrad     TN", 1, 0, 512, 2048, 4096),
    ("wgrad     TN", 1, 0, 2048, 512, 4096), ("fused qkv NN", 0, 0, 4096, 1536, 512),
]


# what a launch costs by itself, one tile per SM with a short and with a long reduction (steady-state rate of the
# TMA ring per SM), and the same through a pure-L2 operand set
DIAG = [
    ("1 tile      ", 0, 1, 128, 128, 32), ("132 tiles k=1 blk", 0, 1, 16896, 128, 32),
    ("132 tiles K=320 ", 0, 1, 16896, 128, 320), ("132 tiles K=3200", 0, 1, 16896, 128, 3200),
    ("132 tiles K=320 BN256", 0, 1, 16896, 256, 320), ("132 tiles K=3200 BN256", 0, 1, 16896, 256, 3200),
    ("4 rounds K=320", 0, 1, 75776, 128, 320), ("4 rounds K=320 MN-B", 0, 0, 75776, 128, 320),
]


def time_shape(ta, tb, m, n, k, reps, act=None, bias=False):
    dev = torch.device("cuda")
    a_shape = (k, m) if ta else (m, k)
    b_shape = (n, k) if tb else (k, n)
    per_set = 4 * (m * k + m * n)
    nsets = max(2, min(64, (160 << 20) // per_set + 1))
    a_bufs = [torch.randn(a_shape, device=dev) for _ in range(nsets)]
    c_bufs = [torch.empty(m, n, device=dev) for _ in range(nsets)]
    b_op = torch.randn(b_shape, device=dev)
    bias_t = torch.randn(n, device=dev) if bias else None
    for i in range(3):
        ops.gemm(a_bufs[i % nsets], b_op, c_bufs[i % nsets], bool(ta), bool(tb), bias_t, act)
    torch.cuda.synchronize()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    graph = torch.cuda.CUDAGraph()            # replayed: no host gaps between the launches
    with torch.cuda.graph(graph):
        for i in range(reps):
            ops.gemm(a_bufs[i % nsets], b_op, c_bufs[i % nsets], bool(ta), bool(tb), bias_t, act)
    graph.replay()
    torch.cuda.synchronize()
    start.record()
    graph.replay()
    stop.record()
    torch.cuda.synchronize()
    return start.elapsed_time(stop) * 1e3 / reps     # us per launch


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--set", default="all")
    args = ap.parse_args()
    peaks = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                        "MEASURED_PEAKS.json")))
    hbm = peaks["hbm_gbs"] * 1e9
    shapes = []
    if args.set in ("ende", "all"):
        shapes += [("ende",) + s for s in ENDE]
    if args.set in ("transformer", "all"):
        shapes += [("transformer",) + s for s in TRANSFORMER]
    if args.set in ("diag", "all"):
        shapes += [("diag",) + s for s in DIAG]
    print("NMB200_TC_BN =", os.environ.get("NMB200_TC_BN", "(auto)"))
    for group, label, ta, tb, m, n, k in shapes:
        us = time_shape(ta, tb, m, n, k, args.reps)
        flop = 2.0 * m * n * k
        floor_us = 4.0 * (m * k + k * n + m * n) / hbm * 1e6
        print("{:12s} {} {:6d} x {:5d} x {:6d}  {:8.1f} us  {:7.1f} TF/s   hbm floor {:6.1f} us".format(
            group, label, m, n, k, us, flop / us * 1e-6, floor_us), flush=True)


if __name__ == "__main__":
    main()
