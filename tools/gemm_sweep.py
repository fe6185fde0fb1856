"""Per-shape GPU time of nm_gemm for the products of the en-de and Transformer training steps.

Every shape is launched back to back REPS times between two CUDA events, operands rotating through enough
buffer sets to exceed the 50 MB L2 (so A and C come from / go to HBM as they do inside a step, while the
small weight operand stays L2-resident as it does inside a step).  Prints one line per shape:
time per launch through ops.gemm (an MN-major TF32 operand therefore includes its K-major copy), TFLOP/s, and
the HBM floor (bytes of A, B and C once each at the device-to-device copy rate measured in the same run).

--kmajor times every product with an MN-major TF32 operand two ways: nm_gemm reading the operands as stored
(the kernel's producer threads transpose every tile) and nm_gemm on K-major copies made by nm_transpose_tf32,
with each copy on a line of its own (time, GB/s against the copy rate).

    python tools/gemm_sweep.py [--reps 50] [--set ende|transformer|diag|all] [--kmajor]
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from neuralmonkey_b200 import lib, ops  # noqa: E402

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
# the products with MN-major TF32 operands (--kmajor): weight gradients X^T.dY and forward projections X.W with W
# stored [in, out]; en-de: GRU kernels (x, h: 300 -> 2H / H), attention keys 600 -> 600, query 300 -> 600,
# output projection 1200 -> 300; Transformer: its dense layers and the tied-embedding products of the loss
ENDE_MN = [
    ("wgrad     TN", 1, 0, 300, 600, 12800), ("wgrad     TN", 1, 0, 300, 300, 12800),
    ("wgrad     TN", 1, 0, 600, 600, 12800), ("wgrad     TN", 1, 0, 1200, 300, 12800),
    ("proj fwd  NN", 0, 0, 12800, 600, 300), ("proj fwd  NN", 0, 0, 12800, 300, 300),
    ("proj fwd  NN", 0, 0, 12800, 600, 600), ("proj fwd  NN", 0, 0, 12800, 300, 1200),
]
TRANSFORMER_MN = [
    ("wgrad     TN", 1, 0, 512, 512, 4096), ("wgrad     TN", 1, 0, 512, 2048, 4096),
    ("wgrad     TN", 1, 0, 2048, 512, 4096), ("emb wgrad TN", 1, 0, 32000, 512, 4096),
    ("qkv/out   NN", 0, 0, 4096, 512, 512), ("ffn in    NN", 0, 0, 4096, 2048, 512),
    ("ffn out   NN", 0, 0, 4096, 512, 2048), ("emb dgrad NN", 0, 0, 4096, 512, 32000),
]


# what a launch costs by itself, one tile per SM with a short and with a long reduction (steady-state rate of the
# TMA ring per SM), and the same through a pure-L2 operand set
DIAG = [
    ("1 tile      ", 0, 1, 128, 128, 32), ("132 tiles k=1 blk", 0, 1, 16896, 128, 32),
    ("132 tiles K=320 ", 0, 1, 16896, 128, 320), ("132 tiles K=3200", 0, 1, 16896, 128, 3200),
    ("132 tiles K=320 BN256", 0, 1, 16896, 256, 320), ("132 tiles K=3200 BN256", 0, 1, 16896, 256, 3200),
    ("4 rounds K=320", 0, 1, 75776, 128, 320), ("4 rounds K=320 MN-B", 0, 0, 75776, 128, 320),
]


def _operands(ta, tb, m, n, k):
    """Operand sets rotating through more memory than the 50 MB L2 (A and C), one B operand."""
    dev = torch.device("cuda")
    a_shape = (k, m) if ta else (m, k)
    b_shape = (n, k) if tb else (k, n)
    per_set = 4 * (m * k + m * n)
    nsets = max(2, min(64, (160 << 20) // per_set + 1))
    a_bufs = [torch.randn(a_shape, device=dev) for _ in range(nsets)]
    c_bufs = [torch.empty(m, n, device=dev) for _ in range(nsets)]
    return a_bufs, torch.randn(b_shape, device=dev), c_bufs


def _graph_us(launch, reps):
    """Device time per call of launch(i), i = 0 .. reps-1 captured in one CUDA graph (no host gaps)."""
    for i in range(3):
        launch(i)
    torch.cuda.synchronize()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for i in range(reps):
            launch(i)
    graph.replay()
    torch.cuda.synchronize()
    start.record()
    graph.replay()
    stop.record()
    torch.cuda.synchronize()
    return start.elapsed_time(stop) * 1e3 / reps


def time_shape(ta, tb, m, n, k, reps, act=None, bias=False):
    a_bufs, b_op, c_bufs = _operands(ta, tb, m, n, k)
    bias_t = torch.randn(n, device="cuda") if bias else None
    return _graph_us(lambda i: ops.gemm(a_bufs[i % len(a_bufs)], b_op, c_bufs[i % len(a_bufs)], bool(ta), bool(tb),
                                        bias_t, act), reps)


def copy_gbs():
    """Device-to-device copy rate of 512 MB (read + write), the HBM yardstick of this run."""
    src = torch.empty(128 << 20, device="cuda")
    dst = torch.empty_like(src)
    us = _graph_us(lambda i: dst.copy_(src), 10)
    return 2 * src.numel() * 4 / (us * 1e-6) / 1e9


def _transpose(src, dst):
    rows, cols = src.shape
    lib.call("nm_transpose_tf32", lib.ptr(src), src.stride(0), lib.ptr(dst), dst.stride(0), rows, cols, lib.stream())


def time_kmajor(ta, tb, m, n, k, reps):
    """One product with MN-major TF32 operands two ways: nm_gemm reading them as stored (the producer threads
    transpose every tile), and nm_transpose_tf32 + nm_gemm on the K-major copies.  Returns
    (us as stored, us of the K-major product, [(operand, us, bytes)] of the copies)."""
    a_bufs, b_op, c_bufs = _operands(ta, tb, m, n, k)
    nsets = len(a_bufs)

    def direct(i):
        a, c = a_bufs[i % nsets], c_bufs[i % nsets]
        lib.call("nm_gemm", int(ta), int(tb), m, n, k, lib.ptr(a), a.stride(0), lib.ptr(b_op), b_op.stride(0),
                 lib.ptr(c), n, None, 0, 0.0, lib.GEMM_AUTO, lib.stream())
    us_direct = _graph_us(direct, reps)
    a_k = [ops.kmajor_tf32(a) for a in a_bufs] if ta else a_bufs
    b_k = ops.kmajor_tf32(b_op) if not tb else b_op
    us_kmajor = _graph_us(lambda i: ops.gemm(a_k[i % nsets], b_k, c_bufs[i % nsets], False, True), reps)
    copies = []
    if ta:
        copies.append(("A", _graph_us(lambda i: _transpose(a_bufs[i % nsets], a_k[i % nsets]), reps),
                       2 * 4 * m * k))
    if not tb:
        copies.append(("B", _graph_us(lambda i: _transpose(b_op, b_k), reps), 2 * 4 * n * k))
    return us_direct, us_kmajor, copies


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--set", default="all")
    ap.add_argument("--kmajor", action="store_true",
                    help="MN-major TF32 products: as stored vs nm_transpose_tf32 + K-major, copies on their own lines")
    args = ap.parse_args()
    print("device: {}".format(torch.cuda.get_device_name(0)))
    gbs = copy_gbs()
    print("device-to-device copy: {:.0f} GB/s".format(gbs), flush=True)
    groups = {"ende": ENDE_MN if args.kmajor else ENDE, "transformer": TRANSFORMER_MN if args.kmajor else TRANSFORMER,
              "diag": [] if args.kmajor else DIAG}
    shapes = [(g,) + s for g in ("ende", "transformer", "diag") if args.set in (g, "all") for s in groups[g]]
    for group, label, ta, tb, m, n, k in shapes:
        flop = 2.0 * m * n * k
        head = "{:12s} {} {:6d} x {:5d} x {:6d}".format(group, label, m, n, k)
        if not args.kmajor:
            us = time_shape(ta, tb, m, n, k, args.reps)
            floor_us = 4.0 * (m * k + k * n + m * n) / (gbs * 1e9) * 1e6
            print("{}  {:8.1f} us  {:7.1f} TF/s   hbm floor {:6.1f} us".format(head, us, flop / us * 1e-6, floor_us),
                  flush=True)
            continue
        us_mn, us_k, copies = time_kmajor(ta, tb, m, n, k, args.reps)
        us_copies = sum(us for _, us, _ in copies)
        print("{}  as stored   {:8.1f} us  {:7.1f} TF/s".format(head, us_mn, flop / us_mn * 1e-6))
        print("{}  K-major     {:8.1f} us  {:7.1f} TF/s".format(head, us_k, flop / us_k * 1e-6))
        for name, us, nbytes in copies:
            print("{}  copy of {}   {:8.1f} us  {:7.0f} GB/s ({:.0%} of the copy rate)".format(
                head, name, us, nbytes / (us * 1e-6) / 1e9, nbytes / (us * 1e-6) / 1e9 / gbs))
        print("{}  copies + K-major {:8.1f} us  ({:.2f}x as stored)".format(head, us_copies + us_k,
                                                                          us_mn / (us_copies + us_k)), flush=True)


if __name__ == "__main__":
    main()
