"""Time the fp16 vocabulary gradient products through the C ABI at the en-de bench shape (M = 12800 target tokens,
K = 300, V = 32000) and at M = 2048, with CUDA events over many launches after warm-up:

    dX      = P16 [M,V] . W16 [K,V]^T * row_scale[m]         nm_gemm_f16     (M x K x V, both operands K-major)
    [dW;db] += alpha * XS16 [M,K+1]^T . P16 [M,V]            nm_gemm_f16_tn  (K+1 x V x M, both MN-major)

the latter into a strided view of a flat buffer, as ops._LogitsXent16 does.  Prints ms per call and TFLOP/s against
the 989 TFLOP/s fp16 data-sheet peak (dense, 700 W); the card's name and power limit are read in the same process.

    python tools/vocab_bwd_bench.py
"""
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PEAK_TFLOPS = 989.0
SHAPES = [(12800, 300, 32000), (2048, 300, 32000)]
WARMUP, ITERS = 10, 50


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name(0)


def time_calls(fn):
    for _ in range(WARMUP):
        fn()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(ITERS):
        fn()
    stop.record()
    torch.cuda.synchronize()
    return start.elapsed_time(stop) / ITERS


def main():
    from neuralmonkey_b200 import lib
    lib.load()
    print("device:", card())
    g = torch.Generator(device="cuda").manual_seed(0)
    p = lib.ptr
    for m, k, v in SHAPES:
        vpad, k1pad = (v + 7) // 8 * 8, (k + 1 + 7) // 8 * 8
        p16 = (torch.rand(m, vpad, device="cuda", generator=g) * 2e-4).half()
        w16 = (torch.randn(k, vpad, device="cuda", generator=g) * 0.1).half()
        xs16 = (torch.randn(m, k1pad, device="cuda", generator=g) * 0.5).half()
        row_scale = torch.rand(m, device="cuda", generator=g)
        alpha = torch.ones(1, device="cuda")
        dx = torch.empty(m, k, device="cuda")
        flat = torch.zeros(k * v + v + 4, device="cuda")
        sink_aug = torch.as_strided(flat, (k + 1, v), (v, 1), 3)     # not 16-byte aligned, as a parameter slice

        def dX():
            lib.call("nm_gemm_f16", m, k, v, p(p16), vpad, p(w16), vpad, p(dx), k, None, p(row_scale), 0.0, 0,
                     lib.stream())

        def dW():
            lib.call("nm_gemm_f16_tn", k + 1, v, m, p(xs16), k1pad, p(p16), vpad, p(sink_aug), v, p(alpha), 1.0,
                     lib.stream())

        t_x, t_w = time_calls(dX), time_calls(dW)
        for name, t, flops in (("dX", t_x, 2.0 * m * k * v), ("dW+db", t_w, 2.0 * m * (k + 1) * v)):
            print("M={:6d} K={:4d} V={:6d}  {:6s}: {:.4f} ms  {:.1f} TFLOP/s ({:.1%} of {:.0f})".format(
                m, k, v, name, t, flops / t / 1e9, flops / t / 1e9 / PEAK_TFLOPS, PEAK_TFLOPS))
        print("M={:6d} K={:4d} V={:6d}  dX + dW+db: {:.4f} ms".format(m, k, v, t_x + t_w))


if __name__ == "__main__":
    main()
