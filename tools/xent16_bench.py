"""Time the fp16 vocabulary cross-entropy entry points (nm_logits_xent_fwd16, nm_logits_xent_bwd16) at the en-de
bench shape (M = 12800 target tokens, K = 300, V = 32000), at M = 2048 and at K = 512 (longer K: the generic-GEMM
instances), with CUDA events over many launches after warm-up.  Prints ms per call, TFLOP/s against the
989 TFLOP/s fp16 data-sheet peak (dense, 700 W) and, for the backward, the GB/s of the P16 write; the card's
name and power limit are read in the same process.

    python tools/xent16_bench.py
"""
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PEAK_TFLOPS = 989.0
SHAPES = [(12800, 300, 32000), (2048, 300, 32000), (12800, 512, 32000)]
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
    for m, k, v in SHAPES:
        kpad, vpad = (k + 7) // 8 * 8, (v + 7) // 8 * 8
        x16 = (torch.randn(m, kpad, device="cuda", generator=g) * 0.5).half()
        wt16 = (torch.randn(v, kpad, device="cuda", generator=g) * 0.1).half()
        b = torch.randn(v, device="cuda", generator=g) * 0.1
        targets = torch.randint(0, v, (m,), device="cuda", generator=g)
        mask = torch.ones(m, device="cuda")
        lse, xent = torch.empty(m, device="cuda"), torch.empty(m, device="cuda")
        argmax = torch.empty(m, device="cuda", dtype=torch.int64)
        part = torch.empty(lib.load().nm_logits_xent_scratch(m, v), device="cuda")
        dl16 = torch.empty(m, vpad, device="cuda", dtype=torch.float16)
        p = lib.ptr

        def fwd():
            lib.call("nm_logits_xent_fwd16", p(x16), kpad, p(wt16), kpad, p(b), 1, p(targets), p(mask), p(lse),
                     p(xent), p(argmax), p(part), None, v, m, v, k, lib.stream())

        def bwd():
            lib.call("nm_logits_xent_bwd16", p(x16), kpad, p(wt16), kpad, p(b), 1, p(targets), p(mask), p(lse),
                     p(dl16), vpad, m, v, k, lib.stream())

        flops = 2.0 * m * v * k
        t_f = time_calls(fwd)
        t_b = time_calls(bwd)
        for name, t in (("fwd16", t_f), ("bwd16", t_b)):
            line = "M={:6d} K={:4d} V={:6d}  {}: {:.4f} ms  {:.1f} TFLOP/s ({:.1%} of {:.0f})".format(
                m, k, v, name, t, flops / t / 1e9, flops / t / 1e9 / PEAK_TFLOPS, PEAK_TFLOPS)
            if name == "bwd16":
                line += "  P16 write {:.0f} GB/s".format(2.0 * m * v / t / 1e6)
            print(line)
        print("M={:6d} K={:4d} V={:6d}  fwd16 + bwd16: {:.4f} ms".format(m, k, v, t_f + t_b))


if __name__ == "__main__":
    main()
