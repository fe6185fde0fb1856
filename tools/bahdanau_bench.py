"""Time the Bahdanau attention entry points, nm_bahdanau_fwd and nm_bahdanau_bwd, through the C ABI with CUDA
events over many calls after warm-up, at three shapes (B, Tx, NQ, A, C):

    en-de        (256,  50, 50, 600, 600)   the training step bench.py measures, source mask on
    captioning   ( 32, 196, 16, 512, 512)   tests/captioning.ini scaled, as bench_workloads.py runs it
    en-de NQ=1   (256,  50,  1, 600, 600)   one query step (step-wise decoding, RL sampling passes)

Each pass evaluates tanh(k + q) for B*NQ*Tx*A elements: the forward once, the backward's key-gradient kernel once
more.  The SFU floor of one pass is elements x SFU operations per element / (SMs x 16 per clock x max SM clock);
it is printed for one SFU operation per element (the reciprocal of the factorised tanh) as a fraction of the
measured time.  The card's name, power limit and clocks are read in the same process.

    python tools/bahdanau_bench.py [--lib path/to/libnmb200.so] [--iters N]

--lib times another build of the library (for example the parent commit's) with the same inputs.
"""
import argparse
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SHAPES = [("en-de", (256, 50, 50, 600, 600)), ("captioning", (32, 196, 16, 512, 512)),
          ("en-de NQ=1", (256, 50, 1, 600, 600))]
WARMUP = 20
SFU_PER_CLOCK_PER_SM = 16


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
        name, power, _clk, max_clk = [s.strip() for s in out.strip().splitlines()[0].split(",")]
        return "{}, power limit {} W, max SM clock {} MHz".format(name, power, max_clk), float(max_clk)
    except (OSError, subprocess.SubprocessError, IndexError, ValueError):
        return torch.cuda.get_device_name(0), 1980.0


def time_calls(fn, iters):
    for _ in range(WARMUP):
        fn()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(iters):
        fn()
    stop.record()
    torch.cuda.synchronize()
    return start.elapsed_time(stop) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="libnmb200.so to load instead of the in-tree build")
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--kernels", action="store_true", help="also list each kernel's time (torch.profiler)")
    args = ap.parse_args()
    from neuralmonkey_b200 import lib
    if args.lib:
        lib.LIB_PATH = os.path.abspath(args.lib)
    lib.load()
    desc, max_mhz = card()
    sms = lib.device_info()["sm_count"]
    print("device: {} ({} SMs); library: {}".format(desc, sms, lib.LIB_PATH))
    p, st = lib.ptr, lib.stream()
    g = torch.Generator(device="cuda").manual_seed(0)
    for label, (b, tx, nq, a, c) in SHAPES:
        keys = torch.randn(b, tx, a, device="cuda", generator=g)
        values = torch.randn(b, tx, c, device="cuda", generator=g)
        qproj = torch.randn(b, nq, a, device="cuda", generator=g)
        v = torch.randn(a, device="cuda", generator=g) * 0.3
        bias = torch.zeros(1, device="cuda")
        lens = torch.randint(1, tx + 1, (b,), device="cuda", generator=g)
        lens[0] = tx
        mask = (torch.arange(tx, device="cuda").unsqueeze(0) < lens.unsqueeze(1)).float()
        energies, weights = torch.empty(b, nq, tx, device="cuda"), torch.empty(b, nq, tx, device="cuda")
        ctx = torch.empty(b, nq, c, device="cuda")
        dctx = torch.randn(b, nq, c, device="cuda", generator=g)
        dkeys, dvalues, dq = torch.empty_like(keys), torch.empty_like(values), torch.empty_like(qproj)
        dv, db, work = torch.zeros(a, device="cuda"), torch.zeros(1, device="cuda"), torch.empty(b * nq * tx,
                                                                                                   device="cuda")

        def fwd():
            lib.call("nm_bahdanau_fwd", p(keys), p(values), p(mask), p(qproj), p(v), p(bias), p(energies),
                     p(weights), p(ctx), b, tx, nq, a, c, st)

        def bwd():
            lib.call("nm_bahdanau_bwd", p(keys), p(values), p(mask), p(qproj), p(v), p(energies), p(weights),
                     p(dctx), p(dkeys), p(dvalues), p(dq), p(dv), p(db), p(work), b, tx, nq, a, c, st)

        t_f, t_b = time_calls(fwd, args.iters), time_calls(bwd, args.iters)
        floor = b * nq * tx * a / (sms * SFU_PER_CLOCK_PER_SM * max_mhz * 1e3)   # ms, 1 SFU op per element
        print("{:11s} B={:3d} Tx={:3d} NQ={:2d} A={:3d} C={:3d}  fwd {:.4f} ms  bwd {:.4f} ms  pair {:.4f} ms  "
              "SFU floor {:.4f} ms per pass: fwd at {:.0%}, bwd at {:.0%}".format(
                  label, b, tx, nq, a, c, t_f, t_b, t_f + t_b, floor, floor / t_f, floor / t_b))
        if args.kernels:
            print("  " + kernel_times(lambda: (fwd(), bwd()), args.iters))


def kernel_times(fn, iters):
    """Mean device time per call of each kernel fn launches, from torch.profiler (a separate pass: tracing slows
    the host, not the kernels)."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    times = {}
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            name = ev.name.split("(")[0].split("<")[0].replace("void ", "").replace("nm::", "")
            times[name] = times.get(name, 0.0) + ev.device_time / 1e3 / iters
    return "  ".join("{} {:.4f} ms".format(n, t) for n, t in sorted(times.items(), key=lambda x: -x[1]))


if __name__ == "__main__":
    main()
