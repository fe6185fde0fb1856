"""Time coverage attention (ops.coverage_attention: nm_coverage_attention_fwd / _bwd) forward and forward plus
backward at the en-de training shape (B=256, Tx=50, NQ=50, A=C=600) and the captioning shape (B=32, Tx=196 regions,
NQ=16, A=C=512), against

    K4 floor        nm_bahdanau_* at the same shape, attention without coverage
    eager torch     the coverage scan composed of fp32 torch operations (tests/coverage_oracle.py's arithmetic)

and the time of one decoding step (NQ = 1, continuing from a running coverage).  The fertility is computed once
outside the timed calls, as the model part caches it per batch.  Variants alternate within each round and every
round is repeated; the median over rounds is printed, in ms per call, from CUDA events around `--iters` calls after
warm-up.  The card's name and power limit are read in the same process.

    python tools/coverage_bench.py [--iters N] [--rounds R]
"""
import argparse
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SHAPES = {"en-de": (256, 50, 50, 600, 600), "captioning": (32, 196, 16, 512, 512)}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name(0)


def eager(keys, values, mask, fert, qproj, v, cw, cov_in=None):
    total = torch.zeros_like(fert) if cov_in is None else cov_in
    contexts = []
    for q in range(qproj.shape[1]):
        cov = total / fert * mask
        e = (v * torch.tanh(keys + qproj[:, q].unsqueeze(1) + cw * cov.unsqueeze(-1))).sum(-1)
        w = torch.softmax(e, -1) * mask
        w = w / (w.sum(-1, keepdim=True) + 1e-8)
        contexts.append(torch.bmm(w.unsqueeze(1), values))
        total = total + w
    return torch.cat(contexts, 1)


def bench_shape(name, dims, iters, rounds):
    from neuralmonkey_b200 import ops
    bsz, tx, nq, a, c = dims
    dev = torch.device("cuda")
    gen = torch.Generator(device=dev).manual_seed(0)

    def r(*shape, scale=1.0):
        return (torch.randn(*shape, device=dev, generator=gen) * scale).requires_grad_()
    keys, values, qproj = r(bsz, tx, a, scale=0.5), r(bsz, tx, c), r(bsz, nq, a, scale=0.5)
    v, cw, bias = r(a, scale=0.1), r(a, scale=0.1), r(1, scale=0.1)
    lengths = torch.randint(tx // 2, tx + 1, (bsz,), device=dev, generator=gen)
    mask = (torch.arange(tx, device=dev)[None] < lengths[:, None]).float()
    with torch.no_grad():
        fert = ops.coverage_fertility(values, torch.randn(c, device=dev, generator=gen) * 0.05, 5)
    fert.requires_grad_()
    cov_in = torch.rand(bsz, tx, device=dev, generator=gen)
    step_q = qproj[:, :1].detach().contiguous()
    dctx = torch.randn(bsz, nq, c, device=dev, generator=gen)

    variants = [("coverage", lambda: ops.coverage_attention(keys, values, mask, fert, qproj, v, cw)[0]),
                ("K4 floor", lambda: ops.bahdanau_attention(keys, values, mask, qproj, v, bias)[0]),
                ("eager torch", lambda: eager(keys, values, mask, fert, qproj, v, cw))]

    def fwd(fn):
        with torch.no_grad():
            fn()

    def fwd_bwd(fn):
        fn().backward(dctx)

    def one_step():
        with torch.no_grad():
            ops.coverage_attention(keys, values, mask, fert, step_q, v, cw, cov_in)

    runs = [(n, m, (lambda fn=fn, run=run: run(fn))) for n, fn in variants
            for m, run in (("fwd", fwd), ("fwd+bwd", fwd_bwd))] + [("coverage NQ=1 step", "fwd", one_step)]
    times = {(n, m): [] for n, m, _ in runs}
    for _n, _m, fn in runs:
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    for _ in range(rounds):
        for n, m, fn in runs:
            start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            for _ in range(iters):
                fn()
            stop.record()
            stop.synchronize()
            times[(n, m)].append(start.elapsed_time(stop) / iters)
    print("{}: B={} Tx={} NQ={} A={} C={}; median of {} rounds x {} calls, ms per call".format(
        name, bsz, tx, nq, a, c, rounds, iters))
    for n, m, _ in runs:
        ts = times[(n, m)]
        print("  {:20s} {:8s} {:9.3f}   (spread {:.3f}-{:.3f})".format(n, m, statistics.median(ts), min(ts), max(ts)))


def main():
    parser = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    parser.add_argument("--iters", type=int, default=20)
    parser.add_argument("--rounds", type=int, default=5)
    args = parser.parse_args()
    from neuralmonkey_b200 import build
    build.build()
    print("card: {}".format(card()))
    for name, dims in SHAPES.items():
        bench_shape(name, dims, args.iters, args.rounds)


if __name__ == "__main__":
    main()
