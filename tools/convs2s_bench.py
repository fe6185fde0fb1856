"""Time one ConvS2S encoder layer (csrc/glu_conv.cu through `ops.conv1d_glu_residual`: conv1d SAME + bias + GLU +
residual) against the cuDNN composition of the same maths under autograd - `F.conv1d` with TF32 allowed, `F.glu`,
the add - forward and forward+backward, at the sizes a user runs, and a 6-layer F = 512 encoder stack the same way.
The two sides alternate in the same process.  TFLOP/s count the convolution's products only (2 * B*T * k*F * 2F per
forward, three times that per forward+backward); the share of peak is over the 495 TFLOP/s TF32 data-sheet figure of
the H100 SXM.  Prints a table and one JSON line; the card's name and power limit are read in the same run.

    python tools/convs2s_bench.py [--iters 50]
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as Fn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

TF32_PEAK_TFLOPS = 495.0
SHAPES = [(64, 50, 512, 3), (32, 100, 512, 5), (128, 30, 256, 3), (16, 10, 10, 5)]
STACK = (64, 50, 512, 3, 6)      # B, T, F, k, layers


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power = [s.strip() for s in out.split(",")]
    return name, power


def timed(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(iters):
        fn()
    ev1.record()
    ev1.synchronize()
    return ev0.elapsed_time(ev1) / iters


def cudnn_layer(x, w_oik, b):
    """[B,T,F] -> [B,T,F] over NCL F.conv1d: the same SAME padding ((k-1)//2 before, the rest after)."""
    k = w_oik.shape[2]
    before = (k - 1) // 2
    xc = Fn.pad(x.transpose(1, 2), (before, k - 1 - before))
    return Fn.glu(Fn.conv1d(xc, w_oik, b), dim=1).transpose(1, 2) + x


def main():
    parser = argparse.ArgumentParser()
    parser.add_argument("--iters", type=int, default=50)
    args = parser.parse_args()
    from neuralmonkey_b200 import ops
    torch.backends.cudnn.allow_tf32 = True
    torch.backends.cuda.matmul.allow_tf32 = True
    name, power = card()
    rows = []
    cases = [s + (1,) for s in SHAPES] + [STACK]
    for b, t, f, k, layers in cases:
        gen = torch.Generator(device="cuda").manual_seed(0)
        x = torch.randn(b, t, f, device="cuda", generator=gen, requires_grad=True)
        ws = [(torch.randn(k, f, 2 * f, device="cuda", generator=gen) * (4.0 / f) ** 0.5).requires_grad_()
              for _ in range(layers)]
        bs = [torch.zeros(2 * f, device="cuda", requires_grad=True) for _ in range(layers)]
        # cuDNN's own layout [2F, F, k], made once outside the timed region
        wc = [w.detach().permute(2, 1, 0).contiguous().requires_grad_() for w in ws]
        bc = [bb.detach().clone().requires_grad_() for bb in bs]
        dy = torch.randn(b, t, f, device="cuda", generator=gen)

        def ours():
            h = x
            for w, bb in zip(ws, bs):
                h = ops.conv1d_glu_residual(h, w, bb)
            return h

        def theirs():
            h = x
            for w, bb in zip(wc, bc):
                h = cudnn_layer(h, w, bb)
            return h

        def fwd(fn):
            def run():
                with torch.no_grad():
                    fn()
            return run

        def fwd_bwd(fn):
            def run():
                fn().backward(dy)
            return run

        with torch.no_grad():
            want = theirs()
            diff = float((ours() - want).abs().max() / want.abs().max())
        flops = 2.0 * b * t * k * f * 2 * f * layers
        times = {}
        for _ in range(2):          # alternate the two sides twice; keep the faster of each
            for key, fn in (("ours_fwd", fwd(ours)), ("cudnn_fwd", fwd(theirs)), ("ours_fb", fwd_bwd(ours)),
                            ("cudnn_fb", fwd_bwd(theirs))):
                ms = timed(fn, args.iters)
                times[key] = min(times.get(key, ms), ms)
        row = {"B": b, "T": t, "F": f, "k": k, "layers": layers, "max_rel_diff": diff}
        for key, ms in times.items():
            mult = 1 if key.endswith("fwd") else 3
            row[key + "_ms"] = round(ms, 4)
            row[key + "_tflops"] = round(mult * flops / ms / 1e9, 2)
            row[key + "_peak_share"] = round(mult * flops / ms / 1e9 / TF32_PEAK_TFLOPS, 4)
        row["fwd_ratio_to_cudnn"] = round(times["ours_fwd"] / times["cudnn_fwd"], 3)
        row["fb_ratio_to_cudnn"] = round(times["ours_fb"] / times["cudnn_fb"], 3)
        rows.append(row)

    print("{} at a {} power limit; ms per call, ratio = ours / cuDNN composition (< 1: faster)".format(name, power))
    print("{:>22} {:>9} {:>9} {:>7} {:>7} {:>6} {:>9} {:>9} {:>7} {:>6}".format(
        "B,T,F,k x layers", "fwd ms", "cudnn", "TFLOP/s", "peak", "ratio", "f+b ms", "cudnn", "TFLOP/s", "ratio"))
    for r in rows:
        print("{:>22} {:>9.4f} {:>9.4f} {:>7.1f} {:>6.1%} {:>6.2f} {:>9.4f} {:>9.4f} {:>7.1f} {:>6.2f}".format(
            "{},{},{},{} x {}".format(r["B"], r["T"], r["F"], r["k"], r["layers"]), r["ours_fwd_ms"],
            r["cudnn_fwd_ms"], r["ours_fwd_tflops"], r["ours_fwd_peak_share"], r["fwd_ratio_to_cudnn"],
            r["ours_fb_ms"], r["cudnn_fb_ms"], r["ours_fb_tflops"], r["fb_ratio_to_cudnn"]))
    sweep = kblock_sweep(ops, args.iters)
    print("forward per 32-wide k-block and CTA at B=64, T=50, F=512 (k = 1 -> 5, {} CTAs on {} SMs, 1 CTA per SM): "
          "{:.2f} us; the same block's wgmma products at the TF32 peak would take {:.2f} us".format(
              sweep["ctas"], sweep["sms"], sweep["us_per_kblock"], sweep["us_per_kblock_at_peak"]))
    print(json.dumps({"card": name, "power_limit": power, "rows": rows, "kblock_sweep": sweep}))


def kblock_sweep(ops, iters):
    """Forward time against the filter width at a fixed grid: the slope is what one CTA spends per 32-wide k-block
    (the wgmma forward runs 128 x 128 tiles, one CTA per SM at its register count)."""
    b, t, f = 64, 50, 512
    ms = {}
    for k in (1, 5):
        x = torch.randn(b, t, f, device="cuda")
        w = torch.randn(k, f, 2 * f, device="cuda") * (4.0 / f) ** 0.5
        bias = torch.zeros(2 * f, device="cuda")

        def run():
            with torch.no_grad():
                ops.conv1d_glu_residual(x, w, bias)
        ms[k] = min(timed(run, iters) for _ in range(2))
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ctas = -(-b * t // 128) * -(-f // 64)
    waves = -(-ctas // sms)
    kblocks = (5 - 1) * f // 32
    flop_per_kblock = 2.0 * 128 * 128 * 32
    return {"ms_k1": round(ms[1], 4), "ms_k5": round(ms[5], 4), "ctas": ctas, "sms": sms,
            "us_per_kblock": (ms[5] - ms[1]) * 1e3 / (kblocks * waves),
            "us_per_kblock_at_peak": flop_per_kblock / (TF32_PEAK_TFLOPS * 1e12 / sms) * 1e6}


if __name__ == "__main__":
    main()
