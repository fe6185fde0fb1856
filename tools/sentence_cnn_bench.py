"""Device times of the character-level sentence encoder at the shape of Lee, Cho & Hofmann (2017): B = 64 sentences
of 400 characters, 128-wide character embeddings, filter widths 1-8 with 200-300 filters each (2100 channels),
segments of 5, 4 highway layers.  The GRU is run at rnn_size 256: the cluster GRU covers H <= 320 (the paper uses 512).

  conv      the eight convolutions + bias + ReLU + segment max, forward and forward + backward, against cuDNN's
            conv1d + ReLU + max_pool1d (TF32 allowed) at the same shape
  highway   one highway layer forward + backward, against the PyTorch composition (TF32 matmuls)
  encoder   one SentenceCNNEncoder forward + backward, on the wgmma (TF32) engine and the exact fp32 one

CUDA events around `--iters` calls after `--warmup` calls; the card's name and power limit are read in the same run.

    python tools/sentence_cnn_bench.py [--iters 20] [--warmup 5] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

B, T, E, S, DEPTH, RNN = 64, 400, 128, 5, 4, 256
FILTERS = [(1, 200), (2, 200), (3, 250), (4, 250), (5, 300), (6, 300), (7, 300), (8, 300)]
D = sum(n for _, n in FILTERS)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters


def conv_flops():
    return sum(2.0 * B * T * k * E * n for k, n in FILTERS)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sentence_cnn_bench needs a CUDA device")
    from neuralmonkey_b200 import ops, runtime
    from neuralmonkey_b200.encoders import SentenceCNNEncoder
    from neuralmonkey_b200.model.sequence import Sequence
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(B, T, E, device="cuda", generator=g)
    ws = [(torch.randn(k, E, n, device="cuda", generator=g) * (1.0 / (k * E) ** 0.5), torch.zeros(n, device="cuda"))
          for k, n in FILTERS]
    res = {"card": card(), "shape": dict(B=B, T=T, E=E, filters=FILTERS, segment=S, highway=DEPTH, rnn_size=RNN)}

    # -- convolutions + ReLU + segment max ---------------------------------------------------------------------------
    def ours_conv(train):
        xi = x.detach().requires_grad_(train)
        params = [(w.detach().requires_grad_(train), b.detach().requires_grad_(train)) for w, b in ws]
        out = torch.cat([ops.pool2d(ops.conv1d(xi, w, b, "same", "relu").unsqueeze(2), S, S, "same", "max").squeeze(2)
                         for w, b in params], 2)
        if train:
            out.backward(torch.ones_like(out))
        return out

    wt = [(w.permute(2, 1, 0).contiguous(), b) for w, b in ws]

    def cudnn_conv(train):
        xi = x.detach().transpose(1, 2).contiguous().requires_grad_(train)
        outs = []
        for (k, _), (w, b) in zip(FILTERS, wt):
            w, b = w.detach().requires_grad_(train), b.detach().requires_grad_(train)
            pb = (k - 1) // 2
            y = F.relu(F.conv1d(F.pad(xi, (pb, k - 1 - pb)), w, b))
            tp = -(-T // S)
            pad = (tp - 1) * S + S - T
            outs.append(F.max_pool1d(F.pad(y, (pad // 2, pad - pad // 2), value=float("-inf")), S, S))
        out = torch.cat(outs, 1)
        if train:
            out.backward(torch.ones_like(out))
        return out

    flops = conv_flops()
    for name, fn in (("ours", ours_conv), ("cudnn", cudnn_conv)):
        f_ms = timed(lambda: fn(False), args.iters, args.warmup)
        fb_ms = timed(lambda: fn(True), args.iters, args.warmup)
        res["conv_" + name] = {"fwd_ms": round(f_ms, 3), "fwd_bwd_ms": round(fb_ms, 3),
                               "fwd_tflops": round(flops / f_ms / 1e9, 1),
                               "fwd_bwd_tflops": round(3 * flops / fb_ms / 1e9, 1)}

    # -- one highway layer ----------------------------------------------------------------------------------------
    n_rows = B * (-(-T // S))
    h = torch.randn(n_rows, D, device="cuda", generator=g)
    wh, wtr = (torch.randn(D, D, device="cuda", generator=g) / D ** 0.5 for _ in range(2))
    bh, bt = torch.full((D,), -1.0, device="cuda"), torch.full((D,), -1.0, device="cuda")

    def ours_highway():
        hi, a, c, p, q = (t.detach().requires_grad_(True) for t in (h, wh, wtr, bh, bt))
        y = ops.highway_gate(ops.linear(hi, a, p), ops.linear(hi, c, q), hi)
        y.backward(torch.ones_like(y))

    def torch_highway():
        hi, a, c, p, q = (t.detach().requires_grad_(True) for t in (h, wh, wtr, bh, bt))
        gate = torch.sigmoid(hi @ c + q)
        y = torch.relu(hi @ a + p) * gate + hi * (1 - gate)
        y.backward(torch.ones_like(y))

    hw_flops = 3 * 2 * 2.0 * n_rows * D * D
    for name, fn in (("ours", ours_highway), ("torch", torch_highway)):
        ms = timed(fn, args.iters, args.warmup)
        res["highway_" + name] = {"fwd_bwd_ms": round(ms, 3), "tflops": round(hw_flops / ms / 1e9, 1)}

    # -- the whole encoder -----------------------------------------------------------------------------------------
    mask = torch.ones(B, T, device="cuda")
    mask[B // 2:, T - 57:] = 0
    states = x * mask.unsqueeze(-1)

    class Inputs(Sequence):
        temporal_states = property(lambda self: states)
        temporal_mask = property(lambda self: mask)
        dimension = property(lambda self: E)

    runtime.reset()
    enc = SentenceCNNEncoder(name="enc", input_sequence=Inputs("inputs"), segment_size=S, highway_depth=DEPTH,
                             rnn_size=RNN, filters=FILTERS)
    enc.ensure_declared()
    runtime.arena().finalize(runtime.device())
    enc.train_mode = True

    def encoder_step():
        enc.reset_batch()
        out = enc.temporal_states
        loss = out.sum() + enc.output.sum()
        loss.backward()
        runtime.arena().fold_autograd_grads()

    for engine in ("auto", "simt"):
        ops.set_gemm_backend(engine)
        ms = timed(encoder_step, args.iters, args.warmup)
        res["encoder_" + ("tf32" if engine == "auto" else "exact_fp32")] = {"fwd_bwd_ms": round(ms, 3)}
    ops.set_gemm_backend("auto")
    line = json.dumps(res)
    print(line)
    if args.json:
        with open(args.json, "w") as handle:
            handle.write(line + "\n")


if __name__ == "__main__":
    main()
