"""Time the CNN encoder's convolutions (csrc/cnn.cu on the kernels of csrc/conv_igemm.cuh: forward, data gradient,
weight gradient) at tests/str.ini's own shapes and at a CRNN-like stack, next to cuDNN (torch.nn.functional.conv2d with TF32 allowed, alternating with ours in the same
process, as a comparison point only), and one full training step of the str.ini model.  Prints a table and one JSON
line; the card's name and power limit are read in the same run.

    python tools/cnn_bench.py [--iters 50]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

TF32_PEAK_TFLOPS = 495.0      # H100 SXM data sheet, dense TF32

# (label, N, H, W, Cin, Cout, k, padding)
LAYERS = [
    ("str C3 1->4 valid", 4, 32, 256, 1, 4, 3, "valid"),
    ("str R proj 4->12 1x1", 4, 15, 127, 4, 12, 1, "same"),
    ("str R conv_a 4->12", 4, 15, 127, 4, 12, 3, "same"),
    ("str R conv_b 12->12", 4, 15, 127, 12, 12, 3, "same"),
    ("crnn 1->64", 64, 32, 256, 1, 64, 3, "same"),
    ("crnn 64->128", 64, 16, 128, 64, 128, 3, "same"),
    ("crnn 128->256", 64, 8, 64, 128, 256, 3, "same"),
    ("crnn 256->256", 64, 8, 64, 256, 256, 3, "same"),
]


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power = [s.strip() for s in out.split(",")]
    return name, power


def timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(iters):
        fn()
    ev1.record()
    ev1.synchronize()
    return ev0.elapsed_time(ev1) / iters


def layer_calls(n, h, w, cin, cout, k, pad):
    from neuralmonkey_b200 import lib, ops
    from neuralmonkey_b200.lib import call, ptr
    pt, pb = ops.conv_pads(k, pad)
    ho, wo = h + pt + pb - k + 1, w + pt + pb - k + 1
    x = torch.randn(n, h, w, cin, device="cuda")
    wt = torch.randn(k, k, cin, cout, device="cuda") / (k * cin ** 0.5)
    b = torch.randn(cout, device="cuda")
    y = torch.empty(n, ho, wo, cout, device="cuda")
    dy = torch.randn(n, ho, wo, cout, device="cuda")
    dx = torch.empty_like(x)
    dw, db = torch.zeros_like(wt), torch.zeros_like(b)
    be = ops._conv_backend()
    ws = torch.empty(ops.conv_wgrad_workspace(n, h, w, cin, cout, k, pt, pb, be), device="cuda")
    ours = {
        "fwd": lambda: call("nm_conv2d_fwd", ptr(x), ptr(wt), ptr(b), ptr(y), n, h, w, cin, cout, k, pt, pb, pt, pb, 0,
                            0, be, lib.stream()),
        "dgrad": lambda: call("nm_conv2d_fwd", ptr(dy), ptr(wt), None, ptr(dx), n, ho, wo, cout, cin, k, k - 1 - pt,
                              k - 1 - pb, k - 1 - pt, k - 1 - pb, 1, 0, be, lib.stream()),
        "wgrad": lambda: call("nm_conv2d_wgrad", ptr(x), ptr(dy), ptr(dw), ptr(db), ptr(ws), ws.numel(), n, h, w, cin,
                              cout, k, pt, pb, pt, pb, be, lib.stream()),
    }
    # cuDNN on the same NHWC memory (channels_last views), explicit TF-style padding
    xn = x.permute(0, 3, 1, 2)
    wn = wt.permute(3, 2, 0, 1).contiguous(memory_format=torch.channels_last)
    dyn = dy.permute(0, 3, 1, 2)
    xpad = torch.nn.functional.pad(xn, (pt, pb, pt, pb)).contiguous(memory_format=torch.channels_last)

    def cud_bwd(mask):
        return torch.ops.aten.convolution_backward(dyn, xpad, wn, [cout], [1, 1], [0, 0], [1, 1], False, [0, 0], 1,
                                                   mask)
    cudnn = {
        "fwd": lambda: torch.nn.functional.conv2d(xpad, wn, b),
        "dgrad": lambda: cud_bwd([True, False, False]),
        "wgrad": lambda: cud_bwd([False, True, True]),
    }
    flops = 2.0 * n * ho * wo * cout * k * k * cin
    return ours, cudnn, flops


def str_step_ms(iters):
    from neuralmonkey_b200 import runtime, tf
    from neuralmonkey_b200.attention import Attention
    from neuralmonkey_b200.dataset import BatchingScheme, Dataset
    from neuralmonkey_b200.decoders.decoder import Decoder
    from neuralmonkey_b200.encoders import RecurrentEncoder
    from neuralmonkey_b200.encoders.cnn_encoder import CNNEncoder, CNNTemporalView
    from neuralmonkey_b200.trainers import CrossEntropyTrainer
    from neuralmonkey_b200.vocabulary import Vocabulary
    out = {}
    for graph in (False, True):
        runtime.reset()
        cnn = CNNEncoder(name="cnn", data_id="images", batch_normalize=True, image_height=32, image_width=256,
                         pixel_dim=1, dropout_keep_prob=0.5,
                         convolutions=[("C", 3, 1, "valid", 4), ("M", 2, 2, "same"), ("R", 3, 12),
                                       ("A", 2, 1, "same")])
        view = CNNTemporalView(name="cnn_in_time", cnn=cnn)
        enc = RecurrentEncoder(name="encoder", input_sequence=view, rnn_layers=[(256,)])
        att = Attention(name="attention_sentence_encoder", encoder=enc)
        dec = Decoder(name="decoder", encoders=[enc], attentions=[att], rnn_size=9, embedding_size=9,
                      dropout_keep_prob=0.5, data_id="target_chars", max_output_len=10,
                      vocabulary=Vocabulary(list("abcdefghijklmnopqrstuvwxyz")))
        trainer = CrossEntropyTrainer(decoders=[dec], l2_weight=1e-8, clip_norm=1.0, use_cuda_graph=graph,
                                      optimizer=tf.train.AdadeltaOptimizer(learning_rate=1e-4, epsilon=1e-6, rho=0.95))
        parts = (cnn, view, enc, att, dec)
        for part in parts:
            part.ensure_declared()
        runtime.arena().finalize(runtime.device())
        rng = np.random.RandomState(0)
        images = [rng.randint(0, 256, size=(32, 256, 1)).astype(np.float64) for _ in range(4)]
        words = [list("scene"), list("text"), list("recognition"[:8]), list("ocr")]
        data = Dataset("bench", {"images": lambda: iter(images), "target_chars": lambda: iter(words)},
                       BatchingScheme(batch_size=4))

        def step():
            for part in parts:
                part.feed_dict(data, train=True)
            trainer.train_step()
        for _ in range(3):
            step()
        torch.cuda.synchronize()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        for _ in range(iters):
            step()
        ev1.record()
        ev1.synchronize()
        out["graph" if graph else "eager"] = ev0.elapsed_time(ev1) / iters
    runtime.reset()
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("cnn_bench.py needs a GPU")
    torch.backends.cudnn.allow_tf32 = True
    torch.backends.cuda.matmul.allow_tf32 = True
    name, power = card()
    rows = []
    print("{} at power limit {}".format(name, power))
    print("{:<22} {:>5} {:>9} {:>9} {:>8} {:>7} {:>7}".format("layer", "pass", "ours ms", "cuDNN ms", "TFLOP/s",
                                                              "% peak", "ratio"))
    for label, *shape in LAYERS:
        ours, cudnn, flops = layer_calls(*shape)
        for kind in ("fwd", "dgrad", "wgrad"):
            t_ours, t_cud = [], []
            for _ in range(3):                       # alternate the two, take each one's best round
                t_ours.append(timed(ours[kind], args.iters))
                t_cud.append(timed(cudnn[kind], args.iters))
            a, c = min(t_ours), min(t_cud)
            tflops = flops / (a * 1e-3) / 1e12
            rows.append({"layer": label, "pass": kind, "ours_ms": a, "cudnn_ms": c, "tflops": tflops,
                         "peak_share": tflops / TF32_PEAK_TFLOPS})
            print("{:<22} {:>5} {:>9.4f} {:>9.4f} {:>8.2f} {:>6.1f}% {:>7.2f}".format(
                label, kind, a, c, tflops, 100 * tflops / TF32_PEAK_TFLOPS, a / c))
    step = str_step_ms(max(10, args.iters // 2))
    print("str.ini model, one training step (batch 4): eager {:.2f} ms, CUDA graph {:.2f} ms".format(
        step["eager"], step["graph"]))
    print(json.dumps({"card": name, "power_limit": power, "layers": rows, "str_step_ms": step}))


if __name__ == "__main__":
    main()
