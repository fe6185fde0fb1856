"""Time the sentence classification kernels (csrc/classify.cu, and the Kim-CNN convolution on nm_gemm) at the shapes
of a realistic classifier - B=256 sentences of T=50 words, a bidirectional GRU of 300 (D=600), self-attentive
pooling with hidden 350 and R=30 heads, a Kim CNN over E=300 embeddings with filters (3,100), (4,100), (5,100) -
next to the PyTorch composition of the same maths (alternating in the same process, as a comparison point only),
and one training step of that whole classifier (MLP [512], Adam), with its forward+backward part alone.  Shares of peak: HBM bandwidth for the
pooling kernels (bytes the algorithm must move over 3.35 TB/s), TF32 for the CNN products (495 TFLOP/s); both are
data-sheet figures of the H100 SXM.  Prints a table and one JSON line; the card's name and power limit are read in
the same run.

    python tools/classifier_bench.py [--iters 50]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_TBS = 3.35
TF32_PEAK_TFLOPS = 495.0
B, T, D, R, HIDDEN, E, FILTERS, MLP = 256, 50, 600, 30, 350, 300, (3, 4, 5), 512


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


def fwd_bwd(fn, leaves, douts):
    def run():
        for x in leaves:
            x.grad = None
        outs = fn()
        outs = outs if isinstance(outs, tuple) else (outs,)
        torch.autograd.backward([o for o, d in zip(outs, douts) if d is not None], [d for d in douts if d is not None])
    return run


def torch_max_pool(x, m):
    mm = m.unsqueeze(-1)
    return (x * mm + 1e-15 * (1 - mm)).amax(1)


def torch_mean_pool(x, m):
    return (x * m.unsqueeze(-1)).sum(1) / (m.sum(1, keepdim=True) + 1e-8)


def torch_attentive(e, m, v):
    w = torch.softmax(e, 1) * m.unsqueeze(-1)
    w = w / (w.sum(1, keepdim=True) + 1e-8)
    return w, w.transpose(1, 2) @ v


def torch_conv(x, w, b):
    y = torch.nn.functional.conv1d(x.transpose(1, 2), w.permute(2, 1, 0), b)
    return torch.relu(y).amax(2)


def kernels(iters):
    from neuralmonkey_b200 import ops
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    gen = torch.Generator(device="cuda").manual_seed(0)
    lengths = torch.randint(5, T + 1, (B,), device="cuda", generator=gen)
    mask = (torch.arange(T, device="cuda")[None] < lengths[:, None]).float()
    x = torch.randn(B, T, D, device="cuda", generator=gen, requires_grad=True)
    dy = torch.randn(B, D, device="cuda", generator=gen)
    rows = []
    io = 4 * B * T * D
    for label, ours, theirs, nbytes_f, nbytes_b in (
            ("max pool", ops.seq_max_pool, torch_max_pool, io + 4 * B * T, 2 * io + 4 * B * T),
            ("mean pool", ops.seq_mean_pool, torch_mean_pool, io + 4 * B * T, io + 4 * B * T)):
        f_ours, f_theirs = timed(lambda: ours(x, mask), iters), timed(lambda: theirs(x, mask), iters)
        b_ours = timed(fwd_bwd(lambda: ours(x, mask), [x], [dy]), iters)
        b_theirs = timed(fwd_bwd(lambda: theirs(x, mask), [x], [dy]), iters)
        rows.append((label, "fwd", f_ours, f_theirs, "HBM", nbytes_f / (f_ours * 1e-3) / (HBM_TBS * 1e12)))
        rows.append((label, "fwd+bwd", b_ours, b_theirs, "HBM",
                     (nbytes_f + nbytes_b) / (b_ours * 1e-3) / (HBM_TBS * 1e12)))
    e = torch.randn(B, T, R, device="cuda", generator=gen, requires_grad=True)
    dw, dout = torch.randn(B, T, R, device="cuda", generator=gen), torch.randn(B, R, D, device="cuda", generator=gen)
    att_bytes = io + 4 * (2 * B * T * R + B * R * D)
    f_ours = timed(lambda: ops.attentive_pool(e, mask, x), iters)
    f_theirs = timed(lambda: torch_attentive(e, mask, x), iters)
    b_ours = timed(fwd_bwd(lambda: ops.attentive_pool(e, mask, x), [e, x], [dw, dout]), iters)
    b_theirs = timed(fwd_bwd(lambda: torch_attentive(e, mask, x), [e, x], [dw, dout]), iters)
    rows.append(("attentive pool R=30", "fwd", f_ours, f_theirs, "HBM", att_bytes / (f_ours * 1e-3) / (HBM_TBS * 1e12)))
    rows.append(("attentive pool R=30", "fwd+bwd", b_ours, b_theirs, "HBM",
                 3 * att_bytes / (b_ours * 1e-3) / (HBM_TBS * 1e12)))
    emb = torch.randn(B, T, E, device="cuda", generator=gen, requires_grad=True)
    for width in FILTERS:
        w = (torch.randn(width, E, 100, device="cuda", generator=gen) * 0.05).requires_grad_()
        bias = torch.zeros(100, device="cuda", requires_grad=True)
        dpool = torch.randn(B, 100, device="cuda", generator=gen)
        flops = 2.0 * (B * T - width + 1) * width * E * 100
        f_ours = timed(lambda: ops.conv1d_max_pool(emb, w, bias), iters)
        f_theirs = timed(lambda: torch_conv(emb, w, bias), iters)
        b_ours = timed(fwd_bwd(lambda: ops.conv1d_max_pool(emb, w, bias), [emb, w, bias], [dpool]), iters)
        b_theirs = timed(fwd_bwd(lambda: torch_conv(emb, w, bias), [emb, w, bias], [dpool]), iters)
        label = "kim cnn w={} E=300 F=100".format(width)
        rows.append((label, "fwd", f_ours, f_theirs, "TF32", flops / (f_ours * 1e-3) / (TF32_PEAK_TFLOPS * 1e12)))
        rows.append((label, "fwd+bwd", b_ours, b_theirs, "TF32",
                     3 * flops / (b_ours * 1e-3) / (TF32_PEAK_TFLOPS * 1e12)))
    pred = torch.randn(B, 1, device="cuda", generator=gen, requires_grad=True)
    target = torch.randn(B, device="cuda", generator=gen)
    one = torch.ones((), device="cuda")
    rows.append(("squared error B=256", "fwd+bwd",
                 timed(fwd_bwd(lambda: ops.squared_error(pred, target), [pred], [one]), iters),
                 timed(fwd_bwd(lambda: ((pred - target[:, None]) ** 2).mean(), [pred], [one]), iters), "-", None))
    return rows


class _Data:
    def __init__(self, series):
        self.series = series

    def __len__(self):
        return len(next(iter(self.series.values())))

    def get_series(self, name):
        return self.series[name]

    def maybe_get_series(self, name):
        return self.series.get(name)


def training_pass(iters):
    """(one training step: forward, backward and the Adam update of `CrossEntropyTrainer`, forward + backward
    alone) of the whole classifier, in ms."""
    from neuralmonkey_b200 import runtime, tf
    from neuralmonkey_b200.trainers import CrossEntropyTrainer
    from neuralmonkey_b200.decoders.classifier import Classifier
    from neuralmonkey_b200.encoders.attentive import AttentiveEncoder
    from neuralmonkey_b200.encoders.pooling import SequenceMaxPooling
    from neuralmonkey_b200.encoders.recurrent import SentenceEncoder
    from neuralmonkey_b200.encoders.sequence_cnn_encoder import SequenceCNNEncoder
    from neuralmonkey_b200.vocabulary import Vocabulary
    words = Vocabulary(["w{}".format(i) for i in range(10000)])
    enc = SentenceEncoder(name="enc", vocabulary=words, data_id="source", embedding_size=E, rnn_size=D // 2)
    att = AttentiveEncoder(name="att", input_sequence=enc, hidden_size=HIDDEN, num_heads=R)
    maxp = SequenceMaxPooling(name="maxp", input_sequence=enc)
    cnn = SequenceCNNEncoder(name="cnn", vocabulary=words, data_id="source", embedding_size=E,
                             filters=[(w, 100) for w in FILTERS])
    clf = Classifier(name="clf", encoders=[att, maxp, cnn], vocabulary=Vocabulary(["c{}".format(i) for i in range(5)]),
                     data_id="label", layers=[MLP], dropout_keep_prob=0.5)
    parts = [enc.input_sequence, enc, att, maxp, cnn, clf]
    trainer = CrossEntropyTrainer(decoders=[clf], l2_weight=1e-8, clip_norm=1.0,
                                  optimizer=tf.AdamOptimizer(learning_rate=1e-4))
    for p in trainer.parameterizeds:
        p.ensure_declared()
    runtime.arena().finalize(runtime.device())
    rng = np.random.RandomState(0)
    data = _Data({"source": [["w{}".format(i) for i in rng.randint(0, 10000, size=rng.randint(T // 2, T + 1))]
                             for _ in range(B - 1)] + [["w1"] * T],
                  "label": [["c{}".format(rng.randint(5))] for _ in range(B)]})

    def feed():
        for p in parts:
            p.feed_dict(data, train=True)

    def step():
        feed()
        trainer.train_step()

    def forward_backward():
        feed()
        clf.loss_sum_and_count[0].backward()
    return timed(step, iters), timed(forward_backward, iters)


def main():
    parser = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    parser.add_argument("--iters", type=int, default=50)
    args = parser.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("classifier_bench needs a GPU")
    name, power = card()
    rows = kernels(args.iters)
    step_ms, fwd_bwd_ms = training_pass(max(5, args.iters // 5))
    print("{} at a {} power limit; ms per call, torch = the PyTorch composition of the same maths".format(name, power))
    print("{:26s} {:8s} {:>8s} {:>8s} {:>6s} {:>8s}".format("kernel", "pass", "ours", "torch", "x", "%peak"))
    for label, kind, ours, theirs, bound, share in rows:
        print("{:26s} {:8s} {:8.3f} {:8.3f} {:6.2f} {:>8s}".format(
            label, kind, ours, theirs, ours / theirs, "-" if share is None else "{:.1f} {}".format(100 * share, bound)))
    print("classifier training step (B={}, T={}): {:.2f} ms, forward+backward alone {:.2f} ms".format(
        B, T, step_ms, fwd_bwd_ms))
    print(json.dumps({"card": name, "power_limit": power, "step_ms": step_ms, "forward_backward_ms": fwd_bwd_ms,
                      "kernels": [{"kernel": r[0], "pass": r[1], "ours_ms": r[2], "torch_ms": r[3],
                                   "peak_bound": r[4], "share_of_peak": r[5]} for r in rows]}))


if __name__ == "__main__":
    main()
