"""Time supervised attention at the en-de training shape (B=256, Tx=50, NQ=50, A=C=600):

    alignment loss      ops.alignment_xent forward + backward (nm_alignment_xent_fwd / _bwd), and the share of the
                        3.35 TB/s HBM3 data-sheet bandwidth its compulsory bytes, 3*B*NQ*Tx*4 (energies and targets
                        read, energy gradient written), take over the measured time
    K4 backward         nm_bahdanau_bwd with and without de_in
    training step       one CrossEntropyTrainer step of the en-de-shaped model (vocabularies of 32000, sizes of
                        bench_models.ENDE_INI) with the decoder alone and with the decoder plus a WordAlignmentDecoder
                        (weights 1 and 1e-3), both eager

The kernel variants alternate within each round and every round is repeated (the two models, sharing one parameter
arena, are timed one after the other); the median over rounds is printed, in ms per call, from CUDA events around
`--iters` calls after warm-up.  The card's name and power limit are read in the same
process.

    python tools/alignment_bench.py [--iters N] [--rounds R]
"""
import argparse
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

B, TX, NQ, A, C = 256, 50, 50, 600, 600
HBM_BYTES_PER_S = 3.35e12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name(0)


def timed(runs, iters, rounds):
    for _n, fn in runs:
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    times = {n: [] for n, _ in runs}
    for _ in range(rounds):
        for n, fn in runs:
            start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            for _ in range(iters):
                fn()
            stop.record()
            stop.synchronize()
            times[n].append(start.elapsed_time(stop) / iters)
    for n, _ in runs:
        ts = times[n]
        print("  {:34s} {:9.4f} ms   (spread {:.4f}-{:.4f})".format(n, statistics.median(ts), min(ts), max(ts)))
    return {n: statistics.median(ts) for n, ts in times.items()}


def bench_kernels(iters, rounds):
    from neuralmonkey_b200 import lib, ops
    dev = torch.device("cuda")
    gen = torch.Generator(device=dev).manual_seed(0)
    energies = (torch.randn(B, NQ, TX, device=dev, generator=gen) * 2).requires_grad_()
    target = torch.rand(B, NQ, TX, device=dev, generator=gen)
    pad = (torch.rand(B, NQ, device=dev, generator=gen) < 0.9).float()

    def xent():
        ops.alignment_xent(energies, target, pad).backward()

    keys, values = torch.randn(B, TX, A, device=dev, generator=gen) * 0.5, torch.randn(B, TX, C, device=dev,
                                                                                         generator=gen)
    qproj, v, bias = torch.randn(B, NQ, A, device=dev, generator=gen) * 0.5, torch.randn(A, device=dev) * 0.1, \
        torch.zeros(1, device=dev)
    mask = torch.ones(B, TX, device=dev)
    e, w, ctx = (torch.empty(B, NQ, n, device=dev) for n in (TX, TX, C))
    p, st = lib.ptr, lib.stream()
    lib.call("nm_bahdanau_fwd", p(keys), p(values), p(mask), p(qproj), p(v), p(bias), p(e), p(w), p(ctx), B, TX, NQ,
             A, C, st)
    dctx, de_in = torch.randn(B, NQ, C, device=dev, generator=gen), torch.randn(B, NQ, TX, device=dev, generator=gen)
    dk, dval, dq = torch.empty_like(keys), torch.empty_like(values), torch.empty_like(qproj)
    dv, db, work = torch.zeros(A, device=dev), torch.zeros(1, device=dev), torch.empty(B * NQ * TX, device=dev)

    def k4_bwd(grad_e):
        lib.call("nm_bahdanau_bwd", p(keys), p(values), p(mask), p(qproj), p(v), p(e), p(w), p(dctx), p(grad_e),
                 p(dk), p(dval), p(dq), p(dv), p(db), p(work), B, TX, NQ, A, C, st)

    print("kernels: B={} Tx={} NQ={} A={} C={}; median of {} rounds x {} calls".format(B, TX, NQ, A, C, rounds,
                                                                                        iters))
    t = timed([("alignment loss fwd+bwd", xent), ("nm_bahdanau_bwd without de_in", lambda: k4_bwd(None)),
               ("nm_bahdanau_bwd with de_in", lambda: k4_bwd(de_in))], iters, rounds)
    nbytes = 3 * B * NQ * TX * 4
    ms = t["alignment loss fwd+bwd"]
    print("  alignment loss: {:.2f} MB compulsory, {:.1f} GB/s, {:.1%} of 3.35 TB/s".format(
        nbytes / 1e6, nbytes / (ms * 1e-3) / 1e9, nbytes / (ms * 1e-3) / HBM_BYTES_PER_S))


def bench_step(iters, rounds):
    from neuralmonkey_b200 import runtime, tf
    from neuralmonkey_b200.attention import Attention
    from neuralmonkey_b200.decoders import Decoder
    from neuralmonkey_b200.decoders.word_alignment_decoder import WordAlignmentDecoder
    from neuralmonkey_b200.encoders import SentenceEncoder
    from neuralmonkey_b200.trainers import CrossEntropyTrainer
    from neuralmonkey_b200.vocabulary import Vocabulary

    rng = np.random.RandomState(0)
    src = torch.from_numpy(rng.randint(4, 32000, size=(B, TX))).long()
    tgt = torch.from_numpy(rng.randint(4, 32000, size=(B, NQ))).long()
    tgt[:, -1] = 2
    ali = (rng.rand(B, NQ, TX) < 0.05).astype(np.float32)
    print("en-de training step (eager), B={} Tx={} T={}; one model at a time:".format(B, TX, NQ))
    for with_alignment in (False, True):
        runtime.reset()
        enc = SentenceEncoder(name="encoder", vocabulary=Vocabulary(["s{}".format(i) for i in range(31996)]),
                              data_id="source", embedding_size=300, rnn_size=300, max_input_len=TX)
        att = Attention(name="attention", encoder=enc)
        dec = Decoder(encoders=[enc], vocabulary=Vocabulary(["t{}".format(i) for i in range(31996)]),
                      data_id="target", name="decoder", max_output_len=NQ, rnn_size=300, embedding_size=300,
                      attentions=[att])
        decoders = [dec]
        if with_alignment:
            decoders.append(WordAlignmentDecoder(encoder=enc, decoder=dec, data_id="ali", name="alignment"))
        trainer = CrossEntropyTrainer(decoders=decoders, decoder_weights=[1., 1e-3][:len(decoders)],
                                      optimizer=tf.AdamOptimizer(learning_rate=1e-4))
        for part in trainer.parameterizeds:
            part.ensure_declared()
        runtime.arena().finalize(runtime.device())

        def step(enc=enc, att=att, dec=dec, decoders=decoders, trainer=trainer):
            enc.input_sequence.feed_ids([src], train=True)
            for part in (enc, att):
                part.reset_batch()
                part.train_mode = True
                part.batch_size = B
            dec.feed_ids(tgt, B, train=True)
            if len(decoders) > 1:
                decoders[1].reset_batch()
                decoders[1].train_mode, decoders[1].batch_size = True, B
                decoders[1]._alignment_host = ali         # pylint: disable=protected-access
            trainer.train_step()
        timed([("training step, decoder{}".format(" + alignment" if with_alignment else " alone"), step)], iters,
              rounds)


def main():
    parser = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    parser.add_argument("--iters", type=int, default=20)
    parser.add_argument("--rounds", type=int, default=5)
    args = parser.parse_args()
    from neuralmonkey_b200 import build
    build.build()
    print("card: {}".format(card()))
    bench_kernels(args.iters, args.rounds)
    bench_step(max(1, args.iters // 4), args.rounds)


if __name__ == "__main__":
    main()
