"""Time the joint multi-source attention (ops.joint_attention: nm_joint_attention_fwd / _bwd) forward and forward
plus backward at a multimodal training shape: B = 64 sentences, NQ = 30 decoder steps, a 40-token text encoder
beside 196 image regions, A = C = 512.

    flat J=0        the flat combination without the sentinel (Tx = 236 in two segments)
    flat sentinel   the same with the sentinel as one per-query candidate
    hier            the hierarchical combination over two K4 children (Tx = 40 and 196) and the sentinel (J = 3)
    K4 floor        nm_bahdanau_* at the same Tx = 236 with no candidates
    eager torch     the flat sentinel math composed of fp32 torch operations

Variants alternate within each round and every round is repeated; the median over rounds is printed, in ms per
call, from CUDA events around `--iters` calls after warm-up.  The card's name and power limit are read in the same
process.

    python tools/multiattention_bench.py [--iters N] [--rounds R]
"""
import argparse
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

B, NQ, TEXT, REGIONS, A, C = 64, 30, 40, 196, 512, 512


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name(0)


def eager(keys, values, mask, seg_ends, seg_bias, ckeys, cvalues, cand_bias, qproj, v):
    bias = torch.cat([seg_bias[s].expand(e - (seg_ends[s - 1] if s else 0)) for s, e in enumerate(seg_ends)])
    e = torch.cat([(v * torch.tanh(keys.unsqueeze(1) + qproj.unsqueeze(2))).sum(-1) + bias,
                   (v * torch.tanh(ckeys + qproj.unsqueeze(2))).sum(-1) + cand_bias], -1)
    w = torch.softmax(e, -1) * torch.cat([mask, mask.new_ones(mask.shape[0], ckeys.shape[2])], 1).unsqueeze(1)
    w = w / (w.sum(-1, keepdim=True) + 1e-8)
    tx = keys.shape[1]
    return (torch.einsum("bqt,btc->bqc", w[..., :tx], values)
            + torch.einsum("bqj,bqjc->bqc", w[..., tx:], cvalues)), w


def main():
    parser = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    parser.add_argument("--iters", type=int, default=50)
    parser.add_argument("--rounds", type=int, default=5)
    args = parser.parse_args()
    from neuralmonkey_b200 import build, ops
    build.build()
    dev = torch.device("cuda")
    gen = torch.Generator(device=dev).manual_seed(0)

    def r(*shape, scale=1.0):
        return (torch.randn(*shape, device=dev, generator=gen) * scale).requires_grad_()
    tx = TEXT + REGIONS
    keys, values = r(B, tx, A, scale=0.5), r(B, tx, C)
    lengths = torch.randint(10, TEXT + 1, (B,), device=dev, generator=gen)
    mask = torch.cat([(torch.arange(TEXT, device=dev)[None] < lengths[:, None]).float(),
                      torch.ones(B, REGIONS, device=dev)], 1)
    seg_bias, qproj, v = r(2, scale=0.1), r(B, NQ, A, scale=0.5), r(A, scale=0.1)
    ckeys, cvalues, cand_bias = r(B, NQ, 1, A, scale=0.5), r(B, NQ, 1, C), r(1, scale=0.1)
    hkeys, hvalues, hbias = r(B, NQ, 3, A, scale=0.5), r(B, NQ, 3, C), r(3, scale=0.1)
    k4_bias = r(1, scale=0.1)
    text_k, text_v, img_k, img_v = r(B, TEXT, A, scale=0.5), r(B, TEXT, C), r(B, REGIONS, A, scale=0.5), r(B, REGIONS, C)
    ends = [TEXT, tx]
    dctx = torch.randn(B, NQ, C, device=dev, generator=gen)

    def flat0():
        return ops.joint_attention(keys, values, mask, ends, seg_bias, None, None, None, qproj, v)[0]

    def flat_sentinel():
        return ops.joint_attention(keys, values, mask, ends, seg_bias, ckeys, cvalues, cand_bias, qproj, v)[0]

    def hier():
        c_text = ops.bahdanau_attention(text_k, text_v, mask[:, :TEXT], qproj, v, k4_bias)[0]
        c_img = ops.bahdanau_attention(img_k, img_v, None, qproj, v, k4_bias)[0]
        ck = torch.stack([c_text, c_img, hkeys[:, :, 2]], 2)
        return ops.joint_attention(None, None, None, [], None, ck, hvalues, hbias, qproj, v)[0]

    def k4():
        return ops.bahdanau_attention(keys, values, mask, qproj, v, k4_bias)[0]

    def torch_eager():
        return eager(keys, values, mask, ends, seg_bias, ckeys, cvalues, cand_bias, qproj, v)[0]

    variants = [("flat J=0", flat0), ("K4 floor", k4), ("flat sentinel", flat_sentinel), ("hier", hier),
                ("eager torch", torch_eager)]

    def fwd(fn):
        with torch.no_grad():
            fn()

    def fwd_bwd(fn):
        out = fn()
        out.backward(dctx)

    times = {(name, mode): [] for name, _ in variants for mode in ("fwd", "fwd+bwd")}
    for name, fn in variants:
        for _ in range(3):
            fwd(fn)
            fwd_bwd(fn)
    torch.cuda.synchronize()
    for _ in range(args.rounds):
        for name, fn in variants:
            for mode, run in (("fwd", fwd), ("fwd+bwd", fwd_bwd)):
                start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                start.record()
                for _ in range(args.iters):
                    run(fn)
                stop.record()
                stop.synchronize()
                times[(name, mode)].append(start.elapsed_time(stop) / args.iters)
    print("card: {}".format(card()))
    print("shape: B={} NQ={} Tx={}+{} A={} C={}; median of {} rounds x {} calls, ms per call".format(
        B, NQ, TEXT, REGIONS, A, C, args.rounds, args.iters))
    for name, _ in variants:
        print("{:14s} fwd {:8.3f}   fwd+bwd {:8.3f}   (spread fwd {:.3f}-{:.3f})".format(
            name, statistics.median(times[(name, "fwd")]), statistics.median(times[(name, "fwd+bwd")]),
            min(times[(name, "fwd")]), max(times[(name, "fwd")])))


if __name__ == "__main__":
    main()
