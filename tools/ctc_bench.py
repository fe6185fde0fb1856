"""Times the CTC kernels against PyTorch's CUDA CTC loss on the shapes of a character-level speech model.

For each shape (B, T, C, L) it prints one JSON line with:
  - ours_ms: `ops.ctc_loss` forward + backward (logits -> per-sentence loss -> dlogits);
  - torch_ms: `log_softmax` + `torch.nn.functional.ctc_loss(reduction="none")` forward + backward;
  - loss_max_rel_diff: the largest relative difference between the two implementations' losses;
  - greedy_ms: `ops.ctc_greedy_decode`;
  - bwd_ms, bwd_hbm_bound_ms, bwd_hbm_fraction: our backward call alone, the time its compulsory HBM traffic
    (logits read + dlogits written, B*T*C*4 bytes each) takes at the data sheet's 3.35 TB/s, and their ratio;
  - bwd_workspace_mb: what the backward additionally moves through its workspace (the fp64 alpha lattice read,
    the per-class occupancies written and read back), which that bound leaves out.
Sentences with no alignment count as loss 0 on both sides (`zero_infinity=True` for PyTorch).
Times are CUDA-event means over --iters calls after --warmup calls.  The first line names the card and its power
limit, read in the same run.

    python tools/ctc_bench.py [--iters 50] [--warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from neuralmonkey_b200 import ops  # noqa: E402

SHAPES = [(32, 200, 29, 60), (32, 800, 29, 200), (16, 1600, 29, 400), (32, 400, 1025, 60),
          (8, 2048, 3, 1000)]      # the last: two label classes, each repeated ~500 times in one sentence
HBM_BYTES_PER_S = 3.35e12      # H100 SXM data sheet


def _card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True)
    name, power = (out.stdout.strip().splitlines() or [","])[0].split(",")[:2]
    return {"gpu": name.strip(), "power_limit": power.strip()}


def _time(fn, iters: int, warmup: int) -> float:
    for _ in range(warmup):
        fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / iters


def _inputs(bsz, t_max, classes, max_label, seed=0):
    gen = torch.Generator().manual_seed(seed)
    logits = torch.randn(bsz, t_max, classes, generator=gen)
    frames = torch.randint(t_max * 3 // 4, t_max + 1, (bsz,), generator=gen, dtype=torch.int32)
    frames[0] = t_max
    lengths = torch.randint(max_label // 2, max_label + 1, (bsz,), generator=gen, dtype=torch.int32)
    lengths[0] = max_label
    labels = torch.randint(0, classes - 1, (bsz, max_label), generator=gen)
    return logits.cuda(), frames.cuda(), labels.cuda(), lengths.cuda()


def bench_shape(bsz, t_max, classes, max_label, iters, warmup) -> dict:
    logits, frames, labels, lengths = _inputs(bsz, t_max, classes, max_label)
    grad = torch.ones(bsz, device="cuda")

    def ours():
        x = logits.detach().requires_grad_(True)
        loss = ops.ctc_loss(x, frames, labels, lengths, True)
        loss.backward(grad)
        return loss

    def reference():
        x = logits.detach().requires_grad_(True)
        loss = torch.nn.functional.ctc_loss(torch.log_softmax(x, -1).transpose(0, 1), labels, frames.long(),
                                            lengths.long(), blank=classes - 1, reduction="none", zero_infinity=True)
        loss.backward(grad)
        return loss

    a, b = ours().detach(), reference().detach()
    rel = float(((a - b).abs() / b.abs().clamp_min(1e-6)).max())

    x = logits.detach().requires_grad_(True)
    loss = ops.ctc_loss(x, frames, labels, lengths, True)

    def backward_only():
        torch.autograd.backward(loss, grad, retain_graph=True)

    bwd_ms = _time(backward_only, iters, warmup)
    bound_ms = 2 * bsz * t_max * classes * 4 / HBM_BYTES_PER_S * 1e3
    workspace_bytes = bsz * t_max * ((2 * max_label + 1) * 8 + 2 * (max_label + 1) * 4)
    return {"shape": {"B": bsz, "T": t_max, "C": classes, "L": max_label},
            "ours_ms": round(_time(ours, iters, warmup), 4),
            "torch_ms": round(_time(reference, iters, warmup), 4),
            "loss_max_rel_diff": rel,
            "greedy_ms": round(_time(lambda: ops.ctc_greedy_decode(logits, frames, True), iters, warmup), 4),
            "bwd_ms": round(bwd_ms, 4), "bwd_hbm_bound_ms": round(bound_ms, 4),
            "bwd_hbm_fraction": round(bound_ms / bwd_ms, 4), "bwd_workspace_mb": round(workspace_bytes / 1e6, 1)}


def main() -> None:
    parser = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    parser.add_argument("--iters", type=int, default=50)
    parser.add_argument("--warmup", type=int, default=5)
    args = parser.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ctc_bench.py needs a CUDA device")
    print(json.dumps(_card()), flush=True)
    for shape in SHAPES:
        print(json.dumps(bench_shape(*shape, args.iters, args.warmup)), flush=True)


if __name__ == "__main__":
    main()
