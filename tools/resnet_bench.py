"""Time the frozen resnet_v2_50 forward to block4 (ImageNet encoder, nm_conv2d_bn_fwd on the kernels of
csrc/conv_igemm.cuh) at batch 32 and 128 on 229x229 images, on both engines, next to the same network through cuDNN
(torch.nn.functional.conv2d with TF32 allowed, NHWC channels-last, alternating with ours in the same process, as a
comparison point only).  FLOPs are counted from the convolution shapes.  `--profile` adds a torch.profiler
per-kernel table from a separate run.  Prints a table and one JSON line; the card's name and power limit are read in
the same run.

    python tools/resnet_bench.py [--iters 10] [--profile]
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tests import resnet_oracle as RO  # noqa: E402

NET, LAYER = "resnet_v2_50", "resnet_v2_50/block4"


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
    except (OSError, subprocess.CalledProcessError):
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def conv_flops(size):
    """2 * N-free multiply-adds of every convolution up to block4 at a size x size input, per image."""
    total, side = 0, (size + 6 - 7) // 2 + 1
    total += 2 * side * side * 7 * 7 * 3 * 64
    side = -(-side // 2)
    for _scope, din, depth, bd, stride, _last in RO.units(NET):
        if din != depth:
            total += 2 * side * side * din * depth
        total += 2 * side * side * din * bd
        out = (side + 2 - 3) // stride + 1
        total += 2 * out * out * 9 * bd * bd
        total += 2 * out * out * bd * depth
        side = out
    return total


def ours(params):
    """The encoder's forward on the engine the GEMM backend selects at call time."""
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.encoders import ImageNet
    runtime.reset()
    enc = ImageNet(name="imagenet", data_id="images", network_type=NET, spatial_layer=LAYER)
    enc.ensure_declared()
    arena = runtime.arena()
    arena.finalize(runtime.device())
    arena.load_dict({n: params[n] for n in arena.order})

    def run(images):
        enc.feed_images(images)
        return enc.spatial_states
    return run


def cudnn(params):
    """The same network in NCHW-logical, channels-last tensors through cuDNN; batch norm folded per call as ours."""
    p = {n: v.cuda() for n, v in params.items()}
    w = {n: v.permute(3, 2, 0, 1).contiguous(memory_format=torch.channels_last) for n, v in p.items()
         if n.endswith("/weights")}

    def bn(x, scope, relu=True):
        scale = p[scope + "/gamma"] * torch.rsqrt(p[scope + "/moving_variance"] + RO.EPS)
        shift = p[scope + "/beta"] - p[scope + "/moving_mean"] * scale
        y = x * scale.view(1, -1, 1, 1) + shift.view(1, -1, 1, 1)
        return torch.relu(y) if relu else y

    def conv(x, name, stride=1, bias=None):
        k = w[name].shape[2]
        b, a = (k - 1) // 2, k - 1 - (k - 1) // 2
        if k > 1:
            x = F.pad(x, (b, a, b, a))
        return F.conv2d(x, w[name], bias, stride=stride)

    def run(images):
        x = images.permute(0, 3, 1, 2)
        x = conv(x, NET + "/conv1/weights", 2, p[NET + "/conv1/biases"])
        x = F.max_pool2d(F.pad(x, (1, 1, 1, 1), value=float("-inf")), 3, 2, ceil_mode=False)
        for scope, din, depth, _bd, stride, _last in RO.units(NET):
            pre = bn(x, scope + "/preact")
            sc = (conv(pre, scope + "/shortcut/weights", stride, p[scope + "/shortcut/biases"]) if din != depth
                  else x[:, :, ::stride, ::stride])
            h = bn(conv(pre, scope + "/conv1/weights"), scope + "/conv1/BatchNorm")
            h = bn(conv(h, scope + "/conv2/weights", stride), scope + "/conv2/BatchNorm")
            x = sc + conv(h, scope + "/conv3/weights", 1, p[scope + "/conv3/biases"])
        return x
    return run


def time_ms(fn, images, iters):
    fn(images)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        fn(images)
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batches", default="32,128")
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    torch.backends.cudnn.allow_tf32 = True
    torch.backends.cuda.matmul.allow_tf32 = True
    name, power = card()
    params = {n: v.float() for n, v in RO.random_params(NET, seed=1).items()}
    flops = conv_flops(229)
    from neuralmonkey_b200 import ops
    enc = ours(params)
    rows = []
    for batch in [int(b) for b in args.batches.split(",")]:
        images = torch.rand(batch, 229, 229, 3, device="cuda") * 2 - 1
        fns = {"tf32 (ours)": (enc, "auto"), "fp32 exact (ours)": (enc, "simt"), "cuDNN tf32": (cudnn(params), "auto")}
        best = {k: float("inf") for k in fns}
        for _ in range(args.rounds):      # alternate the implementations, keep each one's best round
            for label, (fn, backend) in fns.items():
                ops.set_gemm_backend(backend)
                best[label] = min(best[label], time_ms(fn, images, args.iters))
        ops.set_gemm_backend("auto")
        for label, ms in best.items():
            rows.append({"batch": batch, "impl": label, "ms": round(ms, 3),
                         "tflops": round(flops * batch / (ms * 1e-3) / 1e12, 1)})
            print("batch {:4d}  {:18s} {:9.2f} ms  {:6.1f} TFLOP/s".format(batch, label, ms, rows[-1]["tflops"]))
    print("card: {}, power limit {}; {:.2f} GFLOP per 229x229 image to block4".format(name, power, flops / 1e9))
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        ops.set_gemm_backend("auto")
        fn = enc
        images = torch.rand(32, 229, 229, 3, device="cuda") * 2 - 1
        fn(images)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                fn(images)
            torch.cuda.synchronize()
        print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=15))
    print(json.dumps({"bench": "resnet_v2_50_block4_forward", "card": name, "power_limit": power,
                      "gflop_per_image": round(flops / 1e9, 3), "rows": rows}))


if __name__ == "__main__":
    main()
