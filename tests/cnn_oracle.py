"""fp64 restatement of the CNN encoder's operations (reference: encoders/cnn_encoder.py, TF 1.x tf.layers), for the
tests.  Every function has the signature of its `neuralmonkey_b200.ops` counterpart, so the host tests can run the
model part over these in place of the kernels, and the GPU tests can compare the kernels with them.

What is restated of TensorFlow 1.x (not available to check against here):
  * conv2d: stride 1; `same` pads k-1 pixels, (k-1)//2 before and the rest after (the odd pixel bottom / right).
  * batch_normalization(momentum=0.99, epsilon=1e-3, center, scale) on 4-D input runs the fused kernel: training
    normalizes with the batch mean and the BIASED batch variance, and moves moving_variance toward the
    Bessel-corrected (unbiased) one; evaluation uses the moving statistics.
  * max / average pooling: `valid` drops what does not fill a window; `same` pads like conv2d, max ignores the
    padding and average divides by the number of pixels inside the image; the max-pool gradient goes to the first
    maximal pixel of the window.
  * AdadeltaOptimizer: accum = rho accum + (1-rho) g^2; update = sqrt(accum_update + eps) / sqrt(accum + eps) g;
    accum_update = rho accum_update + (1-rho) update^2; var -= lr update.
"""
from typing import Dict, Optional, Tuple

import torch
import torch.nn.functional as F


def conv_pads(k: int, padding: str) -> Tuple[int, int]:
    if padding == "valid":
        return 0, 0
    if padding == "same":
        return (k - 1) // 2, k - 1 - (k - 1) // 2
    raise ValueError(padding)


def conv2d(x, w, b, padding, act=None):
    """NHWC x, HWIO w."""
    pt, pb = conv_pads(w.shape[0], padding)
    xn = F.pad(x.permute(0, 3, 1, 2), (pt, pb, pt, pb))
    y = F.conv2d(xn, w.permute(3, 2, 0, 1))
    y = y.permute(0, 2, 3, 1)
    if b is not None:
        y = y + b
    return torch.relu(y) if act == "relu" else y


def batch_norm(x, gamma, beta, moving_mean, moving_var, training, relu=False, momentum=0.99, eps=1e-3):
    dims = tuple(range(x.dim() - 1))
    if training:
        mean = x.mean(dim=dims)
        var = ((x - mean) ** 2).mean(dim=dims)
        p = x.numel() // x.shape[-1]
        with torch.no_grad():
            # through .data: the update is invisible to autograd, as the kernel's is (the arena's variables share
            # one version counter)
            unbiased = var * p / max(p - 1, 1)
            moving_mean.data.copy_((momentum * moving_mean.double() + (1 - momentum) * mean.double()).to(moving_mean))
            moving_var.data.copy_((momentum * moving_var.double() + (1 - momentum) * unbiased.double()).to(moving_var))
    else:
        mean, var = moving_mean.to(x.dtype), moving_var.to(x.dtype)
    y = gamma * (x - mean) / torch.sqrt(var + eps) + beta
    return torch.relu(y) if relu else y


def pool_out(size: int, k: int, stride: int, padding: str) -> int:
    return -(-size // stride) if padding == "same" else (size - k) // stride + 1


def pool2d(x, k, stride, padding, kind):
    n, h, w, c = x.shape
    xn = x.permute(0, 3, 1, 2)
    if padding == "same":
        ho, wo = pool_out(h, k, stride, padding), pool_out(w, k, stride, padding)
        ph, pw = max((ho - 1) * stride + k - h, 0), max((wo - 1) * stride + k - w, 0)
        pads = (pw // 2, pw - pw // 2, ph // 2, ph - ph // 2)
    else:
        pads = (0, 0, 0, 0)
    if kind == "max":
        y = F.max_pool2d(F.pad(xn, pads, value=float("-inf")), k, stride)
    else:
        total = F.avg_pool2d(F.pad(xn, pads), k, stride, divisor_override=1)
        count = F.avg_pool2d(F.pad(torch.ones_like(xn[:, :1]), pads), k, stride, divisor_override=1)
        y = total / count
    return y.permute(0, 2, 3, 1)


def linear(x, w, b=None, act=None):
    y = x @ w
    if b is not None:
        y = y + b
    return torch.relu(y) if act == "relu" else y


def adadelta_step(params: Dict[str, torch.Tensor], grads: Dict[str, torch.Tensor],
                  accum: Dict[str, torch.Tensor], accum_update: Dict[str, torch.Tensor], lr: float, rho: float,
                  eps: float, clip_norm: Optional[float] = None) -> None:
    """In place, per tensor, after tf.clip_by_norm (the reference trainer's per-gradient clipping)."""
    for name, g in grads.items():
        if clip_norm:
            norm = torch.sqrt((g * g).sum())
            g = g * clip_norm / torch.maximum(norm, torch.tensor(clip_norm, dtype=g.dtype))
        accum[name] = rho * accum[name] + (1 - rho) * g * g
        update = torch.sqrt(accum_update[name] + eps) / torch.sqrt(accum[name] + eps) * g
        accum_update[name] = rho * accum_update[name] + (1 - rho) * update * update
        params[name] = params[name] - lr * update


def cnn_encoder(p: Dict[str, torch.Tensor], name: str, convolutions, images: torch.Tensor, batch_normalize: bool,
                train: bool, fully_connected=None) -> Dict[str, torch.Tensor]:
    """The reference's CNNEncoder.image_processing_layers / output (cnn_encoder.py:111-197) over `images` (already
    divided by 255), variables from `p` by their TF names; the moving statistics in `p` are updated in training.
    Dropout is left out (keep_prob 1)."""
    scope = name + "/convolutions/"

    def conv(s, x, pad):
        return conv2d(x, p[s + "/conv2d/kernel"], p[s + "/conv2d/bias"], pad)

    def bn(s, x, relu):
        if not batch_normalize:
            return torch.relu(x) if relu else x
        b = s + "/batch_normalization/"
        return batch_norm(x, p[b + "gamma"], p[b + "beta"], p[b + "moving_mean"], p[b + "moving_variance"], train,
                          relu)

    x = images
    mask = torch.sign(images.sum(dim=3, keepdim=True))
    channels = images.shape[3]
    for i, spec in enumerate(convolutions):
        if spec[0] == "C":
            k, stride, pad, cout = spec[1:]
            s = scope + "layer_{}_convolution".format(i)
            x = bn(s, conv(s, x, pad), True)
            mask = pool2d(mask, k, stride, pad, "max")
            channels = cout
        elif spec[0] in ("M", "A"):
            k, stride = spec[1], spec[2]
            x = pool2d(x, k, stride, "valid", "max" if spec[0] == "M" else "avg")
            mask = pool2d(mask, k, stride, "valid", "max")
        else:
            k, cout = spec[1], spec[2]
            s = scope + "layer_{}_resnet_block".format(i)
            before = x if cout == channels else bn(s + "/project_input", conv(s + "/project_input", x, "same"), False)
            after = conv(s + "/conv_a", bn(s + "/conv_a", x, True), "same")
            after = conv(s + "/conv_b", bn(s + "/conv_b", after, True), "same")
            x = after + before
            channels = cout
    if fully_connected is None:
        output = x.mean(dim=(1, 2))
    else:
        output = x.reshape(x.shape[0], -1)
        for i in range(len(fully_connected)):
            output = linear(output, p[name + "/mlp/mlp_layer_{}/kernel".format(i)],
                            p[name + "/mlp/mlp_layer_{}/bias".format(i)], "relu")
    b, h, w, c = x.shape
    return {"spatial_states": x, "spatial_mask": mask, "output": output,
            "temporal_states": x.permute(0, 2, 1, 3).reshape(b, w, h * c),
            "temporal_mask": (mask.squeeze(3).sum(dim=1) > 0).to(x.dtype)}
