"""fp64 restatement of slim's ResNet-v2 feature extractor (nets/resnet_v2.py, nets/resnet_utils.py) in inference
mode with `global_pool=False, num_classes=None`, the way the reference's ImageNet encoder calls it.  Written with
torch.nn.functional only, without importing the port:
  * `conv2d_same(x, k, s)`: SAME at s = 1; at s > 1 explicit F.pad by (k-1)//2 before and the rest after, then VALID;
  * SAME max pooling pads with -inf, TF's way (the odd pixel after);
  * batch norm: y = (x - moving_mean) / sqrt(moving_variance + 1e-5) * gamma + beta.
Tensors are NHWC at the interface, filters HWIO, as in the slim checkpoints."""
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F

BLOCKS = {"resnet_v2_50": ((64, 3, 2), (128, 4, 2), (256, 6, 2), (512, 3, 1)),
          "resnet_v2_101": ((64, 3, 2), (128, 4, 2), (256, 23, 2), (512, 3, 1)),
          "resnet_v2_152": ((64, 3, 2), (128, 8, 2), (256, 36, 2), (512, 3, 1))}
EPS = 1e-5


def conv2d_same(x: torch.Tensor, w: torch.Tensor, stride: int, bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    """x NCHW, w HWIO."""
    k = w.shape[0]
    before, after = (k - 1) // 2, k - 1 - (k - 1) // 2   # at stride 1 these are SAME's pads too
    x = F.pad(x, (before, after, before, after))
    return F.conv2d(x, w.permute(3, 2, 0, 1), bias, stride=stride)


def conv2d_bn(x, w, stride=1, pads=(0, 0), in_scale=None, in_shift=None, out_scale=None, out_shift=None, bias=None,
              res=None, res_stride=1, act=None) -> torch.Tensor:
    """What nm_conv2d_bn_fwd computes, in fp64 over NHWC x and HWIO w: the input prologue is applied before the zero
    padding; y = act(z + res[:, ::res_stride, ::res_stride]), z = conv * out_scale + out_shift or conv + bias."""
    def c(t):
        return t.double().view(1, -1, 1, 1)
    a = x.double().permute(0, 3, 1, 2)
    if in_scale is not None:
        a = torch.relu(a * c(in_scale) + c(in_shift))
    a = F.pad(a, (pads[0], pads[1], pads[0], pads[1]))
    z = F.conv2d(a, w.double().permute(3, 2, 0, 1), stride=stride)
    if out_scale is not None:
        z = z * c(out_scale) + c(out_shift)
    elif bias is not None:
        z = z + c(bias)
    z = z.permute(0, 2, 3, 1)
    if res is not None:
        z = z + res.double()[:, ::res_stride, ::res_stride]
    return torch.relu(z) if act == "relu" else z


def max_pool_same(x: torch.Tensor, k: int, stride: int) -> torch.Tensor:
    h, w = x.shape[2], x.shape[3]
    ho, wo = -(-h // stride), -(-w // stride)
    ph, pw = max((ho - 1) * stride + k - h, 0), max((wo - 1) * stride + k - w, 0)
    x = F.pad(x, (pw // 2, pw - pw // 2, ph // 2, ph - ph // 2), value=float("-inf"))
    return F.max_pool2d(x, k, stride)


def batch_norm(x: torch.Tensor, p: Dict[str, torch.Tensor], scope: str) -> torch.Tensor:
    def c(name):
        return p[scope + "/" + name].view(1, -1, 1, 1)
    return (x - c("moving_mean")) / torch.sqrt(c("moving_variance") + EPS) * c("gamma") + c("beta")


def units(net: str) -> List[Tuple[str, int, int, int, int, bool]]:
    out, depth_in = [], 64
    for b, (base, count, stride) in enumerate(BLOCKS[net], 1):
        for u in range(1, count + 1):
            out.append(("{}/block{}/unit_{}/bottleneck_v2".format(net, b, u), depth_in, 4 * base, base,
                        stride if u == count else 1, u == count))
            depth_in = 4 * base
    return out


def end_point_names(net: str) -> List[str]:
    names = [net + "/conv1"]
    for scope, din, depth, _bd, _s, last in units(net):
        names += ([scope + "/shortcut"] if din != depth else []) + [scope + "/" + c for c in ("conv1", "conv2", "conv3")]
        names.append(scope)
        if last:
            names.append(scope.rsplit("/", 2)[0])
    return names


def variable_shapes(net: str) -> Dict[str, Tuple[int, ...]]:
    out = {net + "/conv1/weights": (7, 7, 3, 64), net + "/conv1/biases": (64,)}
    for scope, din, depth, bd, _s, _last in units(net):
        for v in ("beta", "gamma", "moving_mean", "moving_variance"):
            out["{}/preact/{}".format(scope, v)] = (din,)
            out["{}/conv1/BatchNorm/{}".format(scope, v)] = (bd,)
            out["{}/conv2/BatchNorm/{}".format(scope, v)] = (bd,)
        if din != depth:
            out[scope + "/shortcut/weights"] = (1, 1, din, depth)
            out[scope + "/shortcut/biases"] = (depth,)
        out[scope + "/conv1/weights"] = (1, 1, din, bd)
        out[scope + "/conv2/weights"] = (3, 3, bd, bd)
        out[scope + "/conv3/weights"] = (1, 1, bd, depth)
        out[scope + "/conv3/biases"] = (depth,)
    return out


def resnet_v2(p: Dict[str, torch.Tensor], net: str, images: torch.Tensor,
              stop: Optional[str] = None) -> Dict[str, torch.Tensor]:
    """Every end point (NHWC) up to and including `stop` (all of them when None)."""
    points = {}

    def emit(name, t):
        points[name] = t.permute(0, 2, 3, 1)
        return name == stop

    x = images.permute(0, 3, 1, 2)
    x = conv2d_same(x, p[net + "/conv1/weights"], 2, p[net + "/conv1/biases"])
    if emit(net + "/conv1", x):
        return points
    x = max_pool_same(x, 3, 2)
    for scope, din, depth, _bd, stride, last in units(net):
        preact = torch.relu(batch_norm(x, p, scope + "/preact"))
        if din == depth:
            shortcut = x[:, :, ::stride, ::stride]
        else:
            shortcut = conv2d_same(preact, p[scope + "/shortcut/weights"], stride, p[scope + "/shortcut/biases"])
            if emit(scope + "/shortcut", shortcut):
                return points
        h = torch.relu(batch_norm(conv2d_same(preact, p[scope + "/conv1/weights"], 1), p, scope + "/conv1/BatchNorm"))
        if emit(scope + "/conv1", h):
            return points
        h = torch.relu(batch_norm(conv2d_same(h, p[scope + "/conv2/weights"], stride), p,
                                  scope + "/conv2/BatchNorm"))
        if emit(scope + "/conv2", h):
            return points
        h = conv2d_same(h, p[scope + "/conv3/weights"], 1, p[scope + "/conv3/biases"])
        if emit(scope + "/conv3", h):
            return points
        x = shortcut + h
        if emit(scope, x):
            return points
        if last and emit(scope.rsplit("/", 2)[0], x):
            return points
    return points


def random_params(net: str, seed: int = 0, dtype: torch.dtype = torch.float64) -> Dict[str, torch.Tensor]:
    """He-scaled filters, small biases, batch-norm statistics that keep activations O(1) through the network."""
    gen = torch.Generator().manual_seed(seed)
    out = {}
    for name, shape in variable_shapes(net).items():
        if name.endswith("/weights"):
            fan_in = shape[0] * shape[1] * shape[2]
            t = torch.randn(shape, generator=gen, dtype=torch.float64) * (2.0 / fan_in) ** 0.5
        elif name.endswith("/gamma"):
            t = 0.5 + 0.5 * torch.rand(shape, generator=gen, dtype=torch.float64)
        elif name.endswith("/moving_variance"):
            t = 0.5 + torch.rand(shape, generator=gen, dtype=torch.float64)
        else:
            t = 0.1 * torch.randn(shape, generator=gen, dtype=torch.float64)
        out[name] = t.to(dtype)
    return out
