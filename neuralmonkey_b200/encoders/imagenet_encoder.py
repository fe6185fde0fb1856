"""Pre-trained ImageNet encoder (reference: neuralmonkey/encoders/imagenet_encoder.py:16-258).

The reference imports the network definition from a checkout of tensorflow/models
(`research/slim/nets`, a third-party dependency that is not vendored) and runs it frozen
(`tf.stop_gradient`, :212,234).  What the hot path uses of it is the VGG convolution stack up
to a convolutional endpoint (tests/captioning.ini: `vgg_16/conv5/conv5_3`, [B,14,14,512]),
restated here from the published slim `nets/vgg.py`: blocks of 3x3/SAME conv + bias + ReLU
with 64-128-256-512-512 channels (2,2,3,3,3 convs for VGG-16; 2,2,4,4,4 for VGG-19), each
followed by a 2x2/2 max pool; variables `<net>/convB/convB_I/{weights,biases}` in HWIO
layout, which is the checkpoint layout.

The ResNet-v2 networks restate the published slim `nets/resnet_v2.py` / `nets/resnet_utils.py`
(`resnet_arg_scope`, `conv2d_same`, `bottleneck_v2`, `resnet_v2_block`) at the reference's 229x229
input, in inference mode (`is_training=False`, `global_pool=False`, `num_classes=None`):
  * root: `conv1` = 7x7/2 `conv2d_same` with 64 outputs and biases, no batch norm or activation,
    then `pool1`, a 3x3/2 SAME max pool (not an end point);
  * blocks (base_depth, units, stride): (64, 3, 2), (128, 4 | 4 | 8, 2), (256, 6 | 23 | 36, 2),
    (512, 3, 1) for 50 | 101 | 152; each unit has depth 4*base_depth and depth_bottleneck base_depth,
    the block's stride sits on its last unit;
  * unit: preact = relu(BN(x)); shortcut = x[:, ::s, ::s] when depth == depth_in, else a 1x1/s conv
    of preact with biases; conv1 = relu(BN(conv1x1(preact))); conv2 = relu(BN(conv2d_same(conv1, 3,
    s))); conv3 = conv1x1(conv2) with biases; output = shortcut + conv3;
  * batch norm: scale=True, epsilon=1e-5, the moving statistics; conv weights HWIO, no biases unless
    stated;
  * `conv2d_same(k, s)`: a SAME conv at s = 1, else explicit pads (k-1)//2 before and the rest after,
    then a VALID conv;
  * end points in slim's order: `<net>/conv1`, per unit `.../bottleneck_v2/{shortcut, conv1, conv2,
    conv3}` (shortcut only where it is a conv) and `.../bottleneck_v2`, per block `<net>/blockB`;
    `postnorm` follows block4 but is not an end point.
Batch-norm scale and shift are recomputed from the variables on every forward pass, so loading new
values takes effect at once.  The fully connected endpoints (fc6-fc8) and AlexNet are outside the
path (SURVEY.md section 8, a13).
"""
from typing import Any, Dict, List, Optional, Tuple

import numpy as np
import torch

from neuralmonkey_b200 import ops, runtime
from neuralmonkey_b200.decorators import tensor
from neuralmonkey_b200.model.model_part import ModelPart
from neuralmonkey_b200.model.parameterized import InitializerSpecs
from neuralmonkey_b200.model.stateful import SpatialStatefulWithOutput
from neuralmonkey_b200.params import ones_initializer, variance_scaling_initializer, zeros_initializer

VGG_BLOCKS = {"vgg_16": (2, 2, 3, 3, 3), "vgg_19": (2, 2, 4, 4, 4)}
VGG_CHANNELS = (64, 128, 256, 512, 512)
SUPPORTED_NETWORKS = ["alexnet_v2", "vgg_16", "vgg_19", "resnet_v2_50", "resnet_v2_101",
                      "resnet_v2_152"]
# (base_depth, units, stride) of block1..block4
RESNET_BLOCKS = {"resnet_v2_50": ((64, 3, 2), (128, 4, 2), (256, 6, 2), (512, 3, 1)),
                 "resnet_v2_101": ((64, 3, 2), (128, 4, 2), (256, 23, 2), (512, 3, 1)),
                 "resnet_v2_152": ((64, 3, 2), (128, 8, 2), (256, 36, 2), (512, 3, 1))}
BUILT_NETWORKS = sorted(VGG_BLOCKS) + sorted(RESNET_BLOCKS)
RESNET_BN_EPSILON = 1e-5


def vgg_layers(network_type: str) -> List[Tuple[str, str, int, int]]:
    """[(endpoint, kind, cin, cout)] in execution order."""
    layers = []
    cin = 3
    for block, (convs, cout) in enumerate(zip(VGG_BLOCKS[network_type], VGG_CHANNELS), 1):
        for i in range(1, convs + 1):
            layers.append(("{}/conv{}/conv{}_{}".format(network_type, block, block, i), "conv", cin, cout))
            cin = cout
        layers.append(("{}/pool{}".format(network_type, block), "pool", cout, cout))
    return layers


def resnet_units(network_type: str) -> List[Tuple[str, int, int, int, int, bool]]:
    """[(scope, depth_in, depth, depth_bottleneck, stride, last of its block)] of every bottleneck unit."""
    units = []
    depth_in = 64
    for block, (base, count, stride) in enumerate(RESNET_BLOCKS[network_type], 1):
        for unit in range(1, count + 1):
            scope = "{}/block{}/unit_{}/bottleneck_v2".format(network_type, block, unit)
            units.append((scope, depth_in, 4 * base, base, stride if unit == count else 1, unit == count))
            depth_in = 4 * base
    return units


def resnet_layers(network_type: str) -> List[Tuple[str, int, List[Tuple[str, List[int]]]]]:
    """[(end point, channels, [(variable, shape)] it adds)] in slim's end-point order."""
    def bn(scope, c):
        return [(scope + "/" + v, [c]) for v in ("beta", "gamma", "moving_mean", "moving_variance")]
    layers = [(network_type + "/conv1", 64, [(network_type + "/conv1/weights", [7, 7, 3, 64]),
                                             (network_type + "/conv1/biases", [64])])]
    for scope, din, depth, bd, _stride, last in resnet_units(network_type):
        preact = bn(scope + "/preact", din)
        if din != depth:
            layers.append((scope + "/shortcut", depth, preact + [(scope + "/shortcut/weights", [1, 1, din, depth]),
                                                                 (scope + "/shortcut/biases", [depth])]))
            preact = []
        layers.append((scope + "/conv1", bd,
                       preact + [(scope + "/conv1/weights", [1, 1, din, bd])] + bn(scope + "/conv1/BatchNorm", bd)))
        layers.append((scope + "/conv2", bd,
                       [(scope + "/conv2/weights", [3, 3, bd, bd])] + bn(scope + "/conv2/BatchNorm", bd)))
        layers.append((scope + "/conv3", depth, [(scope + "/conv3/weights", [1, 1, bd, depth]),
                                                 (scope + "/conv3/biases", [depth])]))
        layers.append((scope, depth, []))
        if last:
            layers.append((scope.rsplit("/", 2)[0], depth, []))
    return layers


def conv2d_same_pads(k: int) -> Tuple[int, int]:
    """The pads of slim's conv2d_same: SAME at stride 1, the same pads before a VALID conv at any stride."""
    return (k - 1) // 2, k - 1 - (k - 1) // 2


class ImageNet(ModelPart, SpatialStatefulWithOutput):
    # pylint: disable=too-many-arguments
    def __init__(self, name: str, data_id: str, network_type: str, slim_models_path: str = None,
                 load_checkpoint: str = None, spatial_layer: str = None, encoded_layer: str = None,
                 initializers: InitializerSpecs = None) -> None:
        ModelPart.__init__(self, name, load_checkpoint=load_checkpoint, initializers=initializers,
                           save_checkpoint=None)
        self.data_id = data_id
        self.network_type = network_type
        self.spatial_layer = spatial_layer
        self.encoded_layer = encoded_layer
        if self.network_type not in SUPPORTED_NETWORKS:
            raise ValueError("Network '{}' is not among the supported ones ({})".format(
                self.network_type, ", ".join(SUPPORTED_NETWORKS)))
        if self.network_type not in BUILT_NETWORKS:
            raise NotImplementedError("Only the {} networks are built (got '{}')".format(
                ", ".join(BUILT_NETWORKS), self.network_type))
        self.resnet = self.network_type in RESNET_BLOCKS
        if self.resnet:
            self.height, self.width = 229, 229
            self._resnet_layers = resnet_layers(network_type)
            endpoints = [l[0] for l in self._resnet_layers]
        else:
            self.height, self.width = 224, 224
            self._layers = vgg_layers(network_type)
            endpoints = [l[0] for l in self._layers]
        if self.spatial_layer is not None and self.spatial_layer not in endpoints:
            raise ValueError("Network '{}' does not contain endpoint '{}'".format(
                self.network_type, self.spatial_layer))
        if self.encoded_layer is not None:
            raise NotImplementedError("encoded_layer endpoints (fc6-fc8) are outside the hot path; "
                                      "leave it unset to average the convolutional maps")
        self._images = None  # type: Optional[torch.Tensor]

    def declare_variables(self) -> None:
        # slim networks live in their own top-level scope, independently of `name` (:113-114);
        # frozen: not trainable, so they sit behind the trainable prefix of the arena
        if self.resnet:
            for endpoint, _channels, variables in self._resnet_layers:
                for var, shape in variables:
                    init = (variance_scaling_initializer(2.0, "fan_in", "normal") if var.endswith("/weights")
                            else ones_initializer() if var.endswith(("/gamma", "/moving_variance"))
                            else zeros_initializer())
                    self.declare(var, shape, init, trainable=False, absolute=True)
                if endpoint == self.spatial_layer:
                    break
            return
        for endpoint, kind, cin, cout in self._layers:
            if kind != "conv":
                continue
            self.declare(endpoint + "/weights", [3, 3, cin, cout],
                         variance_scaling_initializer(2.0, "fan_in", "normal"), trainable=False,
                         absolute=True)
            self.declare(endpoint + "/biases", [cout], zeros_initializer(), trainable=False,
                         absolute=True)
            if endpoint == self.spatial_layer:
                break

    @property
    def input_types(self) -> Dict[str, Any]:
        return {self.data_id: float}

    @property
    def input_shapes(self) -> Dict[str, Any]:
        return {self.data_id: [None, self.height, self.width, 3]}

    def feed_dict(self, dataset, train: bool = False) -> Dict[str, Any]:
        fd = ModelPart.feed_dict(self, dataset, train)
        images = np.array(list(dataset.get_series(self.data_id)), dtype=np.float32)
        if images.shape[1:] != (self.height, self.width, 3):
            raise ValueError("ImageNet '{}' expects images of shape {}, got {}".format(
                self.name, (self.height, self.width, 3), images.shape[1:]))
        self.feed_images(torch.from_numpy(images), train)
        fd[self.data_id] = images
        return fd

    def feed_images(self, images: torch.Tensor, train: bool = False) -> None:
        """[batch, H, W, 3] float32 (any H, W divisible by the pooling the endpoint needs)."""
        self.reset_batch()
        self.train_mode = bool(train)
        self.batch_size = int(images.shape[0])
        self._images = runtime.to_device(images)

    def static_inputs(self) -> Dict[str, Any]:
        return {"images": self._images} if self._images is not None else {}

    def bind_static(self, tensors: Dict[str, Any]) -> None:
        self.reset_batch()
        if tensors:
            self._images = tensors["images"]

    @tensor
    def input_image(self) -> torch.Tensor:
        return self._images

    def _v(self, name: str) -> torch.Tensor:
        return self.var(name, absolute=True)

    def _bn(self, scope: str) -> Tuple[torch.Tensor, torch.Tensor]:
        """(scale, shift) of an inference-mode batch norm: y = x * scale + shift."""
        scale = self._v(scope + "/gamma") * torch.rsqrt(self._v(scope + "/moving_variance") + RESNET_BN_EPSILON)
        return scale, torch.addcmul(self._v(scope + "/beta"), self._v(scope + "/moving_mean"), scale, value=-1.0)

    def _resnet_end_points(self) -> Dict[str, torch.Tensor]:
        """The end points up to spatial_layer.  A unit's residual add runs inside its conv3, so a unit that is
        passed through keeps no separate conv3 end point; the preactivation runs inside the gathers of the
        convolutions that read it."""
        net, stop = self.network_type, self.spatial_layer
        points = {}
        x = ops.conv2d_bn_fwd(self.input_image, self._v(net + "/conv1/weights"), stride=2, pads=conv2d_same_pads(7),
                              bias=self._v(net + "/conv1/biases"))
        points[net + "/conv1"] = x
        if stop == net + "/conv1":
            return points
        x = ops.pool2d(x, 3, 2, "same", "max")
        for scope, din, depth, _bd, stride, last in resnet_units(net):
            pre_scale, pre_shift = self._bn(scope + "/preact")
            if din != depth:
                shortcut = ops.conv2d_bn_fwd(x, self._v(scope + "/shortcut/weights"), stride=stride,
                                             in_scale=pre_scale, in_shift=pre_shift,
                                             bias=self._v(scope + "/shortcut/biases"))
                points[scope + "/shortcut"] = shortcut
                if stop == scope + "/shortcut":
                    return points
                res_stride = 1
            else:
                shortcut, res_stride = x, stride
            scale, shift = self._bn(scope + "/conv1/BatchNorm")
            h = ops.conv2d_bn_fwd(x, self._v(scope + "/conv1/weights"), in_scale=pre_scale, in_shift=pre_shift,
                                  out_scale=scale, out_shift=shift, act="relu")
            points[scope + "/conv1"] = h
            if stop == scope + "/conv1":
                return points
            scale, shift = self._bn(scope + "/conv2/BatchNorm")
            h = ops.conv2d_bn_fwd(h, self._v(scope + "/conv2/weights"), stride=stride, pads=conv2d_same_pads(3),
                                  out_scale=scale, out_shift=shift, act="relu")
            points[scope + "/conv2"] = h
            if stop == scope + "/conv2":
                return points
            if stop == scope + "/conv3":
                points[stop] = ops.conv2d_bn_fwd(h, self._v(scope + "/conv3/weights"),
                                                 bias=self._v(scope + "/conv3/biases"))
                return points
            x = ops.conv2d_bn_fwd(h, self._v(scope + "/conv3/weights"), bias=self._v(scope + "/conv3/biases"),
                                  res=shortcut, res_stride=res_stride)
            points[scope] = x
            block = scope.rsplit("/", 2)[0]
            if last:
                points[block] = x
            if stop in (scope, block if last else None):
                return points
        return points

    @tensor
    def end_points(self) -> Dict[str, torch.Tensor]:
        if self.resnet:
            return self._resnet_end_points()
        points = {}
        x = self.input_image
        for endpoint, kind, _cin, _cout in self._layers:
            if kind == "conv":
                x = ops.conv3x3_bias_relu(x, self.var(endpoint + "/weights", absolute=True),
                                          self.var(endpoint + "/biases", absolute=True))
            else:
                x = ops.maxpool2x2(x)
            points[endpoint] = x
            if endpoint == self.spatial_layer:
                break
        return points

    @tensor
    def spatial_states(self) -> Optional[torch.Tensor]:
        if self.spatial_layer is None:
            return None
        return self.end_points[self.spatial_layer].detach()

    @tensor
    def spatial_mask(self) -> Optional[torch.Tensor]:
        if self.spatial_layer is None:
            return None
        s = self.spatial_states
        return torch.ones(s.shape[:3], device=s.device, dtype=torch.float32)

    @tensor
    def output(self) -> torch.Tensor:
        return self.spatial_states.mean(dim=(1, 2))

    @property
    def dimension(self) -> int:
        if self.resnet:
            for endpoint, channels, _variables in self._resnet_layers:
                if endpoint == self.spatial_layer:
                    return channels
            raise ValueError("spatial_layer is not set")
        for endpoint, _kind, _cin, cout in self._layers:
            if endpoint == self.spatial_layer:
                return cout
        raise ValueError("spatial_layer is not set")
