"""Trainable CNN image encoder (reference: neuralmonkey/encoders/cnn_encoder.py:28-355).

`CNNEncoder` runs a stack of layers over NHWC images, each given by a tuple:
    ("C", kernel_size, stride, padding, out_channels)  convolution + [batch norm] + ReLU
    ("M" / "A", pool_size, stride, padding)            max / average pooling
    ("R", kernel_size, out_channels)                   pre-activation residual block (needs batch_normalize)
and `CNNTemporalView` slices its last map left to right into a sequence (scene-text recognition, tests/str.ini).

The reference's quirks are kept, since checkpoints and configs depend on them:
  * `plain_convolution` (:209-241) never applies the stride to the convolution; it only strides the mask's max
    pooling.  A stride > 1 therefore gives a mask smaller than the states: that layer is refused here with a
    ValueError at build time instead of failing later on a shape mismatch.
  * `pooling` (:289-320) ignores its padding argument (after checking it) and always pools `valid`.
  * a residual block (:244-286) passes its input mask through unchanged.
Batch normalization moves its moving statistics in every forward pass made in training mode (`ops.batch_norm`, in
the same launch as the batch statistics).  The reference moves them when its trainer runs the UPDATE_OPS together
with the train op, which is once per forward pass in every trainer but `DelayedUpdateTrainer`: that one runs them
only with the update, so with `batches_per_update` > 1 it moves them once per update (from the last batch) where this
encoder moves them once per batch.
Convolutions, batch normalization and pooling are the sm_90a kernels of `csrc/cnn.cu` (`ops.conv2d`,
`ops.batch_norm`, `ops.pool2d`).
"""
from typing import Any, Dict, List, Optional, Tuple

import numpy as np
import torch

from neuralmonkey_b200 import distributed, ops, runtime
from neuralmonkey_b200.decorators import tensor
from neuralmonkey_b200.model.model_part import ModelPart
from neuralmonkey_b200.model.parameterized import InitializerSpecs
from neuralmonkey_b200.model.stateful import SpatialStatefulWithOutput, TemporalStatefulWithOutput
from neuralmonkey_b200.nn.utils import dropout
from neuralmonkey_b200.params import (ones_initializer, variance_scaling_initializer,
                                      zeros_initializer)
from neuralmonkey_b200.typecheck import check_argument_types

# tf.layers defaults: glorot-uniform kernels, zero biases; batch_normalization(momentum=0.99, epsilon=1e-3)
_GLOROT = variance_scaling_initializer(1.0, "fan_avg", "uniform")
BN_MOMENTUM = 0.99
BN_EPSILON = 1e-3


def _is_int(v: Any) -> bool:
    return isinstance(v, int) and not isinstance(v, bool)


def _check_spec(spec: Any, i: int) -> None:
    """The reference's checks of one layer tuple (check_argument_types inside each layer function)."""
    if not isinstance(spec, (tuple, list)) or not spec:
        raise ValueError("Specification of convolutional layer number {} must be a tuple, was {}".format(i, spec))
    kind = spec[0]
    if kind == "C":
        if len(spec) != 5 or not (_is_int(spec[1]) and _is_int(spec[2]) and isinstance(spec[3], str)
                                  and _is_int(spec[4])):
            raise ValueError(
                "Specification of a convolutional layer (number {} in config) needs to have 5 members: "
                '"C", kernel size, stride, padding, output channels, was {}'.format(i, spec))
        if spec[3] not in ("same", "valid"):
            raise ValueError("Padding must be 'same' or 'valid', was '{}' in layer {}.".format(spec[3], i + 1))
        if spec[1] < 1 or spec[2] < 1 or spec[4] < 1:
            raise ValueError("Kernel size, stride and channels of layer {} must be positive, was {}".format(
                i + 1, spec))
    elif kind in ("M", "A"):
        if len(spec) != 4 or not (_is_int(spec[1]) and _is_int(spec[2]) and isinstance(spec[3], str)):
            raise ValueError(
                "Specification of a max-pooling layer (number {} in config) needs to have 3 members: "
                '"M", pool size, stride, padding, was {}'.format(i, spec))
        if spec[3] not in ("same", "valid"):
            raise ValueError("Padding must be 'same' or 'valid', was '{}' in layer {}.".format(spec[3], i + 1))
        if spec[1] < 1 or spec[2] < 1:
            raise ValueError("Pool size and stride of layer {} must be positive, was {}".format(i + 1, spec))
    elif kind == "R":
        if len(spec) != 3 or not (_is_int(spec[1]) and _is_int(spec[2])):
            raise ValueError(
                "Specification of a residual block (number {} in config) needs to have 3 members: "
                '"R", kernel size, channels; was {}'.format(i, spec))
        if spec[1] < 1 or spec[2] < 1:
            raise ValueError("Kernel size and channels of layer {} must be positive, was {}".format(i + 1, spec))
    else:
        raise ValueError("Unknown type of convoutional layer #{}: '{}'".format(i + 1, kind))


def layer_shapes(convolutions: List[Tuple], height: int, width: int, channels: int,
                 batch_normalize: bool) -> List[Tuple[Tuple[int, int, int], Tuple[int, int]]]:
    """[((H, W, C) of the states, (H, W) of the mask)] after every layer; raises ValueError for a spec the
    reference rejects, and for a layer whose states and mask come out with different shapes."""
    h, w, c = height, width, channels
    out = []
    for i, spec in enumerate(convolutions):
        _check_spec(spec, i)
        kind = spec[0]
        if kind == "C":
            k, stride, pad, cout = spec[1:]
            if pad == "valid":
                if h < k or w < k:
                    raise ValueError("Layer {} ({}): the {}x{} map is smaller than the window".format(i + 1, spec, h, w))
                sh, sw = h - k + 1, w - k + 1
            else:
                sh, sw = h, w
            mh, mw = ops.pool_out(h, k, stride, pad), ops.pool_out(w, k, stride, pad)
            if (sh, sw) != (mh, mw):
                raise ValueError(
                    "Layer {} ({}): the convolution ignores its stride (as the reference's plain_convolution "
                    "does) but the mask is pooled with it, so the states would be {}x{} and the mask {}x{}".format(
                        i + 1, spec, sh, sw, mh, mw))
            h, w, c = sh, sw, cout
        elif kind in ("M", "A"):
            k, stride = spec[1], spec[2]
            if h < k or w < k:
                raise ValueError("Layer {} ({}): the {}x{} map is smaller than the window".format(i + 1, spec, h, w))
            h, w = ops.pool_out(h, k, stride, "valid"), ops.pool_out(w, k, stride, "valid")
        else:
            if not batch_normalize:
                raise ValueError("Using ResNet blocks requires batch normalization to be turned on.")
            c = spec[2]
        out.append(((h, w, c), (h, w)))
    return out


class CNNEncoder(ModelPart, SpatialStatefulWithOutput):
    """An image encoder: convolutions, pooling and residual blocks over [batch, height, width, pixel_dim]."""

    # pylint: disable=too-many-arguments
    def __init__(self, name: str, data_id: str, convolutions: List[Tuple], image_height: int, image_width: int,
                 pixel_dim: int, fully_connected: List[int] = None, batch_normalize: bool = False,
                 dropout_keep_prob: float = 0.5, reuse: ModelPart = None, save_checkpoint: str = None,
                 load_checkpoint: str = None, initializers: InitializerSpecs = None) -> None:
        check_argument_types()
        ModelPart.__init__(self, name, reuse, save_checkpoint, load_checkpoint, initializers)
        self.data_id = data_id
        self.dropout_keep_prob = dropout_keep_prob
        self.image_height = image_height
        self.image_width = image_width
        self.pixel_dim = pixel_dim
        self.convolutions = [tuple(c) if isinstance(c, list) else c for c in convolutions]
        self.fully_connected = fully_connected
        self.batch_normalize = batch_normalize
        self.shapes = layer_shapes(self.convolutions, image_height, image_width, pixel_dim, batch_normalize)
        if not self.shapes:
            raise ValueError("CNNEncoder '{}' needs at least one layer".format(name))
        self._images = None  # type: Optional[torch.Tensor]

    # -- variables -----------------------------------------------------------------------------
    def _declare_conv(self, scope: str, k: int, cin: int, cout: int) -> None:
        self.declare(scope + "/conv2d/kernel", [k, k, cin, cout], _GLOROT)
        self.declare(scope + "/conv2d/bias", [cout], zeros_initializer())

    def _declare_bn(self, scope: str, channels: int) -> None:
        if not self.batch_normalize:
            return
        bn = scope + "/batch_normalization/"
        self.declare(bn + "gamma", [channels], ones_initializer())
        self.declare(bn + "beta", [channels], zeros_initializer())
        # saved with the model, updated by the forward pass in training, never trained (no gradient, no L2)
        self.declare(bn + "moving_mean", [channels], zeros_initializer(), trainable=False)
        self.declare(bn + "moving_variance", [channels], ones_initializer(), trainable=False)

    def declare_variables(self) -> None:
        channels = self.pixel_dim
        for i, spec in enumerate(self.convolutions):
            if spec[0] == "C":
                scope = "convolutions/layer_{}_convolution".format(i)
                self._declare_conv(scope, spec[1], channels, spec[4])
                self._declare_bn(scope, spec[4])
                channels = spec[4]
            elif spec[0] == "R":
                scope = "convolutions/layer_{}_resnet_block".format(i)
                k, cout = spec[1], spec[2]
                if cout != channels:
                    self._declare_conv(scope + "/project_input", 1, channels, cout)
                    self._declare_bn(scope + "/project_input", cout)
                self._declare_bn(scope + "/conv_a", channels)
                self._declare_conv(scope + "/conv_a", k, channels, cout)
                self._declare_bn(scope + "/conv_b", cout)
                self._declare_conv(scope + "/conv_b", k, cout, cout)
                channels = cout
        if self.fully_connected is not None:
            (h, w, c), _ = self.shapes[-1]
            size = h * w * c
            for i, units in enumerate(self.fully_connected):
                self.declare("mlp/mlp_layer_{}/kernel".format(i), [size, units], _GLOROT)
                self.declare("mlp/mlp_layer_{}/bias".format(i), [units], zeros_initializer())
                size = units

    # -- feeding -------------------------------------------------------------------------------
    @property
    def input_types(self) -> Dict[str, Any]:
        return {self.data_id: float}

    @property
    def input_shapes(self) -> Dict[str, Any]:
        return {self.data_id: [None, self.image_height, self.image_width, self.pixel_dim]}

    def feed_dict(self, dataset, train: bool = False) -> Dict[str, Any]:
        fd = ModelPart.feed_dict(self, dataset, train)
        images = np.array(list(dataset.get_series(self.data_id)), dtype=np.float32)
        expected = (self.image_height, self.image_width, self.pixel_dim)
        if images.shape[1:] != expected:
            raise ValueError("CNNEncoder '{}' expects images of shape {}, got {}".format(
                self.name, expected, images.shape[1:]))
        images = images / np.float32(255.0)
        self.feed_images(torch.from_numpy(images), train)
        fd[self.data_id] = images
        return fd

    def feed_images(self, images: torch.Tensor, train: bool = False) -> None:
        """[batch, height, width, pixel_dim] float32, already divided by 255."""
        if self.batch_normalize and train and distributed.world_size() > 1:
            raise RuntimeError(
                "CNNEncoder '{}' normalizes with the statistics of each rank's batch: data-parallel ranks would "
                "each update with different statistics and could not reproduce the single-GPU step; train it on "
                "one rank".format(self.name))
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

    # -- the network ---------------------------------------------------------------------------
    @tensor
    def image_input(self) -> torch.Tensor:
        return self._images

    @tensor
    def image_mask(self) -> torch.Tensor:
        """1 where the pixel is non-zero in some channel: sign(sum over channels), [B, H, W, 1]."""
        return torch.sign(self.image_input.sum(dim=3, keepdim=True))

    def _conv(self, scope: str, x: torch.Tensor, padding: str, act: Optional[str] = None) -> torch.Tensor:
        return ops.conv2d(x, self.var(scope + "/conv2d/kernel"), self.var(scope + "/conv2d/bias"), padding, act)

    def _bn(self, scope: str, x: torch.Tensor, relu: bool) -> torch.Tensor:
        """batch_norm_callback (+ the ReLU that follows it, fused); without batch_normalize only the ReLU."""
        if not self.batch_normalize:
            return torch.relu(x) if relu else x
        bn = scope + "/batch_normalization/"
        return ops.batch_norm(x, self.var(bn + "gamma"), self.var(bn + "beta"), self.var(bn + "moving_mean"),
                              self.var(bn + "moving_variance"), self.train_mode, relu, BN_MOMENTUM, BN_EPSILON)

    @tensor
    def image_processing_layers(self) -> List[Tuple[torch.Tensor, torch.Tensor]]:
        x, mask = self.image_input, self.image_mask
        channels = self.pixel_dim
        layers = []
        for i, spec in enumerate(self.convolutions):
            if spec[0] == "C":
                k, stride, pad, cout = spec[1:]
                scope = "convolutions/layer_{}_convolution".format(i)
                if self.batch_normalize:
                    x = self._bn(scope, self._conv(scope, x, pad), relu=True)
                else:
                    x = self._conv(scope, x, pad, act="relu")
                mask = ops.pool2d(mask, k, stride, pad, "max")
                channels = cout
            elif spec[0] in ("M", "A"):
                k, stride = spec[1], spec[2]
                x = ops.pool2d(x, k, stride, "valid", "max" if spec[0] == "M" else "avg")
                mask = ops.pool2d(mask, k, stride, "valid", "max")
            else:
                k, cout = spec[1], spec[2]
                scope = "convolutions/layer_{}_resnet_block".format(i)
                if cout == channels:
                    before = x
                else:
                    before = self._bn(scope + "/project_input", self._conv(scope + "/project_input", x, "same"),
                                      relu=False)
                after = self._conv(scope + "/conv_a", self._bn(scope + "/conv_a", x, relu=True), "same")
                after = self._conv(scope + "/conv_b", self._bn(scope + "/conv_b", after, relu=True), "same")
                x = after + before
                channels = cout
            layers.append((x, mask))
        return layers

    @tensor
    def spatial_states(self) -> torch.Tensor:
        return self.image_processing_layers[-1][0]

    @tensor
    def spatial_mask(self) -> torch.Tensor:
        """[B, H', W', 1], as the reference returns it."""
        return self.image_processing_layers[-1][1]

    @tensor
    def output(self) -> torch.Tensor:
        """Mean of the last map over height and width, or the fully connected layers (ReLU + dropout after
        each) over the flattened map."""
        states = self.spatial_states
        if self.fully_connected is None:
            return states.mean(dim=(1, 2))
        x = states.reshape(states.shape[0], -1)
        for i in range(len(self.fully_connected)):
            x = ops.linear(x, self.var("mlp/mlp_layer_{}/kernel".format(i)),
                           self.var("mlp/mlp_layer_{}/bias".format(i)), act="relu")
            x = dropout(x, self.dropout_keep_prob, self.train_mode)
        return x

    @property
    def dimension(self) -> int:
        return self.shapes[-1][0][2]


class CNNTemporalView(ModelPart, TemporalStatefulWithOutput):
    """Slice the convolutional maps left to right: time = width, state = the column's height x channels."""

    def __init__(self, name: str, cnn: CNNEncoder) -> None:
        check_argument_types()
        ModelPart.__init__(self, name, save_checkpoint=None, load_checkpoint=None)
        self._cnn = cnn

    @tensor
    def output(self) -> torch.Tensor:
        return self._cnn.output

    @tensor
    def temporal_states(self) -> torch.Tensor:
        states = self._cnn.spatial_states
        b, h, w, c = states.shape
        return states.permute(0, 2, 1, 3).reshape(b, w, h * c)

    @tensor
    def temporal_mask(self) -> torch.Tensor:
        """1 for columns with at least one unmasked row."""
        summed = self._cnn.spatial_mask.squeeze(3).sum(dim=1)
        return (summed > 0).to(torch.float32)

    @property
    def dimension(self) -> int:
        (h, _w, c), _ = self._cnn.shapes[-1]
        return h * c

    @property
    def dependencies(self) -> List[str]:
        return super().dependencies + ["_cnn"]
