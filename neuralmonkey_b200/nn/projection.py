"""Multilayer projection (reference: neuralmonkey/nn/projection.py:38-57): dense layers with the activation and
dropout after EVERY layer, shared by the deep-output MLP of the RNN decoder, `MultilayerPerceptron` and
`SequenceRegressor`.  Layer i's variables are `<scope>/mlp_layer_<i>/kernel` and `.../bias` of the owning part."""
from typing import List

import torch

from neuralmonkey_b200 import ops
from neuralmonkey_b200.nn.utils import dropout
from neuralmonkey_b200.params import zeros_initializer


def activation_name(activation_fn) -> str:
    if callable(activation_fn):
        activation_fn = getattr(activation_fn, "__name__", str(activation_fn))
    if activation_fn not in ("tanh", "relu", "sigmoid"):
        raise ValueError("Unsupported activation {}".format(activation_fn))
    return activation_fn


def declare_multilayer_projection(part, scope: str, in_size: int, layer_sizes: List[int]) -> int:
    """Declare the layers on `part`; returns the width of the last one (in_size without layers)."""
    for i, width in enumerate(layer_sizes):
        pre = "{}/mlp_layer_{}/".format(scope, i)
        part.declare(pre + "kernel", [in_size, width])
        part.declare(pre + "bias", [width], zeros_initializer())
        in_size = width
    return in_size


def multilayer_projection(part, x: torch.Tensor, scope: str, layer_sizes: List[int], activation: str,
                          dropout_keep_prob: float, train_mode: bool) -> torch.Tensor:
    for i in range(len(layer_sizes)):
        pre = "{}/mlp_layer_{}/".format(scope, i)
        x = dropout(ops.linear(x, part.var(pre + "kernel"), part.var(pre + "bias"), act=activation),
                    dropout_keep_prob, train_mode)
    return x
