"""Deep-output projections (reference: neuralmonkey/decoders/output_projection.py:76-188).

An OutputProjection maps (cell output, embedded input, contexts) of ANY number of rows to the
vector the vocabulary projection consumes; in training the rows are all T*B positions at
once.  It declares its variables under the decoder's `attention_decoder/` scope.
"""
from typing import List, Tuple

import torch

from neuralmonkey_b200 import ops
from neuralmonkey_b200.nn.utils import dropout
from neuralmonkey_b200.params import zeros_initializer


class OutputProjection:
    size = 0

    def declare(self, decoder, in_size: int) -> None:
        raise NotImplementedError

    def __call__(self, decoder, prev_state: torch.Tensor, prev_output: torch.Tensor,
                 ctx_tensors: List[torch.Tensor], train_mode: bool) -> torch.Tensor:
        raise NotImplementedError


class _Nonlinear(OutputProjection):
    def __init__(self, output_size: int, activation: str, dropout_keep_prob: float) -> None:
        self.size = output_size
        self.activation = activation
        self.dropout_keep_prob = dropout_keep_prob

    def declare(self, decoder, in_size):
        decoder.declare("attention_decoder/dense/kernel", [in_size, self.size])
        decoder.declare("attention_decoder/dense/bias", [self.size], zeros_initializer())

    def __call__(self, decoder, prev_state, prev_output, ctx_tensors, train_mode):
        cat = torch.cat([prev_state, prev_output] + list(ctx_tensors), -1)
        y = ops.linear(cat, decoder.var("attention_decoder/dense/kernel"),
                       decoder.var("attention_decoder/dense/bias"), act=self.activation)
        return dropout(y, self.dropout_keep_prob, train_mode)


class _Maxout(OutputProjection):
    def __init__(self, maxout_size: int, dropout_keep_prob: float) -> None:
        self.size = maxout_size
        self.dropout_keep_prob = dropout_keep_prob

    def declare(self, decoder, in_size):
        pre = "attention_decoder/MaxoutProjection/MaxoutProjection/"
        decoder.declare(pre + "kernel", [in_size, 2 * self.size])
        decoder.declare(pre + "bias", [2 * self.size], zeros_initializer())

    def __call__(self, decoder, prev_state, prev_output, ctx_tensors, train_mode):
        pre = "attention_decoder/MaxoutProjection/MaxoutProjection/"
        cat = torch.cat([prev_state, prev_output] + list(ctx_tensors), -1)
        z = ops.linear(cat, decoder.var(pre + "kernel"), decoder.var(pre + "bias"))
        return dropout(ops.maxout(z), self.dropout_keep_prob, train_mode)


def nonlinear_output(output_size: int, activation_fn: str = "tanh",
                     dropout_keep_prob: float = 1.0) -> Tuple[OutputProjection, int]:
    """activation(dense([state; emb; ctx])) (output_projection.py:115-130)."""
    if callable(activation_fn):
        activation_fn = getattr(activation_fn, "__name__", str(activation_fn))
    if activation_fn not in ("tanh", "relu", "sigmoid"):
        raise ValueError("Unsupported activation {}".format(activation_fn))
    return _Nonlinear(output_size, activation_fn, dropout_keep_prob), output_size


def maxout_output(maxout_size: int, dropout_keep_prob: float = 1.0) -> Tuple[OutputProjection, int]:
    """Maxout deep output (output_projection.py:133-160): dense to 2*size, then
    max(first half, second half) as nn/projection.py:7-35 actually computes."""
    return _Maxout(maxout_size, dropout_keep_prob), maxout_size


class _Nematus(OutputProjection):
    def __init__(self, output_size: int, activation: str, dropout_keep_prob: float) -> None:
        self.size, self.activation, self.dropout_keep_prob = output_size, activation, dropout_keep_prob

    _PARTS = ("rnn_state", "prev_out", "context")

    def declare(self, decoder, in_size):
        ctx_size = in_size - decoder.rnn_size - decoder.embedding_size
        for name, width in zip(self._PARTS, (decoder.rnn_size, decoder.embedding_size, ctx_size)):
            decoder.declare("attention_decoder/{}/kernel".format(name), [width, self.size])
            decoder.declare("attention_decoder/{}/bias".format(name), [self.size], zeros_initializer())

    def __call__(self, decoder, prev_state, prev_output, ctx_tensors, train_mode):
        ctx = ctx_tensors[0] if len(ctx_tensors) == 1 else torch.cat(list(ctx_tensors), -1)
        total = None
        for name, x in zip(self._PARTS, (prev_state, prev_output, ctx)):
            y = ops.linear(x, decoder.var("attention_decoder/{}/kernel".format(name)),
                           decoder.var("attention_decoder/{}/bias".format(name)))
            total = y if total is None else total + y
        return dropout(getattr(torch, self.activation)(total), self.dropout_keep_prob, train_mode)


class _MLP(OutputProjection):
    def __init__(self, layer_sizes: List[int], activation: str, dropout_keep_prob: float) -> None:
        self.layer_sizes, self.size = list(layer_sizes), layer_sizes[-1]
        self.activation, self.dropout_keep_prob = activation, dropout_keep_prob

    def declare(self, decoder, in_size):
        for i, width in enumerate(self.layer_sizes):
            pre = "attention_decoder/deep_output_mlp/mlp_layer_{}/".format(i)
            decoder.declare(pre + "kernel", [in_size, width])
            decoder.declare(pre + "bias", [width], zeros_initializer())
            in_size = width

    def __call__(self, decoder, prev_state, prev_output, ctx_tensors, train_mode):
        x = torch.cat([prev_state, prev_output] + list(ctx_tensors), -1)
        for i in range(len(self.layer_sizes)):
            pre = "attention_decoder/deep_output_mlp/mlp_layer_{}/".format(i)
            # multilayer_projection (nn/projection.py:38-57): activation and dropout after EVERY layer
            x = dropout(ops.linear(x, decoder.var(pre + "kernel"), decoder.var(pre + "bias"), act=self.activation),
                        self.dropout_keep_prob, train_mode)
        return x


def _activation_name(activation_fn) -> str:
    if callable(activation_fn):
        activation_fn = getattr(activation_fn, "__name__", str(activation_fn))
    if activation_fn not in ("tanh", "relu", "sigmoid"):
        raise ValueError("Unsupported activation {}".format(activation_fn))
    return activation_fn


def nematus_output(output_size: int, activation_fn: str = "tanh",
                   dropout_keep_prob: float = 1.0) -> Tuple[OutputProjection, int]:
    """activation(dense(state) + dense(embedding) + dense(contexts)) (output_projection.py:76-112)."""
    return _Nematus(output_size, _activation_name(activation_fn), dropout_keep_prob), output_size


def mlp_output(layer_sizes: List[int], activation: str = "tanh",
               dropout_keep_prob: float = 1.0) -> Tuple[OutputProjection, int]:
    """A multilayer perceptron over [state; embedding; contexts] (output_projection.py:163-188)."""
    return _MLP(layer_sizes, _activation_name(activation), dropout_keep_prob), layer_sizes[-1]
