"""Convolutional seq2seq encoder of Gehring et al. (2017), http://arxiv.org/abs/1705.03122 (reference:
neuralmonkey/encoders/facebook_conv.py).

The embedded input plus a learned position table (clipped to the batch's length) goes through a dense layer to
`conv_features` channels, then `encoder_layers` residual convolutions: conv1d over time (SAME padding) to
2 * conv_features channels, the gated linear unit and the input added back, each one call of
`ops.conv1d_glu_residual` (the K19 kernels).  A second dense layer of the ordered embeddings is added to the last
layer's output.  `output` is the max over every position, padding included, as the reference's `reduce_max` is.

`dropout_keep_prob` is accepted and ignored: the reference stores it and never applies it."""
import numpy as np
import torch

from neuralmonkey_b200 import ops
from neuralmonkey_b200.decorators import tensor
from neuralmonkey_b200.logging import log
from neuralmonkey_b200.model.model_part import ModelPart
from neuralmonkey_b200.model.parameterized import InitializerSpecs
from neuralmonkey_b200.model.sequence import EmbeddedSequence
from neuralmonkey_b200.model.stateful import TemporalStatefulWithOutput
from neuralmonkey_b200.params import normal_initializer, variance_scaling_initializer, zeros_initializer
from neuralmonkey_b200.typecheck import check_argument_types

# tf.get_variable's default (glorot uniform) and tf.layers.dense's kernel initializer
_GLOROT = variance_scaling_initializer(1.0, "fan_avg", "uniform")


class SentenceEncoder(ModelPart, TemporalStatefulWithOutput):

    # pylint: disable=too-many-arguments
    def __init__(self, name: str, input_sequence: EmbeddedSequence, conv_features: int, encoder_layers: int,
                 kernel_width: int = 5, dropout_keep_prob: float = 1.0, reuse: ModelPart = None,
                 save_checkpoint: str = None, load_checkpoint: str = None,
                 initializers: InitializerSpecs = None) -> None:
        check_argument_types()
        ModelPart.__init__(self, name, reuse, save_checkpoint, load_checkpoint, initializers)
        self.input_sequence = input_sequence
        self.encoder_layers = encoder_layers
        self.conv_features = conv_features
        self.kernel_width = kernel_width
        self.dropout_keep_prob = dropout_keep_prob

        if conv_features <= 0:
            raise ValueError("Number of features must be a positive integer.")
        if encoder_layers <= 0:
            raise ValueError("Number of encoder layers must be a positive integer.")
        if self.input_sequence.max_length is None:
            raise ValueError("Input sequence must have a maximum length for "
                             "positional embeddings with this encoder")
        self.max_input_length = self.input_sequence.max_length
        log("Initializing convolutional seq2seq encoder, name {}".format(self.name))

    def declare_variables(self) -> None:
        self.input_sequence.ensure_declared()
        emb, feats = self.input_sequence.dimension, self.conv_features
        self.declare("input_projection/order_embeddings", [self.max_input_length, emb], _GLOROT)
        for scope in ("order_and_embed", "input_to_final_state"):
            self.declare(scope + "/kernel", [emb, feats], _GLOROT)
            self.declare(scope + "/bias", [feats], zeros_initializer())
        for layer in range(self.encoder_layers):
            scope = "encoder_conv_{}/".format(layer)
            # initialized as described in the paper
            self.declare(scope + "convolution_filters", [self.kernel_width, feats, 2 * feats],
                         normal_initializer(stddev=float(np.sqrt(4 / feats))))
            self.declare(scope + "conv_bias", [2 * feats], zeros_initializer())

    @property
    def dimension(self) -> int:
        return self.conv_features

    @tensor
    def ordered_embedded_inputs(self) -> torch.Tensor:
        """[batch, time, embedding]: the embedded input plus the position table clipped to the batch's length."""
        states = self.input_sequence.temporal_states
        return states + self.var("input_projection/order_embeddings")[:states.shape[1]].unsqueeze(0)

    @tensor
    def temporal_states(self) -> torch.Tensor:
        inputs = self.ordered_embedded_inputs
        convolutions = ops.linear(inputs, self.var("order_and_embed/kernel"), self.var("order_and_embed/bias"))
        for layer in range(self.encoder_layers):
            scope = "encoder_conv_{}/".format(layer)
            convolutions = ops.conv1d_glu_residual(convolutions, self.var(scope + "convolution_filters"),
                                                   self.var(scope + "conv_bias"))
        return convolutions + ops.linear(inputs, self.var("input_to_final_state/kernel"),
                                         self.var("input_to_final_state/bias"))

    @tensor
    def output(self) -> torch.Tensor:
        return ops.seq_max_pool(self.temporal_states, None)

    @tensor
    def temporal_mask(self) -> torch.Tensor:
        return self.input_sequence.temporal_mask
