"""Fully character-level sentence encoder of Lee, Cho & Hofmann (2017) (reference:
neuralmonkey/encoders/sentence_cnn_encoder.py, DESIGN.md §7d).

Over the embedded characters: dropout, then per filter (width w, n channels) a SAME convolution + bias + ReLU over
every position up to the batch's length (`ops.conv1d`), a max over offset segments of `segment_size` positions
(`ops.pool2d` with TF's SAME geometry on a [B, T, 1, n] view), the banks concatenated in filter order; then
`highway_depth` highway layers and a bidirectional GRU over ceil(length / segment_size) segments.  `temporal_mask`
is the same SAME max pool over the input mask, which can admit segments the GRU never ran: both are kept as the
reference computes them."""
from typing import List, Tuple

import torch

from neuralmonkey_b200 import ops
from neuralmonkey_b200.decorators import tensor
from neuralmonkey_b200.encoders.recurrent import gru_cell_tensors, gru_cell_variables
from neuralmonkey_b200.model.model_part import ModelPart
from neuralmonkey_b200.model.parameterized import InitializerSpecs
from neuralmonkey_b200.model.sequence import Sequence
from neuralmonkey_b200.model.stateful import TemporalStatefulWithOutput
from neuralmonkey_b200.nn.highway import declare_highway, highway
from neuralmonkey_b200.nn.utils import dropout
from neuralmonkey_b200.params import variance_scaling_initializer, zeros_initializer
from neuralmonkey_b200.typecheck import check_argument_types

_GLOROT = variance_scaling_initializer(1.0, "fan_avg", "uniform")
_CELLS = ("bidirectional_rnn/fw/OrthoGRUCell", "bidirectional_rnn/bw/OrthoGRUCell")


# pylint: disable=too-many-instance-attributes
class SentenceCNNEncoder(ModelPart, TemporalStatefulWithOutput):
    """Recurrent over convolutional encoder: a CNN with segment max-pooling and highway layers, then a
    bidirectional GRU over the segments."""

    # pylint: disable=too-many-arguments
    def __init__(self, name: str, input_sequence: Sequence, segment_size: int, highway_depth: int, rnn_size: int,
                 filters: List[Tuple[int, int]], dropout_keep_prob: float = 1.0, use_noisy_activations: bool = False,
                 reuse: ModelPart = None, save_checkpoint: str = None, load_checkpoint: str = None,
                 initializers: InitializerSpecs = None) -> None:
        ModelPart.__init__(self, name, reuse, save_checkpoint, load_checkpoint, initializers)
        check_argument_types()
        self.input_sequence = input_sequence
        self.segment_size = segment_size
        self.highway_depth = highway_depth
        self.rnn_size = rnn_size
        self.filters = filters
        self.dropout_keep_prob = dropout_keep_prob
        self.use_noisy_activations = use_noisy_activations

        # the reference's checks and messages (sentence_cnn_encoder.py:79-101)
        if dropout_keep_prob <= 0. or dropout_keep_prob > 1.:
            raise ValueError("Dropout keep probability must be in (0; 1], was {}".format(dropout_keep_prob))
        if rnn_size <= 0:
            raise ValueError("RNN size must be a positive integer.")
        if highway_depth <= 0:
            raise ValueError("Highway depth must be a positive integer.")
        if segment_size <= 0:
            raise ValueError("Segment size be a positive integer.")
        if not filters:
            raise ValueError("You must specify convolutional filters.")
        for filter_size, num_filters in self.filters:
            if filter_size <= 0:
                raise ValueError("Filter size must be a positive integer.")
            if num_filters <= 0:
                raise ValueError("Number of filters must be a positive int.")
        if use_noisy_activations:
            # nn/noisy_gru_cell.py:33-39,83: both gates call tf.get_variable("p") in the one scope `Gates`, and
            # tf.layers.dense is handed a Python list, so the reference cannot build this cell
            raise NotImplementedError("SentenceCNNEncoder: use_noisy_activations=True is not supported; the "
                                      "reference's NoisyGRUCell cannot be built")

    @property
    def cnn_size(self) -> int:
        return sum(num_filters for _, num_filters in self.filters)

    @property
    def dimension(self) -> int:
        return 2 * self.rnn_size

    def declare_variables(self) -> None:
        if hasattr(self.input_sequence, "ensure_declared"):
            self.input_sequence.ensure_declared()
        in_dim = self.input_sequence.dimension
        for filter_size, num_filters in self.filters:
            scope = "conv-maxpool-{}/".format(filter_size)
            self.declare(scope + "conv_W", [filter_size, in_dim, num_filters], _GLOROT)
            self.declare(scope + "conv_bias", [num_filters], zeros_initializer())
        for i in range(self.highway_depth):
            declare_highway(self, "highway_layer_{}".format(i), self.cnn_size)
        for scope in _CELLS:
            gru_cell_variables(self, scope, self.cnn_size, self.rnn_size)

    def _segment_max(self, x: torch.Tensor) -> torch.Tensor:
        """tf.nn.max_pool over time, ksize = strides = segment_size, SAME: [B, T, C] -> [B, ceil(T/s), C]."""
        s = self.segment_size
        return ops.pool2d(x.unsqueeze(2), s, s, "same", "max").squeeze(2)

    @tensor
    def cnn_encoded(self) -> torch.Tensor:
        """[B, ceil(T/s), sum of the filter counts]: convolutions, ReLU and segment max (lines 104-143)."""
        dropped = dropout(self.input_sequence.temporal_states, self.dropout_keep_prob, self.train_mode)
        pooled = []
        for filter_size, _ in self.filters:
            scope = "conv-maxpool-{}/".format(filter_size)
            conv = ops.conv1d(dropped, self.var(scope + "conv_W"), self.var(scope + "conv_bias"), "same", "relu")
            pooled.append(self._segment_max(conv))
        return pooled[0] if len(pooled) == 1 else torch.cat(pooled, 2)

    @tensor
    def highway_layer(self) -> torch.Tensor:
        """The highway layers over every segment (lines 146-158)."""
        encoded = self.cnn_encoded
        layer = encoded.reshape(-1, encoded.shape[-1])
        for i in range(self.highway_depth):
            layer = highway(self, "highway_layer_{}".format(i), layer)
        return layer.view(encoded.shape)

    @tensor
    def bidirectional_rnn(self) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
        """(out_fw, final_fw, out_bw, final_bw) over ceil(lengths / segment_size) segments (lines 161-172)."""
        s = self.segment_size
        seq_lens = torch.div(self.input_sequence.lengths + (s - 1), s, rounding_mode="floor").to(torch.int32)
        return ops.gru_bilayer(self.highway_layer, seq_lens, gru_cell_tensors(self, _CELLS[0]),
                               gru_cell_tensors(self, _CELLS[1]))

    @tensor
    def temporal_states(self) -> torch.Tensor:
        out_fw, _, out_bw, _ = self.bidirectional_rnn
        return torch.cat([out_fw, out_bw], 2)

    @tensor
    def output(self) -> torch.Tensor:
        _, final_fw, _, final_bw = self.bidirectional_rnn
        return torch.cat([final_fw, final_bw], 1)

    @tensor
    def temporal_mask(self) -> torch.Tensor:
        """The segment max of the input mask (lines 187-196)."""
        return self._segment_max(self.input_sequence.temporal_mask.to(torch.float32).unsqueeze(-1)).squeeze(-1)
