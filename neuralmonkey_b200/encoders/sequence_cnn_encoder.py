"""Convolutional sentence encoder of Kim (2014) (reference: neuralmonkey/encoders/sequence_cnn_encoder.py).

Per filter (width w, F channels): conv1d over the embedded words (VALID), bias, ReLU and the max over time, on
`ops.conv1d_max_pool` (nm_gemm per filter tap + the K18 max over time).  The outputs are concatenated in filter
order.  The reference pools over every window, padding included, and so does this encoder; a batch shorter than
a filter is refused with ValueError, where TF would reduce over an empty axis."""
from typing import Any, Dict, List, Tuple

import torch

from neuralmonkey_b200 import ops, runtime
from neuralmonkey_b200.decorators import tensor
from neuralmonkey_b200.model.model_part import ModelPart
from neuralmonkey_b200.model.parameterized import InitializerSpecs
from neuralmonkey_b200.model.stateful import Stateful
from neuralmonkey_b200.nn.utils import dropout
from neuralmonkey_b200.params import variance_scaling_initializer, zeros_initializer
from neuralmonkey_b200.typecheck import check_argument_types
from neuralmonkey_b200.vocabulary import Vocabulary, pad_batch, sentence_mask

_GLOROT = variance_scaling_initializer(1.0, "fan_avg", "uniform")


class SequenceCNNEncoder(ModelPart, Stateful):
    """Encoder processing a sequence using a CNN."""

    # pylint: disable=too-many-arguments
    def __init__(self, name: str, vocabulary: Vocabulary, data_id: str, embedding_size: int,
                 filters: List[Tuple[int, int]], max_input_len: int = None, dropout_keep_prob: float = 1.0,
                 reuse: ModelPart = None, save_checkpoint: str = None, load_checkpoint: str = None,
                 initializers: InitializerSpecs = None) -> None:
        check_argument_types()
        ModelPart.__init__(self, name, reuse, save_checkpoint, load_checkpoint, initializers)
        self.vocabulary = vocabulary
        self.data_id = data_id
        self.max_input_len = max_input_len
        self.embedding_size = embedding_size
        self.dropout_keep_prob = dropout_keep_prob
        self.filters = [tuple(f) for f in filters]
        if any(len(f) != 2 or f[0] < 1 or f[1] < 1 for f in self.filters):
            raise ValueError("filters must be (size, channels) pairs of positive integers, got {}".format(filters))
        self._ids = None  # type: Any

    def declare_variables(self) -> None:
        self.declare("input_projection/word_embeddings", [len(self.vocabulary), self.embedding_size], _GLOROT)
        for size, channels in self.filters:
            scope = "conv-maxpool-{}/".format(size)
            self.declare(scope + "conv_W", [size, self.embedding_size, channels], _GLOROT)
            self.declare(scope + "conv_bias", [channels], zeros_initializer())

    @property
    def input_types(self) -> Dict[str, Any]:
        return {self.data_id: str}

    @property
    def input_shapes(self) -> Dict[str, Any]:
        return {self.data_id: [None, None]}

    def feed_dict(self, dataset, train: bool = False) -> Dict[str, Any]:
        fd = ModelPart.feed_dict(self, dataset, train)
        padded = pad_batch(list(dataset.get_series(self.data_id)), self.max_input_len)
        fd[self.data_id] = padded
        self._ids = runtime.to_device(self.vocabulary.strings_to_indices(padded))
        return fd

    def static_inputs(self) -> Dict[str, Any]:
        return {"ids": self._ids} if self._ids is not None else {}

    def bind_static(self, tensors: Dict[str, Any]) -> None:
        self.reset_batch()
        if tensors:
            self._ids = tensors["ids"]

    @tensor
    def inputs(self) -> torch.Tensor:
        """[batch, time] int64 word ids."""
        return self._ids

    @tensor
    def input_mask(self) -> torch.Tensor:
        return sentence_mask(self.inputs)

    @tensor
    def embedded_inputs(self) -> torch.Tensor:
        return dropout(ops.embed(self.inputs, self.var("input_projection/word_embeddings")),
                       self.dropout_keep_prob, self.train_mode)

    @tensor
    def output(self) -> torch.Tensor:
        pooled = [ops.conv1d_max_pool(self.embedded_inputs, self.var("conv-maxpool-{}/conv_W".format(size)),
                                      self.var("conv-maxpool-{}/conv_bias".format(size)))
                  for size, _ in self.filters]
        return pooled[0] if len(pooled) == 1 else torch.cat(pooled, 1)

    @property
    def dimension(self) -> int:
        return sum(channels for _, channels in self.filters)
