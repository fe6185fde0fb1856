"""Pooling of a sequence over time (reference: neuralmonkey/encoders/pooling.py): the [batch, dimension] `output`
of a temporal encoder, on the K18 kernels (`ops.seq_max_pool`, `ops.seq_mean_pool`)."""
import torch

from neuralmonkey_b200 import ops
from neuralmonkey_b200.decorators import tensor
from neuralmonkey_b200.model.model_part import ModelPart
from neuralmonkey_b200.model.parameterized import InitializerSpecs
from neuralmonkey_b200.model.stateful import Stateful, TemporalStateful
from neuralmonkey_b200.typecheck import check_argument_types


class SequencePooling(ModelPart, Stateful):
    """An abstract pooling layer over a sequence."""

    def __init__(self, name: str, input_sequence: TemporalStateful, reuse: ModelPart = None,
                 save_checkpoint: str = None, load_checkpoint: str = None,
                 initializers: InitializerSpecs = None) -> None:
        check_argument_types()
        ModelPart.__init__(self, name, reuse, save_checkpoint, load_checkpoint, initializers)
        self.input_sequence = input_sequence

    @property
    def dimension(self) -> int:
        return self.input_sequence.dimension


class SequenceMaxPooling(SequencePooling):
    """reduce_max(states*mask + 1e-15*(1-mask)) over time: a sentence whose valid states are all negative pools to
    1e-15, as in the reference.  A batch without any valid position raises ValueError (the reference's assert)."""

    @tensor
    def output(self) -> torch.Tensor:
        return ops.seq_max_pool(self.input_sequence.temporal_states, self.input_sequence.temporal_mask)


class SequenceAveragePooling(SequencePooling):
    """sum(states*mask) / (sum(mask) + 1e-8) over time."""

    @tensor
    def output(self) -> torch.Tensor:
        return ops.seq_mean_pool(self.input_sequence.temporal_states, self.input_sequence.temporal_mask)
