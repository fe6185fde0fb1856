"""Structured self-attentive sentence embedding (reference: neuralmonkey/encoders/attentive.py; Lin et al. 2017,
https://arxiv.org/abs/1703.03130).

R = `num_heads` attention distributions over the (dropped-out) input states: energies = S2(tanh(S1(states))),
both dense layers without bias (`ops.linear`), then per head a softmax over all positions, times the mask and
renormalised with +1e-8, and the [batch, R, state] matrix weights^T . states (`ops.attentive_pool`, one K18 kernel
per direction).  The matrix is `temporal_states` (time = heads, mask all ones); `output` is it flattened and,
with `output_size`, projected."""
from typing import Optional

import torch

from neuralmonkey_b200 import ops
from neuralmonkey_b200.decorators import tensor
from neuralmonkey_b200.model.model_part import ModelPart
from neuralmonkey_b200.model.parameterized import InitializerSpecs
from neuralmonkey_b200.model.stateful import TemporalStateful, TemporalStatefulWithOutput
from neuralmonkey_b200.nn.utils import dropout
from neuralmonkey_b200.params import zeros_initializer
from neuralmonkey_b200.typecheck import check_argument_types


class AttentiveEncoder(ModelPart, TemporalStatefulWithOutput):
    """An encoder with attention over the input and a fixed-dimension output."""

    # pylint: disable=too-many-arguments
    def __init__(self, name: str, input_sequence: TemporalStateful, hidden_size: int, num_heads: int,
                 output_size: int = None, state_proj_size: int = None, dropout_keep_prob: float = 1.0,
                 reuse: ModelPart = None, save_checkpoint: str = None, load_checkpoint: str = None,
                 initializers: InitializerSpecs = None) -> None:
        check_argument_types()
        ModelPart.__init__(self, name, reuse, save_checkpoint, load_checkpoint, initializers)
        self.input_sequence = input_sequence
        self.hidden_size = hidden_size
        self.num_heads = num_heads
        self.output_size = output_size
        self.state_proj_size = state_proj_size
        self.dropout_keep_prob = dropout_keep_prob
        if self.dropout_keep_prob <= 0.0 or self.dropout_keep_prob > 1.0:
            raise ValueError("Dropout keep prob must be inside (0,1].")

    def declare_variables(self) -> None:
        dim = self.input_sequence.dimension
        self.declare("S1/kernel", [dim, self.hidden_size])
        self.declare("S2/kernel", [self.hidden_size, self.num_heads])
        if self.state_proj_size is not None:
            self.declare("state_projection/kernel", [dim, self.state_proj_size])
            self.declare("state_projection/bias", [self.state_proj_size], zeros_initializer())
        if self.output_size is not None:
            self.declare("output_projection/kernel", [self.num_heads * self._state_size, self.output_size])
            self.declare("output_projection/bias", [self.output_size], zeros_initializer())

    @property
    def _state_size(self) -> int:
        return self.state_proj_size if self.state_proj_size is not None else self.input_sequence.dimension

    @tensor
    def _attention_states_dropped(self) -> torch.Tensor:
        return dropout(self.input_sequence.temporal_states, self.dropout_keep_prob, self.train_mode)

    @tensor
    def _pooled(self):
        states = self._attention_states_dropped
        hidden = ops.linear(states, self.var("S1/kernel"), None, act="tanh")
        energies = ops.linear(hidden, self.var("S2/kernel"))
        if self.state_proj_size is not None:
            states = ops.linear(states, self.var("state_projection/kernel"), self.var("state_projection/bias"))
        return ops.attentive_pool(energies, self._mask, states)

    @property
    def _mask(self) -> Optional[torch.Tensor]:
        return getattr(self.input_sequence, "temporal_mask", None)

    @property
    def attention_weights(self) -> torch.Tensor:
        """[batch, time, num_heads]."""
        return self._pooled[0]

    @property
    def temporal_states(self) -> torch.Tensor:
        """[batch, num_heads, state size]."""
        return self._pooled[1]

    @tensor
    def temporal_mask(self) -> torch.Tensor:
        states = self.temporal_states
        return torch.ones(states.shape[:2], device=states.device, dtype=torch.float32)

    @tensor
    def output(self) -> torch.Tensor:
        out = self.temporal_states.reshape(-1, self.num_heads * self._state_size)
        if self.output_size is not None:
            out = ops.linear(out, self.var("output_projection/kernel"), self.var("output_projection/bias"))
        return out

    @property
    def dimension(self) -> int:
        return self._state_size

    @property
    def output_dimension(self) -> int:
        return self.output_size if self.output_size is not None else self.num_heads * self._state_size
