"""Bahdanau (MLP) attention (reference: neuralmonkey/attention/feed_forward.py:23-189).

The score/softmax/mask/renormalise/context chain is the fused K4 kernel; the key projection
`hidden_features` (the reference's 1x1 conv) is one tensor-core GEMM per batch, computed
once and shared by every decoder step.
"""
from typing import Optional, Tuple

import torch

from neuralmonkey_b200.typecheck import check_argument_types
from neuralmonkey_b200 import ops
from neuralmonkey_b200.attention.base_attention import (
    Attendable, BaseAttention, empty_attention_loop_state, get_attention_mask,
    get_attention_states)
from neuralmonkey_b200.attention.namedtuples import AttentionLoopState
from neuralmonkey_b200.decorators import tensor
from neuralmonkey_b200.model.model_part import ModelPart
from neuralmonkey_b200.model.parameterized import InitializerSpecs
from neuralmonkey_b200.model.stateful import SpatialStateful, TemporalStateful
from neuralmonkey_b200.nn.utils import dropout
from neuralmonkey_b200.params import zeros_initializer


class Attention(BaseAttention):
    # pylint: disable=too-many-arguments
    def __init__(self, name: str, encoder: Attendable, dropout_keep_prob: float = 1.0,
                 state_size: int = None, reuse: ModelPart = None, save_checkpoint: str = None,
                 load_checkpoint: str = None, initializers: InitializerSpecs = None) -> None:
        check_argument_types()
        BaseAttention.__init__(self, name, reuse, save_checkpoint, load_checkpoint, initializers)
        self.encoder = encoder
        self.dropout_keep_prob = dropout_keep_prob
        self._state_size = state_size
        self.query_state_size = None  # set by the decoder that uses this attention

    @property
    def context_vector_size(self) -> int:
        return self.encoder.dimension

    @property
    def state_size(self) -> int:
        if self._state_size is not None:
            return self._state_size
        return self.context_vector_size

    def set_query_size(self, size: int) -> None:
        """The reference infers it from the first query tensor (feed_forward.py:131); variables
        here are declared before any batch is seen, so the decoder announces it."""
        if self.query_state_size is not None and self.query_state_size != size:
            raise ValueError("Attention '{}' used with query sizes {} and {}".format(
                self.name, self.query_state_size, size))
        self.query_state_size = size

    def declare_variables(self) -> None:
        if self.query_state_size is None:
            raise ValueError("Attention '{}' is not used by any decoder".format(self.name))
        self.declare("Attention/attn_query_projection", [self.query_state_size, self.state_size])
        self.declare("attn_key_projection", [self.context_vector_size, self.state_size])
        self.declare("attn_similarity_v", [self.state_size])
        self.declare("attn_projection_bias", [self.state_size], zeros_initializer())
        self.declare("attn_bias", [1], zeros_initializer())

    @tensor
    def attention_states(self) -> torch.Tensor:
        return dropout(get_attention_states(self.encoder), self.dropout_keep_prob, self.train_mode)

    @tensor
    def attention_mask(self) -> Optional[torch.Tensor]:
        return get_attention_mask(self.encoder)

    @tensor
    def hidden_features(self) -> torch.Tensor:
        """U_a . states, [batch, time, state_size] (feed_forward.py:111-118)."""
        return ops.linear(self.attention_states, self.var("attn_key_projection"))

    def _operands(self, queries: torch.Tensor):
        y = ops.linear(queries, self.var("Attention/attn_query_projection"),
                       self.var("attn_projection_bias"))
        keys, values, mask = self.hidden_features, self.attention_states, self.attention_mask
        if queries.shape[0] != keys.shape[0]:
            keys, values, mask = self._beam_tiled(queries.shape[0])
        return keys, values, mask, y, self.var("attn_similarity_v"), self.var("attn_bias")

    def attention_sequence(self, queries: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """All query steps at once: queries [batch, NQ, query_size] ->
        (contexts [batch, NQ, ctx], weights [batch, NQ, time])."""
        return ops.bahdanau_attention(*self._operands(queries))

    def attention_sequence_energies(self, queries: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """`attention_sequence` that also returns the pre-softmax energies [batch, NQ, time] of the same evaluation,
        differentiable (the reference's attention logits, feed_forward.py:136-137)."""
        return ops.bahdanau_attention_energies(*self._operands(queries))

    def _beam_tiled(self, rows: int):
        """Keys / values / mask repeated beam-minor for a BeamSearchDecoder parent.  The
        reference relies on broadcasting, which only works for batch size 1
        (beam_search_decoder.py docstring); tiling gives the same numbers there and extends
        to any batch."""
        cache = self.__dict__.setdefault("_batch_cache", {})
        key = ("beam_tiled", rows)
        if key not in cache:
            bsz = self.hidden_features.shape[0]
            if rows % bsz != 0:
                raise ValueError("Attention '{}': {} query rows over a batch of {}".format(
                    self.name, rows, bsz))
            rep = rows // bsz
            mask = self.attention_mask
            cache[key] = (self.hidden_features.repeat_interleave(rep, 0),
                          self.attention_states.repeat_interleave(rep, 0),
                          mask.repeat_interleave(rep, 0) if mask is not None else None)
        return cache[key]

    def attention(self, query: torch.Tensor, decoder_prev_state: torch.Tensor,
                  decoder_input: torch.Tensor,
                  loop_state: AttentionLoopState) -> Tuple[torch.Tensor, AttentionLoopState]:
        """One decoder step (feed_forward.py:125-166)."""
        ctx, weights = self.attention_sequence(query.unsqueeze(1))
        context, weights = ctx[:, 0], weights[:, 0]
        next_loop_state = AttentionLoopState(
            contexts=torch.cat([loop_state.contexts, context.unsqueeze(0)], 0),
            weights=torch.cat([loop_state.weights, weights.unsqueeze(0)], 0))
        return context, next_loop_state

    def initial_loop_state(self) -> AttentionLoopState:
        states = self.attention_states
        return empty_attention_loop_state(states.shape[0], states.shape[1], self.context_vector_size)

    def finalize_loop(self, key: str, last_loop_state: AttentionLoopState) -> None:
        self.histories[key] = last_loop_state.weights
