"""Multi-head scaled dot-product attention
(reference: neuralmonkey/attention/scaled_dot_product.py:24-226).

`attention()` = q/k/v projections (bias-free by default) -> K8 core (`ops.mha_core`:
scaling, causal and key masks with the reference's -1e9 semantics, softmax, PV) -> output
projection.  With one head the reference applies no projections at all (:171-179,217-223).
Variables are declared by the owning model part under `<scope>/{query,keys,vals,output}_proj`.
"""
from typing import List, Optional, Tuple

import torch

from neuralmonkey_b200 import ops
from neuralmonkey_b200.attention.base_attention import (Attendable, BaseAttention, get_attention_mask,
                                                         get_attention_states)
from neuralmonkey_b200.attention.namedtuples import MultiHeadLoopState
from neuralmonkey_b200.decorators import tensor
from neuralmonkey_b200.model.model_part import ModelPart
from neuralmonkey_b200.model.parameterized import InitializerSpecs
from neuralmonkey_b200.nn.utils import dropout, dropout_mask
from neuralmonkey_b200.params import variance_scaling_initializer, zeros_initializer
from neuralmonkey_b200.typecheck import check_argument_types


def declare_attention(part, scope: str, q_dim: int, kv_dim: int, num_heads: int,
                      use_bias: bool = False) -> None:
    """Variables of one `attention()` call site (tf.layers.dense names)."""
    if num_heads <= 1:
        return
    for name, in_dim in (("query_proj", q_dim), ("keys_proj", kv_dim), ("vals_proj", kv_dim),
                         ("output_proj", q_dim)):
        part.declare("{}/{}/kernel".format(scope, name), [in_dim, q_dim])
        if use_bias:
            part.declare("{}/{}/bias".format(scope, name), [q_dim], zeros_initializer())


def attention(part, scope: str, queries: torch.Tensor, keys: torch.Tensor, values: torch.Tensor,
              keys_mask: Optional[torch.Tensor], num_heads: int, masked: bool = False,
              attention_dropout_keep_prob: float = 1.0, train_mode: bool = False,
              use_bias: bool = False) -> Tuple[torch.Tensor, torch.Tensor]:
    """Returns (context [batch, time_q, dim], weights [batch, heads, time_q, time_k])."""
    if num_heads <= 0:
        raise ValueError("Number of heads must be greater than zero.")
    q_dim = queries.shape[-1]
    if q_dim != keys.shape[-1]:
        raise ValueError("Queries and keys do not match in the last dimension. Queries: {}, Keys: {}"
                         .format(q_dim, keys.shape[-1]))
    if keys.shape[1] != values.shape[1]:
        raise ValueError("Keys and values 'time' dimension does not match. Keys: {}, Values: {}"
                         .format(keys.shape[1], values.shape[1]))
    if q_dim % num_heads != 0:
        raise ValueError("Last dimension of the query ({}) should be divisible by the number of "
                         "heads ({})".format(q_dim, num_heads))

    def proj(x, name):
        bias = part.var("{}/{}/bias".format(scope, name)) if use_bias else None
        return ops.linear(x, part.var("{}/{}/kernel".format(scope, name)), bias)

    if num_heads > 1:
        queries, keys, values = proj(queries, "query_proj"), proj(keys, "keys_proj"), proj(values, "vals_proj")
    drop = None
    if attention_dropout_keep_prob < 1.0 and train_mode:
        # dropout on the attention weights (:208-214), inside the fused core: the mask rides along
        drop = dropout_mask((queries.shape[0], num_heads, queries.shape[1], keys.shape[1]),
                            attention_dropout_keep_prob, train_mode, queries.device)
    context, weights = ops.mha_core(queries, keys, values, keys_mask, masked, num_heads, drop)
    if num_heads > 1:
        context = proj(context, "output_proj")
    return context, weights


class MultiHeadAttention(BaseAttention):
    """The attention OBJECT an RNN decoder is given (scaled_dot_product.py:246-383; tests/post-edit.ini):
    `attention()` above with the decoder's cell output as the only query of a step, keys and values from one
    or two encoders.

    The head projections of `n_heads > 1` are `tf.layers.dense` calls made while the decoder's step scope is
    open, so the variables are the DECODER's: `<decoder>/attention_decoder/{query,keys,vals,output}_proj/kernel`
    (two multi-head attentions of one decoder share them through AUTO_REUSE; different sizes collide, as in
    the reference).  The decoder announces itself through `set_step_owner`.  Training does not step (see
    decoders/decoder.py): all T cell outputs are the T queries of ONE `attention()` call; a run-time step is the
    same call with one query per hypothesis."""
    STEP_SCOPE = "attention_decoder"

    # pylint: disable=too-many-arguments
    def __init__(self, name: str, n_heads: int, keys_encoder: Attendable, values_encoder: Attendable = None,
                 dropout_keep_prob: float = 1.0, reuse: ModelPart = None, save_checkpoint: str = None,
                 load_checkpoint: str = None, initializers: InitializerSpecs = None) -> None:
        check_argument_types()
        BaseAttention.__init__(self, name, reuse, save_checkpoint, load_checkpoint, initializers)
        self.n_heads = n_heads
        self.dropout_keep_prob = dropout_keep_prob
        self.keys_encoder = keys_encoder
        self.values_encoder = values_encoder if values_encoder is not None else keys_encoder
        if self.n_heads <= 0:
            raise ValueError("Number of heads must be greater than zero.")
        if self.dropout_keep_prob <= 0.0 or self.dropout_keep_prob > 1.0:
            raise ValueError("Dropout keep prob must be inside (0,1].")
        self._default_initializer = variance_scaling_initializer(mode="fan_avg", distribution="uniform")
        self._step_owner = None  # type: Optional[ModelPart]
    # pylint: enable=too-many-arguments

    @property
    def dependencies(self) -> List[str]:
        return BaseAttention.dependencies.fget(self) + ["keys_encoder", "values_encoder"]

    def set_query_size(self, size: int) -> None:
        keys_dim = self.keys_encoder.dimension
        if size != keys_dim:
            raise ValueError("Queries and keys do not match in the last dimension. Queries: {}, Keys: {}"
                             .format(size, keys_dim))
        if size % self.n_heads != 0:
            raise ValueError("Last dimension of the query ({}) should be divisible by the number of heads ({})"
                             .format(size, self.n_heads))
        if self.n_heads == 1 and self.values_encoder.dimension != size:
            raise ValueError("With one head the values are not projected: their dimension ({}) must be the "
                             "queries' ({})".format(self.values_encoder.dimension, size))
        self.query_state_size = size

    def set_step_owner(self, decoder: ModelPart) -> None:
        """The decoder whose step scope holds the head projections; declares them there."""
        if self._step_owner is not None and self._step_owner is not decoder:
            raise ValueError("Attention '{}' is used by the decoders '{}' and '{}'".format(
                self.name, self._step_owner.name, decoder.name))
        self._step_owner = decoder
        if self.query_state_size is None:
            raise ValueError("Attention '{}': the decoder did not announce its query size".format(self.name))
        if self.n_heads > 1:
            init = self._default_initializer
            q_dim = self.query_state_size
            for local, in_dim in (("query_proj", q_dim), ("keys_proj", self.keys_encoder.dimension),
                                  ("vals_proj", self.values_encoder.dimension), ("output_proj", q_dim)):
                decoder.declare("{}/{}/kernel".format(self.STEP_SCOPE, local), [in_dim, q_dim], init)

    @tensor
    def attention_keys(self) -> torch.Tensor:
        return get_attention_states(self.keys_encoder)

    @tensor
    def attention_mask(self) -> Optional[torch.Tensor]:
        return get_attention_mask(self.keys_encoder)

    @tensor
    def attention_values(self) -> torch.Tensor:
        return get_attention_states(self.values_encoder)

    @property
    def context_vector_size(self) -> int:
        """The reference reads the values' last dimension (:366-368); with several heads the context leaves
        `output_proj`, whose width is the queries' - the same number whenever the reference's graph builds
        with a projection behind it, and the true width of the context otherwise."""
        if self.n_heads > 1 and self.query_state_size is not None:
            return self.query_state_size
        return self.values_encoder.dimension

    def _operands(self, rows: int):
        """Keys / values / mask, repeated beam-minor when a BeamSearchDecoder parent asks with
        batch x beam query rows (see Attention._beam_tiled)."""
        keys, values, mask = self.attention_keys, self.attention_values, self.attention_mask
        bsz = keys.shape[0]
        if rows == bsz:
            return keys, values, mask
        cache = self.__dict__.setdefault("_batch_cache", {})
        key = ("beam_tiled", rows)
        if key not in cache:
            if rows % bsz != 0:
                raise ValueError("Attention '{}': {} query rows over a batch of {}".format(self.name, rows, bsz))
            rep = rows // bsz
            cache[key] = (keys.repeat_interleave(rep, 0), values.repeat_interleave(rep, 0),
                          mask.repeat_interleave(rep, 0) if mask is not None else None)
        return cache[key]

    def attention_sequence(self, queries: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """queries [batch, NQ, query_size] -> (contexts [batch, NQ, ctx], weights [batch, heads, NQ, time])."""
        if self._step_owner is None:
            raise ValueError("Attention '{}' is not used by any decoder".format(self.name))
        keys, values, mask = self._operands(queries.shape[0])
        return attention(self._step_owner, self.STEP_SCOPE, queries, keys, values, mask, self.n_heads,
                         masked=False, attention_dropout_keep_prob=self.dropout_keep_prob,
                         train_mode=self.train_mode)

    def attention(self, query: torch.Tensor, decoder_prev_state: torch.Tensor, decoder_input: torch.Tensor,
                  loop_state: MultiHeadLoopState) -> Tuple[torch.Tensor, MultiHeadLoopState]:
        """One decoder step (:296-350): the query becomes a one-step sequence."""
        ctx, weights = self.attention_sequence(query.unsqueeze(1))
        context = ctx[:, 0]
        next_loop_state = MultiHeadLoopState(
            contexts=torch.cat([loop_state.contexts, context.unsqueeze(0)], 0),
            head_weights=[torch.cat([loop_state.head_weights[i], weights[:, i, 0].unsqueeze(0)], 0)
                          for i in range(self.n_heads)])
        return context, next_loop_state

    def initial_loop_state(self) -> MultiHeadLoopState:
        keys = self.attention_keys
        dev = keys.device
        return MultiHeadLoopState(
            contexts=torch.zeros(0, keys.shape[0], self.context_vector_size, device=dev),
            head_weights=[torch.zeros(0, keys.shape[0], keys.shape[1], device=dev) for _ in range(self.n_heads)])

    def finalize_loop(self, key: str, last_loop_state: MultiHeadLoopState) -> None:
        for i in range(self.n_heads):
            self.histories["{}_head{}".format(key, i)] = last_loop_state.head_weights[i]

    def record_weights(self, key: str, weights: torch.Tensor) -> None:
        """Weights of a whole pass as `attention_sequence` returns them, [batch, heads, NQ, time]."""
        for i in range(self.n_heads):
            self.histories["{}_head{}".format(key, i)] = weights[:, i].detach().transpose(0, 1)

    def visualize_attention(self, key: str, max_outputs: int = 16) -> None:
        for i in range(self.n_heads):
            head_key = "{}_head{}".format(key, i)
            if head_key not in self.histories:
                raise ValueError("Key {} not among attention histories".format(head_key))


class ScaledDotProdAttention(MultiHeadAttention):
    """One head, no projections (scaled_dot_product.py:386-402; tests/factored.ini, tests/post-edit.ini)."""

    # pylint: disable=too-many-arguments
    def __init__(self, name: str, keys_encoder: Attendable, values_encoder: Attendable = None,
                 dropout_keep_prob: float = 1.0, reuse: ModelPart = None, save_checkpoint: str = None,
                 load_checkpoint: str = None, initializers: InitializerSpecs = None) -> None:
        check_argument_types()
        MultiHeadAttention.__init__(self, name, 1, keys_encoder, values_encoder, dropout_keep_prob, reuse,
                                    save_checkpoint, load_checkpoint, initializers)
    # pylint: enable=too-many-arguments
