"""Transformer decoder (reference: neuralmonkey/decoders/transformer.py:70-520).

Training runs all positions at once (as the reference does, :389-447): inputs are
`[<s>] + targets[:-1]`, embedded by the BASE `embed_input_symbols` - the reference's
position-aware `embed_input_symbol` (singular, :240-256) is never called, so no position
signal reaches the decoder (SURVEY.md trap list) - then depth x (masked self-attention,
encoder attention, feed-forward) and a final LayerNorm; the vocabulary projection +
cross-entropy is the fused kernel of the base class.  At run time `next_state` re-runs the
whole prefix each step exactly like the reference (:485-518); the key mask column of a
position is `not finished` at the time it was appended.
"""
from typing import Any, List, NamedTuple, Tuple, Union

import torch

from neuralmonkey_b200.typecheck import check_argument_types
from neuralmonkey_b200 import ops, runtime
from neuralmonkey_b200.attention.base_attention import (Attendable, get_attention_mask,
                                                        get_attention_states)
from neuralmonkey_b200.attention.scaled_dot_product import attention, declare_attention
from neuralmonkey_b200.attention.transformer_cross_layer import (declare_cross, flat, hierarchical,
                                                                parallel, serial)
from neuralmonkey_b200.decoders.autoregressive import (AutoregressiveDecoder, DecoderFeedables,
                                                       LoopState)
from neuralmonkey_b200.decorators import tensor
from neuralmonkey_b200.encoders.transformer import (declare_feedforward, declare_layer_norm,
                                                    feedforward_sublayer, scoped_layer_norm)
from neuralmonkey_b200.logging import warn
from neuralmonkey_b200.model.model_part import ModelPart
from neuralmonkey_b200.model.parameterized import InitializerSpecs
from neuralmonkey_b200.model.sequence import EmbeddedSequence
from neuralmonkey_b200.nn.utils import dropout
from neuralmonkey_b200.params import (ones_initializer, variance_scaling_initializer,
                                      zeros_initializer)
from neuralmonkey_b200.vocabulary import START_TOKEN_INDEX, Vocabulary

STRATEGIES = ["serial", "parallel", "flat", "hierarchical"]

# `kv_cache`: per layer the projected self-attention keys and values of the prefix
# ([batch, time, dim] each).  Being a feedable, it is re-ordered with the beam by
# BeamSearchDecoder like every other per-hypothesis tensor.
TransformerFeedables = NamedTuple("TransformerFeedables", [
    ("input_sequence", torch.Tensor), ("input_mask", torch.Tensor), ("kv_cache", Any)])


class TransformerDecoder(AutoregressiveDecoder):
    # pylint: disable=too-many-arguments,too-many-locals,too-many-instance-attributes
    def __init__(self, name: str, encoders: List[Attendable], vocabulary: Vocabulary, data_id: str,
                 ff_hidden_size: int, n_heads_self: int, n_heads_enc: Union[List[int], int],
                 depth: int, max_output_len: int, attention_combination_strategy: str = "serial",
                 n_heads_hier: int = None, dropout_keep_prob: float = 1.0, embedding_size: int = None,
                 embeddings_source: EmbeddedSequence = None, tie_embeddings: bool = True,
                 label_smoothing: float = None, self_attention_dropout_keep_prob: float = 1.0,
                 attention_dropout_keep_prob: Union[float, List[float]] = 1.0,
                 use_att_transform_bias: bool = False, supress_unk: bool = False,
                 reuse: ModelPart = None, save_checkpoint: str = None, load_checkpoint: str = None,
                 initializers: InitializerSpecs = None) -> None:
        check_argument_types()
        AutoregressiveDecoder.__init__(
            self, name=name, vocabulary=vocabulary, data_id=data_id, max_output_len=max_output_len,
            dropout_keep_prob=dropout_keep_prob, embedding_size=embedding_size,
            embeddings_source=embeddings_source, tie_embeddings=tie_embeddings,
            label_smoothing=label_smoothing, supress_unk=supress_unk, reuse=reuse,
            save_checkpoint=save_checkpoint, load_checkpoint=load_checkpoint,
            initializers=initializers)
        self.encoders = encoders
        self.ff_hidden_size = ff_hidden_size
        self.n_heads_self = n_heads_self
        if isinstance(n_heads_enc, int):
            if attention_combination_strategy == "flat":
                self.n_heads_enc = [n_heads_enc]
            else:
                self.n_heads_enc = [n_heads_enc for _ in self.encoders]
        else:
            self.n_heads_enc = n_heads_enc
        self.depth = depth
        if isinstance(attention_dropout_keep_prob, float):
            self.attention_dropout_keep_prob = [attention_dropout_keep_prob for _ in encoders]
        else:
            self.attention_dropout_keep_prob = attention_dropout_keep_prob
        self.self_att_dropout_keep_prob = self_attention_dropout_keep_prob
        self.use_att_transform_bias = use_att_transform_bias
        self.attention_combination_strategy = attention_combination_strategy
        self.n_heads_hier = n_heads_hier
        self.encoder_states = lambda: [get_attention_states(e) for e in self.encoders]
        self.encoder_masks = lambda: [get_attention_mask(e) for e in self.encoders]
        if self.attention_combination_strategy not in STRATEGIES:
            raise ValueError("Unknown attention combination strategy '{}'. Allowed: {}.".format(
                self.attention_combination_strategy, ", ".join(STRATEGIES)))
        if self.attention_combination_strategy == "hierarchical" and self.n_heads_hier is None:
            raise ValueError("You must provide n_heads_hier when using the hierarchical attention "
                             "combination strategy.")
        if self.attention_combination_strategy != "hierarchical" and self.n_heads_hier is not None:
            warn("Ignoring n_heads_hier parameter -- use the hierarchical attention combination "
                 "strategy instead.")
        if self.attention_combination_strategy == "flat" and len(self.n_heads_enc) != 1:
            raise ValueError("For the flat attention combination strategy, only a single value is "
                             "permitted in n_heads_enc.")
        if self.attention_combination_strategy in ("flat", "hierarchical"):
            self.use_kv_cache = False      # these strategies decode by re-running the prefix
        self._default_initializer = variance_scaling_initializer(mode="fan_avg", distribution="uniform")

    @property
    def dependencies(self) -> List[str]:
        return AutoregressiveDecoder.dependencies.fget(self) + ["embeddings_source"]

    @property
    def dimension(self) -> int:
        if self.encoders:
            dims = [e.dimension for e in self.encoders]
            for i, enc_dim in enumerate(dims):
                if enc_dim != dims[0]:
                    raise ValueError("Dimension of the {}-th encoder ({}) differs from the dimension "
                                     "of the first one ({}).".format(i, enc_dim, dims[0]))
            if self.embedding_size is not None and self.embedding_size != dims[0]:
                raise ValueError("Model dimension and input embedding size do not match")
            return dims[0]
        if self.embedding_size is None:
            raise ValueError("'embedding_size' must be specified when no encoders are provided")
        return self.embedding_size

    @property
    def output_dimension(self) -> int:
        return self.dimension

    def declare_variables(self) -> None:
        AutoregressiveDecoder.declare_variables(self)
        dim = self.dimension
        for i in range(self.depth):
            scope = "layer_{}".format(i)
            declare_layer_norm(self, scope + "/self_attention", dim)
            declare_attention(self, scope + "/self_attention", dim, dim, self.n_heads_self,
                              self.use_att_transform_bias)
            declare_cross(self, scope + "/encdec_attention", self.attention_combination_strategy, dim,
                          self.n_heads_enc, self.n_heads_hier)
            declare_feedforward(self, scope + "/feedforward", dim, self.ff_hidden_size)
        self.declare("LayerNorm/gamma", [dim], ones_initializer())
        self.declare("LayerNorm/beta", [dim], zeros_initializer())

    # -- the layer stack -------------------------------------------------------------------
    def _stack(self, inputs: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
        states = inputs
        enc_states, enc_masks = self.encoder_states(), self.encoder_masks()
        strategy = self.attention_combination_strategy
        if strategy == "hierarchical":
            def combine(part, scope, queries, states, masks, heads, akps, keep_prob):
                return hierarchical(part, scope, queries, states, masks, heads, self.n_heads_hier, akps, keep_prob)
        else:
            combine = {"serial": serial, "parallel": parallel, "flat": flat}[strategy]
        for i in range(self.depth):
            scope = "layer_{}".format(i)
            normalized = scoped_layer_norm(self, scope + "/self_attention", states)
            ctx, _ = attention(self, scope + "/self_attention", normalized, normalized, normalized,
                               mask, self.n_heads_self, True, self.self_att_dropout_keep_prob,
                               self.train_mode, self.use_att_transform_bias)
            states = dropout(ctx, self.dropout_keep_prob, self.train_mode, residual=states)
            states = combine(self, scope + "/encdec_attention", states, enc_states, enc_masks,
                             self.n_heads_enc, self.attention_dropout_keep_prob,
                             self.dropout_keep_prob)
            states = feedforward_sublayer(self, scope + "/feedforward", states, self.dropout_keep_prob,
                                          self.train_mode)
        return scoped_layer_norm(self, "", states)

    # -- training -----------------------------------------------------------------------------
    @property
    def _train_unk_index(self) -> int:
        """train_loop_result computes the training logits itself (decoders/transformer.py:409-419) and
        never adds the -1e9 <unk> column; `supress_unk` only acts in the run-time loops."""
        return -1

    @tensor
    def train_input_symbols(self) -> torch.Tensor:
        """[batch, time]: <s> followed by the gold symbols but the last (:258-268)."""
        gold = self._train_targets_bm
        go = torch.full((gold.shape[0], 1), START_TOKEN_INDEX, dtype=torch.int64, device=gold.device)
        return torch.cat([go, gold[:, :-1]], dim=1)

    @tensor
    def _train_states_bm(self) -> torch.Tensor:
        input_sequence = self.embed_input_symbols(self.train_input_symbols)
        return self._stack(input_sequence, self._train_mask_bm)

    # -- runtime --------------------------------------------------------------------------------
    # The reference re-runs all layers over the whole prefix at every step and keeps the last
    # position (:485-518).  Position j of a causal stack depends only on positions <= j and on the
    # key-mask entries appended up to j, none of which change later, so the states of the prefix
    # computed at earlier steps are exactly what the recomputation would produce: the projected
    # self-attention keys / values of the prefix are cached per layer and a step runs the stack on
    # the NEW position only - O(t) instead of O(t^2) work per step.  `use_kv_cache=False` restores
    # the reference's schedule (used by the parity tests as the cross-check).
    use_kv_cache = True

    def get_initial_feedables(self) -> DecoderFeedables:
        feedables = AutoregressiveDecoder.get_initial_feedables(self)
        dev = runtime.device()
        cache = None
        if self.use_kv_cache:
            cache = [torch.zeros(self.batch_size, 0, self.dimension, device=dev)
                     for _ in range(2 * self.depth)]
        return feedables._replace(other=TransformerFeedables(
            input_sequence=torch.zeros(self.batch_size, 0, self.dimension, device=dev),
            input_mask=torch.zeros(self.batch_size, 0, 1, device=dev), kv_cache=cache))

    def _cross_kv(self, layer: int, enc_index: int, states: torch.Tensor):
        """Projected encoder keys / values of one (layer, encoder): fixed for a whole decode."""
        cache = self.__dict__.setdefault("_batch_cache", {})
        key = ("cross_kv", layer, enc_index, states.data_ptr(), tuple(states.shape))
        if key not in cache:
            scope = "layer_{}/encdec_attention/enc_{}".format(layer, enc_index)
            if self.n_heads_enc[enc_index] > 1:
                cache[key] = (ops.linear(states, self.var(scope + "/keys_proj/kernel")),
                              ops.linear(states, self.var(scope + "/vals_proj/kernel")))
            else:
                cache[key] = (states, states)
        return cache[key]

    def _project(self, scope: str, name: str, x: torch.Tensor, heads: int, bias: bool) -> torch.Tensor:
        if heads <= 1:
            return x
        b = self.var("{}/{}/bias".format(scope, name)) if bias else None
        return ops.linear(x, self.var("{}/{}/kernel".format(scope, name)), b)

    def _step_cached(self, new_input: torch.Tensor, mask: torch.Tensor, kv_cache, static_pos=None):
        """One position through the stack.  new_input [batch, 1, dim]; mask [batch, t] incl. the
        new position; kv_cache as in TransformerFeedables.  Returns (state [batch, dim], cache').

        With `static_pos` (int64 device tensor [1]) the caches are full-length buffers
        [batch, max_time, dim] updated in place at that position, and `mask` covers max_time with
        zeros beyond it (masked keys get probability exactly 0): every shape is independent of the
        step, which is what lets BeamSearchDecoder replay one CUDA graph per step."""
        states = new_input
        enc_states, enc_masks = self.encoder_states(), self.encoder_masks()
        new_cache = []
        for i in range(self.depth):
            scope = "layer_{}".format(i)
            sa = scope + "/self_attention"
            normalized = scoped_layer_norm(self, sa, states)
            bias = self.use_att_transform_bias
            q = self._project(sa, "query_proj", normalized, self.n_heads_self, bias)
            k_new = self._project(sa, "keys_proj", normalized, self.n_heads_self, bias)
            v_new = self._project(sa, "vals_proj", normalized, self.n_heads_self, bias)
            if static_pos is not None:
                keys = kv_cache[2 * i].index_copy_(1, static_pos, k_new)
                vals = kv_cache[2 * i + 1].index_copy_(1, static_pos, v_new)
            else:
                keys = torch.cat([kv_cache[2 * i], k_new], 1)
                vals = torch.cat([kv_cache[2 * i + 1], v_new], 1)
            new_cache += [keys, vals]
            # the new position is the last one: the causal mask lets it see every cached key
            ctx, _ = ops.mha_core(q, keys, vals, mask, False, self.n_heads_self)
            ctx = self._project(sa, "output_proj", ctx, self.n_heads_self, bias)
            states = ctx + states
            cross = scope + "/encdec_attention"
            if self.attention_combination_strategy == "serial":
                for j, (es, em) in enumerate(zip(enc_states, enc_masks)):
                    cs = "{}/enc_{}".format(cross, j)
                    heads = self.n_heads_enc[j]
                    normalized = scoped_layer_norm(self, cs, states)
                    ek, ev = self._cross_kv(i, j, es)
                    q = self._project(cs, "query_proj", normalized, heads, False)
                    ctx, _ = ops.mha_core(q, ek, ev, em, False, heads)
                    states = self._project(cs, "output_proj", ctx, heads, False) + states
            else:
                normalized = scoped_layer_norm(self, cross, states)
                total = states
                for j, (es, em) in enumerate(zip(enc_states, enc_masks)):
                    cs = "{}/enc_{}".format(cross, j)
                    heads = self.n_heads_enc[j]
                    ek, ev = self._cross_kv(i, j, es)
                    q = self._project(cs, "query_proj", normalized, heads, False)
                    ctx, _ = ops.mha_core(q, ek, ev, em, False, heads)
                    total = total + self._project(cs, "output_proj", ctx, heads, False)
                states = total
            states = feedforward_sublayer(self, scope + "/feedforward", states, 1.0, False)
        return scoped_layer_norm(self, "", states)[:, 0, :].contiguous(), new_cache

    def next_state(self, loop_state: LoopState) -> Tuple[torch.Tensor, Any, Any]:
        feedables = loop_state.feedables
        tr = feedables.other
        new_input = feedables.embedded_input.unsqueeze(1)
        input_sequence = torch.cat([tr.input_sequence, new_input], dim=1)
        unfinished = (~feedables.finished).to(torch.float32)
        input_mask = torch.cat([tr.input_mask, unfinished.view(-1, 1, 1)], dim=1)
        if tr.kv_cache is not None and not self.train_mode:
            output_state, cache = self._step_cached(new_input, input_mask.squeeze(-1), tr.kv_cache)
        else:
            cache = tr.kv_cache
            states = self._stack(input_sequence, input_mask.squeeze(-1))
            output_state = states[:, -1, :].contiguous()
        return (output_state,
                TransformerFeedables(input_sequence=input_sequence, input_mask=input_mask, kv_cache=cache),
                loop_state.histories.other)
