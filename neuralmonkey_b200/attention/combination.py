"""Attention combination strategies for multi-source decoders (reference: neuralmonkey/attention/combination.py).

Flat combination (Libovicky & Helcl 2017, eqs. 8-10) projects the states of every encoder into one space and
takes one distribution over all of them, optionally with the sentinel (Lu et al. 2017) as one more position.
Hierarchical combination (eqs. 6-7) takes a context from each child attention and a second distribution over
those contexts and the sentinel.  Both are one `ops.joint_attention` call per pass: the flat keys are the
encoders' projections side by side along time, one segment (and energy bias) per encoder, and the sentinel and
the child contexts are per-query candidates.

Variable names are the reference's.  Those the reference creates inside `attention()` (`tf.layers.dense` under
`attention_<name>`) are made while the decoder's step scope is open, so they are the decoder's:
`<decoder>/attention_decoder/attention_<name>/...`; the decoder announces itself through `set_step_owner`.
"""
from typing import Any, List, Optional, Tuple

import torch

from neuralmonkey_b200.typecheck import check_argument_types
from neuralmonkey_b200 import ops
from neuralmonkey_b200.attention.base_attention import (
    Attendable, BaseAttention, empty_attention_loop_state, get_attention_mask, get_attention_states)
from neuralmonkey_b200.attention.coverage import CoverageAttention
from neuralmonkey_b200.attention.namedtuples import AttentionLoopState, HierarchicalLoopState
from neuralmonkey_b200.decorators import tensor
from neuralmonkey_b200.model.model_part import ModelPart
from neuralmonkey_b200.model.parameterized import InitializerSpecs
from neuralmonkey_b200.params import normal_initializer, zeros_initializer


class MultiAttention(BaseAttention):
    """Base class for attention combination (combination.py:33-103)."""
    STEP_SCOPE = "attention_decoder"
    # the decoder passes the per-step previous cell output and embedded input (the sentinel's inputs)
    wants_sentinel_inputs = True

    # pylint: disable=unused-argument,too-many-arguments
    def __init__(self, name: str, attention_state_size: int, share_attn_projections: bool = False,
                 use_sentinels: bool = False, reuse: ModelPart = None, save_checkpoint: str = None,
                 load_checkpoint: str = None, initializers: InitializerSpecs = None) -> None:
        BaseAttention.__init__(self, name, reuse, save_checkpoint, load_checkpoint, initializers)
        self.attention_state_size = attention_state_size
        self._share_projections = share_attn_projections
        self._use_sentinels = use_sentinels
        self.att_scope_name = "attention_{}".format(name)
        self._step_owner = None  # type: Optional[ModelPart]
        self._input_size = None  # type: Optional[int]
        if attention_state_size <= 0:
            raise ValueError("attention_state_size must be positive, not {}".format(attention_state_size))
    # pylint: enable=unused-argument,too-many-arguments

    @property
    def attn_size(self) -> int:
        return self.attention_state_size

    def declare_variables(self) -> None:
        self.declare("attn_v", [1, 1, self.attention_state_size], normal_initializer(stddev=0.001))

    def _attn_v(self) -> torch.Tensor:
        """attn_v [1, 1, A] as the vector the kernel takes, keeping the arena's gradient sink of the variable.
        (The segment and candidate biases are separate scalar variables that the op takes stacked, so their
        gradients reach the arena through autograd.)"""
        var = self.var("attn_v")
        flat = var.view(-1)
        if getattr(var, "nm_grad", None) is not None:
            flat.nm_grad = var.nm_grad.view(-1)
        return flat

    def set_query_size(self, size: int) -> None:
        if self.query_state_size is not None and self.query_state_size != size:
            raise ValueError("Attention '{}' used with query sizes {} and {}".format(
                self.name, self.query_state_size, size))
        self.query_state_size = size

    # -- the variables tf.layers.dense / get_variable create inside attention() -----------------------
    def _step_name(self, local: str) -> str:
        return "{}/{}/{}".format(self.STEP_SCOPE, self.att_scope_name, local)

    def _declare_dense(self, local: str, in_size: int, out_size: int = None) -> None:
        out_size = self.attention_state_size if out_size is None else out_size
        self._step_owner.declare(self._step_name(local + "/kernel"), [in_size, out_size])
        self._step_owner.declare(self._step_name(local + "/bias"), [out_size], zeros_initializer())

    def _dense(self, x: torch.Tensor, local: str, act: str = None) -> torch.Tensor:
        return ops.linear(x, self._step_owner.var(self._step_name(local + "/kernel")),
                          self._step_owner.var(self._step_name(local + "/bias")), act=act)

    def _declare_vector_logit(self, scope: str, in_size: int) -> None:
        """The variables of `_vector_logit` (combination.py:74-103)."""
        self._step_owner.declare(self._step_name("{}_logit/vector_bias".format(scope)), [], zeros_initializer())
        self._declare_dense("{}_logit/vector_projection".format(scope), in_size)
        if not self._share_projections:
            self._declare_dense("{}_logit/vector_ctx_proj".format(scope), in_size)

    def set_step_owner(self, decoder: ModelPart) -> None:
        """The decoder whose step scope holds the variables made inside `attention()`; declares them there."""
        if self._step_owner is not None and self._step_owner is not decoder:
            raise ValueError("Attention '{}' is used by the decoders '{}' and '{}'".format(
                self.name, self._step_owner.name, decoder.name))
        if self.query_state_size is None:
            raise ValueError("Attention '{}': the decoder did not announce its query size".format(self.name))
        if self._step_owner is decoder:
            return
        self._step_owner = decoder
        self._input_size = decoder.embedding_size
        self._declare_dense("dense", self.query_state_size)
        if self._use_sentinels:
            self._declare_dense("sentinel/dense", self.query_state_size + self._input_size, self.query_state_size)
            self._declare_vector_logit("sentinel", self.query_state_size)
        self._declare_step_variables()

    def _declare_step_variables(self) -> None:
        pass

    def _check_owner(self) -> None:
        if self._step_owner is None:
            raise ValueError("Attention '{}' is not used by any decoder".format(self.name))

    def _sentinel(self, queries, prev_outputs, inputs) -> torch.Tensor:
        """sigmoid(dense([prev_state, input])) * state (combination.py:330-342), per query step."""
        if prev_outputs is None or inputs is None:
            raise ValueError("Attention '{}' uses the sentinel: it needs the decoder's previous outputs and "
                             "inputs".format(self.name))
        gate = self._dense(torch.cat([prev_outputs, inputs], -1), "sentinel/dense", act="sigmoid")
        return gate * queries

    def _vector_candidate(self, value: torch.Tensor, scope: str, ctx_local: Optional[str]):
        """(logit key [.., A], context value [.., A]) of one vector (`_vector_logit`); `ctx_local` names the
        value's projection, None for the logit projection itself."""
        key = self._dense(value, "{}_logit/vector_projection".format(scope))
        return key, (key if ctx_local is None else self._dense(value, ctx_local))

    def _vector_bias(self, scope: str) -> torch.Tensor:
        return self._step_owner.var(self._step_name("{}_logit/vector_bias".format(scope))).reshape(1)

    def attention(self, query: torch.Tensor, decoder_prev_state: torch.Tensor, decoder_input: torch.Tensor,
                  loop_state: Any) -> Tuple[torch.Tensor, Any]:
        raise NotImplementedError("Abstract method")

    def attention_sequence(self, queries: torch.Tensor, prev_outputs: torch.Tensor = None,
                           inputs: torch.Tensor = None) -> Tuple[torch.Tensor, torch.Tensor]:
        raise NotImplementedError("Abstract method")

    def _step(self, query, decoder_prev_state, decoder_input):
        """One decoder step as a one-query sequence: (context [B, ctx], weights [B, L])."""
        prev = decoder_prev_state.unsqueeze(1) if decoder_prev_state is not None else None
        inp = decoder_input.unsqueeze(1) if decoder_input is not None else None
        ctx, weights = self.attention_sequence(query.unsqueeze(1), prev, inp)
        return ctx[:, 0], weights[:, 0]


def _append(loop_state: AttentionLoopState, context: torch.Tensor, weights: torch.Tensor) -> AttentionLoopState:
    return AttentionLoopState(contexts=torch.cat([loop_state.contexts, context.unsqueeze(0)], 0),
                              weights=torch.cat([loop_state.weights, weights.unsqueeze(0)], 0))


class FlatMultiAttention(MultiAttention):
    """Flat attention combination (combination.py:106-327)."""

    # pylint: disable=too-many-arguments
    def __init__(self, name: str, encoders: List[Attendable], attention_state_size: int,
                 share_attn_projections: bool = False, use_sentinels: bool = False, reuse: ModelPart = None,
                 save_checkpoint: str = None, load_checkpoint: str = None,
                 initializers: InitializerSpecs = None) -> None:
        check_argument_types()
        MultiAttention.__init__(self, name=name, attention_state_size=attention_state_size,
                                share_attn_projections=share_attn_projections, use_sentinels=use_sentinels,
                                reuse=reuse, save_checkpoint=save_checkpoint, load_checkpoint=load_checkpoint,
                                initializers=initializers)
        if not encoders:
            raise ValueError("FlatMultiAttention '{}' needs at least one encoder".format(name))
        self._encoders = encoders
    # pylint: enable=too-many-arguments

    @property
    def dependencies(self) -> List[str]:
        return MultiAttention.dependencies.fget(self) + ["_encoders"]

    @property
    def context_vector_size(self) -> int:
        return self.attention_state_size

    def declare_variables(self) -> None:
        MultiAttention.declare_variables(self)
        scopes = ["logits_projections"] + ([] if self._share_projections else ["context_projections"])
        for scope in scopes:
            for i, enc in enumerate(self._encoders):
                self.declare("{}/proj_matrix_{}".format(scope, i), [enc.dimension, self.attention_state_size],
                             normal_initializer(stddev=0.001))
                self.declare("{}/proj_bias_{}".format(scope, i), [self.attention_state_size], zeros_initializer())
        for i in range(len(self._encoders)):
            self.declare("attn_bias_{}".format(i), [], zeros_initializer())

    def _projections(self, scope: str) -> torch.Tensor:
        """Every encoder's projection, side by side along time: [B, sum T_i, A]."""
        parts = [ops.linear(get_attention_states(enc), self.var("{}/proj_matrix_{}".format(scope, i)),
                            self.var("{}/proj_bias_{}".format(scope, i)))
                 for i, enc in enumerate(self._encoders)]
        return parts[0] if len(parts) == 1 else torch.cat(parts, 1)

    @tensor
    def _flat(self):
        """(keys, values, mask, segment ends) over all encoders, once per batch.  Spatial encoders are flattened
        over (h, w) and get all-ones masks."""
        keys = self._projections("logits_projections")
        values = keys if self._share_projections else self._projections("context_projections")
        masks, ends = [], []
        for enc in self._encoders:
            states = get_attention_states(enc)
            mask = get_attention_mask(enc)
            masks.append(mask if mask is not None else states.new_ones(states.shape[:2]))
            ends.append((ends[-1] if ends else 0) + states.shape[1])
        mask = masks[0] if len(masks) == 1 else torch.cat(masks, 1)
        return keys, values, mask.contiguous(), ends

    def _operands(self, rows: int):
        """Keys / values / mask, repeated beam-minor when a BeamSearchDecoder parent asks with batch x beam query
        rows, as `Attention._beam_tiled` does.  The reference tiles beam-major (`tf.tile`, combination.py:300-312)
        while the beam search lays hypotheses out beam-minor (row b * beam + k), so the two agree only at batch
        size 1; repeating each sentence's rows keeps every hypothesis with its own sentence at any batch size."""
        keys, values, mask, ends = self._flat
        bsz = keys.shape[0]
        if rows == bsz:
            return keys, values, mask, ends
        cache = self.__dict__.setdefault("_batch_cache", {})
        key = ("beam_tiled", rows)
        if key not in cache:
            if rows % bsz != 0:
                raise ValueError("Attention '{}': {} query rows over a batch of {}".format(self.name, rows, bsz))
            rep = rows // bsz
            cache[key] = (keys.repeat_interleave(rep, 0), values.repeat_interleave(rep, 0),
                          mask.repeat_interleave(rep, 0), ends)
        return cache[key]

    def attention_sequence(self, queries: torch.Tensor, prev_outputs: torch.Tensor = None,
                           inputs: torch.Tensor = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """All query steps at once: queries [B, NQ, query_size] (and for the sentinel the previous cell outputs and
        the inputs of each step, [B, NQ, .]) -> (contexts [B, NQ, A], weights [B, NQ, sum T_i (+1)])."""
        self._check_owner()
        qproj = self._dense(queries, "dense")
        keys, values, mask, ends = self._operands(queries.shape[0])
        seg_bias = torch.stack([self.var("attn_bias_{}".format(i)) for i in range(len(self._encoders))])
        ckeys = cvalues = cand_bias = None
        if self._use_sentinels:
            sentinel = self._sentinel(queries, prev_outputs, inputs)
            ctx_local = None if self._share_projections else "sentinel_logit/vector_ctx_proj"
            ckeys, cvalues = self._vector_candidate(sentinel, "sentinel", ctx_local)
            ckeys, cvalues = ckeys.unsqueeze(2), cvalues.unsqueeze(2)
            cand_bias = self._vector_bias("sentinel")
        return ops.joint_attention(keys, values, mask, ends, seg_bias, ckeys, cvalues, cand_bias, qproj,
                                   self._attn_v())

    def attention(self, query: torch.Tensor, decoder_prev_state: torch.Tensor, decoder_input: torch.Tensor,
                  loop_state: AttentionLoopState) -> Tuple[torch.Tensor, AttentionLoopState]:
        """One decoder step (combination.py:240-296)."""
        context, weights = self._step(query, decoder_prev_state, decoder_input)
        return context, _append(loop_state, context, weights)

    def initial_loop_state(self) -> AttentionLoopState:
        keys = self._flat[0]
        return empty_attention_loop_state(keys.shape[0], keys.shape[1] + int(self._use_sentinels),
                                          self.context_vector_size)

    def finalize_loop(self, key: str, last_loop_state: AttentionLoopState) -> None:
        self.histories[key] = last_loop_state.weights


class HierarchicalMultiAttention(MultiAttention):
    """Hierarchical attention combination (combination.py:345-475)."""

    # pylint: disable=too-many-arguments
    def __init__(self, name: str, attentions: List[BaseAttention], attention_state_size: int, use_sentinels: bool,
                 share_attn_projections: bool, reuse: ModelPart = None, save_checkpoint: str = None,
                 load_checkpoint: str = None, initializers: InitializerSpecs = None) -> None:
        check_argument_types()
        MultiAttention.__init__(self, name=name, attention_state_size=attention_state_size,
                                use_sentinels=use_sentinels, share_attn_projections=share_attn_projections,
                                reuse=reuse, save_checkpoint=save_checkpoint, load_checkpoint=load_checkpoint,
                                initializers=initializers)
        if not attentions:
            raise ValueError("HierarchicalMultiAttention '{}' needs at least one attention".format(name))
        for att in attentions:
            if isinstance(att, CoverageAttention):
                raise ValueError("HierarchicalMultiAttention '{}': child '{}' is a CoverageAttention, whose energies "
                                 "read its loop state; the children are queried without one".format(name, att.name))
        self.attentions = attentions
    # pylint: enable=too-many-arguments

    @property
    def context_vector_size(self) -> int:
        return self.attention_state_size

    def set_query_size(self, size: int) -> None:
        """The decoder only sees this wrapper: the children are queried with the same cell output."""
        MultiAttention.set_query_size(self, size)
        for att in self.attentions:
            if hasattr(att, "set_query_size"):
                att.set_query_size(size)

    def declare_variables(self) -> None:
        MultiAttention.declare_variables(self)
        for att in self.attentions:
            att.ensure_declared()

    def set_step_owner(self, decoder: ModelPart) -> None:
        MultiAttention.set_step_owner(self, decoder)
        for att in self.attentions:
            if hasattr(att, "set_step_owner"):
                att.set_step_owner(decoder)

    def _declare_step_variables(self) -> None:
        for att in self.attentions:
            self._declare_vector_logit(att.name, att.context_vector_size)
        if not self._share_projections:
            for att in self.attentions:
                self._declare_dense("proj_attn_{}".format(att.name), att.context_vector_size)
            if self._use_sentinels:
                self._declare_dense("proj_sentinel", self.query_state_size)

    def _child_sequence(self, att, queries, prev_outputs, inputs):
        if getattr(att, "wants_sentinel_inputs", False):
            return att.attention_sequence(queries, prev_outputs, inputs)
        return att.attention_sequence(queries)

    def _combine(self, queries, contexts, sentinel):
        """The second-level attention over the child contexts [B, NQ, C_i] (and the sentinel)."""
        keys, values = [], []
        for att, ctx in zip(self.attentions, contexts):
            ctx_local = None if self._share_projections else "proj_attn_{}".format(att.name)
            k, v = self._vector_candidate(ctx, att.name, ctx_local)
            keys.append(k)
            values.append(v)
        biases = [self._vector_bias(att.name) for att in self.attentions]
        if sentinel is not None:
            k, v = self._vector_candidate(sentinel, "sentinel", None if self._share_projections else "proj_sentinel")
            keys.append(k)
            values.append(v)
            biases.append(self._vector_bias("sentinel"))
        qproj = self._dense(queries, "dense")
        return ops.joint_attention(None, None, None, [], None, torch.stack(keys, 2), torch.stack(values, 2),
                                   torch.cat(biases), qproj, self._attn_v())

    def attention_sequence(self, queries: torch.Tensor, prev_outputs: torch.Tensor = None,
                           inputs: torch.Tensor = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """All query steps at once -> (contexts [B, NQ, A], weights [B, NQ, N (+1)]).  The children's weights
        are recorded in their own histories by the caller's `record_weights` only for stepped loops; here they
        are dropped with the children's contexts kept."""
        self._check_owner()
        contexts = [self._child_sequence(att, queries, prev_outputs, inputs)[0] for att in self.attentions]
        sentinel = self._sentinel(queries, prev_outputs, inputs) if self._use_sentinels else None
        return self._combine(queries, contexts, sentinel)

    def attention(self, query: torch.Tensor, decoder_prev_state: torch.Tensor, decoder_input: torch.Tensor,
                  loop_state: HierarchicalLoopState) -> Tuple[torch.Tensor, HierarchicalLoopState]:
        """One decoder step (combination.py:394-463): each child attends with its own loop state."""
        self._check_owner()
        contexts, child_states = [], []
        for att, state in zip(self.attentions, loop_state.child_loop_states):
            ctx, new_state = att.attention(query, decoder_prev_state, decoder_input, state)
            contexts.append(ctx.unsqueeze(1))
            child_states.append(new_state)
        sentinel = None
        if self._use_sentinels:
            if decoder_prev_state is None or decoder_input is None:
                raise ValueError("Attention '{}' uses the sentinel: it needs the decoder's previous outputs and "
                                 "inputs".format(self.name))
            sentinel = self._sentinel(query.unsqueeze(1), decoder_prev_state.unsqueeze(1),
                                      decoder_input.unsqueeze(1))
        ctx, weights = self._combine(query.unsqueeze(1), contexts, sentinel)
        context, weights = ctx[:, 0], weights[:, 0]
        return context, HierarchicalLoopState(child_loop_states=child_states,
                                              loop_state=_append(loop_state.loop_state, context, weights))

    def initial_loop_state(self) -> HierarchicalLoopState:
        children = [a.initial_loop_state() for a in self.attentions]
        bsz = children[0].contexts.shape[1] if children else 0
        return HierarchicalLoopState(
            child_loop_states=children,
            loop_state=empty_attention_loop_state(bsz, len(self.attentions) + int(self._use_sentinels),
                                                  self.context_vector_size))

    def finalize_loop(self, key: str, last_loop_state: HierarchicalLoopState) -> None:
        for att, state in zip(self.attentions, last_loop_state.child_loop_states):
            att.finalize_loop(key, state)
        self.histories[key] = last_loop_state.loop_state.weights
