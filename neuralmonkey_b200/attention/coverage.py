"""Coverage attention of Tu et al. (2016), "Modeling Coverage for Neural Machine Translation", arxiv.org/abs/1601.04811
(reference: neuralmonkey/attention/coverage.py).

The feed-forward attention of Bahdanau et al. with one more term in the energies: the coverage of each encoder
position, the sum of the attention weights it received at the earlier decoder steps over its fertility,

    fert[b,t] = 1e-8 + max_fertility * sigmoid(states[b,t] . fertility_matrix)
    cov[b,q,t] = (sum_{q'<q} w[b,q',t]) / fert[b,t] * mask[b,t]
    e[b,q,t]  = sum_a v[a] * tanh(keys[b,t,a] + y[b,q,a] + coverage_matrix[a] * cov[b,q,t])

with no energy bias (`attn_bias` is never created).  The energies depend on the earlier steps' weights but not on
the decoder's state, so all teacher-forced steps still run in one call, `ops.coverage_attention`, a scan over the
steps; decoding carries the running sum in the loop state and continues the scan one step per call.

The reference computes the sum as `weights_in_time.size()` > 0 ? reduce_sum(weights_in_time, 0) : 0 over the loop
state's weights (coverage.py:52-56).  Those weights are a plain tensor grown by `tf.concat`, which has no `size()`
method, so the reference class cannot build its graph as written.  This port implements what the expression
states: the sum of the previous steps' weights, 0 at the first step.
"""
from typing import NamedTuple, Optional, Tuple

import torch

from neuralmonkey_b200.typecheck import check_argument_types
from neuralmonkey_b200 import ops
from neuralmonkey_b200.attention.base_attention import Attendable
from neuralmonkey_b200.attention.feed_forward import Attention
from neuralmonkey_b200.decorators import tensor
from neuralmonkey_b200.model.model_part import ModelPart
from neuralmonkey_b200.model.parameterized import InitializerSpecs
from neuralmonkey_b200.params import zeros_initializer

# AttentionLoopState with the running sum of the weights so far, [batch, time]
CoverageLoopState = NamedTuple("CoverageLoopState", [("contexts", torch.Tensor), ("weights", torch.Tensor),
                                                     ("coverage", torch.Tensor)])


def _flat(var: torch.Tensor) -> torch.Tensor:
    """A [1, ..., 1, N] variable as the [N] vector the kernels take, keeping its gradient sink in the arena."""
    flat = var.view(-1)
    if getattr(var, "nm_grad", None) is not None:
        flat.nm_grad = var.nm_grad.view(-1)
    return flat


class CoverageAttention(Attention):
    # pylint: disable=too-many-arguments
    def __init__(self, name: str, encoder: Attendable, dropout_keep_prob: float = 1.0, state_size: int = None,
                 max_fertility: int = 5, reuse: ModelPart = None, save_checkpoint: str = None,
                 load_checkpoint: str = None, initializers: InitializerSpecs = None) -> None:
        check_argument_types()
        Attention.__init__(self, name, encoder, dropout_keep_prob, state_size, reuse, save_checkpoint,
                           load_checkpoint, initializers)
        self.max_fertility = max_fertility
    # pylint: enable=too-many-arguments

    def declare_variables(self) -> None:
        if self.query_state_size is None:
            raise ValueError("Attention '{}' is not used by any decoder".format(self.name))
        self.declare("Attention/attn_query_projection", [self.query_state_size, self.state_size])
        self.declare("attn_key_projection", [self.context_vector_size, self.state_size])
        self.declare("attn_similarity_v", [self.state_size])
        self.declare("attn_projection_bias", [self.state_size], zeros_initializer())
        self.declare("coverage_matrix", [1, 1, 1, self.state_size])
        self.declare("fertility_matrix", [1, 1, self.context_vector_size])

    @tensor
    def fertility(self) -> torch.Tensor:
        """[batch, time] (coverage.py:47-50)."""
        return ops.coverage_fertility(self.attention_states, _flat(self.var("fertility_matrix")),
                                      self.max_fertility)

    def coverage_scan(self, queries: torch.Tensor,
                      coverage: Optional[torch.Tensor]) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """Consecutive steps from the running sum `coverage` [batch, time] (None: the first step): queries
        [batch, NQ, query_size] -> (contexts [batch, NQ, ctx], weights [batch, NQ, time], the running sum after
        the last step)."""
        y = ops.linear(queries, self.var("Attention/attn_query_projection"), self.var("attn_projection_bias"))
        keys, values, mask, fert = self.hidden_features, self.attention_states, self.attention_mask, self.fertility
        if queries.shape[0] != keys.shape[0]:
            keys, values, mask = self._beam_tiled(queries.shape[0])
            fert = fert.repeat_interleave(queries.shape[0] // fert.shape[0], 0)
        return ops.coverage_attention(keys, values, mask, fert, y, self.var("attn_similarity_v"),
                                      _flat(self.var("coverage_matrix")), coverage)

    def attention_sequence(self, queries: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """All query steps of a pass, from zero coverage."""
        ctx, weights, _ = self.coverage_scan(queries, None)
        return ctx, weights

    def attention(self, query: torch.Tensor, decoder_prev_state: torch.Tensor, decoder_input: torch.Tensor,
                  loop_state: CoverageLoopState) -> Tuple[torch.Tensor, CoverageLoopState]:
        """One decoder step (coverage.py:52-61 in feed_forward.py:125-166)."""
        ctx, weights, coverage = self.coverage_scan(query.unsqueeze(1), loop_state.coverage)
        context, weights = ctx[:, 0], weights[:, 0]
        return context, CoverageLoopState(
            contexts=torch.cat([loop_state.contexts, context.unsqueeze(0)], 0),
            weights=torch.cat([loop_state.weights, weights.unsqueeze(0)], 0),
            coverage=coverage)

    def initial_loop_state(self) -> CoverageLoopState:
        state = Attention.initial_loop_state(self)
        return CoverageLoopState(contexts=state.contexts, weights=state.weights, coverage=None)
