"""RNN attention decoder (reference: neuralmonkey/decoders/decoder.py:67-396).

Training does not step: with `attention_on_input=False` and no conditional GRU (the
defaults, and what the five target configs use) the attention context never feeds back
into the recurrence (decoder.py:264-277,288-297), so
  1. the GRU runs over all gold inputs as one K2 sequence kernel,
  2. all T queries attend in one K4 launch,
  3. the deep-output projection is one GEMM over T*B rows,
and the base class adds the fused vocabulary projection + loss.  The runtime (greedy / beam)
path steps through `next_state`, using the same kernels with T = 1.

Variants (SURVEY.md 8(f) N4, see nn/variants.py; GPU-verified by tests/test_gpu_variants.py): with `conditional_gru`
or `rnn_cell="NematusGRU"` the context feeds the recurrence, so training steps through time with the
same `_variant_step` the runtime uses (teacher-forced inputs), one set of T = 1 launches per step.
"""
from typing import Any, Dict, List, NamedTuple, Tuple

import torch

from neuralmonkey_b200.typecheck import check_argument_types
from neuralmonkey_b200 import ops, runtime
from neuralmonkey_b200.attention.base_attention import BaseAttention
from neuralmonkey_b200.attention.coverage import CoverageAttention
from neuralmonkey_b200.decoders.autoregressive import AutoregressiveDecoder, LoopState
from neuralmonkey_b200.decoders.encoder_projection import (
    EncoderProjection, concat_encoder_projection, empty_initial_state, linear_encoder_projection)
from neuralmonkey_b200.decoders.output_projection import OutputProjection, nonlinear_output
from neuralmonkey_b200.decorators import tensor
from neuralmonkey_b200.encoders.recurrent import gru_cell_tensors, gru_cell_variables
from neuralmonkey_b200.logging import log
from neuralmonkey_b200.model.model_part import ModelPart
from neuralmonkey_b200.model.parameterized import InitializerSpecs
from neuralmonkey_b200.model.sequence import EmbeddedSequence
from neuralmonkey_b200.model.stateful import Stateful
from neuralmonkey_b200.nn.utils import dropout, dropout_mask
from neuralmonkey_b200.nn.variants import LSTMCell, NematusGRUCell
from neuralmonkey_b200.vocabulary import END_TOKEN_INDEX, START_TOKEN_INDEX, Vocabulary

RNN_CELL_TYPES = ("NematusGRU", "GRU", "LSTM")

RNNFeedables = NamedTuple("RNNFeedables", [
    ("prev_rnn_state", torch.Tensor), ("prev_rnn_output", torch.Tensor),
    ("prev_contexts", List[torch.Tensor])])
RNNHistories = NamedTuple("RNNHistories", [
    ("rnn_outputs", Any), ("attention_histories", List[Any])])


class Decoder(AutoregressiveDecoder):
    # pylint: disable=too-many-arguments,too-many-locals,too-many-instance-attributes
    def __init__(self, encoders: List[Stateful], vocabulary: Vocabulary, data_id: str, name: str,
                 max_output_len: int, dropout_keep_prob: float = 1.0, embedding_size: int = None,
                 embeddings_source: EmbeddedSequence = None, tie_embeddings: bool = False,
                 label_smoothing: float = None, rnn_size: int = None,
                 output_projection=None, encoder_projection: EncoderProjection = None,
                 attentions: List[BaseAttention] = None, attention_on_input: bool = False,
                 rnn_cell: str = "GRU", conditional_gru: bool = False, supress_unk: bool = False,
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
        self._output_projection_spec = output_projection
        self._conditional_gru = conditional_gru
        self._attention_on_input = attention_on_input
        self._rnn_cell_str = rnn_cell
        self._rnn_size = rnn_size
        self._encoder_projection = encoder_projection
        self.attentions = list(attentions) if attentions is not None else []

        if not rnn_size and not encoder_projection and not encoders:
            raise ValueError("No RNN size, no encoders and no encoder_projection specified")
        if self._rnn_cell_str not in RNN_CELL_TYPES:
            raise ValueError("RNN cell must be a either 'GRU', 'LSTM', or 'NematusGRU'. Not {}"
                             .format(self._rnn_cell_str))
        if attention_on_input:
            # the reference itself cannot build this option: input_plus_attention reads
            # `feedables.prev_contexts` (decoder.py:273), which does not exist (the contexts are in
            # `feedables.other`) - tests/test_oracle_vs_reference_code.py records the AttributeError
            raise NotImplementedError("attention_on_input=True fails in the reference while the graph is "
                                      "built (decoders/decoder.py:273); it is not supported here either")
        self._stepwise = self._rnn_cell_str != "GRU" or conditional_gru
        for att in self.attentions:
            if hasattr(att, "set_query_size"):
                att.set_query_size(self.rnn_size)

    # -- static configuration ------------------------------------------------------------
    @property
    def encoder_projection(self) -> EncoderProjection:
        if self._encoder_projection is not None:
            return self._encoder_projection
        if not self.encoders:
            log("No direct encoder input. Using empty initial state")
            return empty_initial_state
        if self._rnn_size is None:
            log("No rnn_size or encoder_projection: Using concatenation of encoded states")
            return concat_encoder_projection
        if not hasattr(self, "_default_projection"):
            log("Using linear projection of encoders as the initial state")
            self._default_projection = linear_encoder_projection(self.dropout_keep_prob)
        return self._default_projection

    @property
    def rnn_size(self) -> int:
        if self._rnn_size is not None:
            return self._rnn_size
        if self._encoder_projection is None:
            assert self.encoders
            return sum(e.dimension for e in self.encoders)
        raise ValueError("Cannot infer RNN size.")

    @property
    def output_projection_spec(self) -> Tuple[OutputProjection, int]:
        if not hasattr(self, "_out_proj"):
            if self._output_projection_spec is None:
                log("No output projection specified - using tanh projection")
                self._out_proj = nonlinear_output(self.rnn_size, "tanh")
            elif isinstance(self._output_projection_spec, tuple):
                self._out_proj = self._output_projection_spec
            else:
                self._out_proj = (self._output_projection_spec, self.rnn_size)
        return self._out_proj

    @property
    def output_projection(self) -> OutputProjection:
        return self.output_projection_spec[0]

    @property
    def output_dimension(self) -> int:
        return self.output_projection_spec[1]

    @property
    def _nematus_cells(self):
        """(first cell, conditional cell or None) - _get_rnn_cell / _get_conditional_gru_cell
        (decoder.py:253-262): the conditional cell carries its bias on the state side."""
        if "_nematus_cells_cache" not in self.__dict__:
            ctx_size = sum(a.context_vector_size for a in self.attentions)
            first = NematusGRUCell(self, "attention_decoder/nematus_gru_cell", self.embedding_size, self.rnn_size)
            cond = (NematusGRUCell(self, self._COND_SCOPE, ctx_size, self.rnn_size, use_state_bias=True,
                                   use_input_bias=False) if self._conditional_gru else None)
            self.__dict__["_nematus_cells_cache"] = (first, cond)
        return self.__dict__["_nematus_cells_cache"]

    @property
    def _lstm_cell(self) -> LSTMCell:
        return LSTMCell(self, "attention_decoder/lstm_cell", self.embedding_size, self.rnn_size)

    _CELL_SCOPE = "attention_decoder/OrthoGRUCell"
    _COND_SCOPE = "attention_decoder/cond_gru_2_cell"      # the scope decoder.py:324 passes

    def declare_variables(self) -> None:
        AutoregressiveDecoder.declare_variables(self)
        if self.embedding_size != self.output_dimension:
            raise ValueError("The dimension ({}) of the output projection must be same as the "
                             "dimension of the input embedding ({})"
                             .format(self.output_dimension, self.embedding_size))
        self.encoder_projection.declare(self, self.rnn_size, self.encoders)
        ctx_size = sum(a.context_vector_size for a in self.attentions)
        if self._rnn_cell_str == "LSTM":
            self._lstm_cell.declare()
        elif self._rnn_cell_str == "NematusGRU":
            for cell in self._nematus_cells:
                if cell is not None:
                    cell.declare()
        else:
            gru_cell_variables(self, self._CELL_SCOPE, self.embedding_size, self.rnn_size)
            if self._conditional_gru:
                gru_cell_variables(self, self._COND_SCOPE, ctx_size, self.rnn_size)
        self.output_projection.declare(self, self.rnn_size + self.embedding_size + ctx_size)
        for att in self.attentions:
            att.ensure_declared()
            if hasattr(att, "set_step_owner"):       # head projections live in this decoder's step scope
                att.set_step_owner(self)

    # -- initial state ---------------------------------------------------------------------
    @tensor
    def initial_state(self) -> torch.Tensor:
        """dropout(encoder_projection(...)) (decoder.py:226-252): with the default linear
        projection dropout is applied twice, inside the projection and here."""
        init = dropout(self.encoder_projection(self, self.train_mode, self.rnn_size, self.encoders),
                       self.dropout_keep_prob, self.train_mode)
        if init.dim() == 1:
            init = init.unsqueeze(0).expand(self.batch_size, -1).contiguous()
        return init

    @staticmethod
    def _attend_sequence(att, queries, prev_outputs, inputs):
        """att.attention_sequence over queries [B, NQ, rnn]; attentions that declare `wants_sentinel_inputs`
        (attention.combination) also get each query step's previous cell output and embedded input
        [B, NQ, .], which `next_state` hands to `attention()` at run time."""
        if getattr(att, "wants_sentinel_inputs", False):
            return att.attention_sequence(queries, prev_outputs, inputs)
        return att.attention_sequence(queries)

    def _step_attend(self, prev_output, rnn_input, coverage):
        """`attend(att, query)` of one teacher-forced or differentiable step: prev_output is what the step
        received (the (c, h) pair of an LSTM), rnn_input the step's embedded input.  `coverage` maps each coverage
        attention (by id) to its running sum of weights, absent before the first step; `attend` advances it."""
        prev_h = prev_output[1] if isinstance(prev_output, tuple) else prev_output

        def attend(att, query):
            if isinstance(att, CoverageAttention):
                ctx, w, coverage[id(att)] = att.coverage_scan(query.unsqueeze(1), coverage.get(id(att)))
                return ctx[:, 0], w
            ctx, w = self._attend_sequence(att, query.unsqueeze(1), prev_h.unsqueeze(1), rnn_input.unsqueeze(1))
            return ctx[:, 0], w
        return attend

    # -- variants: one step of decoder.py:279-358 with the context inside the recurrence ---------
    def _variant_step(self, rnn_input: torch.Tensor, prev_output: torch.Tensor, attend):
        """(output, dropped cell output, dropped contexts, attention results) of one step.
        `attend(att, query)` runs one attention.  Order as in the reference: first cell -> attention
        queried with its RAW output -> (conditional cell over the raw contexts, state = first cell's
        output) -> dropout on contexts and on the cell output -> deep output."""
        next_c = None
        if self._rnn_cell_str == "LSTM":
            # the LSTM branch (decoder.py:326-339): the loop carries (prev_rnn_state = c, prev_rnn_output = h);
            # `prev_output` is that pair here.  The conditional cell belongs to the GRU branch only.
            next_c, cell_output = self._lstm_cell(rnn_input, prev_output[0], prev_output[1])
        elif self._rnn_cell_str == "NematusGRU":
            cell_output = self._nematus_cells[0](rnn_input, prev_output)
        else:
            cell_output = ops.gru_layer(rnn_input.unsqueeze(1), *gru_cell_tensors(self, self._CELL_SCOPE),
                                        h0=prev_output)[2][:, 0]
        attended = [attend(att, cell_output) for att in self.attentions]
        contexts = [a[0] for a in attended]
        if self._conditional_gru and next_c is None:
            cond_input = contexts[0] if len(contexts) == 1 else torch.cat(contexts, -1)
            if self._rnn_cell_str == "NematusGRU":
                cell_output = self._nematus_cells[1](cond_input, cell_output)
            else:
                cell_output = ops.gru_layer(cond_input.unsqueeze(1), *gru_cell_tensors(self, self._COND_SCOPE),
                                            h0=cell_output)[2][:, 0]
        contexts = [dropout(ctx, self.dropout_keep_prob, self.train_mode) for ctx in contexts]
        cell_output = dropout(cell_output, self.dropout_keep_prob, self.train_mode)
        output = self.output_projection(self, cell_output, rnn_input, contexts, self.train_mode)
        return output, (cell_output if next_c is None else (next_c, cell_output)), contexts, attended

    def _train_pass_stepwise(self):
        fed = self._train_step_inputs_bm
        emb = self.embed_input_symbols(fed)                # [B,T,E]
        prev = self.initial_state
        if self._rnn_cell_str == "LSTM":
            prev = (prev, prev)
        outputs, cells, weights, coverage = [], [], [[] for _ in self.attentions], {}
        for t in range(fed.shape[1]):       # one query per sentence and step: NQ = 1
            out, prev, _ctx, attended = self._variant_step(emb[:, t], prev,
                                                           self._step_attend(prev, emb[:, t], coverage))
            outputs.append(out)
            cells.append(prev[1] if isinstance(prev, tuple) else prev)
            for hist, (_c, w) in zip(weights, attended):
                hist.append(w)
        weights = [torch.cat(hist, dim=-2) for hist in weights]     # the query axis is the one before time
        for att, w in zip(self.attentions, weights):
            att.record_weights("{}_train".format(self.name), w)
        return torch.stack(outputs, 1), torch.stack(cells, 1), weights

    # -- training: all steps at once ------------------------------------------------------
    @tensor
    def _train_pass(self):
        if self._stepwise:
            return self._train_pass_stepwise()
        fed = self._train_step_inputs_bm                   # [B,T] symbols fed at each step
        bsz, steps = fed.shape
        emb = self.embed_input_symbols(fed)                # [B,T,E] (dropout inside)
        mask = dropout_mask((bsz, steps, self.rnn_size), self.dropout_keep_prob, self.train_mode,
                            emb.device)
        dropped, _final, raw = ops.gru_layer(emb, *gru_cell_tensors(self, self._CELL_SCOPE),
                                             h0=self.initial_state, drop_mask=mask)
        # the previous output each step hands to the attention: the initial state, then the dropped cell outputs
        prev_outputs = None
        if any(getattr(att, "wants_sentinel_inputs", False) for att in self.attentions):
            prev_outputs = torch.cat([self.initial_state.unsqueeze(1), dropped[:, :-1]], 1)
        contexts, weights = [], []
        for att in self.attentions:
            ctx, w = self._attend_sequence(att, raw, prev_outputs, emb)   # queries = cell outputs BEFORE dropout
            contexts.append(dropout(ctx, self.dropout_keep_prob, self.train_mode))
            weights.append(w)
        out = self.output_projection(self, dropped, emb, contexts, self.train_mode)  # [B,T,O]
        for att, w in zip(self.attentions, weights):
            att.record_weights("{}_train".format(self.name), w)
        return out, dropped, weights

    @property
    def _train_states_bm(self) -> torch.Tensor:
        return self._train_pass[0]

    @property
    def train_rnn_outputs(self) -> torch.Tensor:
        """[time, batch, rnn_size] history of (dropped-out) cell outputs."""
        return self._train_pass[1].transpose(0, 1)

    # -- the decoding loop under autograd (the reinforcement-learning objectives) ----------------------------
    def differentiable_loop(self, sample: bool = False, temperature: float = 1.,
                            sample_index: int = 0) -> Dict[str, torch.Tensor]:
        """decoding_loop(train_mode=False, sample, temperature) as the reference's RL objectives differentiate it
        (trainers/rl_trainer.py:120-140, self_critical_objective.py:56-92): the loop runs inside the training
        graph, so decoder dropout is active in training and the gradient passes through the same masks that chose
        the symbols.  Each step computes its output state with autograd through `_variant_step` (as the step-wise
        training pass does), projects it to logits without autograd and chooses the next symbol: the first-index
        argmax, or a draw from softmax(logits / temperature) (`ops.sample_logits_step`, `sample_index` selects an
        independent stream); then symbols *= unfinished, finished |= symbols == </s> (get_body,
        autoregressive.py:446-517).  The loop stops when every row has finished or after max_output_len steps.

        Returns time-major {"states" [T,B,O] (differentiable), "symbols" [T,B], "argmax" [T,B] (the unmasked argmax
        of the step's logits), "mask" [T,B] (not finished after the step)}; `loop_nll` gives the per-position
        negative log-likelihoods of chosen symbols."""
        if temperature <= 0:
            raise ValueError("The softmax temperature must be positive")
        dev = runtime.device()
        symbols = torch.full((self.batch_size,), START_TOKEN_INDEX, dtype=torch.int64, device=dev)
        finished = torch.zeros(self.batch_size, dtype=torch.bool, device=dev)
        prev = self.initial_state
        if self._rnn_cell_str == "LSTM":
            prev = (prev, prev)

        states, chosen, argmaxes, masks, coverage = [], [], [], [], {}
        for step in range(self.max_output_len):
            emb = self.embed_input_symbols(symbols)
            out, prev, _ctx, _attended = self._variant_step(emb, prev, self._step_attend(prev, emb, coverage))
            with torch.no_grad():
                logits, _lse, argmax = self.state_to_logits(out.detach(), keep_logits=sample)
                if sample:
                    symbols, finished = ops.sample_logits_step(logits, temperature, finished, self._unk_index, step,
                                                               sample_index)
                else:
                    symbols = argmax * (~finished).to(torch.int64)
                    finished = finished | (symbols == END_TOKEN_INDEX)
            states.append(out)
            chosen.append(symbols)
            argmaxes.append(argmax)
            masks.append(~finished)
            if bool(finished.all()):
                break
        return {"states": torch.stack(states, 0), "symbols": torch.stack(chosen, 0),
                "argmax": torch.stack(argmaxes, 0), "mask": torch.stack(masks, 0)}

    def loop_nll(self, states: torch.Tensor, targets: torch.Tensor, temperature: float = 1.):
        """-log softmax(logits / temperature)[target] of states [T,B,O] (from `differentiable_loop`) at targets
        [T,B]: one batched `ops.logits_xent`, differentiable in the states and the projection.  Returns
        (nll [T,B], first-index argmax of the logits [T,B]).  Like the reference (autoregressive.py:492-493) the
        temperature divides the whole projection; the -1e9 <unk> column is not divided, which changes nothing, as
        its exponential is 0 either way."""
        steps, bsz, dim = states.shape
        w, b = self.decoding_w, self.decoding_b
        if temperature != 1.:
            w = w / temperature
            b = b / temperature if b is not None else None
        ones = torch.ones(steps * bsz, device=states.device, dtype=torch.float32)
        nll, _lse, argmax, _ = ops.logits_xent(states.reshape(steps * bsz, dim), w, b,
                                               targets.reshape(-1).contiguous(), ones, self._unk_index,
                                               self._w_transposed)
        return nll.view(steps, bsz), argmax.view(steps, bsz)

    # -- runtime: one step ----------------------------------------------------------------
    def get_initial_feedables(self):
        feedables = AutoregressiveDecoder.get_initial_feedables(self)
        dev = runtime.device()
        rnn_feedables = RNNFeedables(
            prev_contexts=[torch.zeros(self.batch_size, a.context_vector_size, device=dev)
                           for a in self.attentions],
            prev_rnn_state=self.initial_state, prev_rnn_output=self.initial_state)
        return feedables._replace(other=rnn_feedables)

    def get_initial_histories(self):
        histories = AutoregressiveDecoder.get_initial_histories(self)
        rnn_histories = RNNHistories(
            rnn_outputs=[],
            attention_histories=[a.initial_loop_state() for a in self.attentions if a is not None])
        return histories._replace(other=rnn_histories)

    def reorder_attention_states(self, histories, gather):
        """`histories` (of this decoder's loop state) with the running coverage of every coverage attention
        passed through `gather` - the beam search's re-ordering of rows to the selected hypotheses.  The other
        histories are not read by the next step and stay as they are."""
        if not any(isinstance(att, CoverageAttention) for att in self.attentions):
            return histories
        states = [state._replace(coverage=gather(state.coverage))
                  if isinstance(att, CoverageAttention) and state.coverage is not None else state
                  for att, state in zip(self.attentions, histories.other.attention_histories)]
        return histories._replace(other=histories.other._replace(attention_histories=states))

    def next_state(self, loop_state: LoopState) -> Tuple[torch.Tensor, Any, Any]:
        """Decoder.next_state, GRU branch (decoder.py:279-358)."""
        rnn_feedables = loop_state.feedables.other
        rnn_histories = loop_state.histories.other
        rnn_input = loop_state.feedables.embedded_input
        if self._stepwise:
            states = iter(rnn_histories.attention_histories)
            prev = rnn_feedables.prev_rnn_output
            if self._rnn_cell_str == "LSTM":
                prev = (rnn_feedables.prev_rnn_state, rnn_feedables.prev_rnn_output)
            output, carried, contexts, attended = self._variant_step(
                rnn_input, prev,
                lambda att, query: att.attention(query, rnn_feedables.prev_rnn_output, rnn_input, next(states)))
            next_state, cell_output = carried if isinstance(carried, tuple) else (carried, carried)
            rnn_histories.rnn_outputs.append(cell_output)
            return (output,
                    RNNFeedables(prev_rnn_state=next_state, prev_rnn_output=cell_output,
                                 prev_contexts=list(contexts)),
                    RNNHistories(rnn_outputs=rnn_histories.rnn_outputs,
                                 attention_histories=[a[1] for a in attended]))
        mask = dropout_mask((rnn_input.shape[0], 1, self.rnn_size), self.dropout_keep_prob,
                            self.train_mode, rnn_input.device)
        dropped, _fin, raw = ops.gru_layer(rnn_input.unsqueeze(1),
                                           *gru_cell_tensors(self, self._CELL_SCOPE),
                                           h0=rnn_feedables.prev_rnn_output, drop_mask=mask)
        cell_output_raw, cell_output = raw[:, 0], dropped[:, 0]
        contexts, att_loop_states = [], []
        for att, att_state in zip(self.attentions, rnn_histories.attention_histories):
            ctx, new_state = att.attention(cell_output_raw, rnn_feedables.prev_rnn_output, rnn_input,
                                           att_state)
            contexts.append(dropout(ctx, self.dropout_keep_prob, self.train_mode))
            att_loop_states.append(new_state)
        output = self.output_projection(self, cell_output, loop_state.feedables.embedded_input,
                                        contexts, self.train_mode)
        new_feedables = RNNFeedables(prev_rnn_state=cell_output, prev_rnn_output=cell_output,
                                     prev_contexts=list(contexts))
        rnn_histories.rnn_outputs.append(cell_output)
        new_histories = RNNHistories(rnn_outputs=rnn_histories.rnn_outputs,
                                     attention_histories=att_loop_states)
        return output, new_feedables, new_histories

    # -- runtime: the whole greedy loop on the fused step kernel -------------------------------------
    use_fused_decoding = True

    @property
    def decode_engine(self):
        """The RNNDecodeEngine of this decoder, or None when its structure is outside what the fused
        step covers (decoders/rnn_decode.py)."""
        from neuralmonkey_b200.decoders import rnn_decode
        if not self.use_fused_decoding or not rnn_decode.supported(self):
            return None
        if "_decode_engine" not in self.__dict__:
            self.__dict__["_decode_engine"] = rnn_decode.RNNDecodeEngine(self)
        return self.__dict__["_decode_engine"]

    @tensor
    def _runtime(self):
        engine = self.decode_engine
        if (engine is None or (self.train_mode and self.dropout_keep_prob < 1.0)
                or not engine.fits(self.batch_size, 1)):
            return AutoregressiveDecoder._runtime.fget(self)
        gold = gold_mask = None
        if self._train_ids_host is not None:
            gold, gold_mask = self.train_inputs, self.train_mask
        res = engine.greedy(self.max_output_len, gold, gold_mask)
        key = "{}_run".format(self.name)
        self.attentions[0].histories[key] = res["weights"]
        self.attentions[0].visualize_attention(key)
        return {"logits": None, "output_states": res["output_states"], "symbols": res["symbols"],
                "mask": res["mask"], "argmax": res["argmax"], "lse": res["lse"], "xent": res["xent"],
                "rnn_outputs": res["rnn_outputs"], "contexts": res["contexts"]}

    def finalize_loop(self, final_loop_state: LoopState, train_mode: bool) -> None:
        for att_state, attn_obj in zip(final_loop_state.histories.other.attention_histories,
                                       self.attentions):
            key = "{}_{}".format(self.name, "train" if train_mode else "run")
            attn_obj.finalize_loop(key, att_state)
            if not train_mode:
                attn_obj.visualize_attention(key)
