"""Beam search decoder (reference: neuralmonkey/decoders/beam_search_decoder.py:44-560).

Same algorithm and loop-state structures as the reference (GNMT length penalty, eq. 14 of
arxiv.org/abs/1609.08144): the parent decoder's step runs once to score the first token,
then each beam step = K12 kernel (`ops.beam_step`: finished-row masking, hypothesis scores,
top-k over beam*vocabulary, bookkeeping gathers - beam_search_decoder.py:440-496) + one row
gather per decoder feedable (`ops.beam_gather` = tf_utils.gather_flat) + one parent decoder
step on the re-ordered beam.  The host loop reads one device flag per step (all finished).

Differences kept deliberately small: decoder *histories* (logits/attention weights of every
step) are not re-gathered each step - the reference never finalises them for beam search
either (:372-374) - and only the last step's logits are kept alive, so a beam of 12 over a
32k vocabulary does not hold steps*batch*beam*V floats.  Ensembling, which the reference does by
re-feeding the loop state one step at a time (`max_steps` placeholder, beamsearch_runner.py:48-78), is
`ensemble_outputs`: the same schedule in one loop.
"""
from typing import Any, List, NamedTuple

import torch

from neuralmonkey_b200.typecheck import check_argument_types
from neuralmonkey_b200 import ops, runtime
from neuralmonkey_b200.decoders.autoregressive import (AutoregressiveDecoder, DecoderFeedables,
                                                       LoopState)
from neuralmonkey_b200.decorators import tensor
from neuralmonkey_b200.model.model_part import ModelPart
from neuralmonkey_b200.vocabulary import END_TOKEN_INDEX, Vocabulary

INF = 1e9  # beam_search_decoder.py:43

SearchState = NamedTuple("SearchState", [
    ("logprob_sum", torch.Tensor), ("prev_logprobs", torch.Tensor), ("lengths", torch.Tensor),
    ("finished", torch.Tensor)])
SearchResults = NamedTuple("SearchResults", [("scores", torch.Tensor), ("token_ids", torch.Tensor)])
BeamSearchLoopState = NamedTuple("BeamSearchLoopState", [
    ("search_state", SearchState), ("search_results", SearchResults),
    ("decoder_loop_state", LoopState)])
BeamSearchOutput = NamedTuple("BeamSearchOutput", [
    ("last_search_step_output", SearchResults), ("last_dec_loop_state", LoopState),
    ("last_search_state", SearchState), ("attention_loop_states", List[Any])])


def map_structure(fn, obj):
    """tf.contrib.framework.nest.map_structure over tuples / lists of tensors."""
    if torch.is_tensor(obj):
        return fn(obj)
    if isinstance(obj, tuple) and hasattr(obj, "_fields"):
        return type(obj)(*[map_structure(fn, o) for o in obj])
    if isinstance(obj, (list, tuple)):
        return type(obj)(map_structure(fn, o) for o in obj)
    return obj


class BeamSearchDecoder(ModelPart):
    def __init__(self, name: str, parent_decoder: AutoregressiveDecoder, beam_size: int,
                 max_steps: int, length_normalization: float) -> None:
        check_argument_types()
        ModelPart.__init__(self, name)
        self.parent_decoder = parent_decoder
        self.beam_size = beam_size
        self.length_normalization = length_normalization
        self.max_steps_int = max_steps
        self.max_steps = max_steps
        if beam_size < 1:
            raise ValueError("Beam size must be a positive integer.")

    @property
    def vocabulary(self) -> Vocabulary:
        return self.parent_decoder.vocabulary

    def expand_to_beam(self, val: torch.Tensor, dim: int = 0) -> torch.Tensor:
        """Copy a tensor along `dim` beam_size times, beam-minor (beam_search_decoder.py:562-590)."""
        if val.dim() <= dim:
            return val
        return val.repeat_interleave(self.beam_size, dim=dim)

    # -- one parent decoder step without history bookkeeping --------------------------------
    def _decoder_step(self, dec_ls: LoopState):
        parent = self.parent_decoder
        feedables = dec_ls.feedables
        output_state, dec_other, hist_other = parent.next_state(dec_ls)
        logits, lse, argmax = parent.state_to_logits(output_state)
        logprobs = ops.log_softmax_from_lse(logits, lse)
        symbols = argmax * (~feedables.finished).to(torch.int64)
        finished = feedables.finished | (symbols == END_TOKEN_INDEX)
        next_feedables = DecoderFeedables(step=feedables.step + 1, finished=finished,
                                          embedded_input=feedables.embedded_input, other=dec_other)
        next_ls = LoopState(histories=dec_ls.histories._replace(other=hist_other),
                            constants=dec_ls.constants, feedables=next_feedables)
        bsz = logprobs.shape[0] // self.beam_size
        return next_ls, logprobs.view(bsz, self.beam_size, -1), symbols

    def get_initial_loop_state(self) -> BeamSearchLoopState:
        parent = self.parent_decoder
        bsz, k, dev = parent.batch_size, self.beam_size, runtime.device()
        dec_init = parent.get_initial_loop_state()
        dec_init = dec_init._replace(
            feedables=map_structure(self.expand_to_beam, dec_init.feedables),
            histories=map_structure(lambda x: self.expand_to_beam(x, 1), dec_init.histories))
        dec_next, logprobs, symbols = self._decoder_step(dec_init)
        logprob_sum = torch.full((bsz, k), -INF, device=dev, dtype=torch.float32)
        logprob_sum[:, 0] = 0.0
        search_state = SearchState(
            logprob_sum=logprob_sum, prev_logprobs=logprobs,
            lengths=torch.zeros(bsz, k, dtype=torch.int32, device=dev),
            finished=torch.zeros(bsz, k, dtype=torch.bool, device=dev))
        search_results = SearchResults(scores=torch.zeros(bsz, k, device=dev),
                                       token_ids=symbols.view(1, bsz, k))
        return BeamSearchLoopState(search_state, search_results, dec_next)

    def _select(self, state: SearchState):
        """Steps (1)-(8) of the beam body on the shared search state: the K12 kernel."""
        return ops.beam_step(state.prev_logprobs, state.logprob_sum, state.lengths,
                             state.finished.to(torch.uint8), self.length_normalization)

    def _advance(self, dec_ls: LoopState, words, beams, finished, bsz: int):
        """Re-order one decoder's feedables to the selected beams, feed the chosen words, step it."""
        k = self.beam_size
        gathered = map_structure(
            lambda x: ops.beam_gather(x, beams, bsz, k)
            if x.dim() >= 1 and x.shape[0] == bsz * k and x.numel() > 0 else x, dec_ls.feedables)
        gathered = gathered._replace(
            embedded_input=self.parent_decoder.embed_input_symbols(words.view(-1)),
            finished=finished.view(-1))
        histories = dec_ls.histories
        reorder = getattr(self.parent_decoder, "reorder_attention_states", None)
        if reorder is not None:     # loop states the next step's attention energies read (coverage)
            histories = reorder(histories, lambda x: ops.beam_gather(x, beams, bsz, k))
        return self._decoder_step(dec_ls._replace(feedables=gathered, histories=histories))

    def decoding_loop(self, initial: BeamSearchLoopState) -> BeamSearchOutput:
        k = self.beam_size
        bsz = initial.search_state.logprob_sum.shape[0]
        dev = runtime.device()
        state, dec_ls = initial.search_state, initial.decoder_loop_state
        scores = initial.search_results.scores
        # token history rows [batch*beam, 1 + max_steps]; re-ordered with the beam each step
        history = torch.zeros(bsz * k, self.max_steps + 1, dtype=torch.int64, device=dev)
        history[:, 0] = initial.search_results.token_ids.reshape(-1)
        written = 1
        # loop_continue_criterion (:330-355): decoder step - 1 < max_steps and not all finished
        while dec_ls.feedables.step - 1 < self.max_steps and not bool(state.finished.all()):
            scores, words, beams, lsum, lens, fin = self._select(state)
            finished = fin.to(torch.bool)
            history = ops.beam_gather(history, beams, bsz, k)
            history[:, written] = words.view(-1)
            written += 1
            dec_ls, logprobs, _ = self._advance(dec_ls, words, beams, finished, bsz)
            state = SearchState(logprob_sum=lsum, prev_logprobs=logprobs, lengths=lens,
                                finished=finished)
        token_ids = history[:, :written].view(bsz, k, written).permute(2, 0, 1).contiguous()
        return BeamSearchOutput(
            last_search_step_output=SearchResults(scores=scores, token_ids=token_ids),
            last_dec_loop_state=dec_ls, last_search_state=state, attention_loop_states=[])

    def ensemble_outputs(self, activate, num_sessions: int) -> BeamSearchOutput:
        """The search over an ensemble (runners/beamsearch_runner.py:44-118 drive it through placeholders
        one step at a time; this is the same schedule in one loop).  `activate(i)` switches the model
        parts to session i.  Every session runs its own decoder (own parameters, own encoder states, own
        recurrent state); the search state is ONE: after each decoder step the sessions' next-token
        log-probabilities are averaged in probability space, logsumexp - log(n) (:50-54), and the next
        selection is made on that average - so all sessions follow the same beam."""
        parent = self.parent_decoder
        k = self.beam_size
        enc_states, enc_masks = parent.encoder_states, parent.encoder_masks
        log_n = float(torch.log(torch.tensor(float(num_sessions))))

        def on_session(index, fn):
            activate(index)
            tiled_states = [self.expand_to_beam(s) for s in enc_states()]
            tiled_masks = [self.expand_to_beam(m) if m is not None else None for m in enc_masks()]
            parent.encoder_states, parent.encoder_masks = (lambda: tiled_states), (lambda: tiled_masks)
            try:
                with torch.no_grad():
                    return fn()
            finally:
                parent.encoder_states, parent.encoder_masks = enc_states, enc_masks

        initial = [on_session(i, self.get_initial_loop_state) for i in range(num_sessions)]
        dec_ls = [init.decoder_loop_state for init in initial]

        def average(logprobs):
            return torch.logsumexp(torch.stack(logprobs, 0), dim=0) - log_n

        state = initial[0].search_state._replace(
            prev_logprobs=average([init.search_state.prev_logprobs for init in initial]))
        scores = initial[0].search_results.scores
        bsz = state.logprob_sum.shape[0]
        history = torch.zeros(bsz * k, self.max_steps + 1, dtype=torch.int64, device=runtime.device())
        history[:, 0] = initial[0].search_results.token_ids.reshape(-1)
        written = 1
        while dec_ls[0].feedables.step - 1 < self.max_steps and not bool(state.finished.all()):
            scores, words, beams, lsum, lens, fin = self._select(state)
            finished = fin.to(torch.bool)
            history = ops.beam_gather(history, beams, bsz, k)
            history[:, written] = words.view(-1)
            written += 1
            stepped = [on_session(i, lambda i=i: self._advance(dec_ls[i], words, beams, finished, bsz))
                       for i in range(num_sessions)]
            dec_ls = [s[0] for s in stepped]
            state = SearchState(logprob_sum=lsum, prev_logprobs=average([s[1] for s in stepped]),
                                lengths=lens, finished=finished)
        token_ids = history[:, :written].view(bsz, k, written).permute(2, 0, 1).contiguous()
        return BeamSearchOutput(
            last_search_step_output=SearchResults(scores=scores, token_ids=token_ids),
            last_dec_loop_state=dec_ls[0], last_search_state=state, attention_loop_states=[])

    # Replay one captured CUDA graph per step when the parent is a Transformer decoder with a KV
    # cache (decoders/beam_graph.py); False falls back to the step-by-step host loop.
    use_cuda_graph = True
    MAX_GRAPHS = 4        # captured (batch, source length) shapes kept alive
    GRAPH_AFTER = 2       # a shape is captured the second time it shows up; one-offs use the loop

    def _graph_outputs(self, tiled_states, tiled_masks) -> BeamSearchOutput:
        from neuralmonkey_b200.decoders.beam_graph import TransformerBeamGraph
        parent = self.parent_decoder
        bsz = parent.batch_size
        key = (bsz, tuple(tuple(s.shape) for s in tiled_states))
        graphs = self.__dict__.setdefault("_graphs", {})
        if key not in graphs:
            while len(graphs) >= self.MAX_GRAPHS:          # bounded: each holds its KV buffers
                graphs.pop(next(iter(graphs)))
            graphs[key] = TransformerBeamGraph(self, bsz, key[1])
        else:
            graphs[key] = graphs.pop(key)                  # most recently used last
        res = graphs[key].run(tiled_states, tiled_masks)
        dev = runtime.device()
        feedables = DecoderFeedables(step=res["steps"] + 1, finished=res["finished"].view(-1),
                                     embedded_input=torch.zeros(0, device=dev), other=None)
        dec_ls = LoopState(histories=parent.get_initial_histories(), constants=None, feedables=feedables)
        return BeamSearchOutput(
            last_search_step_output=SearchResults(scores=res["scores"], token_ids=res["token_ids"]),
            last_dec_loop_state=dec_ls,
            last_search_state=SearchState(logprob_sum=res["logprob_sum"], prev_logprobs=res["logprobs"],
                                          lengths=res["lengths"], finished=res["finished"]),
            attention_loop_states=[])

    use_fused_step = True

    def _fused_outputs(self, engine) -> BeamSearchOutput:
        parent = self.parent_decoder
        res = engine.beam(self.beam_size, self.max_steps, self.length_normalization)
        dev = runtime.device()
        feedables = DecoderFeedables(step=res["steps"] + 1, finished=res["finished"].view(-1),
                                     embedded_input=torch.zeros(0, device=dev), other=None)
        dec_ls = LoopState(histories=parent.get_initial_histories(), constants=None, feedables=feedables)
        logprobs = ops.log_softmax_from_lse(res["logits"].reshape(-1, res["logits"].shape[-1]),
                                            res["lse"].reshape(-1)).view(res["logits"].shape)
        return BeamSearchOutput(
            last_search_step_output=SearchResults(scores=res["scores"], token_ids=res["token_ids"]),
            last_dec_loop_state=dec_ls,
            last_search_state=SearchState(logprob_sum=res["logprob_sum"], prev_logprobs=logprobs,
                                          lengths=res["lengths"], finished=res["finished"]),
            attention_loop_states=[])

    @tensor
    def outputs(self) -> BeamSearchOutput:
        parent = self.parent_decoder
        engine = getattr(parent, "decode_engine", None) if self.use_fused_step else None
        if engine is not None:
            # RNN parent: the fused step kernel follows the beam indices itself and reads the UN-tiled
            # encoder tensors (`group` = beam size), so nothing is tiled or re-gathered here
            return self._fused_outputs(engine)
        enc_states, enc_masks = parent.encoder_states, parent.encoder_masks
        # beam-tiled encoder tensors for the duration of the search (:174-186)
        tiled_states = [self.expand_to_beam(s) for s in enc_states()]
        tiled_masks = [self.expand_to_beam(m) if m is not None else None for m in enc_masks()]
        from neuralmonkey_b200.decoders.transformer import TransformerDecoder
        seen = self.__dict__.setdefault("_shape_seen", {})
        shape_key = (parent.batch_size, tuple(tuple(s.shape) for s in tiled_states))
        seen[shape_key] = seen.get(shape_key, 0) + 1
        if len(seen) > 4096:
            seen.clear()
        if (self.use_cuda_graph and isinstance(parent, TransformerDecoder) and parent.use_kv_cache
                and runtime.device().type == "cuda" and seen[shape_key] >= self.GRAPH_AFTER):
            try:
                with torch.no_grad():
                    return self._graph_outputs(tiled_states, tiled_masks)
            finally:
                parent.encoder_states, parent.encoder_masks = enc_states, enc_masks
        parent.encoder_states = lambda: tiled_states
        parent.encoder_masks = lambda: tiled_masks
        try:
            with torch.no_grad():
                result = self.decoding_loop(self.get_initial_loop_state())
        finally:
            parent.encoder_states, parent.encoder_masks = enc_states, enc_masks
        return result
