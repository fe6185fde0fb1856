"""Autoregressive decoder base (reference: neuralmonkey/decoders/autoregressive.py:28-584).

What the reference expresses as two `tf.while_loop`s is split by what the data allows:

* training (teacher forcing): every step's input is known up front, so subclasses compute
  all output states in one batched pass (`train_output_states`) and the vocabulary
  projection + cross-entropy is ONE fused tensor-core GEMM over all T*B rows
  (`ops.logits_xent`) - the `[T,B,V]` logits are never materialised unless asked for;
* runtime (greedy feedback): a host loop over steps, each step = subclass `next_state` +
  fused logits/argmax kernel; histories are kept as lists and stacked once (the reference
  re-concatenates every history at every step, tf_utils.py:222-235).
"""
from typing import Any, Callable, Dict, List, NamedTuple, Optional, Tuple

import numpy as np
import torch

from neuralmonkey_b200 import ops, runtime
from neuralmonkey_b200.decorators import tensor
from neuralmonkey_b200.logging import warn
from neuralmonkey_b200.model.model_part import ModelPart
from neuralmonkey_b200.model.parameterized import InitializerSpecs
from neuralmonkey_b200.model.sequence import EmbeddedSequence
from neuralmonkey_b200.nn.utils import dropout
from neuralmonkey_b200.params import uniform_initializer, zeros_initializer
from neuralmonkey_b200.vocabulary import (END_TOKEN_INDEX, PAD_TOKEN_INDEX, START_TOKEN_INDEX,
                                          UNK_TOKEN_INDEX, Vocabulary, pad_batch)

# Loop-state tuples of the reference (autoregressive.py:28-113).  `other` carries the
# subclass-specific part (RNNFeedables / TransformerFeedables ...).
DecoderConstants = NamedTuple("DecoderConstants", [("train_inputs", Optional[torch.Tensor])])
DecoderHistories = NamedTuple("DecoderHistories", [
    ("logits", Any), ("output_states", Any), ("output_symbols", Any), ("output_mask", Any),
    ("other", Any)])
DecoderFeedables = NamedTuple("DecoderFeedables", [
    ("step", int), ("finished", torch.Tensor), ("embedded_input", torch.Tensor), ("other", Any)])
LoopState = NamedTuple("LoopState", [
    ("histories", Any), ("constants", Any), ("feedables", Any)])


class AutoregressiveDecoder(ModelPart):
    # pylint: disable=too-many-arguments,too-many-instance-attributes
    def __init__(self, name: str, vocabulary: Vocabulary, data_id: str, max_output_len: int,
                 dropout_keep_prob: float = 1.0, embedding_size: int = None,
                 embeddings_source: EmbeddedSequence = None, tie_embeddings: bool = False,
                 label_smoothing: float = None, supress_unk: bool = False, reuse: ModelPart = None,
                 save_checkpoint: str = None, load_checkpoint: str = None,
                 initializers: InitializerSpecs = None) -> None:
        ModelPart.__init__(self, name, reuse, save_checkpoint, load_checkpoint, initializers)
        self.vocabulary = vocabulary
        self.data_id = data_id
        self.max_output_len = max_output_len
        self.dropout_keep_prob = dropout_keep_prob
        self._embedding_size = embedding_size
        self.embeddings_source = embeddings_source
        self.label_smoothing = label_smoothing
        self.tie_embeddings = tie_embeddings
        self.supress_unk = supress_unk
        # callables so a BeamSearchDecoder can substitute beam-tiled tensors
        self.encoder_states = lambda: []  # type: Callable[[], List[torch.Tensor]]
        self.encoder_masks = lambda: []  # type: Callable[[], List[torch.Tensor]]
        if self.max_output_len <= 0:
            raise ValueError("Maximum sequence length must be a positive integer.")
        if self._embedding_size is not None and self._embedding_size <= 0:
            raise ValueError("Embedding size must be a positive integer.")
        if self.dropout_keep_prob < 0.0 or self.dropout_keep_prob > 1.0:
            raise ValueError("Dropout keep probability must be a real number in the interval [0,1].")
        self._train_ids_host = None  # type: Optional[torch.Tensor]

    # -- static configuration ----------------------------------------------------------
    @property
    def embedding_size(self) -> int:
        if self.embeddings_source is None:
            if self._embedding_size is None:
                raise ValueError(
                    "You must specify either embedding size or the embedded sequence from which "
                    "to reuse the embeddings (e.g. set 'embedding_size' or 'embeddings_source' "
                    "parameter)")
            return self._embedding_size
        if self._embedding_size is not None:
            warn("Overriding the embedding_size parameter with the size of the reused "
                 "embeddings from the encoder.")
        return self.embeddings_source.embedding_sizes[0]

    @property
    def output_dimension(self) -> int:
        raise NotImplementedError("Abstract property")

    def declare_variables(self) -> None:
        if self.embeddings_source is not None:
            self.embeddings_source.ensure_declared()
        else:
            self.declare("word_embeddings", [len(self.vocabulary), self.embedding_size])
        if self.tie_embeddings:
            if self.embedding_size != self.output_dimension:
                raise ValueError("`embedding_size must be equal to the output_projection size when "
                                 "using the `tie_embeddings` option")
        else:
            self.declare("state_to_word_W", [self.output_dimension, len(self.vocabulary)],
                         uniform_initializer(-0.5, 0.5))
            self.declare("state_to_word_b", [len(self.vocabulary)], zeros_initializer())

    @property
    def embedding_matrix(self) -> torch.Tensor:
        if self.embeddings_source is not None:
            return self.embeddings_source.embedding_matrix
        return self.var("word_embeddings")

    @property
    def decoding_w(self) -> torch.Tensor:
        """[output_dimension, V]; with tied embeddings the [V, E] matrix is used transposed
        inside the GEMM (`_w_transposed`), never copied."""
        if self.tie_embeddings:
            return self.embedding_matrix
        return self.var("state_to_word_W")

    @property
    def _w_transposed(self) -> bool:
        return bool(self.tie_embeddings)

    @property
    def decoding_b(self) -> Optional[torch.Tensor]:
        if self.tie_embeddings:
            return None  # tf.zeros constant (autoregressive.py:241-242)
        return self.var("state_to_word_b")

    @property
    def _unk_index(self) -> int:
        return UNK_TOKEN_INDEX if self.supress_unk else -1

    @property
    def _train_unk_index(self) -> int:
        """The <unk> column suppressed in the TRAINING logits: the same as at run time for decoders whose
        training pass goes through get_body (autoregressive.py:450-459)."""
        return self._unk_index

    # -- feeding -------------------------------------------------------------------------
    @property
    def input_types(self) -> Dict[str, Any]:
        return {self.data_id: str}

    @property
    def input_shapes(self) -> Dict[str, Any]:
        return {self.data_id: [None, None]}

    def feed_dict(self, dataset, train: bool = False) -> Dict[str, Any]:
        fd = ModelPart.feed_dict(self, dataset, train)
        sentences = dataset.maybe_get_series(self.data_id)
        if sentences is None and train:
            raise ValueError("When training, you must feed reference sentences")
        self._train_ids_host = None
        if sentences is not None:
            padded = pad_batch(list(sentences), self.max_output_len, add_start_symbol=False,
                               add_end_symbol=True)
            self._train_ids_host = self.vocabulary.strings_to_indices(padded)
            fd[self.data_id] = self._train_ids_host
        return fd

    def feed_ids(self, ids: Optional[torch.Tensor], batch_size: int, train: bool = False) -> None:
        """Feed indexed references ([batch, time] int64 incl. </s>, or None)."""
        self.reset_batch()
        self.train_mode = bool(train)
        self.batch_size = batch_size
        self._train_ids_host = ids.cpu() if ids is not None else None

    def static_inputs(self) -> Dict[str, Any]:
        if self._train_ids_host is None:
            return {}
        return {"targets": self._train_targets_bm, "fed_symbols": self._train_step_inputs_bm}

    def bind_static(self, tensors: Dict[str, Any]) -> None:
        self.reset_batch()
        if tensors:
            self.__dict__["_batch_cache"].update({"_train_targets_bm": tensors["targets"],
                                                  "_train_step_inputs_bm": tensors["fed_symbols"]})

    @tensor
    def _train_targets_bm(self) -> torch.Tensor:
        """[batch, time] int64 gold symbols incl. </s> (batch-major: the layout every training
        kernel works in; the reference's time-major `train_inputs` is a view of it)."""
        if self._train_ids_host is None:
            raise ValueError("Decoder '{}' has no reference series fed".format(self.name))
        return runtime.to_device(self._train_ids_host.contiguous())

    @tensor
    def _train_mask_bm(self) -> torch.Tensor:
        return (self._train_targets_bm != PAD_TOKEN_INDEX).to(torch.float32)

    @tensor
    def train_inputs(self) -> torch.Tensor:
        """[time, batch] int64 (autoregressive.py:199-202)."""
        return self._train_targets_bm.t()

    @tensor
    def train_mask(self) -> torch.Tensor:
        return self._train_mask_bm.t()

    @staticmethod
    def teacher_forcing_inputs(gold: np.ndarray) -> np.ndarray:
        """[batch, time] symbols fed at each training step, from the gold ids [batch, time]: <s>, then
        the gold symbol of the previous step times `unfinished` - i.e. <pad> after the first </s>
        (get_body: logits_to_symbols / is_finished, autoregressive.py:446-475).  Host arithmetic on
        the ids of one batch; the device sees only the result."""
        bsz, steps = gold.shape
        finished = np.zeros(bsz, dtype=bool)
        fed = np.empty((bsz, steps), dtype=np.int64)
        fed[:, 0] = START_TOKEN_INDEX
        for s in range(steps - 1):
            nxt = gold[:, s] * (~finished)
            finished |= (nxt == END_TOKEN_INDEX)
            fed[:, s + 1] = nxt
        return fed

    @tensor
    def _train_step_inputs_bm(self) -> torch.Tensor:
        return runtime.to_device(torch.from_numpy(self.teacher_forcing_inputs(self._train_ids_host.numpy())))

    def embed_input_symbols(self, input_symbols: torch.Tensor) -> torch.Tensor:
        embedded = ops.embed(input_symbols, self.embedding_matrix)
        return dropout(embedded, self.dropout_keep_prob, self.train_mode)

    # -- training tensors ------------------------------------------------------------------
    @property
    def _train_states_bm(self) -> torch.Tensor:
        """[batch, time, output_dimension]: subclasses compute all steps in one pass."""
        raise NotImplementedError("Abstract property")

    @property
    def train_output_states(self) -> torch.Tensor:
        """[time, batch, output_dimension] (a transposed view)."""
        return self._train_states_bm.transpose(0, 1)

    @tensor
    def _train_xent_result(self):
        states = self._train_states_bm
        bsz, steps, dim = states.shape
        targets = self._train_targets_bm[:, :steps]
        weights = self._train_mask_bm[:, :steps]
        if self.label_smoothing:
            # What the reference computes (autoregressive.py:294-310, SURVEY.md trap 14): tf.losses.
            # softmax_cross_entropy reduces the smoothed cross-entropies to ONE scalar - their mean over
            # ALL positions, padding (target <pad>) included - and sequence_loss multiplies it by the mask.
            flat = states.reshape(bsz * steps, dim)
            every = torch.ones(bsz * steps, device=flat.device, dtype=torch.float32)
            plain, lse, argmax, _ = ops.logits_xent(flat, self.decoding_w, self.decoding_b,
                                                    targets.reshape(-1), every, self._train_unk_index,
                                                    self._w_transposed)
            term = ops.smoothing_term(flat, self.decoding_w, self.decoding_b, targets.reshape(-1),
                                      self._train_unk_index, self._w_transposed)
            scalar = (plain + float(self.label_smoothing) * term).mean()
            return scalar * weights, lse.view(bsz, steps), argmax.view(bsz, steps)
        xent, lse, argmax, _ = ops.logits_xent(
            states.reshape(bsz * steps, dim), self.decoding_w, self.decoding_b,
            targets.reshape(-1), weights.reshape(-1), self._train_unk_index, self._w_transposed)
        return xent.view(bsz, steps), lse.view(bsz, steps), argmax.view(bsz, steps)

    @tensor
    def train_xents(self) -> torch.Tensor:
        """[batch, time] masked cross-entropies (autoregressive.py:292-310)."""
        return self._train_xent_result[0]

    @tensor
    def train_loss(self) -> torch.Tensor:
        """sum(xent) / sum(mask) (autoregressive.py:312-316)."""
        return self._train_xent_result[0].sum() / self._train_mask_bm.sum()

    @tensor
    def train_xent_sum(self) -> torch.Tensor:
        """Un-normalised sum of cross-entropies: what data-parallel ranks exchange."""
        return self._train_xent_result[0].sum()

    @property
    def cost(self) -> torch.Tensor:
        return self.train_loss

    @tensor
    def train_logits(self) -> torch.Tensor:
        """[time, batch, V]; materialised only when a runner asks for it."""
        states = self._train_states_bm.detach()
        bsz, steps, dim = states.shape
        _, _, _, logits = ops.logits_xent(
            states.reshape(bsz * steps, dim), self.decoding_w.detach(),
            self.decoding_b.detach() if self.decoding_b is not None else None,
            self._train_targets_bm[:, :steps].reshape(-1),
            self._train_mask_bm[:, :steps].reshape(-1), self._train_unk_index, self._w_transposed,
            keep_logits=True)
        return logits.view(bsz, steps, -1).transpose(0, 1)

    @tensor
    def train_logprobs(self) -> torch.Tensor:
        logits = self.train_logits.transpose(0, 1).contiguous()  # [B,T,V]
        lse = self._train_xent_result[1].detach()
        return ops.log_softmax_from_lse(logits.reshape(-1, logits.shape[-1]),
                                        lse.reshape(-1)).view(logits.shape).transpose(0, 1)

    # -- runtime (greedy) loop ------------------------------------------------------------
    def get_initial_feedables(self) -> DecoderFeedables:
        dev = runtime.device()
        go = torch.full((self.batch_size,), START_TOKEN_INDEX, dtype=torch.int64, device=dev)
        return DecoderFeedables(
            step=0, finished=torch.zeros(self.batch_size, dtype=torch.bool, device=dev),
            embedded_input=self.embed_input_symbols(go), other=None)

    def get_initial_histories(self) -> DecoderHistories:
        return DecoderHistories(logits=[], output_states=[], output_symbols=[], output_mask=[],
                                other=None)

    def get_initial_loop_state(self) -> LoopState:
        return LoopState(histories=self.get_initial_histories(),
                         constants=DecoderConstants(train_inputs=None),
                         feedables=self.get_initial_feedables())

    def next_state(self, loop_state: LoopState) -> Tuple[torch.Tensor, Any, Any]:
        """One decoder step: (output state [batch, output_dimension], feedables.other,
        histories.other)."""
        raise NotImplementedError("Abstract method.")

    def state_to_logits(self, state: torch.Tensor, keep_logits: bool = True):
        """logits (+ -1e9 on <unk>), their logsumexp and first-index argmax, in one fused
        kernel (autoregressive.py:450-459,470)."""
        bsz = state.shape[0]
        dev = state.device
        dummy_t = torch.zeros(bsz, dtype=torch.int64, device=dev)
        dummy_w = torch.zeros(bsz, dtype=torch.float32, device=dev)
        _, lse, argmax, logits = ops.logits_xent(state, self.decoding_w, self.decoding_b, dummy_t,
                                                 dummy_w, self._unk_index, self._w_transposed,
                                                 keep_logits=keep_logits)
        return logits, lse, argmax

    def body(self, loop_state: LoopState) -> LoopState:
        """get_body(train_mode=False) (autoregressive.py:482-517)."""
        feedables = loop_state.feedables
        histories = loop_state.histories
        output_state, dec_other, hist_other = self.next_state(loop_state)
        logits, _lse, argmax = self.state_to_logits(output_state)
        next_symbols = argmax * (~feedables.finished).to(torch.int64)
        finished = feedables.finished | (next_symbols == END_TOKEN_INDEX)
        next_feedables = DecoderFeedables(
            step=feedables.step + 1, finished=finished,
            embedded_input=self.embed_input_symbols(next_symbols), other=dec_other)
        histories.logits.append(logits)
        histories.output_states.append(output_state)
        histories.output_symbols.append(next_symbols)
        histories.output_mask.append(~finished)
        next_histories = histories._replace(other=hist_other)
        return LoopState(histories=next_histories, constants=loop_state.constants,
                         feedables=next_feedables)

    def get_body(self, train_mode: bool, sample: bool = False, temperature: float = 1.):
        """The loop body as a callable over a LoopState (autoregressive.py:442-517).  Run time without
        sampling at temperature 1 is `body` (fused logits + argmax).  `sample=True` draws the next symbols from
        softmax(logits / temperature) - tf.multinomial over the logits, what the RL trainer's sampling pass asks
        for (trainers/rl_trainer.py:124) - and a temperature other than 1 divides the logits that enter the
        histories, as the reference does before choosing the symbols.  The teacher-forced pass is not stepped
        in this package (`train_logits` & co. come from whole-sequence kernels), so `train_mode=True` is
        refused here."""
        if train_mode:
            raise NotImplementedError(
                "the teacher-forced pass is not stepped: use train_logits / train_output_states / train_xents")
        if not sample and float(temperature) == 1.0:
            return self.body
        temperature = float(temperature)

        def body(loop_state: LoopState) -> LoopState:
            feedables = loop_state.feedables
            histories = loop_state.histories
            output_state, dec_other, hist_other = self.next_state(loop_state)
            logits, _lse, argmax = self.state_to_logits(output_state)
            if temperature != 1.0:
                logits = logits / temperature       # argmax is unchanged by a positive scale
            if sample:
                probs = torch.softmax(logits, dim=-1)
                next_symbols = torch.multinomial(probs, num_samples=1).squeeze(1)
            else:
                next_symbols = argmax
            next_symbols = next_symbols * (~feedables.finished).to(torch.int64)
            finished = feedables.finished | (next_symbols == END_TOKEN_INDEX)
            next_feedables = DecoderFeedables(
                step=feedables.step + 1, finished=finished,
                embedded_input=self.embed_input_symbols(next_symbols), other=dec_other)
            histories.logits.append(logits)
            histories.output_states.append(output_state)
            histories.output_symbols.append(next_symbols)
            histories.output_mask.append(~finished)
            return LoopState(histories=histories._replace(other=hist_other), constants=loop_state.constants,
                             feedables=next_feedables)

        return body

    def decoding_loop(self, train_mode: bool, sample: bool = False, temperature: float = 1) -> LoopState:
        """Run the decoding loop with the body of `get_body` until every hypothesis has finished or
        `max_output_len` steps were taken (autoregressive.py:425-437,532-562); the histories are lists of
        per-step tensors (`torch.stack` them time-major)."""
        if temperature <= 0:
            raise ValueError("The softmax temperature must be positive")
        body = self.get_body(train_mode, sample, temperature)
        with torch.no_grad():
            loop_state = self.get_initial_loop_state()
            step = 0
            while step < self.max_output_len:
                loop_state = body(loop_state)
                step += 1
                if bool(loop_state.feedables.finished.all()):
                    break
            self.finalize_loop(loop_state, train_mode)
        return loop_state

    def finalize_loop(self, final_loop_state: LoopState, train_mode: bool) -> None:
        """Post-loop hook (attention histories etc.)."""

    @tensor
    def runtime_loop_result(self) -> LoopState:
        """decoding_loop(train_mode=False) (autoregressive.py:532-562)."""
        # loop_continue_criterion: not all finished and step < max_output_len (:425-437);
        # the all-finished test is one device->host flag per step
        return self.decoding_loop(train_mode=False)

    @tensor
    def _runtime(self) -> Dict[str, Any]:
        """The histories of the greedy loop, stacked time-major.  Subclasses with a fused decoding engine
        override this (decoders/decoder.py); `logits` may then be None: they are re-computed from the
        output states by ONE batched projection when somebody asks for them, `xent` / `argmax` / `lse` come
        from the fused step."""
        hist = self.runtime_loop_result.histories
        return {"logits": torch.stack(hist.logits, 0), "output_states": torch.stack(hist.output_states, 0),
                "symbols": torch.stack(hist.output_symbols, 0), "mask": torch.stack(hist.output_mask, 0)}

    @tensor
    def runtime_logits(self) -> torch.Tensor:
        logits = self._runtime["logits"]
        if logits is None:
            # the same GEMM instances the steps ran, over all steps at once: bit-identical values
            states = self._runtime["output_states"]
            steps, bsz, dim = states.shape
            with torch.no_grad():
                dummy_t = torch.zeros(steps * bsz, dtype=torch.int64, device=states.device)
                dummy_w = torch.zeros(steps * bsz, dtype=torch.float32, device=states.device)
                _, _, _, logits = ops.logits_xent(
                    states.reshape(steps * bsz, dim), self.decoding_w.detach(),
                    self.decoding_b.detach() if self.decoding_b is not None else None, dummy_t, dummy_w,
                    self._unk_index, self._w_transposed, keep_logits=True)
            logits = logits.view(steps, bsz, -1)
        return logits

    @tensor
    def runtime_output_states(self) -> torch.Tensor:
        return self._runtime["output_states"]

    @tensor
    def runtime_mask(self) -> torch.Tensor:
        return self._runtime["mask"]

    @tensor
    def runtime_symbols(self) -> torch.Tensor:
        """[time, batch] greedy symbols (argmax over the full vocabulary, PAD once finished)."""
        return self._runtime["symbols"]

    @tensor
    def runtime_argmax(self) -> torch.Tensor:
        """[time, batch] argmax of the step's logits over the full vocabulary WITHOUT the `* unfinished`
        masking: what GreedyRunner's host-side np.argmax over runtime_logprobs yields (runners/runner.py:49)."""
        arg = self._runtime.get("argmax")
        if arg is not None:
            return arg
        logits = self.runtime_logits
        steps, bsz, vocab = logits.shape
        _lse, _xent, arg = ops.xent_rows(logits.reshape(steps * bsz, vocab), want_argmax=True)
        return arg.view(steps, bsz)

    @tensor
    def decoded(self) -> torch.Tensor:
        """argmax over logits[:, :, 1:] + 1 (autoregressive.py:341-349)."""
        logits = self.runtime_logits
        steps, bsz, vocab = logits.shape
        # columns 1..V-1 of every row: same buffer, pointer advanced by one float, ld = V
        _lse, _xent, arg = ops.xent_rows(logits.reshape(steps * bsz, vocab), want_argmax=True, first_col=1)
        return (arg + 1).view(steps, bsz)

    @tensor
    def _runtime_lse(self) -> torch.Tensor:
        lse = self._runtime.get("lse")
        if lse is not None:
            return lse.reshape(-1)
        logits = self.runtime_logits
        steps, bsz, vocab = logits.shape
        return ops.xent_rows(logits.reshape(steps * bsz, vocab))[0]

    @tensor
    def runtime_logprobs(self) -> torch.Tensor:
        logits = self.runtime_logits
        return ops.log_softmax_from_lse(logits.reshape(-1, logits.shape[-1]),
                                        self._runtime_lse).view(logits.shape)

    @tensor
    def runtime_xents(self) -> torch.Tensor:
        """[batch, min_time] (autoregressive.py:351-366)."""
        xent = self._runtime.get("xent")
        if xent is not None:
            return xent.t()
        logits = self.runtime_logits
        targets = self.train_inputs
        min_time = min(targets.shape[0], logits.shape[0])
        bsz, vocab = logits.shape[1], logits.shape[2]
        lg = logits[:min_time].reshape(min_time * bsz, vocab)
        tg = targets[:min_time].reshape(-1).contiguous()
        wt = self.train_mask[:min_time].reshape(-1).contiguous()
        _lse, xent, _arg = ops.xent_rows(lg, tg, wt)
        return xent.view(min_time, bsz).t()

    @tensor
    def runtime_loss(self) -> torch.Tensor:
        """sum(runtime_xents) / sum(runtime_mask) - the mask excludes the </s> step
        (autoregressive.py:368-371,510-511)."""
        return self.runtime_xents.sum() / self.runtime_mask.to(torch.float32).sum()
