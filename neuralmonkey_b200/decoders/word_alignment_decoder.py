"""Supervised attention from word alignments (reference: neuralmonkey/decoders/word_alignment_decoder.py).

The reference module is marked untested and cannot run: it asks the decoder for `get_attention_object`, which no
longer exists.  What it computes is restated from its code:

* training (:100-108): softmax_cross_entropy_with_logits of the attention energies of the decoder's training pass
  (the pre-softmax scores e of `attention.Attention`, over all encoder positions, padding included) against the fed
  alignment matrices, times the decoder's training padding, summed over steps and sentences;
* run time (:94-98): the attention of the decoder's greedy run, batch-major.  The reference takes the softmax of
  the run-time energies; the decoding step records the masked and renormalised weights instead, so padded encoder
  positions get weight 0 here.

The energies come from the decoder's own attention evaluation (`Decoder.supervise_attention`), so the decoder's
cost and the alignment cost reach the attention's backward kernel in one call.  The loss is `ops.alignment_xent`.
"""
from typing import Any, Dict, List, cast

import numpy as np
import torch

from neuralmonkey_b200 import ops, runtime
from neuralmonkey_b200.decoders.decoder import Decoder
from neuralmonkey_b200.decorators import tensor
from neuralmonkey_b200.logging import warn
from neuralmonkey_b200.model.model_part import ModelPart
from neuralmonkey_b200.model.parameterized import InitializerSpecs
from neuralmonkey_b200.model.sequence import Sequence
from neuralmonkey_b200.model.stateful import TemporalStateful
from neuralmonkey_b200.typecheck import check_argument_types


class WordAlignmentDecoder(ModelPart):
    """A decoder that computes soft alignment from an attentive encoder.

    Loss is computed as cross-entropy against a reference alignment.  It declares no variables.
    """

    # pylint: disable=too-many-arguments
    def __init__(self, encoder: TemporalStateful, decoder: Decoder, data_id: str, name: str,
                 reuse: ModelPart = None, initializers: InitializerSpecs = None) -> None:
        check_argument_types()
        ModelPart.__init__(self, name, reuse, None, None, initializers)
        self.encoder = encoder
        self.decoder = decoder
        self.data_id = data_id
        self.attention = decoder.supervise_attention(encoder)
        self._alignment_host = None     # type: Any
    # pylint: enable=too-many-arguments

    @property
    def dependencies(self) -> List[str]:
        return ModelPart.dependencies.fget(self) + ["decoder"]

    @property
    def enc_input(self) -> Sequence:
        if not isinstance(self.encoder.input_sequence, Sequence):
            raise TypeError("Expected Sequence type in encoder.input_sequence")
        return cast(Sequence, self.encoder.input_sequence)

    @property
    def input_types(self) -> Dict[str, Any]:
        return {self.data_id: np.float32}

    @property
    def input_shapes(self) -> Dict[str, Any]:
        return {self.data_id: [None, self.decoder.max_output_len, self.enc_input.max_length]}

    def feed_dict(self, dataset, train: bool = False) -> Dict[str, Any]:
        fd = ModelPart.feed_dict(self, dataset, train)
        alignment = dataset.maybe_get_series(self.data_id)
        if alignment is None:
            if train:
                warn("Training alignment not present!")
            self._alignment_host = None
        else:
            self._alignment_host = np.asarray(list(alignment), dtype=np.float32)
            fd[self.data_id] = self._alignment_host
        return fd

    @tensor
    def ref_alignment(self) -> torch.Tensor:
        """[batch, max_output_len, encoder input length] fed alignments; zeros when none are fed, as wide as the
        encoder's max_length or, without one, as the batch's encoder states."""
        if self._alignment_host is None:
            width = self.enc_input.max_length
            if width is None:
                width = self.attention.attention_states.shape[1]
            return torch.zeros(self.batch_size, self.decoder.max_output_len, width, device=runtime.device())
        return runtime.to_device(torch.from_numpy(self._alignment_host))

    @property
    def alignment_target(self) -> torch.Tensor:
        """[max_output_len, batch, encoder input length] (word_alignment_decoder.py:59-62)."""
        return self.ref_alignment.transpose(0, 1)

    @tensor
    def train_loss(self) -> torch.Tensor:
        """The summed alignment cross-entropy of the training pass.  Rows of the fed matrices beyond the decoder's
        training steps and columns beyond the batch's encoder states are dropped; missing ones are zero targets."""
        energies = self.decoder.train_attention_energies(self.attention)     # [B, steps, Tx]
        bsz, steps, width = energies.shape
        ref = self.ref_alignment
        if ref.dim() != 3 or ref.shape[0] != bsz:
            raise ValueError("WordAlignmentDecoder '{}': alignments of shape {} for a batch of {}".format(
                self.name, tuple(ref.shape), bsz))
        if tuple(ref.shape) == (bsz, steps, width):
            target = ref
        else:
            target = energies.new_zeros(bsz, steps, width)
            rows, cols = min(steps, ref.shape[1]), min(width, ref.shape[2])
            target[:, :rows, :cols] = ref[:, :rows, :cols]
        pad = self.decoder.train_mask.t()[:, :steps]
        return ops.alignment_xent(energies, target, pad)

    @property
    def cost(self) -> torch.Tensor:
        return self.train_loss

    # GenericTrainer(use_cuda_graph=True) captures a step of one token-mean objective; this cost is a second one
    graph_capturable = False

    @tensor
    def runtime_loss(self) -> torch.Tensor:
        return torch.zeros((), device=runtime.device())

    @tensor
    def decoded(self) -> torch.Tensor:
        """[batch, run steps, encoder states] attention weights of the decoder's greedy run."""
        _ = self.decoder.runtime_symbols        # the greedy run records the histories
        key = "{}_run".format(self.decoder.name)
        if key not in self.attention.histories:
            raise KeyError("Attention has no recorded histories under key '{}'".format(key))
        return self.attention.histories[key].transpose(0, 1)
