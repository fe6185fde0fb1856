"""Initial-state projections (reference: neuralmonkey/decoders/encoder_projection.py:37-145).

An EncoderProjection is a callable (decoder, train_mode, rnn_size, encoders) -> [batch, rnn_size]
plus a `declare(decoder, rnn_size, encoders)` hook naming its variables under the decoder's
`initial_state/` scope.
"""
from typing import Callable, List, Optional

import torch

from neuralmonkey_b200 import ops, runtime
from neuralmonkey_b200.model.stateful import Stateful
from neuralmonkey_b200.nn.utils import dropout
from neuralmonkey_b200.params import block_orthogonal_initializer, zeros_initializer


class EncoderProjection:
    def declare(self, decoder, rnn_size: Optional[int], encoders: List[Stateful]) -> None:
        pass

    def output_size(self, rnn_size: Optional[int], encoders: List[Stateful]) -> int:
        raise NotImplementedError

    def __call__(self, decoder, train_mode: bool, rnn_size: Optional[int],
                 encoders: List[Stateful]) -> torch.Tensor:
        raise NotImplementedError


def _encoder_output_size(enc: Stateful) -> int:
    """Width of `enc.output` (the reference reads it off the tensor's static shape).  It is the part's `dimension`
    except where `dimension` names the width of the input instead (StatefulFiller with a projection)."""
    width = getattr(enc, "output_dimension", None)
    return enc.dimension if width is None else width


class _Empty(EncoderProjection):
    def output_size(self, rnn_size, encoders):
        if rnn_size is None:
            raise ValueError("You must supply rnn_size for this type of encoder projection")
        return rnn_size

    def __call__(self, decoder, train_mode, rnn_size, encoders):
        if rnn_size is None:
            raise ValueError("You must supply rnn_size for this type of encoder projection")
        return torch.zeros(rnn_size, device=runtime.device())


class _Concat(EncoderProjection):
    def output_size(self, rnn_size, encoders):
        if not encoders:
            raise ValueError("There must be at least one encoder for this type of encoder projection")
        size = sum(_encoder_output_size(e) for e in encoders)
        if rnn_size is not None and rnn_size != size:
            raise ValueError("RNN size supplied for concat projection ({}) does not match the size "
                             "of the concatenated vectors ({}).".format(rnn_size, size))
        return size

    def __call__(self, decoder, train_mode, rnn_size, encoders):
        self.output_size(rnn_size, encoders)
        outs = [e.output for e in encoders]
        return outs[0] if len(outs) == 1 else torch.cat(outs, 1)


class _Linear(EncoderProjection):
    def __init__(self, dropout_keep_prob: float) -> None:
        self.dropout_keep_prob = dropout_keep_prob

    def output_size(self, rnn_size, encoders):
        if rnn_size is None:
            raise ValueError("You must supply rnn_size for this type of encoder projection")
        return rnn_size

    def declare(self, decoder, rnn_size, encoders):
        in_size = sum(_encoder_output_size(e) for e in encoders)
        decoder.declare("initial_state/encoders_projection/kernel", [in_size, rnn_size])
        decoder.declare("initial_state/encoders_projection/bias", [rnn_size], zeros_initializer())

    def __call__(self, decoder, train_mode, rnn_size, encoders):
        en_concat = concat_encoder_projection(decoder, train_mode, None, encoders)
        y = ops.linear(en_concat, decoder.var("initial_state/encoders_projection/kernel"),
                       decoder.var("initial_state/encoders_projection/bias"))
        return dropout(y, self.dropout_keep_prob, train_mode)


empty_initial_state = _Empty()
concat_encoder_projection = _Concat()


def linear_encoder_projection(dropout_keep_prob: float) -> EncoderProjection:
    """dropout(dense(concat(encoder outputs), rnn_size)) (encoder_projection.py:47-73)."""
    return _Linear(dropout_keep_prob)


class _Nematus(EncoderProjection):
    def __init__(self, dropout_keep_prob: float) -> None:
        self.dropout_keep_prob = dropout_keep_prob

    def output_size(self, rnn_size, encoders):
        return rnn_size

    @staticmethod
    def _check(encoders):
        if len(encoders) != 1:
            raise ValueError("Exactly one encoder required for this type of projection. {} given."
                             .format(len(encoders)))
        return encoders[0]

    def declare(self, decoder, rnn_size, encoders):
        encoder = self._check(encoders)
        in_size = encoder.dimension
        # orthogonal when square, otherwise the scope default (encoder_projection.py:131-134)
        init = block_orthogonal_initializer() if in_size == rnn_size else None
        decoder.declare("initial_state/encoders_projection/kernel", [in_size, rnn_size], init)
        decoder.declare("initial_state/encoders_projection/bias", [rnn_size], zeros_initializer())

    def __call__(self, decoder, train_mode, rnn_size, encoders):
        encoder = self._check(encoders)
        mask = encoder.temporal_mask
        means = (encoder.temporal_states * mask.unsqueeze(2)).sum(1) / mask.sum(1, keepdim=True)
        y = ops.linear(means.contiguous(), decoder.var("initial_state/encoders_projection/kernel"),
                       decoder.var("initial_state/encoders_projection/bias"), act="tanh")
        return dropout(y, self.dropout_keep_prob, train_mode)


def nematus_projection(dropout_keep_prob: float = 1.0) -> EncoderProjection:
    """tanh(dense(mean of the encoder's states over its unmasked positions))
    (encoder_projection.py:99-145)."""
    return _Nematus(dropout_keep_prob)
