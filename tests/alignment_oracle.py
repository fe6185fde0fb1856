"""Supervised attention restated in torch, for tests/test_host_alignment.py and tests/test_gpu_alignment.py.

* `bahdanau_attention_energies` and `alignment_xent` are CPU stand-ins of the two ops of the same names (the ops
  `tests/cpu_ops.py` does not cover); in fp64 they are also the oracle of the kernels.
* `build` makes a SentenceEncoder + Attention + Decoder + WordAlignmentDecoder with a CrossEntropyTrainer over both;
  `oracle_losses` computes the decoder's training loss and the alignment loss of the same batch with
  `oracle.nm_oracle` from a dict of parameters (fp64 with requires_grad for gradients).
"""
from typing import Dict, Optional

import numpy as np
import torch

from oracle import nm_oracle as O

STAND_INS = ("bahdanau_attention_energies", "alignment_xent")


def bahdanau_attention_energies(keys, values, mask, qproj, v, bias):
    energies = (v * torch.tanh(keys.unsqueeze(1) + qproj.unsqueeze(2))).sum(-1) + bias
    weights = torch.softmax(energies, dim=-1)
    if mask is not None:
        weights = weights * mask.unsqueeze(1)
        weights = weights / (weights.sum(-1, keepdim=True) + 1e-8)
    return torch.einsum("bqt,btc->bqc", weights, values), weights, energies


def alignment_xent(energies, target, pad):
    """sum_{b,q} pad * sum_t target * (logsumexp_t e - e): tf.nn.softmax_cross_entropy_with_logits times the
    padding, summed (word_alignment_decoder.py:100-108)."""
    xent = (target * (torch.logsumexp(energies, -1, keepdim=True) - energies)).sum(-1)
    return (xent * pad).sum()


def crop(ref: torch.Tensor, steps: int, width: int) -> torch.Tensor:
    """The fed [B, rows, cols] alignments as the [B, steps, width] target: extra rows / columns dropped, missing
    ones zero."""
    out = ref.new_zeros(ref.shape[0], steps, width)
    rows, cols = min(steps, ref.shape[1]), min(width, ref.shape[2])
    out[:, :rows, :cols] = ref[:, :rows, :cols]
    return out


# pylint: disable=too-many-arguments,too-many-locals
def build(vs=40, vt=50, es=11, he=7, et=9, hd=8, maxout=9, max_len=8, rnn_cell="GRU", conditional_gru=False,
          weights=(1., 1e-3), lr=1e-4, clip=None, use_cuda_graph=False, dropout_keep_prob=1.0):
    """The shape family of the reference's tests/alignment.ini.  Returns a dict of the parts and the arena."""
    from neuralmonkey_b200 import runtime, tf
    from neuralmonkey_b200.attention import Attention
    from neuralmonkey_b200.decoders import Decoder
    from neuralmonkey_b200.decoders.output_projection import maxout_output
    from neuralmonkey_b200.decoders.word_alignment_decoder import WordAlignmentDecoder
    from neuralmonkey_b200.encoders import SentenceEncoder
    from neuralmonkey_b200.trainers import CrossEntropyTrainer
    from neuralmonkey_b200.vocabulary import Vocabulary

    runtime.reset()
    enc = SentenceEncoder(name="sentence_encoder", vocabulary=Vocabulary(["s{}".format(i) for i in range(vs - 4)]),
                          data_id="source", embedding_size=es, rnn_size=he, max_input_len=max_len)
    att = Attention(name="attention", encoder=enc)
    dec = Decoder(encoders=[enc], vocabulary=Vocabulary(["t{}".format(i) for i in range(vt - 4)]),
                  data_id="target", name="decoder", max_output_len=max_len, rnn_size=hd, embedding_size=et,
                  attentions=[att], output_projection=maxout_output(maxout) if maxout else None, rnn_cell=rnn_cell,
                  conditional_gru=conditional_gru, dropout_keep_prob=dropout_keep_prob)
    ali = WordAlignmentDecoder(encoder=enc, decoder=dec, data_id="ali", name="alignment_decoder")
    decoders = [dec, ali] if weights[1] is not None else [dec]
    trainer = CrossEntropyTrainer(decoders=decoders, decoder_weights=list(weights[:len(decoders)]),
                                  clip_norm=clip, optimizer=tf.AdamOptimizer(learning_rate=lr),
                                  use_cuda_graph=use_cuda_graph)
    for part in trainer.parameterizeds:
        part.ensure_declared()
    runtime.arena().finalize(runtime.device())
    return {"enc": enc, "att": att, "dec": dec, "ali": ali, "trainer": trainer, "arena": runtime.arena(),
            "spec": O.RNNDecoderSpec("decoder", "attention", max_len, "maxout" if maxout else "tanh",
                                     rnn_cell=rnn_cell, conditional_gru=conditional_gru)}


def feed(model, src: torch.Tensor, tgt: Optional[torch.Tensor], alignment: Optional[np.ndarray], train: bool):
    """src [B,Tx] / tgt [B,Ty] int64 ids (tgt with </s>), alignment [B, rows, cols] float32 or None."""
    bsz = src.shape[0]
    model["enc"].input_sequence.feed_ids([src], train=train)
    for part in (model["enc"], model["att"]):
        part.reset_batch()
        part.train_mode = train
        part.batch_size = bsz
    model["dec"].feed_ids(tgt, bsz, train=train)
    model["ali"].feed_dict(FakeDataset(bsz, {} if alignment is None else {"ali": alignment}), train=train)


class FakeDataset:
    """What ModelPart.feed_dict reads of a dataset: its length and its series."""

    def __init__(self, size: int, series: Dict[str, np.ndarray]) -> None:
        self._size = size
        self._series = series

    def __len__(self) -> int:
        return self._size

    def maybe_get_series(self, name: str):
        return iter(self._series[name]) if name in self._series else None


def oracle_losses(p, spec, src, tgt, alignment: Optional[torch.Tensor]):
    """(decoder train_loss, alignment loss) of one batch.  p: parameters by name; the alignment loss reads the
    energies of every teacher-forced step's attention evaluation."""
    enc = O.sentence_encoder(p, "sentence_encoder", src)
    states, mask = enc["temporal_states"], enc["temporal_mask"]
    hidden = O.bahdanau_precompute(p, "attention", states)
    energies = []

    def attend(query):
        y = query @ p["attention/Attention/attn_query_projection"] + p["attention/attn_projection_bias"]
        ctx, weights, e = bahdanau_attention_energies(hidden, states, mask, y.unsqueeze(1),
                                                      p["attention/attn_similarity_v"], p["attention/attn_bias"])
        energies.append(e[:, 0])
        return ctx[:, 0], weights[:, 0]

    odec = O.decoder_train(p, spec, enc, tgt.t(), attend=[attend])
    e = torch.stack(energies, 1)                                # [B, steps, Tx]
    pad = odec["train_mask"].t()[:, :e.shape[1]]
    ref = torch.zeros_like(e) if alignment is None else crop(alignment.to(e.dtype), e.shape[1], e.shape[2])
    return odec["train_loss"], alignment_xent(e, ref, pad), e
