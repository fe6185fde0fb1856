"""Golden vectors from the reference's own `decoders/ctc_decoder.py` (`CTCDecoder`), executed over the numpy
TensorFlow stand-in of tf_numpy_shim.py with the CTC operations it calls backed by the fp64 oracle of
tests/ctc_oracle.py:

  feed_dict        pad_batch(sentences, max_length) fed as `target_tokens`
  train_targets    tf.where(params != PAD) -> SparseTensor (label extraction, row-major order)
  logits           the 1x1 conv2d projection with `state_to_word_W` [D, V+1] / `state_to_word_b`, time-major
  cost             tf.nn.ctc_loss(preprocess_collapse_repeated=merge_repeated_targets,
                   ignore_longer_outputs_than_inputs=True, ctc_merge_repeated=merge_repeated_outputs), summed
  decoded          tf.nn.ctc_greedy_decoder -> sparse_transpose -> sparse_tensor_to_dense(default END)

What this pins is the reference's side of those calls (blank last, V+1 classes, sum reduction, the label
extraction, the time-major transpose, END padding, variable names); the CTC arithmetic itself is the oracle's.

    python tests/golden/make_ctc_golden.py   ->  tests/golden/ctc_golden.npz
"""
import collections
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import tf_numpy_shim as shim  # noqa: E402
from make_host_golden import install_stubs  # noqa: E402
from tests import ctc_oracle as CO  # noqa: E402

SparseTensor = collections.namedtuple("SparseTensor", ["indices", "values", "dense_shape"])
SPECIAL = ["<pad>", "<s>", "</s>", "<unk>"]
WORDS = ["yes", "no", "maybe"]
SENTENCES = [["yes", "no", "no", "yes", "maybe"], ["no"], [], ["maybe", "maybe", "unknown-word"],
             ["yes", "yes", "yes"]]
# (tag, max_length, merge_repeated_targets, merge_repeated_outputs)
CASES = [("default", None, False, True), ("merge_targets", None, True, True), ("no_merge_out", 4, False, False)]


class _Vocabulary:
    """The part of the reference's Vocabulary the decoder uses: its size and the string -> index lookup table
    (unknown words -> <unk>)."""

    def __init__(self, words):
        self.words = SPECIAL + list(words)

    def __len__(self):
        return len(self.words)

    def strings_to_indices(self, sentences):
        index = {w: i for i, w in enumerate(self.words)}
        return shim.t(np.array([[index.get(w, 3) for w in s] for s in np.asarray(sentences)], np.int64))


class _Dataset:
    """The part of the reference's Dataset that feed_dict reads."""

    def __len__(self):
        return len(SENTENCES)

    def maybe_get_series(self, _series_id):
        return iter(SENTENCES)


def _labels(sparse, batch):
    rows = [[] for _ in range(batch)]
    for (b, _), v in zip(np.asarray(sparse.indices), np.asarray(sparse.values)):
        rows[int(b)].append(int(v))
    return rows


def _ctc_loss(labels, inputs, sequence_length, preprocess_collapse_repeated=False,
              ctc_merge_repeated=True, ignore_longer_outputs_than_inputs=False, time_major=True):
    assert ignore_longer_outputs_than_inputs and time_major
    logits = torch.from_numpy(np.transpose(np.asarray(inputs, np.float64), (1, 0, 2)))
    rows = _labels(labels, logits.shape[0])
    if preprocess_collapse_repeated:
        rows = [[x for i, x in enumerate(r) if i == 0 or x != r[i - 1]] for r in rows]
    width = max(1, max(len(r) for r in rows))
    padded = [r + [0] * (width - len(r)) for r in rows]
    loss = CO.ctc_loss(logits, np.asarray(sequence_length), padded, [len(r) for r in rows], ctc_merge_repeated)
    return shim.t(loss.numpy().astype(np.float32))


def _ctc_greedy_decoder(inputs, sequence_length, merge_repeated=True):
    logits = torch.from_numpy(np.transpose(np.asarray(inputs, np.float32), (1, 0, 2)))
    ids, lengths = CO.ctc_greedy_decode(logits, np.asarray(sequence_length), merge_repeated)
    indices = [(b, k) for b in range(len(lengths)) for k in range(int(lengths[b]))]
    values = [int(ids[b, k]) for b, k in indices]
    sparse = SparseTensor(np.array(indices, np.int64).reshape(-1, 2), np.array(values, np.int64),
                          np.array([len(lengths), int(lengths.max()) if len(lengths) else 0], np.int64))
    return [sparse], None


def _sparse_transpose(sp):
    order = sorted(range(len(sp.values)), key=lambda i: (sp.indices[i][1], sp.indices[i][0]))
    return SparseTensor(np.array([[sp.indices[i][1], sp.indices[i][0]] for i in order], np.int64).reshape(-1, 2),
                        np.asarray(sp.values)[order], np.asarray(sp.dense_shape)[::-1].copy())


def _sparse_tensor_to_dense(sp, default_value=0):
    dense = np.full([int(d) for d in sp.dense_shape], default_value, np.int64)
    for (i, j), v in zip(np.asarray(sp.indices), np.asarray(sp.values)):
        dense[i, j] = v
    return shim.t(dense)


def _where(cond, a=None, b=None):
    if a is None:           # tf.where(cond): the coordinates of the true entries, row-major
        return shim.t(np.argwhere(np.asarray(cond)).astype(np.int64))
    return shim.t(np.where(np.asarray(cond), np.asarray(a), np.asarray(b)))


def _cast(x, dtype):
    if isinstance(x, SparseTensor):
        return SparseTensor(x.indices, np.asarray(x.values).astype(dtype), x.dense_shape)
    return shim.t(np.asarray(x).astype(dtype))


def main():
    install_stubs()
    tf = shim.install()
    tf.where = _where
    tf.shape = lambda x, out_type=None: np.array(np.asarray(x).shape, out_type or np.int32)
    tf.SparseTensor = SparseTensor
    tf.cast = _cast
    tf.sparse_transpose = _sparse_transpose
    tf.sparse_tensor_to_dense = _sparse_tensor_to_dense
    tf.random_uniform_initializer = lambda *a, **k: None
    tf.nn.ctc_loss = _ctc_loss
    tf.nn.ctc_greedy_decoder = _ctc_greedy_decoder
    from neuralmonkey.decoders.ctc_decoder import CTCDecoder
    from neuralmonkey.vocabulary import pad_batch

    rng = np.random.RandomState(17)
    batch, t_max, dim = len(SENTENCES), 9, 6
    states = np.asarray(rng.randn(batch, t_max, dim), np.float32)
    lengths = np.array([9, 4, 3, 7, 2], np.int32)       # sentence 4 has more labels than frames: ignored
    vocab = _Vocabulary(WORDS)
    out = {"states": states, "lengths": lengths, "words": np.array(WORDS),
           "sentences": np.array([" ".join(s) for s in SENTENCES])}
    for tag, max_length, merge_targets, merge_outputs in CASES:
        shim.VARIABLES.clear()
        w = np.asarray(rng.uniform(-0.5, 0.5, (dim, len(vocab) + 1)), np.float32)
        bias = np.asarray(rng.randn(len(vocab) + 1) * 0.1, np.float32)
        shim.VARIABLES["decoder/state_to_word_W"], shim.VARIABLES["decoder/state_to_word_b"] = w, bias
        dec = object.__new__(CTCDecoder)
        dec.__dict__.update(dict(
            _variable_scope=shim.VarScope("decoder"), _reuse=None, _name="decoder",
            encoder=types.SimpleNamespace(temporal_states=shim.t(states), lengths=shim.t(lengths)),
            vocabulary=vocab, data_id="target", max_length=max_length, merge_repeated_targets=merge_targets,
            merge_repeated_outputs=merge_outputs, beam_width=1, train_mode="train_mode", batch_size="batch_size",
            _dataset={"target": "target_tokens"}))
        fd = dec.feed_dict(_Dataset(), train=True)
        padded = fd["target_tokens"]                     # what the reference feeds into its placeholder
        assert padded == pad_batch(list(SENTENCES), max_length)
        dec.__dict__["_target_tokens_cached_placeholder"] = np.array(padded)
        sparse = dec.train_targets
        key = tag + "_"
        out[key + "W"], out[key + "b"] = w, bias
        out[key + "padded"] = np.array(padded)
        out[key + "label_indices"] = np.asarray(sparse.indices)
        out[key + "label_values"] = np.asarray(sparse.values)
        out[key + "label_shape"] = np.asarray(sparse.dense_shape)
        out[key + "logits"] = np.asarray(dec.logits)
        out[key + "cost"] = np.asarray(dec.cost)
        out[key + "decoded"] = np.asarray(dec.decoded)
        out[key + "variables"] = np.array(sorted(shim.VARIABLES))
    np.savez(os.path.join(HERE, "ctc_golden.npz"), **out)
    print("wrote", os.path.join(HERE, "ctc_golden.npz"), sorted(out))


if __name__ == "__main__":
    main()
