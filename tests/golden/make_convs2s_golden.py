"""Golden vectors from the reference's own convolutional seq2seq encoder, `encoders/facebook_conv.py`
(SentenceEncoder), executed over the numpy TensorFlow stand-in of tf_numpy_shim.py.

The TF ops the module calls that the shim lacks or stubs are restated here in numpy: tf.nn.conv1d (SAME, stride 1:
(k-1)//2 zeros before, the rest after), tf.split, tf.reduce_max, tf.expand_dims and tf.random_normal_initializer.
Variables are drawn on demand by the shim and recorded under their full TF names, so what is pinned is the
reference's side: which layers exist, their names and shapes, where the position table and the residuals enter,
the order of the GLU halves and the max over every position.  The embedded input sequence is fed directly, zero at
the padded positions as the reference's EmbeddedSequence makes it.

    python tests/golden/make_convs2s_golden.py   ->  tests/golden/convs2s_golden.npz   (needs /root/reference)
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REFERENCE = "/root/reference"
sys.path.insert(0, HERE)
import tf_numpy_shim as shim  # noqa: E402
from make_host_golden import install_stubs  # noqa: E402

# tag: (batch lengths, T, embedding size, max_length, conv_features, encoder_layers, kernel_width)
CASES = {
    "padded": ([6, 4, 2], 6, 3, 8, 4, 3, 3),      # a padded batch, 3 layers
    "t1": ([1, 1], 1, 2, 4, 3, 1, 5),             # T = 1
    "short": ([3, 2], 3, 4, 5, 5, 1, 5),          # T < k
    "even": ([5, 3], 5, 3, 6, 6, 3, 4),           # an even k: the extra zero after
    "bpe": ([10, 7, 4, 9], 10, 11, 10, 10, 2, 5), # tests/bpe.ini's encoder (kernel_width left at its default)
}


def _conv1d(value, filters, stride, padding, name=None):
    assert stride == 1 and padding == "SAME"
    x, w = np.asarray(value, np.float64), np.asarray(filters, np.float64)
    width, length = w.shape[0], x.shape[1]
    before = (width - 1) // 2
    padded = np.pad(x, ((0, 0), (before, width - 1 - before), (0, 0)))
    out = np.zeros((x.shape[0], length, w.shape[2]))
    for j in range(width):
        out += padded[:, j:j + length] @ w[j]
    return shim.t(out, np.float32)


def _random_normal_initializer(mean=0.0, stddev=1.0, **kwargs):
    """A marker the patched get_variable below draws from (the shim's own draw ignores initializers)."""
    return ("normal", mean, stddev)


def _install():
    install_stubs()
    tf = shim.install()
    tf.nn.conv1d = _conv1d
    tf.split = lambda value, num, axis=0: [shim.t(p, np.float32) for p in np.split(np.asarray(value), num, axis=axis)]
    tf.reduce_max = lambda x, axis=None: shim.t(np.max(np.asarray(x), axis=axis), np.float32)
    tf.expand_dims = lambda x, axis: shim.t(np.expand_dims(np.asarray(x), axis), np.float32)
    tf.random_normal_initializer = _random_normal_initializer
    shim_get_variable = tf.get_variable

    def get_variable(name=None, shape=None, dtype=None, initializer=None, **kwargs):
        # the shim draws every variable uniformly; a normal initializer is honoured, so the filters have TF's scale
        full = shim._full_name(name)
        if isinstance(initializer, tuple) and full not in shim.VARIABLES:
            shim.VARIABLES[full] = shim.AUTO[0].normal(initializer[1], initializer[2], size=shape).astype(np.float32)
        return shim_get_variable(name, shape=shape, dtype=dtype, initializer=initializer, **kwargs)
    tf.get_variable = get_variable
    # tf_utils.get_variable asks the current experiment for an initializer override; there is none here, and the
    # real neuralmonkey.experiment would import the whole toolkit
    experiment = types.ModuleType("neuralmonkey.experiment")
    current = types.SimpleNamespace(get_initializer=lambda name, default: default)
    experiment.Experiment = types.SimpleNamespace(get_current=lambda: current)
    sys.modules["neuralmonkey.experiment"] = experiment
    sys.path.insert(0, REFERENCE)
    return tf


def _part(cls, name, **attrs):
    """A reference model part without its constructor (no graph, no placeholders)."""
    obj = object.__new__(cls)
    obj.__dict__.update(dict(_variable_scope=shim.VarScope(name), _reuse=None, _name=name, train_mode=False))
    obj.__dict__.update(attrs)
    return obj


def main():
    _install()
    from neuralmonkey.encoders.facebook_conv import SentenceEncoder
    from neuralmonkey.model.stateful import TemporalStateful

    class Sequence(TemporalStateful):
        def __init__(self, states, mask, max_length, emb):
            self._s, self._m = shim.t(states, np.float32), shim.t(mask, np.float32)
            self.max_length, self.embedding_sizes = max_length, [emb]

        @property
        def temporal_states(self):
            return self._s

        @property
        def temporal_mask(self):
            return self._m

    rng = np.random.RandomState(5)
    out = {}
    for tag, (lengths, length, emb, max_len, feats, layers, width) in CASES.items():
        mask = (np.arange(length)[None, :] < np.array(lengths)[:, None]).astype(np.float32)
        states = (rng.randn(len(lengths), length, emb) * mask[:, :, None]).astype(np.float32)
        shim.VARIABLES.clear()
        shim.AUTO[0] = np.random.RandomState(rng.randint(1 << 30))
        enc = _part(SentenceEncoder, tag, input_sequence=Sequence(states, mask, max_len, emb),
                    conv_features=feats, encoder_layers=layers, kernel_width=width, dropout_keep_prob=1.0,
                    max_input_length=max_len)
        out[tag + "_states"], out[tag + "_mask"] = states, mask
        out[tag + "_temporal_states"] = np.asarray(enc.temporal_states, np.float32)
        out[tag + "_output"] = np.asarray(enc.output, np.float32)
        out[tag + "_temporal_mask"] = np.asarray(enc.temporal_mask, np.float32)
        out[tag + "_variable_names"] = np.array(sorted(shim.VARIABLES))
        for name in sorted(shim.VARIABLES):
            out[tag + "_var:" + name] = np.asarray(shim.VARIABLES[name], np.float32)
    np.savez_compressed(os.path.join(HERE, "convs2s_golden.npz"), **out)


if __name__ == "__main__":
    main()
