"""Golden vectors from the reference's own `encoders/sentence_cnn_encoder.py` (`SentenceCNNEncoder`), with its
`nn/highway.py`, `nn/ortho_gru_cell.py` and `nn/utils.py` dropout, executed over the numpy TensorFlow stand-in of
tf_numpy_shim.py.

The TF ops the encoder calls that the shim lacks are restated here in numpy:
  tf.nn.conv1d     stride 1, SAME: (w-1)//2 zeros before each sequence and the rest after
  tf.nn.max_pool   NHWC, any ksize / strides, SAME: ceil(size/stride) windows, (total padding)//2 before, the
                   padding ignored by the max (the shim's own max_pool only covers the exact-division case)
  tf.nn.bias_add, tf.ceil, tf.divide, tf.cast, tf.sigmoid/tf.add/tf.subtract/tf.multiply, tf.matmul
Variables are drawn on demand by the shim and recorded under their full TF names.  Dropout is the shim's
deterministic mask (every second entry of the last axis dropped, the rest scaled by 1/keep_prob).  What this pins is
the reference's side: the padding and window offsets, which positions the convolutions cover, the order of the
concatenation, the highway arithmetic, the GRU's sequence lengths and the pooled mask.

    python tests/golden/make_sentence_cnn_golden.py   ->  tests/golden/sentence_cnn_golden.npz   (needs /root/reference)
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REFERENCE = "/root/reference"
sys.path.insert(0, HERE)
import tf_numpy_shim as shim  # noqa: E402
from make_host_golden import install_stubs  # noqa: E402

E = 5
# (tag, lengths (the first is T), segment_size, filters, highway_depth, rnn_size, keep_prob, train)
CASES = [
    # T = 12, s = 5: offset windows {0..3}, {4..8}, {9..11}; the length-5 sentence has mask [1, 1, 0] but one GRU step
    ("t12_s5", [12, 5, 9], 5, [(1, 4), (2, 3), (3, 5)], 1, 4, 1.0, False),
    ("t10_s5", [10, 7, 3], 5, [(4, 6)], 3, 3, 1.0, False),                    # T divisible by s, one filter
    ("s1", [7, 6, 2], 1, [(5, 3), (2, 2)], 1, 5, 1.0, False),                  # s = 1: no pooling
    ("s_gt_t", [4, 2, 1], 6, [(6, 3), (1, 2)], 3, 3, 1.0, False),             # s > T, a filter wider than T
    ("dropout", [9, 8, 4], 4, [(3, 4), (2, 4)], 2, 4, 0.5, True),             # deterministic dropout mask
]


def _conv1d(value, filters, stride=1, padding="SAME", name=None):
    assert stride == 1 and padding == "SAME"
    x, w = np.asarray(value, np.float64), np.asarray(filters, np.float64)
    width, length = w.shape[0], x.shape[1]
    before = (width - 1) // 2
    xp = np.pad(x, ((0, 0), (before, width - 1 - before), (0, 0)))
    out = np.zeros((x.shape[0], length, w.shape[2]))
    for j in range(width):
        out += xp[:, j:j + length] @ w[j]
    return shim.t(out, np.float32)


def _max_pool(value, ksize, strides, padding, name=None):
    assert padding == "SAME" and ksize[0] == strides[0] == 1 and ksize[3] == strides[3] == 1
    x = np.asarray(value)
    n, h, w, c = x.shape
    out_h, out_w = -(-h // strides[1]), -(-w // strides[2])
    top = max((out_h - 1) * strides[1] + ksize[1] - h, 0) // 2
    left = max((out_w - 1) * strides[2] + ksize[2] - w, 0) // 2
    out = np.zeros((n, out_h, out_w, c), x.dtype)
    for i in range(out_h):
        for j in range(out_w):
            y0, x0 = i * strides[1] - top, j * strides[2] - left
            win = x[:, max(y0, 0):min(y0 + ksize[1], h), max(x0, 0):min(x0 + ksize[2], w)]
            out[:, i, j] = win.max(axis=(1, 2))
    return shim.t(out)


def _install():
    install_stubs()
    tf = shim.install()
    tf.nn.conv1d = _conv1d
    tf.nn.max_pool = _max_pool
    tf.nn.bias_add = lambda x, b: shim.t(np.asarray(x) + np.asarray(b), np.float32)
    tf.ceil = lambda x: shim.t(np.ceil(np.asarray(x)))
    tf.divide = lambda a, b: shim.t(np.asarray(a) / b)
    tf.cast = lambda x, dtype: shim.t(np.asarray(x).astype(dtype))
    tf.add = lambda a, b, name=None: shim.t(np.asarray(a) + np.asarray(b), np.float32)
    tf.subtract = lambda a, b, name=None: shim.t(a - np.asarray(b), np.float32)
    tf.multiply = lambda a, b, name=None: shim.t(np.asarray(a) * np.asarray(b), np.float32)
    tf.sigmoid = lambda x, name=None: shim.t(1.0 / (1.0 + np.exp(-np.asarray(x, np.float32))), np.float32)
    tf.nn.relu = lambda x, name=None: shim.t(np.maximum(np.asarray(x), 0))
    tf.matmul = lambda a, b: shim.t(np.asarray(a) @ np.asarray(b), np.float32)
    tf.variance_scaling_initializer = lambda *a, **k: None
    tf.constant_initializer = lambda *a, **k: None
    sys.path.insert(0, REFERENCE)
    return tf


def main():
    _install()
    from neuralmonkey.encoders.sentence_cnn_encoder import SentenceCNNEncoder
    from neuralmonkey.model.stateful import TemporalStateful

    class Inputs(TemporalStateful):
        def __init__(self, states, mask):
            self._s, self._m = shim.t(states, np.float32), shim.t(mask, np.float32)

        @property
        def temporal_states(self):
            return self._s

        @property
        def temporal_mask(self):
            return self._m

        @property
        def dimension(self):
            return E

    rng = np.random.RandomState(23)
    out = {}
    for tag, lengths, s, filters, depth, rnn, keep, train in CASES:
        t = lengths[0]
        mask = (np.arange(t)[None, :] < np.array(lengths)[:, None]).astype(np.float32)
        states = (rng.randn(len(lengths), t, E) * mask[:, :, None]).astype(np.float32)
        shim.VARIABLES.clear()
        shim.AUTO[0] = np.random.RandomState(rng.randint(1 << 30))
        enc = object.__new__(SentenceCNNEncoder)
        enc.__dict__.update(dict(
            _variable_scope=shim.VarScope("sentence_encoder"), _reuse=None, _name="sentence_encoder",
            input_sequence=Inputs(states, mask), segment_size=s, highway_depth=depth, rnn_size=rnn,
            filters=filters, dropout_keep_prob=keep, use_noisy_activations=False, train_mode=train,
            batch_size=len(lengths)))
        key = tag + "_"
        out[key + "states"], out[key + "mask"] = states, mask
        out[key + "config"] = np.array([s, depth, rnn, keep, float(train)])
        out[key + "filters"] = np.array(filters)
        with shim._scope_cm("sentence_encoder"):
            for name in ("cnn_encoded", "highway_layer", "temporal_states", "output", "temporal_mask"):
                out[key + name] = np.asarray(getattr(enc, name), np.float64)
        for name in sorted(shim.VARIABLES):
            out[key + "var:" + name] = np.asarray(shim.VARIABLES[name])
    path = os.path.join(HERE, "sentence_cnn_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays")


if __name__ == "__main__":
    main()
