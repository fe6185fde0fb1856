"""Golden vectors from the reference's own sentence classification and regression code, executed over the numpy
TensorFlow stand-in of tf_numpy_shim.py: `encoders/pooling.py` (SequenceMaxPooling, SequenceAveragePooling),
`encoders/attentive.py` (AttentiveEncoder), `encoders/sequence_cnn_encoder.py` (SequenceCNNEncoder),
`model/gradient_reversal.py` (the three views), `nn/mlp.py` (MultilayerPerceptron), `decoders/classifier.py`
(Classifier), `decoders/sequence_regressor.py` (SequenceRegressor), and the `collect_results` of
`runners/logits_runner.py` and `runners/regression_runner.py`.

The TF ops those modules call that the shim lacks are restated here in numpy: tf.nn.conv1d (VALID, stride 1),
tf.nn.bias_add, tf.reduce_max, tf.matmul(transpose_a=True), tf.nn.sparse_softmax_cross_entropy_with_logits,
tf.assert_greater (checked), and no-op summaries.  Variables are drawn on demand by the shim and recorded under their
full TF names, so what is pinned is the reference's side: which layers exist, their names and shapes, the order of
the concatenations, where the mask and the 1e-15 padding enter, the renormalisation of the attention weights,
the regression target broadcast and the runners' text formatting.  Sentence and label ids are fed directly
(the vocabulary's TF lookup tables do not exist here).

    python tests/golden/make_classifier_golden.py   ->  tests/golden/classifier_golden.npz   (needs /root/reference)
"""
import contextlib
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REFERENCE = "/root/reference"
sys.path.insert(0, HERE)
import tf_numpy_shim as shim  # noqa: E402
from make_host_golden import install_stubs  # noqa: E402

B, T, D = 4, 6, 5
LENGTHS = [6, 3, 1, 4]          # a padded batch; sentence 1 is all negative, sentence 2 has one position
VOCAB = 9                       # word ids 0..8, 0 = <pad>
E = 4
CNN_FILTERS = [(2, 3), (3, 2), (6, 2)]      # the last one as long as the batch: T == w
CLASSES = 5


def _conv1d(value, filters, stride=1, padding="VALID", name=None):
    assert stride == 1 and padding == "VALID"
    x, w = np.asarray(value, np.float64), np.asarray(filters, np.float64)
    width = w.shape[0]
    length = x.shape[1] - width + 1
    assert length >= 1
    out = np.zeros((x.shape[0], length, w.shape[2]))
    for j in range(width):
        out += x[:, j:j + length] @ w[j]
    return shim.t(out, np.float32)


def _sparse_xent(logits=None, labels=None, **kwargs):
    z = np.asarray(logits, np.float64)
    z = z - z.max(axis=-1, keepdims=True)
    lse = np.log(np.exp(z).sum(axis=-1))
    return shim.t(lse - z[np.arange(z.shape[0]), np.asarray(labels)], np.float32)


def _assert_greater(x, y, **kwargs):
    assert float(np.asarray(x)) > y, "assert_greater failed"


def _matmul(a, b, transpose_a=False, transpose_b=False):
    a, b = np.asarray(a), np.asarray(b)
    if transpose_a:
        a = np.swapaxes(a, -1, -2)
    if transpose_b:
        b = np.swapaxes(b, -1, -2)
    return shim.t(np.matmul(a, b))


def _install():
    install_stubs()
    tf = shim.install()
    tf.nn.conv1d = _conv1d
    tf.nn.bias_add = lambda x, b: shim.t(np.asarray(x) + np.asarray(b))
    tf.reduce_max = lambda x, axis=None: shim.t(np.max(np.asarray(x), axis=axis))
    tf.matmul = _matmul
    tf.nn.sparse_softmax_cross_entropy_with_logits = _sparse_xent
    tf.assert_greater = _assert_greater
    tf.variance_scaling_initializer = lambda *a, **k: None
    tf.summary = types.SimpleNamespace(scalar=lambda *a, **k: None)
    tf.negative = lambda x: shim.t(-np.asarray(x))
    # model/gradient_reversal.py registers a gradient and overrides Identity's in the current graph
    framework = types.ModuleType("tensorflow.python.framework")
    framework.ops = types.SimpleNamespace(RegisterGradient=lambda name: (lambda fn: fn))
    sys.modules["tensorflow.python"] = types.ModuleType("tensorflow.python")
    sys.modules["tensorflow.python.framework"] = framework
    experiment = types.ModuleType("neuralmonkey.experiment")
    graph = types.SimpleNamespace(gradient_override_map=lambda mapping: contextlib.nullcontext())
    current = types.SimpleNamespace(graph=graph, get_initializer=lambda name, default: default)
    experiment.Experiment = types.SimpleNamespace(get_current=lambda: current)
    sys.modules["neuralmonkey.experiment"] = experiment
    sys.path.insert(0, REFERENCE)
    return tf


def _named(value, name):
    """A shim tensor with the `.name` a graph tensor has (the reversal views name their gradient after it)."""
    out = shim.t(value, np.float32)
    out.name = name
    return out


def _part(cls, name, **attrs):
    """A reference model part without its constructor (no graph, no placeholders)."""
    obj = object.__new__(cls)
    obj.__dict__.update(dict(_variable_scope=shim.VarScope(name), _reuse=None, _name=name, train_mode=False))
    obj.__dict__.update(attrs)
    return obj


def main():
    tf = _install()
    from neuralmonkey.model.stateful import Stateful, TemporalStateful, SpatialStateful
    from neuralmonkey.encoders.pooling import SequenceMaxPooling, SequenceAveragePooling
    from neuralmonkey.encoders.attentive import AttentiveEncoder
    from neuralmonkey.encoders.sequence_cnn_encoder import SequenceCNNEncoder
    from neuralmonkey.model.gradient_reversal import StatefulView, TemporalStatefulView, SpatialStatefulView
    from neuralmonkey.nn.mlp import MultilayerPerceptron
    from neuralmonkey.decoders.classifier import Classifier
    from neuralmonkey.decoders.sequence_regressor import SequenceRegressor
    from neuralmonkey.runners.logits_runner import LogitsRunner
    from neuralmonkey.runners.regression_runner import RegressionRunner

    rng = np.random.RandomState(11)
    out = {}
    mask = (np.arange(T)[None, :] < np.array(LENGTHS)[:, None]).astype(np.float32)
    states = rng.randn(B, T, D).astype(np.float32)
    states[1] = -np.abs(states[1]) - 0.1
    states[3, 1] = states[3, 0]                 # an exact tie inside sentence 3
    out.update(states=states, mask=mask)

    class Sequence(TemporalStateful):
        def __init__(self, s, m):
            self._s, self._m = _named(s, "states:0"), _named(m, "mask:0")

        @property
        def temporal_states(self):
            return self._s

        @property
        def temporal_mask(self):
            return self._m

    class Vector(Stateful):
        def __init__(self, v):
            self._v = _named(v, "output:0")

        @property
        def output(self):
            return self._v

    class Map(SpatialStateful):
        @property
        def spatial_states(self):
            return _named(states[:, :, :, None], "map:0")

        @property
        def spatial_mask(self):
            return shim.t(mask[:, :, None], np.float32)

    seq = Sequence(states, mask)

    # -- pooling ----------------------------------------------------------------------------------------------------
    shim.AUTO[0] = np.random.RandomState(1)
    out["maxpool_output"] = np.asarray(_part(SequenceMaxPooling, "maxpool", input_sequence=seq).output)
    out["avgpool_output"] = np.asarray(_part(SequenceAveragePooling, "avgpool", input_sequence=seq).output)

    # -- gradient reversal views: identity forward ------------------------------------------------------------------
    out["view_output"] = np.asarray(StatefulView(Vector(states[:, 0])).output)
    tview = TemporalStatefulView(seq)
    out["tview_states"], out["tview_mask"] = np.asarray(tview.temporal_states), np.asarray(tview.temporal_mask)
    sview = SpatialStatefulView(Map())
    out["sview_states"], out["sview_mask"] = np.asarray(sview.spatial_states), np.asarray(sview.spatial_mask)
    out["view_dependencies"] = np.array(StatefulView(Vector(states[:, 0])).dependencies)

    # -- AttentiveEncoder, with and without the projections ----------------------------------------------------------
    for tag, proj, size in (("att_plain", None, None), ("att_proj", 3, 7)):
        shim.VARIABLES.clear()
        shim.AUTO[0] = np.random.RandomState(rng.randint(1 << 30))
        att = _part(AttentiveEncoder, tag, input_sequence=seq, hidden_size=4, num_heads=3, output_size=size,
                    state_proj_size=proj, dropout_keep_prob=1.0)
        out[tag + "_weights"] = np.asarray(att.attention_weights)
        out[tag + "_temporal_states"] = np.asarray(att.temporal_states)
        out[tag + "_temporal_mask"] = np.asarray(att.temporal_mask)
        out[tag + "_output"] = np.asarray(att.output)
        out[tag + "_variable_names"] = np.array(sorted(shim.VARIABLES))
        for name in sorted(shim.VARIABLES):
            out[tag + "_var:" + name] = np.asarray(shim.VARIABLES[name])

    # -- SequenceCNNEncoder over a padded batch (identical <pad> windows) ---------------------------------------------
    ids = rng.randint(1, VOCAB, size=(B, T))
    ids[np.arange(T)[None, :] >= np.array(LENGTHS)[:, None]] = 0
    out["cnn_ids"] = ids

    class CNN(SequenceCNNEncoder):
        inputs = property(lambda self: shim.t(ids, np.int64))

    shim.VARIABLES.clear()
    shim.AUTO[0] = np.random.RandomState(rng.randint(1 << 30))
    cnn = _part(CNN, "cnn", vocabulary=list(range(VOCAB)), data_id="source", max_input_len=None, embedding_size=E,
                dropout_keep_prob=1.0, filters=CNN_FILTERS)
    out["cnn_output"] = np.asarray(cnn.output)
    out["cnn_variable_names"] = np.array(sorted(shim.VARIABLES))
    for name in sorted(shim.VARIABLES):
        out["cnn_var:" + name] = np.asarray(shim.VARIABLES[name])

    # -- MultilayerPerceptron and Classifier ------------------------------------------------------------------------
    class Labels(list):
        pass

    labels = rng.randint(0, CLASSES, size=B)
    out["labels"] = labels
    feats = [rng.randn(B, 3).astype(np.float32), rng.randn(B, 4).astype(np.float32)]
    out["features_0"], out["features_1"] = feats

    class Clf(Classifier):
        gt_inputs = property(lambda self: shim.t(labels, np.int64))

    for tag, layers in (("clf_layers", [6, 5]), ("clf_nolayers", [])):
        shim.VARIABLES.clear()
        shim.AUTO[0] = np.random.RandomState(rng.randint(1 << 30))
        clf = _part(Clf, tag, encoders=[Vector(f) for f in feats], vocabulary=Labels(range(CLASSES)),
                    data_id="label", layers=layers, activation_fn=tf.nn.relu, dropout_keep_prob=1.0,
                    max_output_len=1)
        out[tag + "_logits"] = np.asarray(clf.decoded_logits)
        out[tag + "_decoded"] = np.asarray(clf.decoded_seq)
        out[tag + "_logprobs"] = np.asarray(clf.runtime_logprobs)
        out[tag + "_loss"] = np.asarray(clf.loss_with_gt_ins)
        out[tag + "_variable_names"] = np.array(sorted(shim.VARIABLES))
        for name in sorted(shim.VARIABLES):
            out[tag + "_var:" + name] = np.asarray(shim.VARIABLES[name])
    # the perceptron alone, outside any part's scope
    shim.VARIABLES.clear()
    shim.AUTO[0] = np.random.RandomState(rng.randint(1 << 30))
    mlp = MultilayerPerceptron(shim.t(feats[0]), [4], 1.0, CLASSES, train_mode=False)
    out["mlp_logits"], out["mlp_classification"] = np.asarray(mlp.logits), np.asarray(mlp.classification)
    out["mlp_variable_names"] = np.array(sorted(shim.VARIABLES))
    for name in sorted(shim.VARIABLES):
        out["mlp_var:" + name] = np.asarray(shim.VARIABLES[name])

    # -- SequenceRegressor --------------------------------------------------------------------------------------------
    targets = rng.randn(B).astype(np.float32)
    out["reg_targets"] = targets

    class Reg(SequenceRegressor):
        train_inputs = property(lambda self: shim.t(targets, np.float32))

    for tag, layers, dim in (("reg_layers", [6, 5], 1), ("reg_nolayers", [], 3)):
        shim.VARIABLES.clear()
        shim.AUTO[0] = np.random.RandomState(rng.randint(1 << 30))
        reg = _part(Reg, tag, encoders=[Vector(f) for f in feats], data_id="value", max_output_len=1,
                    dimension=dim, _layers=layers, _activation_fn=tf.nn.relu, _dropout_keep_prob=1.0)
        out[tag + "_predictions"] = np.asarray(reg.predictions)
        out[tag + "_cost"] = np.asarray(reg.cost)
        out[tag + "_variable_names"] = np.array(sorted(shim.VARIABLES))
        for name in sorted(shim.VARIABLES):
            out[tag + "_var:" + name] = np.asarray(shim.VARIABLES[name])

    # -- the runners' collect_results ------------------------------------------------------------------------------
    logits = rng.randn(1, B, CLASSES).astype(np.float32)
    out["runner_logits"] = logits
    for normalize in (True, False):
        for pick in (None, 0, 3):
            exe = object.__new__(LogitsRunner.Executable)
            got = {}
            exe._executor = types.SimpleNamespace(normalize=normalize, pick_index=pick)
            exe.set_runner_result = lambda outputs, losses: got.update(outputs=outputs, losses=losses)
            exe.collect_results([{"logits": logits, "train_loss": 1.25, "runtime_loss": 2.5}])
            key = "logits_runner_{}_{}".format(int(normalize), "none" if pick is None else pick)
            out[key] = np.array(["\n".join(row) for row in got["outputs"]])
    sessions = [{"prediction": rng.randn(B, 2).astype(np.float32), "mse": 0.5},
                {"prediction": rng.randn(B, 2).astype(np.float32), "mse": 0.25}]
    exe = object.__new__(RegressionRunner.Executable)
    got = {}
    exe._executor = types.SimpleNamespace(postprocess=None)
    exe.set_runner_result = lambda outputs, losses: got.update(outputs=outputs, losses=losses)
    exe.collect_results(sessions)
    out["regression_sessions"] = np.stack([s["prediction"] for s in sessions])
    out["regression_runner_outputs"] = np.array(got["outputs"])
    out["regression_runner_loss"] = np.array(got["losses"])

    np.savez_compressed(os.path.join(HERE, "classifier_golden.npz"), **out)
    print("wrote", os.path.join(HERE, "classifier_golden.npz"), len(out), "arrays")


if __name__ == "__main__":
    main()
