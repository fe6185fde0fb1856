"""Sentence classification and regression on the CPU: the fp64 restatement of tests/classifier_oracle.py and its
quirks, the model parts over that restatement (variable names, shapes, outputs), the runners' formatting and
argument errors, and the reference's tests/classifier.ini and tests/regressor.ini through `neuralmonkey-train`
(inputs from tests/golden/reference_experiments_classifier.json).  The kernels are tested in
tests/test_gpu_classifier.py."""
import os
import sys

import numpy as np
import pytest
import torch

from tests import classifier_oracle as CLO
from tests import cpu_ops
from tests.golden.make_classifier_bundle import unpack
from tests.helpers import training_log_values

pytestmark = [pytest.mark.filterwarnings("ignore:Converting a tensor with requires_grad")]


@pytest.fixture
def cpu_model(monkeypatch):
    from neuralmonkey_b200 import ops, runtime
    from neuralmonkey_b200.trainers.generic_trainer import GenericTrainer
    for op in cpu_ops.STAND_INS:
        monkeypatch.setattr(ops, op, getattr(cpu_ops, op))
    for op in CLO.STAND_INS:
        monkeypatch.setattr(ops, op, getattr(CLO, op))
    monkeypatch.setattr(runtime, "_device", torch.device("cpu"))
    monkeypatch.setattr(GenericTrainer, "_adam_kernel", cpu_ops.adam_kernel)
    yield
    runtime.reset()


# -- the restatement's quirks ---------------------------------------------------------------------------------------
def test_max_pool_of_an_all_negative_sentence_is_1e_15():
    x = -torch.rand(2, 4, 3, dtype=torch.float64) - 0.5
    mask = torch.tensor([[1, 1, 0, 0], [1, 1, 1, 1]], dtype=torch.float64)
    y = CLO.seq_max_pool(x, mask)
    assert torch.all(y[0] == 1e-15)
    assert torch.equal(y[1], x[1].amax(0))


def test_max_pool_splits_the_gradient_among_ties():
    x = torch.tensor([[[2.0], [2.0], [1.0], [2.0]]], dtype=torch.float64, requires_grad=True)
    mask = torch.tensor([[1.0, 1.0, 1.0, 0.0]], dtype=torch.float64)
    CLO.seq_max_pool(x, mask).sum().backward()
    # the masked 2.0 reads as 1e-15: the gradient is split between the two valid maxima only
    assert torch.allclose(x.grad[0, :, 0], torch.tensor([0.5, 0.5, 0.0, 0.0], dtype=torch.float64))


def test_max_pool_refuses_an_empty_batch():
    with pytest.raises(ValueError, match="mask sum"):
        CLO.seq_max_pool(torch.zeros(2, 3, 1), torch.zeros(2, 3))


def test_conv1d_max_pool_is_the_windowed_product():
    torch.manual_seed(0)
    x, w, b = torch.randn(2, 5, 3, dtype=torch.float64), torch.randn(2, 3, 4, dtype=torch.float64), torch.randn(4)
    want = torch.stack([torch.relu(torch.stack([x[i, t:t + 2].reshape(-1) @ w.reshape(6, 4) + b.double()
                                                for t in range(4)])).amax(0) for i in range(2)])
    assert torch.allclose(CLO.conv1d_max_pool(x, w, b.double()), want)
    with pytest.raises(ValueError, match="shorter than the filter"):
        CLO.conv1d_max_pool(x[:, :1], w, b.double())


def test_attentive_weights_renormalise_over_the_mask():
    torch.manual_seed(0)
    e, v = torch.randn(2, 4, 3, dtype=torch.float64), torch.randn(2, 4, 5, dtype=torch.float64)
    mask = torch.tensor([[1, 1, 0, 0], [1, 1, 1, 1]], dtype=torch.float64)
    w, out = CLO.attentive_pool(e, mask, v)
    assert torch.all(w[0, 2:] == 0)
    assert torch.allclose(w.sum(1), torch.ones(2, 3, dtype=torch.float64))
    assert out.shape == (2, 3, 5)


# -- argument errors ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("keep", [0.0, 1.5, -0.1])
def test_attentive_encoder_refuses_keep_prob_outside_unit_interval(cpu_model, keep):
    from neuralmonkey_b200.encoders.attentive import AttentiveEncoder
    with pytest.raises(ValueError, match=r"inside \(0,1\]"):
        AttentiveEncoder(name="att", input_sequence=_sentence_encoder(), hidden_size=3, num_heads=2,
                         dropout_keep_prob=keep)


def test_logits_runner_argument_errors(cpu_model):
    from neuralmonkey_b200.runners import LogitsRunner
    clf = _classifier([_sentence_encoder()])
    with pytest.raises(ValueError, match="not both"):
        LogitsRunner("out", clf, pick_index=1, pick_value="7")
    with pytest.raises(ValueError, match="is not in vocabulary"):
        LogitsRunner("out", clf, pick_value="no-such-label")
    assert LogitsRunner("out", clf, pick_value="7").pick_index == clf.vocabulary.index_to_word.index("7")


# -- model parts over the restatement -------------------------------------------------------------------------------
def _vocab(words):
    from neuralmonkey_b200.vocabulary import Vocabulary
    return Vocabulary(list(words))


def _sentence_encoder(name="enc"):
    from neuralmonkey_b200.encoders.recurrent import SentenceEncoder
    return SentenceEncoder(name=name, vocabulary=_vocab("abcdef"), data_id="source", embedding_size=5, rnn_size=4)


def _classifier(encoders, layers=(6,), name="clf"):
    from neuralmonkey_b200.decoders.classifier import Classifier
    return Classifier(name=name, encoders=encoders, vocabulary=_vocab(["6", "7", "8"]), data_id="label",
                      layers=list(layers), dropout_keep_prob=1.0)


class _Data:
    def __init__(self, series):
        self.series = series

    def __len__(self):
        return len(next(iter(self.series.values())))

    def get_series(self, name):
        return self.series[name]

    def maybe_get_series(self, name):
        return self.series.get(name)


SENTENCES = [["a", "b", "c"], ["d"], ["e", "f", "a", "b", "c"]]


def test_classifier_stack_variables_and_outputs(cpu_model):
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.encoders.attentive import AttentiveEncoder
    from neuralmonkey_b200.encoders.pooling import SequenceAveragePooling, SequenceMaxPooling
    from neuralmonkey_b200.encoders.sequence_cnn_encoder import SequenceCNNEncoder
    from neuralmonkey_b200.model.gradient_reversal import StatefulView
    enc = _sentence_encoder()
    att = AttentiveEncoder(name="att", input_sequence=enc, hidden_size=3, num_heads=2, output_size=7,
                           state_proj_size=5)
    att_plain = AttentiveEncoder(name="att_plain", input_sequence=enc, hidden_size=3, num_heads=2)
    maxp = SequenceMaxPooling(name="maxp", input_sequence=enc)
    avgp = SequenceAveragePooling(name="avgp", input_sequence=enc)
    cnn = SequenceCNNEncoder(name="cnn", vocabulary=_vocab("abcdef"), data_id="source", embedding_size=4,
                             filters=[(2, 3), (3, 2)])
    clf = _classifier([att, att_plain, maxp, avgp, cnn], layers=(6, 5))
    adv = _classifier([StatefulView(maxp)], layers=(), name="adv")
    for part in (clf, adv):
        part.ensure_declared()
    for part in (enc, att, att_plain, cnn):
        part.ensure_declared()
    arena = runtime.arena()
    arena.finalize(runtime.device())
    shapes = {n: tuple(arena.get(n).shape) for n in arena.order}
    assert shapes["att/S1/kernel"] == (8, 3) and shapes["att/S2/kernel"] == (3, 2)
    assert shapes["att/state_projection/kernel"] == (8, 5) and shapes["att/output_projection/kernel"] == (10, 7)
    assert "att_plain/output_projection/kernel" not in shapes
    assert shapes["cnn/input_projection/word_embeddings"] == (len(cnn.vocabulary), 4)
    assert shapes["cnn/conv-maxpool-2/conv_W"] == (2, 4, 3) and shapes["cnn/conv-maxpool-3/conv_bias"] == (2,)
    width = 7 + 2 * 8 + 8 + 8 + 5
    assert shapes["clf/multilayer_perceptron/deep_output_mlp/mlp_layer_0/kernel"] == (width, 6)
    assert shapes["clf/multilayer_perceptron/deep_output_mlp/mlp_layer_1/bias"] == (5,)
    assert shapes["clf/multilayer_perceptron/classification_layer/kernel"] == (5, len(clf.vocabulary))
    assert shapes["adv/multilayer_perceptron/classification_layer/kernel"] == (8, len(adv.vocabulary))

    data = _Data({"source": SENTENCES, "label": [["7"], ["8"], ["6"]]})
    for part in (enc.input_sequence, enc, att, att_plain, maxp, avgp, cnn, clf, adv):
        part.feed_dict(data, train=False)
    states = enc.temporal_states
    assert maxp.output.shape == avgp.output.shape == (3, states.shape[2])
    assert torch.equal(att.temporal_mask, torch.ones(3, 2))
    assert att.attention_weights.shape == (3, states.shape[1], 2) and att.output.shape == (3, 7)
    assert att_plain.output.shape == (3, 16)
    assert cnn.output.shape == (3, 5)
    assert clf.decoded.shape == (1, 3) and clf.decoded_logits.shape == (1, 3, len(clf.vocabulary))
    logits = clf.decoded_logits[0].double()
    assert torch.allclose(clf.runtime_logprobs[0].double(), torch.log_softmax(logits, -1), atol=1e-6)
    want = torch.nn.functional.cross_entropy(logits, clf.gt_inputs)
    assert torch.allclose(clf.train_loss.double(), want, atol=1e-6)
    loss_sum, count = clf.loss_sum_and_count
    assert float(count) == 3.0 and torch.allclose(loss_sum / count, clf.cost)
    # the reversal view: identity forward, negated gradient backward
    x = torch.randn(3, 8, requires_grad=True)
    from neuralmonkey_b200.model.gradient_reversal import reverse_gradient
    (reverse_gradient(x) * 2).sum().backward()
    assert torch.equal(x.grad, torch.full((3, 8), -2.0))


def test_regressor_outputs_and_names(cpu_model):
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.decoders.sequence_regressor import SequenceRegressor
    for layers, dim in (([4, 3], 1), (None, 2)):
        runtime.reset()
        enc = _sentence_encoder()
        reg = SequenceRegressor(name="reg", encoders=[enc], data_id="value", layers=layers, dimension=dim)
        enc.ensure_declared()
        reg.ensure_declared()
        arena = runtime.arena()
        arena.finalize(runtime.device())
        names = set(arena.order)
        assert ("reg/mlp/mlp_layer_1/kernel" in names) == (layers is not None)
        assert tuple(arena.get("reg/output_projection/kernel").shape) == ((3 if layers else 8), dim)
        data = _Data({"source": SENTENCES, "value": [[1.0, 9.0], [2.0], [3.0]]})
        enc.input_sequence.feed_dict(data, train=False)
        enc.feed_dict(data, train=False)
        reg.feed_dict(data, train=False)
        pred = reg.predictions.double()
        assert pred.shape == (3, dim)
        want = ((pred - torch.tensor([1.0, 2.0, 3.0], dtype=torch.float64)[:, None]) ** 2).mean()
        assert torch.allclose(reg.cost.double(), want)


# -- the reference's INIs, unchanged --------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["classifier", "regressor"])
def test_reference_ini_trains_over_the_stand_ins(cpu_model, monkeypatch, tmp_path, name):
    from neuralmonkey_b200 import runtime
    monkeypatch.setenv("NEURALMONKEY_STRICT", "1")
    unpack(str(tmp_path / "tree"))
    monkeypatch.chdir(tmp_path / "tree")
    out = str(tmp_path / name)
    monkeypatch.setattr(sys, "argv", ["neuralmonkey-train", "tests/{}.ini".format(name), "-s",
                                      'main.output="{}"'.format(out)])
    try:
        from neuralmonkey_b200.train import main
        main()
    finally:
        runtime.reset()
    log_text = open(os.path.join(out, "experiment.log")).read()
    assert "Training finished" in log_text and "Validation (epoch" in log_text
    assert ("classification/Accuracy" if name == "classifier" else "regression/MeanSquaredError") in log_text
    losses = training_log_values(log_text, "classification/train_xent" if name == "classifier" else "regression/mse")
    assert losses and all(np.isfinite(losses))


# -- against the reference's own code (tests/golden/make_classifier_golden.py -> classifier_golden.npz) --------------
def _np(x):
    return torch.from_numpy(np.asarray(x)).double()


def test_oracle_against_the_reference_code():
    """The fp64 restatement against the reference's poolings, AttentiveEncoder, SequenceCNNEncoder,
    MultilayerPerceptron, Classifier and SequenceRegressor."""
    g = CLO.golden()
    states, mask = _np(g["states"]), _np(g["mask"])
    assert torch.allclose(CLO.seq_max_pool(states, mask), _np(g["maxpool_output"]), rtol=1e-6, atol=1e-12)
    assert np.all(g["maxpool_output"][1] == np.float32(1e-15))          # the all-negative sentence
    assert torch.allclose(CLO.seq_mean_pool(states, mask), _np(g["avgpool_output"]), rtol=1e-6, atol=1e-7)
    for tag in ("att_plain", "att_proj"):
        v = {n.split("/", 1)[1]: _np(a) for n, a in CLO.golden_variables(g, tag).items()}
        energies = torch.tanh(states @ v["S1/kernel"]) @ v["S2/kernel"]
        proj = states if tag == "att_plain" else states @ v["state_projection/kernel"] + v["state_projection/bias"]
        weights, pooled = CLO.attentive_pool(energies, mask, proj)
        out = pooled.reshape(pooled.shape[0], -1)
        if tag == "att_proj":
            out = out @ v["output_projection/kernel"] + v["output_projection/bias"]
        for name, got in (("weights", weights), ("temporal_states", pooled), ("output", out)):
            assert torch.allclose(got, _np(g[tag + "_" + name]), rtol=1e-5, atol=1e-6), (tag, name)
    v = {n.split("/", 1)[1]: _np(a) for n, a in CLO.golden_variables(g, "cnn").items()}
    emb = v["input_projection/word_embeddings"][torch.from_numpy(g["cnn_ids"])]
    pooled = torch.cat([CLO.conv1d_max_pool(emb, v["conv-maxpool-{}/conv_W".format(w)],
                                            v["conv-maxpool-{}/conv_bias".format(w)]) for w in (2, 3, 6)], 1)
    assert torch.allclose(pooled, _np(g["cnn_output"]), rtol=1e-5, atol=1e-6)
    feats = torch.cat([_np(g["features_0"]), _np(g["features_1"])], 1)
    for tag, layers in (("clf_layers", 2), ("clf_nolayers", 0)):
        v = {n.split("/", 2)[2]: _np(a) for n, a in CLO.golden_variables(g, tag).items()}
        x = feats
        for i in range(layers):
            x = torch.relu(x @ v["deep_output_mlp/mlp_layer_{}/kernel".format(i)]
                           + v["deep_output_mlp/mlp_layer_{}/bias".format(i)])
        logits = x @ v["classification_layer/kernel"] + v["classification_layer/bias"]
        assert torch.allclose(logits, _np(g[tag + "_logits"])[0], rtol=1e-5, atol=1e-6), tag
        loss = torch.nn.functional.cross_entropy(logits, torch.from_numpy(g["labels"]))
        assert abs(float(loss) - float(g[tag + "_loss"])) < 1e-5, tag
        assert torch.equal(logits.argmax(1), torch.from_numpy(g[tag + "_decoded"][0]))
    for tag, layers in (("reg_layers", 2), ("reg_nolayers", 0)):
        v = {n.split("/", 1)[1]: _np(a) for n, a in CLO.golden_variables(g, tag).items()}
        x = feats
        for i in range(layers):
            x = torch.relu(x @ v["mlp/mlp_layer_{}/kernel".format(i)] + v["mlp/mlp_layer_{}/bias".format(i)])
        pred = x @ v["output_projection/kernel"] + v["output_projection/bias"]
        assert torch.allclose(pred, _np(g[tag + "_predictions"]), rtol=1e-5, atol=1e-6), tag
        assert abs(float(CLO.squared_error(pred, _np(g["reg_targets"]))) - float(g[tag + "_cost"])) < 1e-5, tag


@pytest.mark.parametrize("tag", CLO.MODEL_CASES)
def test_model_parts_against_the_reference_code(cpu_model, tag):
    """The model parts over the stand-ins, with the golden's variables loaded BY NAME: the same variable names and
    shapes as the reference's graph and the same outputs."""
    g = CLO.golden()
    got = CLO.golden_model_outputs(g, tag, "cpu")
    for name, value in got.items():
        want = _np(g[tag + "_" + name] if tag not in ("maxpool", "avgpool") else g[tag + "_output"])
        assert value.shape == want.shape, (tag, name)
        assert torch.allclose(value.double(), want, rtol=1e-5, atol=1e-6), (tag, name)


def test_views_against_the_reference_code():
    """Identity forward through the gradient-reversal views, masks passed through, the wrapped object among the
    dependencies; the gradient is negated."""
    from neuralmonkey_b200.model.gradient_reversal import SpatialStatefulView, StatefulView, TemporalStatefulView
    from neuralmonkey_b200.model.stateful import SpatialStateful, Stateful, TemporalStateful
    g = CLO.golden()
    states = torch.from_numpy(g["states"]).requires_grad_()
    mask = torch.from_numpy(g["mask"])

    class Seq(TemporalStateful):
        temporal_states = property(lambda self: states)
        temporal_mask = property(lambda self: mask)

    class Vec(Stateful):
        output = property(lambda self: states[:, 0])

    class Map(SpatialStateful):
        spatial_states = property(lambda self: states[:, :, :, None])
        spatial_mask = property(lambda self: mask[:, :, None])

    view = StatefulView(Vec())
    assert torch.equal(view.output.detach(), torch.from_numpy(g["view_output"]))
    assert "_reversed_object" in view.dependencies and str(g["view_dependencies"][-1]) == "_reversed_object"
    tview, sview = TemporalStatefulView(Seq()), SpatialStatefulView(Map())
    assert torch.equal(tview.temporal_states.detach(), torch.from_numpy(g["tview_states"]))
    assert torch.equal(tview.temporal_mask, torch.from_numpy(g["tview_mask"]))
    assert torch.equal(sview.spatial_states.detach(), torch.from_numpy(g["sview_states"]))
    assert torch.equal(sview.spatial_mask, torch.from_numpy(g["sview_mask"]))
    (tview.temporal_states.sum() + view.output.sum()).backward()
    want = -torch.ones_like(states)
    want[:, 0] -= 1
    assert torch.equal(states.grad, want)


@pytest.mark.parametrize("normalize", [True, False])
@pytest.mark.parametrize("pick", [None, 0, 3])
def test_logits_runner_against_the_reference_code(normalize, pick):
    from neuralmonkey_b200.runners.logits_runner import LogitsRunner
    g = CLO.golden()
    exe = LogitsRunner.Executable.__new__(LogitsRunner.Executable)
    exe._executor = type("E", (), dict(normalize=normalize, pick_index=pick, output_series="d",
                                       loss_names=["a", "b"]))()
    got = {}
    exe.set_runner_result = lambda outputs, losses: got.update(outputs=outputs, losses=losses)
    exe.collect_results([{"logits": g["runner_logits"], "train_loss": 1.25, "runtime_loss": 2.5}])
    key = "logits_runner_{}_{}".format(int(normalize), "none" if pick is None else pick)
    assert ["\n".join(row) for row in got["outputs"]] == [str(s) for s in g[key]]
    assert got["losses"] == [1.25, 2.5]


def test_regression_runner_against_the_reference_code():
    from neuralmonkey_b200.runners.regression_runner import RegressionRunner
    g = CLO.golden()
    exe = RegressionRunner.Executable.__new__(RegressionRunner.Executable)
    exe._executor = type("E", (), dict(postprocess=None, output_series="r", loss_names=["mse"]))()
    got = {}
    exe.set_runner_result = lambda outputs, losses: got.update(outputs=outputs, losses=losses)
    exe.collect_results([{"prediction": p, "mse": m} for p, m in zip(g["regression_sessions"], (0.5, 0.25))])
    assert np.array_equal(np.array(got["outputs"]), g["regression_runner_outputs"])
    assert got["losses"] == list(g["regression_runner_loss"])
