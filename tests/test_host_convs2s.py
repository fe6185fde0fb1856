"""The convolutional seq2seq encoder on the CPU: the fp64 restatement of tests/convs2s_oracle.py against the
reference's own code, the model part over the stand-ins (variable names, shapes, initializers, outputs), its
constructor errors, and the two commands of the reference's tests_run.sh that train tests/bpe.ini through
`neuralmonkey-train` (inputs from tests/golden/reference_experiments_bpe.json).  The kernels are tested in
tests/test_gpu_convs2s.py."""
import os
import sys

import numpy as np
import pytest
import torch

from tests import convs2s_oracle as CSO
from tests import cpu_ops
from tests.golden.make_bpe_bundle import unpack
from tests.helpers import training_log_values
from tests.test_host_cnn import _adadelta_stand_in

pytestmark = [pytest.mark.filterwarnings("ignore:Converting a tensor with requires_grad")]


@pytest.fixture
def cpu_model(monkeypatch):
    from neuralmonkey_b200 import ops, runtime
    from neuralmonkey_b200.trainers.generic_trainer import GenericTrainer
    for op in cpu_ops.STAND_INS:
        monkeypatch.setattr(ops, op, getattr(cpu_ops, op))
    for op in CSO.STAND_INS:
        monkeypatch.setattr(ops, op, getattr(CSO, op))
    monkeypatch.setattr(runtime, "_device", torch.device("cpu"))
    monkeypatch.setattr(GenericTrainer, "_adam_kernel", _adadelta_stand_in)
    yield
    runtime.reset()


def _np(x):
    return torch.from_numpy(np.asarray(x)).double()


def _sequence(max_length=10, embedding_size=11):
    from neuralmonkey_b200.model.sequence import EmbeddedSequence
    from neuralmonkey_b200.vocabulary import Vocabulary
    return EmbeddedSequence(name="encoder_input", vocabulary=Vocabulary(["w{}".format(i) for i in range(20)]),
                            data_id="source", embedding_size=embedding_size, max_length=max_length)


# -- the restatement ------------------------------------------------------------------------------------------------
def test_same_padding_puts_the_extra_zero_after():
    x = torch.arange(1.0, 6.0, dtype=torch.float64).view(1, 5, 1)
    w = torch.zeros(4, 1, 1, dtype=torch.float64)
    w[0] = 1.0              # tap 0 reads position t - (4-1)//2 = t - 1
    assert torch.equal(CSO.conv1d_same(x, w).view(-1), torch.tensor([0.0, 1, 2, 3, 4], dtype=torch.float64))
    w.zero_()
    w[3] = 1.0              # tap 3 reads t + 2, zero past the end
    assert torch.equal(CSO.conv1d_same(x, w).view(-1), torch.tensor([3.0, 4, 5, 0, 0], dtype=torch.float64))


@pytest.mark.parametrize("tag", CSO.CASES)
def test_oracle_against_the_reference_code(tag):
    g = CSO.golden()
    layers = CSO.SHAPES[tag][1]
    variables = {n: _np(v) for n, v in CSO.golden_variables(g, tag).items()}
    states, output = CSO.encoder(_np(g[tag + "_states"]), variables, layers, prefix=tag + "/")
    assert torch.allclose(states, _np(g[tag + "_temporal_states"]), rtol=1e-5, atol=1e-5)
    assert torch.allclose(output, _np(g[tag + "_output"]), rtol=1e-5, atol=1e-5)


# -- the model part -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag", CSO.CASES)
def test_model_part_against_the_reference_code(cpu_model, tag):
    """Over the stand-ins, with the golden's variables loaded BY NAME: the reference's names and shapes, its
    temporal states, its max over every position (padding included) and the input's mask."""
    g = CSO.golden()
    got = CSO.golden_model_outputs(g, tag, "cpu")
    for name, value in got.items():
        want = _np(g[tag + "_" + name])
        assert value.shape == want.shape, (tag, name)
        assert torch.allclose(value.double(), want, rtol=1e-5, atol=1e-5), (tag, name)


def test_variables_names_shapes_and_initializers(cpu_model):
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.encoders.facebook_conv import SentenceEncoder
    seq = _sequence(max_length=40, embedding_size=30)
    enc = SentenceEncoder(name="sentence_encoder", input_sequence=seq, conv_features=64, encoder_layers=2,
                          dropout_keep_prob=0.5)
    enc.ensure_declared()
    arena = runtime.arena()
    arena.finalize(runtime.device())
    shapes = {n: tuple(arena.get(n).shape) for n in arena.order if n.startswith("sentence_encoder/")}
    assert shapes == {
        "sentence_encoder/input_projection/order_embeddings": (40, 30),
        "sentence_encoder/order_and_embed/kernel": (30, 64),
        "sentence_encoder/order_and_embed/bias": (64,),
        "sentence_encoder/encoder_conv_0/convolution_filters": (5, 64, 128),
        "sentence_encoder/encoder_conv_0/conv_bias": (128,),
        "sentence_encoder/encoder_conv_1/convolution_filters": (5, 64, 128),
        "sentence_encoder/encoder_conv_1/conv_bias": (128,),
        "sentence_encoder/input_to_final_state/kernel": (30, 64),
        "sentence_encoder/input_to_final_state/bias": (64,)}
    assert enc.dimension == 64
    # glorot uniform: |x| <= sqrt(6 / (fan_in + fan_out)), variance 2 / (fan_in + fan_out); not normal(0.001)
    order = arena.get("sentence_encoder/input_projection/order_embeddings").double()
    limit = (6.0 / 70) ** 0.5
    assert float(order.abs().max()) <= limit and float(order.abs().max()) > 0.8 * limit
    assert abs(float(order.var()) - 2.0 / 70) < 0.2 * 2.0 / 70
    filters = arena.get("sentence_encoder/encoder_conv_1/convolution_filters").double()
    assert abs(float(filters.std()) - (4 / 64) ** 0.5) < 0.02 * (4 / 64) ** 0.5
    assert abs(float(filters.mean())) < 0.01
    for name in ("encoder_conv_0/conv_bias", "order_and_embed/bias", "input_to_final_state/bias"):
        assert float(arena.get("sentence_encoder/" + name).abs().max()) == 0.0


@pytest.mark.parametrize("kwargs,message", [
    ({"conv_features": 0}, "Number of features must be a positive integer"),
    ({"conv_features": -3}, "Number of features must be a positive integer"),
    ({"encoder_layers": 0}, "Number of encoder layers must be a positive integer"),
])
def test_constructor_errors(cpu_model, kwargs, message):
    from neuralmonkey_b200.encoders.facebook_conv import SentenceEncoder
    args = dict(name="enc", input_sequence=_sequence(), conv_features=10, encoder_layers=2)
    args.update(kwargs)
    with pytest.raises(ValueError, match=message):
        SentenceEncoder(**args)


def test_constructor_refuses_a_sequence_without_max_length(cpu_model):
    from neuralmonkey_b200.encoders.facebook_conv import SentenceEncoder
    with pytest.raises(ValueError, match="must have a maximum length"):
        SentenceEncoder(name="enc", input_sequence=_sequence(max_length=None), conv_features=10, encoder_layers=2)


# -- the reference's tests_run.sh, its two bpe.ini commands in order ------------------------------------------------
def _train(monkeypatch, strict, argv):
    from neuralmonkey_b200 import runtime
    monkeypatch.setenv("NEURALMONKEY_STRICT", strict)
    monkeypatch.setattr(sys, "argv", ["neuralmonkey-train"] + argv)
    try:
        from neuralmonkey_b200.train import main
        main()
    finally:
        runtime.reset()


def test_reference_bpe_commands_train_over_the_stand_ins(cpu_model, monkeypatch, tmp_path):
    unpack(str(tmp_path))
    monkeypatch.chdir(tmp_path)
    _train(monkeypatch, "", ["tests/bpe.ini"])
    first = open("tests/outputs/bpe/experiment.log").read()
    assert "Training finished" in first and "Validation (epoch" in first
    assert os.path.exists("tests/outputs/bpe/variables.data.index") or any(
        f.startswith("variables.data") for f in os.listdir("tests/outputs/bpe"))
    losses = training_log_values(first, "target_greedy/train_xent")
    assert losses and all(np.isfinite(losses))

    second_out = str(tmp_path / "frozen")
    _train(monkeypatch, "1", ["tests/bpe.ini", "-s", "decoder.encoders=[<encoder_output_frozen>]",
                              "-s", "attention.encoder=<encoder_states_frozen>",
                              "-s", 'main.initial_variables=["tests/outputs/bpe/variables.data"]',
                              "-s", 'main.output="{}"'.format(second_out)])
    second = open(os.path.join(second_out, "experiment.log")).read()
    assert "Training finished" in second
    assert "tests/outputs/bpe/variables.data" in second
