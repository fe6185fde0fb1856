"""The character-level sentence encoder's host side on the CPU: the fp64 restatement of tests/sentence_cnn_oracle.py
against the reference's own class (tests/golden/sentence_cnn_golden.npz), the model part over that restatement
(variable names, outputs, gradients, dropout placement), the reference's constructor tables, the refusal of noisy
activations, and the reference's tests/small_sent_cnn.ini through `neuralmonkey-train` (inputs from the bundles
under tests/golden/).  The kernels are tested in tests/test_gpu_sentence_cnn.py."""
import copy
import os
import sys

import numpy as np
import pytest
import torch

from tests import cpu_ops
from tests import sentence_cnn_oracle as SO
from tests.helpers import training_log_values

pytestmark = [pytest.mark.filterwarnings("ignore:Converting a tensor with requires_grad")]


@pytest.fixture
def cpu_model(monkeypatch):
    from neuralmonkey_b200 import ops, runtime
    from neuralmonkey_b200.trainers.generic_trainer import GenericTrainer
    for op in cpu_ops.STAND_INS:
        monkeypatch.setattr(ops, op, getattr(cpu_ops, op))
    for op in SO.STAND_INS:
        monkeypatch.setattr(ops, op, getattr(SO, op))
    monkeypatch.setattr(runtime, "_device", torch.device("cpu"))
    monkeypatch.setattr(GenericTrainer, "_adam_kernel", cpu_ops.adam_kernel)
    yield
    runtime.reset()


def deterministic_dropout(monkeypatch):
    """The golden's deterministic dropout mask in place of the random one."""
    from neuralmonkey_b200.nn import utils

    def mask(shape, keep_prob, train_mode, device):
        if keep_prob >= 1.0 or not train_mode:
            return None
        return SO.feature_dropout_mask(shape, keep_prob).to(device=device, dtype=torch.float32)
    monkeypatch.setattr(utils, "dropout_mask", mask)


def _close(got, want, rtol, atol=0.0):
    return got.shape == want.shape and bool(torch.allclose(got, want, rtol=rtol, atol=atol))


# -- the restatement against the reference's class -------------------------------------------------------------------
@pytest.mark.parametrize("tag", SO.CASES)
def test_oracle_against_the_reference_code(tag):
    g = SO.golden()
    out, _, _ = SO.oracle_case(g, tag)
    for name in SO.OUTPUTS:
        want = torch.from_numpy(g[tag + "_" + name])
        # the stand-in rounds its dense outputs to fp32
        assert _close(out[name], want, 1e-6, 1e-6), (tag, name, float((out[name] - want).abs().max()))


def test_golden_pins_the_offset_windows_and_the_short_sequence_length():
    """At T = 12 and s = 5 the windows are {0..3}, {4..8}, {9..11}; the length-5 sentence gets the pooled mask
    [1, 1, 0] but one GRU step, so its second segment is admitted by the mask and zero in temporal_states."""
    g = SO.golden()
    assert g["t12_s5_temporal_mask"].tolist() == [[1, 1, 1], [1, 1, 0], [1, 1, 0]]
    ts = g["t12_s5_temporal_states"]
    assert np.all(ts[1, 1:] == 0) and np.any(ts[1, 0] != 0)
    x = torch.arange(12, dtype=torch.float64).view(1, 12, 1)
    assert SO.segment_max(x, 5).view(-1).tolist() == [3.0, 8.0, 11.0]
    assert SO.segment_max(x[:, :4], 6).view(-1).tolist() == [3.0]


# -- the model part over the restatement -------------------------------------------------------------------------------
@pytest.mark.parametrize("tag", SO.CASES)
def test_model_part_against_the_reference_code(cpu_model, monkeypatch, tag):
    """The model part over the stand-ins, with the golden's variables loaded BY NAME: the reference's variable names
    and shapes, the same outputs, and the gradients of the fp64 restatement."""
    deterministic_dropout(monkeypatch)
    g = SO.golden()
    got, grads, dstates = SO.model_case(g, tag, "cpu")
    want, want_grads, want_dstates = SO.oracle_case(g, tag)
    for name in SO.OUTPUTS:
        assert _close(got[name], torch.from_numpy(g[tag + "_" + name]), 1e-5, 1e-6), (tag, name)
    assert sorted(grads) == sorted(want_grads)
    for name, value in want_grads.items():
        assert _close(grads[name].double(), value, 1e-4, 1e-5), (tag, name)
    assert _close(dstates, want_dstates, 1e-4, 1e-5), tag


def test_variable_names_and_initial_values(cpu_model):
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.encoders import SentenceCNNEncoder
    from neuralmonkey_b200.model.sequence import EmbeddedSequence
    from neuralmonkey_b200.vocabulary import Vocabulary
    seq = EmbeddedSequence("chars", Vocabulary(list("abc")), "source_chars", 11)
    enc = SentenceCNNEncoder(name="sentence_encoder", input_sequence=seq, segment_size=5, highway_depth=2,
                             rnn_size=7, filters=[(1, 13), (2, 13), (3, 13)], dropout_keep_prob=0.5)
    assert enc.dimension == 14
    enc.ensure_declared()
    arena = runtime.arena()
    arena.finalize(runtime.device())
    scope = "sentence_encoder/"
    shapes = {n[len(scope):]: tuple(arena.get(n).shape) for n in arena.order if n.startswith(scope)}
    want = {"conv-maxpool-{}/conv_W".format(w): (w, 11, 13) for w in (1, 2, 3)}
    want.update({"conv-maxpool-{}/conv_bias".format(w): (13,) for w in (1, 2, 3)})
    for i in range(2):
        for gate in "HT":
            want["highway_layer_{}/weight_{}".format(i, gate)] = (39, 39)
            want["highway_layer_{}/bias_{}".format(i, gate)] = (39,)
    for d in ("fw", "bw"):
        pre = "bidirectional_rnn/{}/OrthoGRUCell/".format(d)
        want.update({pre + "gates/kernel": (46, 14), pre + "gates/bias": (14,), pre + "candidate/kernel": (46, 7),
                     pre + "candidate/bias": (7,)})
    assert shapes == want
    # the highway weights take tf.get_variable's default, glorot uniform: |w| <= sqrt(6 / (39 + 39)), spread over the
    # whole interval
    bound = (6.0 / (2 * 39)) ** 0.5
    for i in range(2):
        for gate in "HT":
            w = arena.get(scope + "highway_layer_{}/weight_{}".format(i, gate)).double()
            assert float(w.abs().max()) <= bound + 1e-7
            assert float(w.abs().max()) > 0.9 * bound
            assert abs(float(w.std()) - bound / 3 ** 0.5) < 0.1 * bound
    assert torch.all(arena.get(scope + "highway_layer_1/bias_T") == -1.0)
    assert torch.all(arena.get(scope + "highway_layer_0/bias_H") == -1.0)
    assert torch.all(arena.get(scope + "conv-maxpool-2/conv_bias") == 0.0)
    assert torch.all(arena.get(scope + "bidirectional_rnn/fw/OrthoGRUCell/gates/bias") == 1.0)


# -- under the RNN decoder -------------------------------------------------------------------------------------------
def test_greedy_and_beam_decoding_over_the_encoder(cpu_model):
    """The decoder's Bahdanau attention and initial state read the encoder: greedy decoding and beam search run over
    it, and the best beam of a beam of one is the greedy output."""
    from neuralmonkey_b200.decoders.beam_search_decoder import BeamSearchDecoder
    g = torch.Generator().manual_seed(3)
    src, tgt = SO.ini_batch(g)
    model = SO.build_ini_model()
    model["arena"].load_dict({n: torch.randn(v.shape, generator=g) * 0.3 for n, v in model["arena"].state_dict().items()})
    SO.feed_ini_model(model, src, tgt, False)
    greedy = model["dec"].runtime_symbols
    assert greedy.shape[1] == src.shape[0]
    bs = BeamSearchDecoder(name="bs", parent_decoder=model["dec"], beam_size=1, max_steps=10,
                           length_normalization=0.6)
    bs.use_cuda_graph = False
    SO.feed_ini_model(model, src, None, False)
    bs.reset_batch()
    bs.batch_size = src.shape[0]
    ids = bs.outputs.last_search_step_output.token_ids[1:]
    steps = min(ids.shape[0], greedy.shape[0])
    assert torch.equal(ids[:steps].reshape(steps, -1), greedy[:steps])


@pytest.mark.parametrize("views", [False, True])
def test_gradient_blocking_views(cpu_model, views):
    """Behind StatefulView / TemporalStatefulView the encoder gets no cross-entropy gradient: without L2 its
    variables stay put in an Adam step, while those of the decoder move; without the views they move too."""
    g = torch.Generator().manual_seed(4)
    src, tgt = SO.ini_batch(g)
    model = SO.build_ini_model(views=views, l2_weight=0.0)
    params = {n: torch.randn(v.shape, generator=g) * 0.3 for n, v in model["arena"].state_dict().items()}
    loss, after = SO.ini_step(params, src, tgt, views=views, l2_weight=0.0)
    assert np.isfinite(loss)
    encoder = [n for n in params if n.startswith(("sentence_encoder/", "encoder_input/"))]
    assert len(encoder) == 1 + 2 * 3 + 4 * 3 + 4 * 2     # embeddings, convolutions, highway layers, GRU cells
    moved = {n for n in params if not torch.equal(after[n], params[n])}
    assert moved & {n for n in params if n.startswith("decoder/")}
    assert bool(moved & set(encoder)) != views


# -- the constructor (the reference's neuralmonkey/tests/test_encoders_init.py) --------------------------------------
def _tables():
    from neuralmonkey_b200.encoders import SentenceEncoder
    from neuralmonkey_b200.model.sequence import EmbeddedSequence
    from neuralmonkey_b200.vocabulary import Vocabulary
    vocabulary = Vocabulary(["ich", "bin", "der", "walrus"])
    input_sequence = EmbeddedSequence("seq", vocabulary, "marmelade", 300)
    good = {
        "name": ["cnn_encoder"],
        "input_sequence": [input_sequence],
        "segment_size": [10],
        "highway_depth": [11],
        "rnn_size": [30],
        "filters": [[(2, 10)], [(3, 20), (4, 10)]],
        "dropout_keep_prob": [0.5, 1.],
        "use_noisy_activations": [False],
    }
    bad = {
        "nonexistent": ["ahoj"],
        "name": [None, 1],
        "input_sequence": [0, None, vocabulary],
        "segment_size": [-1, 0, "ahoj", 3.14, vocabulary, None],
        "highway_depth": [-1, "ahoj", 3.14, SentenceEncoder, None],
        "rnn_size": [-1, 0, "ahoj", 3.14, vocabulary, SentenceEncoder, None],
        "filters": ["ahoj", [], [(0, 0)], [(1, 2, 3)], [vocabulary, None], [(None, None)]],
        "dropout_keep_prob": [0.0, 0, -1.0, 2.0, "ahoj", vocabulary, None],
        "use_noisy_activations": [None, SentenceEncoder],
    }
    return good, bad


def _combinations(params):
    keys = sorted(params)
    out = [{}]
    for key in keys:
        out = [dict(o, **{key: v}) for o in out for v in params[key]]
    return out


def test_constructor_tables(cpu_model):
    from neuralmonkey_b200.encoders import SentenceCNNEncoder
    good, bad = _tables()
    base = {k: v[0] for k, v in good.items()}
    n = 0
    for key, values in bad.items():
        for value in values:
            options = copy.copy(base)
            options[key] = value
            if key != "name":
                options["name"] = "{}_{}".format(options["name"], n)
            n += 1
            with pytest.raises(Exception):
                SentenceCNNEncoder(**options)
    combos = _combinations(good)
    assert len(combos) == 4
    for options in combos:
        options["name"] = "{}_{}".format(options["name"], n)
        n += 1
        SentenceCNNEncoder(**options)
    with pytest.raises(TypeError):
        SentenceCNNEncoder()  # pylint: disable=no-value-for-parameter


@pytest.mark.parametrize("key,value,message", [
    ("dropout_keep_prob", 0.0, "Dropout keep probability"), ("rnn_size", 0, "RNN size"),
    ("highway_depth", 0, "Highway depth"), ("segment_size", 0, "Segment size"), ("filters", [], "convolutional filters"),
    ("filters", [(0, 3)], "Filter size"), ("filters", [(3, 0)], "Number of filters"),
])
def test_constructor_messages(cpu_model, key, value, message):
    from neuralmonkey_b200.encoders import SentenceCNNEncoder
    good, _ = _tables()
    options = {k: v[0] for k, v in good.items()}
    options[key] = value
    with pytest.raises(ValueError, match=message):
        SentenceCNNEncoder(**options)


def test_noisy_activations_are_refused(cpu_model):
    from neuralmonkey_b200.encoders import SentenceCNNEncoder
    good, _ = _tables()
    options = {k: v[0] for k, v in good.items()}
    options["use_noisy_activations"] = True
    with pytest.raises(NotImplementedError, match="NoisyGRUCell"):
        SentenceCNNEncoder(**options)


# -- the reference's INI, unchanged ----------------------------------------------------------------------------------
# besides the output directory, only the TER evaluation is dropped: pyter, the third-party package it needs, is absent
TER_DROPPED = 'main.evaluation=[("target", evaluators.BLEU)]'


def test_small_sent_cnn_ini_trains_over_the_stand_ins(cpu_model, monkeypatch, tmp_path):
    from neuralmonkey_b200 import runtime
    from tests.golden.make_sent_cnn_bundle import unpack
    monkeypatch.setenv("NEURALMONKEY_STRICT", "1")
    unpack(str(tmp_path / "tree"))
    monkeypatch.chdir(tmp_path / "tree")
    out = str(tmp_path / "small_sent_cnn")
    monkeypatch.setattr(sys, "argv", ["neuralmonkey-train", "tests/small_sent_cnn.ini", "-s",
                                      'main.output="{}"'.format(out), "-s", TER_DROPPED])
    try:
        from neuralmonkey_b200.train import main
        main()
    finally:
        runtime.reset()
    log_text = open(os.path.join(out, "experiment.log")).read()
    assert "Training finished" in log_text and "Validation (epoch" in log_text
    losses = training_log_values(log_text, "train_xent")
    assert losses and all(np.isfinite(losses))
