"""Supervised attention on the CPU: `WordAlignmentPreprocessor` against the reference's own class, and
`WordAlignmentDecoder` / `WordAlignmentRunner` over the stand-ins of tests/cpu_ops.py and tests/alignment_oracle.py
against the fp64 oracle - the loss, every parameter gradient, cropping, the zero-filled feed, the step-wise variants,
the refusals - and the reference's tests/alignment.ini through `neuralmonkey-train`.  The kernels are tested in
tests/test_gpu_alignment.py."""
import json
import os
import sys

import numpy as np
import pytest
import torch

from tests import alignment_oracle as AO
from tests import cpu_ops
from tests.helpers import random_batch

pytestmark = [pytest.mark.filterwarnings("ignore:Converting a tensor with requires_grad")]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _stand_ins(monkeypatch):
    from neuralmonkey_b200 import ops, runtime
    from neuralmonkey_b200.trainers.generic_trainer import GenericTrainer
    for op in cpu_ops.STAND_INS:
        monkeypatch.setattr(ops, op, getattr(cpu_ops, op))
    for op in AO.STAND_INS:
        monkeypatch.setattr(ops, op, getattr(AO, op))
    monkeypatch.setattr(runtime, "_device", torch.device("cpu"))
    monkeypatch.setattr(GenericTrainer, "_adam_kernel", cpu_ops.adam_kernel)


@pytest.fixture
def cpu_model(monkeypatch):
    from neuralmonkey_b200 import runtime
    _stand_ins(monkeypatch)
    yield
    runtime.reset()


# -- the preprocessor ---------------------------------------------------------------------------------------------------
def test_preprocessor_against_the_reference_code():
    from neuralmonkey_b200.processors.alignment import WordAlignmentPreprocessor
    with open(os.path.join(ROOT, "tests", "golden", "alignment_golden.json"), encoding="utf-8") as handle:
        cases = json.load(handle)["cases"]
    assert len(cases) > 100
    for case in cases:
        pre = WordAlignmentPreprocessor(case["source_len"], case["target_len"], normalize=case["normalize"],
                                        zero_based=case["zero_based"])
        got = pre(case["line"].split())
        assert got.dtype == np.float32 and got.shape == (case["target_len"], case["source_len"])
        np.testing.assert_array_equal(got, np.array(case["matrix"], dtype=np.float32), err_msg=str(case))


def test_preprocessor_normalises_rows_and_keeps_empty_rows_zero():
    from neuralmonkey_b200.processors.alignment import WordAlignmentPreprocessor
    got = WordAlignmentPreprocessor(4, 3)("0-0 1-0/3 2:2 9-1".split())
    np.testing.assert_allclose(got, [[0.25, 0.75, 0, 0], [0, 0, 0, 0], [0, 0, 1, 0]])


# -- the decoder against the fp64 oracle ----------------------------------------------------------------------------
def _params(model, seed=7):
    from tests.helpers import oracle_params_for
    params = oracle_params_for(model, seed=seed)
    model["arena"].load_dict(params)
    return params


def _alignments(bsz, rows, cols, seed=0):
    rng = np.random.RandomState(seed)
    ali = rng.rand(bsz, rows, cols).astype(np.float32)
    ali *= rng.rand(bsz, rows, cols) < 0.4
    ali[0, 0] = 0.                                # a row with all-zero targets
    return ali


def _check_against_oracle(model, params, src, tgt, ali, weight=1e-3):
    """The alignment cost and the gradient of cost_dec + weight * cost_ali for every variable, fp32 stand-ins
    against fp64."""
    dec, ali_dec, arena = model["dec"], model["ali"], model["arena"]
    p64 = {n: v.double().requires_grad_(True) for n, v in params.items()}
    o_dec, o_ali, _ = AO.oracle_losses(p64, model["spec"], src, tgt, None if ali is None else torch.from_numpy(ali))
    assert abs(float(ali_dec.cost) - float(o_ali)) <= 2e-5 * abs(float(o_ali)) + 1e-6
    assert abs(float(dec.cost) - float(o_dec)) <= 2e-5 * abs(float(o_dec)) + 1e-6
    arena.zero_grad()
    model["trainer"]._backward()                   # pylint: disable=protected-access
    (o_dec + weight * o_ali).backward()
    for name, grad in arena.named_grads().items():
        want = p64[name].grad
        want = torch.zeros_like(p64[name]) if want is None else want
        err = float((grad.double() - want.reshape(grad.shape)).norm())
        # attn_bias: the gradient is 0 in exact arithmetic (a softmax does not see a shift), fp32 leaves ~1e-7
        assert err <= 2e-4 * float(want.norm()) + 2e-6, (name, err, float(want.norm()))
    return float(o_ali)


@pytest.mark.parametrize("rnn_cell,conditional", [("GRU", False), ("NematusGRU", False), ("GRU", True)])
def test_loss_and_gradients_against_the_oracle(cpu_model, rnn_cell, conditional):
    model = AO.build(rnn_cell=rnn_cell, conditional_gru=conditional, weights=(1., 0.5))
    params = _params(model)
    src, tgt = random_batch(5, 6, 7, 40, 50, seed=1)
    ali = _alignments(5, 7, 6)
    AO.feed(model, src, tgt, ali, train=True)
    assert _check_against_oracle(model, params, src, tgt, ali, weight=0.5) > 0


@pytest.mark.parametrize("rows,cols", [(8, 8), (3, 2), (9, 4)])
def test_rows_and_columns_are_cropped_or_zero_filled(cpu_model, rows, cols):
    """The batch has 7 training steps over 6 encoder states; the fed matrices are larger, smaller or mixed."""
    model = AO.build()
    params = _params(model)
    src, tgt = random_batch(5, 6, 7, 40, 50, seed=2)
    ali = _alignments(5, rows, cols, seed=3)
    AO.feed(model, src, tgt, ali, train=True)
    _check_against_oracle(model, params, src, tgt, ali)


def test_shapes_of_the_energies_and_the_loss(cpu_model):
    model = AO.build()
    _params(model)
    src, tgt = random_batch(4, 5, 6, 40, 50, seed=4)
    AO.feed(model, src, tgt, _alignments(4, 8, 8), train=True)
    energies = model["dec"].train_attention_energies(model["att"])
    assert energies.shape == (4, 6, 5) and energies.requires_grad
    assert model["ali"].cost.shape == () and float(model["ali"].runtime_loss) == 0.
    assert model["ali"].alignment_target.shape == (8, 4, 8)


def test_missing_alignments_are_zeros_and_warn_in_training(cpu_model, monkeypatch):
    from neuralmonkey_b200.decoders import word_alignment_decoder
    warned = []
    monkeypatch.setattr(word_alignment_decoder, "warn", warned.append)
    model = AO.build()
    params = _params(model)
    src, tgt = random_batch(3, 5, 6, 40, 50, seed=5)
    AO.feed(model, src, tgt, None, train=True)
    assert warned == ["Training alignment not present!"]
    assert model["ali"].ref_alignment.shape == (3, 8, 8) and float(model["ali"].ref_alignment.abs().sum()) == 0.
    assert _check_against_oracle(model, params, src, tgt, None) == 0.
    AO.feed(model, src, tgt, None, train=False)
    assert len(warned) == 1


def test_zero_fill_without_max_length_takes_the_batch_width(cpu_model):
    model = AO.build()
    _params(model)
    model["enc"].input_sequence.max_length = None
    src, tgt = random_batch(3, 5, 6, 40, 50, seed=5)
    AO.feed(model, src, tgt, None, train=False)
    assert model["ali"].ref_alignment.shape == (3, 8, 5)


# -- refusals --------------------------------------------------------------------------------------------------------------
def _encoder(name="enc"):
    from neuralmonkey_b200.encoders import SentenceEncoder
    from neuralmonkey_b200.vocabulary import Vocabulary
    return SentenceEncoder(name=name, vocabulary=Vocabulary(["a", "b"]), data_id="source", embedding_size=4,
                           rnn_size=3, max_input_len=5)


@pytest.mark.parametrize("kind", ["coverage", "scaled_dot", "multi_head"])
def test_a_non_bahdanau_attention_is_refused(cpu_model, kind):
    from neuralmonkey_b200.attention import CoverageAttention
    from neuralmonkey_b200.attention.scaled_dot_product import MultiHeadAttention, ScaledDotProdAttention
    from neuralmonkey_b200.decoders import Decoder
    from neuralmonkey_b200.decoders.word_alignment_decoder import WordAlignmentDecoder
    from neuralmonkey_b200.vocabulary import Vocabulary
    enc = _encoder()
    att, cls = {"coverage": (lambda: CoverageAttention(name="a", encoder=enc), "CoverageAttention"),
                "scaled_dot": (lambda: ScaledDotProdAttention(name="a", keys_encoder=enc), "ScaledDotProdAttention"),
                "multi_head": (lambda: MultiHeadAttention(name="a", n_heads=2, keys_encoder=enc),
                               "MultiHeadAttention")}[kind]
    dec = Decoder(encoders=[enc], vocabulary=Vocabulary(["x"]), data_id="target", name="dec", max_output_len=4,
                  rnn_size=6, embedding_size=6, attentions=[att()])
    with pytest.raises(ValueError, match=cls):
        WordAlignmentDecoder(encoder=enc, decoder=dec, data_id="ali", name="ali")


def test_a_decoder_without_attention_over_the_encoder_is_refused(cpu_model):
    from neuralmonkey_b200.attention import Attention
    from neuralmonkey_b200.decoders import Decoder
    from neuralmonkey_b200.decoders.word_alignment_decoder import WordAlignmentDecoder
    from neuralmonkey_b200.vocabulary import Vocabulary
    enc, other = _encoder(), _encoder("other")
    for attentions in ([], [Attention(name="a", encoder=other)]):
        dec = Decoder(encoders=[enc], vocabulary=Vocabulary(["x"]), data_id="target", name="dec",
                      max_output_len=4, rnn_size=6, embedding_size=6, attentions=attentions)
        with pytest.raises(ValueError, match="no attention over encoder 'enc'"):
            WordAlignmentDecoder(encoder=enc, decoder=dec, data_id="ali", name="ali")


def test_cuda_graph_capture_is_refused(cpu_model):
    with pytest.raises(ValueError, match="use_cuda_graph=True cannot capture.*alignment_decoder"):
        AO.build(use_cuda_graph=True)


# -- run time ------------------------------------------------------------------------------------------------------------
def test_runner_and_decoded_after_a_greedy_run(cpu_model):
    from neuralmonkey_b200.runners import WordAlignmentRunner
    model = AO.build()
    _params(model)
    runner = WordAlignmentRunner("ali", model["att"], model["dec"])
    src, _tgt = random_batch(4, 5, 6, 40, 50, seed=6)
    AO.feed(model, src, None, None, train=False)
    executable = runner.get_executable()
    executable.execute()
    out = executable.result.outputs["ali"]
    steps = model["dec"].runtime_symbols.shape[0]
    assert out.shape == (4, 5, steps) and executable.result.losses == {}
    decoded = model["ali"].decoded
    assert decoded.shape == (4, steps, 5)
    np.testing.assert_allclose(out, decoded.permute(0, 2, 1).numpy())
    # the weights of the greedy run: masked and renormalised
    np.testing.assert_allclose(decoded.sum(-1).numpy(), 1., rtol=1e-5)


def test_runner_without_a_run_history_raises_key_error(cpu_model):
    from neuralmonkey_b200.runners import WordAlignmentRunner
    model = AO.build()
    runner = WordAlignmentRunner("ali", model["att"], model["dec"])
    runner.key = "elsewhere_run"
    src, _tgt = random_batch(2, 5, 6, 40, 50, seed=6)
    AO.feed(model, src, None, None, train=False)
    with pytest.raises(KeyError, match="Attention has no recorded histories under key 'elsewhere_run'"):
        runner.get_executable().execute()


# -- the reference's INI --------------------------------------------------------------------------------------------------
def unpack_alignment_ini(tree: str) -> None:
    from tests.golden.make_reference_bundle import unpack
    unpack(tree)
    with open(os.path.join(ROOT, "tests", "golden", "reference_experiments_alignment.json"), encoding="utf-8") as h:
        for rel, text in json.load(h)["files"].items():
            os.makedirs(os.path.dirname(os.path.join(tree, rel)), exist_ok=True)
            with open(os.path.join(tree, rel), "w", encoding="utf-8") as handle:
                handle.write(text)


# The reference refuses tests/alignment.ini as written: its decoder requires the output projection to be as wide as
# the embeddings (decoders/decoder.py:337-342) and the INI has maxout_size=7 with embedding_size=9.  This port keeps
# that check, so the INI trains with the one override below.
ALIGNMENT_INI_OVERRIDES = ["dec_maxout_output.maxout_size=9"]


def test_alignment_ini_trains(monkeypatch, tmp_path):
    from neuralmonkey_b200 import runtime
    _stand_ins(monkeypatch)
    monkeypatch.setenv("NEURALMONKEY_STRICT", "1")
    unpack_alignment_ini(str(tmp_path / "tree"))
    monkeypatch.chdir(tmp_path / "tree")
    out = str(tmp_path / "alignment")
    argv = ["neuralmonkey-train", "tests/alignment.ini", "-s", 'main.output="{}"'.format(out)]
    for change in ALIGNMENT_INI_OVERRIDES:
        argv += ["-s", change]
    monkeypatch.setattr(sys, "argv", argv)
    try:
        from neuralmonkey_b200.train import main
        main()
    finally:
        runtime.reset()
    log_text = open(os.path.join(out, "experiment.log")).read()
    assert "Training finished" in log_text and "Validation (epoch" in log_text
    assert os.path.exists(os.path.join(out, "variables.data.final"))


def test_alignment_ini_as_written_is_refused_like_the_reference(monkeypatch, tmp_path, capfd):
    from neuralmonkey_b200 import runtime
    _stand_ins(monkeypatch)
    unpack_alignment_ini(str(tmp_path / "tree"))
    monkeypatch.chdir(tmp_path / "tree")
    out = tmp_path / "out"
    monkeypatch.setattr(sys, "argv", ["neuralmonkey-train", "tests/alignment.ini", "-s", 'main.output="{}"'.format(out)])
    try:
        from neuralmonkey_b200.train import main
        with pytest.raises(SystemExit):
            main()
    finally:
        runtime.reset()
    assert ("ValueError: The dimension (7) of the output projection must be same as the dimension of the input "
            "embedding (9)") in capfd.readouterr().err
