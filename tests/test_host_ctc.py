"""CTC on the CPU: the fp64 oracle of tests/ctc_oracle.py against torch's CTC loss and against brute-force
enumeration of every alignment, and the host side of `decoders.ctc_decoder.CTCDecoder` (label extraction,
variables, the projection, the loss and the decoding it hands to the operations) over CPU stand-ins of the two
CTC operations."""
import itertools

import numpy as np
import pytest
import torch

from tests import cpu_ops
from tests import ctc_oracle as CO
from tests.helpers import max_abs, oracle_params_for


def _random_case(seed, bsz, t_max, classes, max_label, merge):
    gen = torch.Generator().manual_seed(seed)
    logits = torch.randn(bsz, t_max, classes, generator=gen, dtype=torch.float64) * 2
    frames = torch.randint(1, t_max + 1, (bsz,), generator=gen)
    labels = torch.randint(0, classes - 1, (bsz, max_label), generator=gen)
    lengths = torch.zeros(bsz, dtype=torch.int32)
    for b in range(bsz):       # the longest label that still fits in the frames, or shorter
        need = 0
        for n in range(max_label + 1):
            need = CO._required_frames(labels[b, :n].tolist(), merge)
            if need > int(frames[b]):
                break
            lengths[b] = n
        lengths[b] = int(torch.randint(0, int(lengths[b]) + 1, (1,), generator=gen)) if b % 2 else lengths[b]
    return logits, frames, labels, lengths


def test_oracle_equals_torch_ctc_loss():
    logits, frames, labels, lengths = _random_case(0, 6, 12, 5, 6, merge=True)
    want = torch.nn.functional.ctc_loss(torch.log_softmax(logits, -1).transpose(0, 1), labels, frames,
                                        lengths.to(torch.int64), blank=4, reduction="none")
    got = CO.ctc_loss(logits, frames, labels, lengths, merge=True)
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-12)


def _brute_force(logits, labels, merge):
    """-log of the summed probability of every path of symbols that maps onto `labels`."""
    t_max, classes = logits.shape
    blank = classes - 1
    probs = torch.softmax(logits, -1)
    total = 0.0
    for path in itertools.product(range(classes), repeat=t_max):
        seq = [k for i, k in enumerate(path) if not (merge and i > 0 and path[i - 1] == k)]
        if [k for k in seq if k != blank] == list(labels):
            total += float(torch.prod(probs[torch.arange(t_max), torch.tensor(path)]))
    return -np.log(total) if total > 0 else None


@pytest.mark.parametrize("merge", [True, False])
def test_oracle_equals_brute_force_enumeration(merge):
    gen = torch.Generator().manual_seed(3)
    cases = [(5, 3, []), (5, 3, [0]), (6, 4, [1, 1]), (6, 4, [0, 2, 0]), (4, 3, [1, 1, 1]), (6, 4, [2, 2, 1, 1]),
             (3, 3, [0, 1, 0, 1])]
    for t_max, classes, lab in cases:
        logits = torch.randn(t_max, classes, generator=gen, dtype=torch.float64)
        want = _brute_force(logits, lab, merge)
        got = CO.ctc_loss(logits[None], [t_max], [lab + [0]], [len(lab)], merge)[0]
        if want is None:         # no alignment: the loss of ignore_longer_outputs_than_inputs
            assert float(got) == 0.0 and CO._required_frames(lab, merge) > t_max
        else:
            assert abs(float(got) - want) < 1e-10, (t_max, classes, lab, float(got), want)


def test_greedy_oracle_ties_and_merging():
    logits = torch.tensor([[[0., 1., 1.], [0., 1., 0.], [0., 0., 2.], [0., 1., 0.], [3., 3., 0.], [0., 0., 0.]]])
    ids, lengths = CO.ctc_greedy_decode(logits, [6], merge=True)      # argmax: 1 1 2 1 0 0 -> 1 1 0
    assert ids.tolist() == [[1, 1, 0, 2, 2, 2]] and lengths.tolist() == [3]
    ids, lengths = CO.ctc_greedy_decode(logits, [6], merge=False)
    assert ids.tolist() == [[1, 1, 1, 0, 0, 2]] and lengths.tolist() == [5]
    ids, lengths = CO.ctc_greedy_decode(logits, [2], merge=True)
    assert ids.tolist() == [[1, 2, 2, 2, 2, 2]] and lengths.tolist() == [1]


# -- the model part over CPU stand-ins of the two CTC operations --------------------------------------------
def ctc_loss_stand_in(logits, frames, labels, label_lengths, merge_repeated):
    return CO.ctc_loss(logits, frames, labels, label_lengths, merge_repeated).to(logits.dtype)


def ctc_greedy_decode_stand_in(logits, frames, merge_repeated):
    return CO.ctc_greedy_decode(logits.detach(), frames, merge_repeated)


@pytest.fixture
def cpu_model(monkeypatch):
    from neuralmonkey_b200 import ops, runtime
    for name in cpu_ops.STAND_INS:
        monkeypatch.setattr(ops, name, getattr(cpu_ops, name))
    monkeypatch.setattr(ops, "ctc_loss", ctc_loss_stand_in)
    monkeypatch.setattr(ops, "ctc_greedy_decode", ctc_greedy_decode_stand_in)
    monkeypatch.setattr(runtime, "_device", torch.device("cpu"))
    yield
    runtime.reset()


def _vocabulary(words):
    from neuralmonkey_b200.vocabulary import Vocabulary
    return Vocabulary(words)


def _model(merge_targets=False, merge_outputs=True, max_length=None):
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.decoders.ctc_decoder import CTCDecoder
    from neuralmonkey_b200.encoders import RecurrentEncoder
    from neuralmonkey_b200.encoders.numpy_stateful_filler import TemporalFiller
    runtime.reset()
    seq = TemporalFiller(name="input_seq", data_id="source", input_size=4)
    enc = RecurrentEncoder(name="audio_encoder", input_sequence=seq, rnn_layers=[(5, "bidirectional"), (6, "forward")])
    dec = CTCDecoder(name="decoder", encoder=enc, vocabulary=_vocabulary(["yes", "no", "maybe"]), data_id="target",
                     max_length=max_length, merge_repeated_targets=merge_targets, merge_repeated_outputs=merge_outputs)
    for part in (seq, enc, dec):
        part.ensure_declared()
    arena = runtime.arena()
    arena.finalize(runtime.device())
    params = oracle_params_for({"arena": arena}, scale=0.5)
    arena.load_dict(params)
    return seq, enc, dec, arena, params


def _feed(parts, features, targets, train=True):
    from neuralmonkey_b200.dataset import BatchingScheme, Dataset
    series = {"source": lambda: iter(features)}
    if targets is not None:
        series["target"] = lambda: iter(targets)
    data = Dataset("toy", series, BatchingScheme(batch_size=len(features)))
    for part in parts:
        part.feed_dict(data, train=train)


TARGETS = [["yes", "no", "no", "yes"], ["no"], [], ["maybe", "maybe", "unknown-word"]]


@pytest.mark.parametrize("merge_targets,merge_outputs", [(False, True), (True, True), (False, False)])
def test_ctc_decoder_against_the_oracle(cpu_model, merge_targets, merge_outputs):
    seq, enc, dec, arena, params = _model(merge_targets, merge_outputs)
    rng = np.random.RandomState(2)
    features = [rng.randn(n, 4).astype(np.float32) for n in (9, 4, 3, 7)]
    _feed((seq, enc, dec), features, TARGETS)
    assert [v for v in arena.order if v.startswith("decoder/")] == ["decoder/state_to_word_W", "decoder/state_to_word_b"]
    assert tuple(arena.get("decoder/state_to_word_W").shape) == (6, 8)      # len(vocabulary) + 1 classes
    # train_targets: the non-<pad> ids in order, <unk> for unknown words; the loss sees them with repeats
    # collapsed when merge_repeated_targets is set
    ids = {w: i for i, w in enumerate(dec.vocabulary._vocabulary)}
    want_targets = [[ids[w] if w in ids else 3 for w in s] for s in TARGETS]
    want_labels = want_targets
    if merge_targets:
        want_labels = [[x for i, x in enumerate(s) if i == 0 or x != s[i - 1]] for s in want_targets]
    for (labels, lengths), want in ((dec.train_targets, want_targets), ((dec._labels, dec._label_lengths), want_labels)):
        assert lengths.tolist() == [len(s) for s in want]
        assert [labels[b, :len(s)].tolist() for b, s in enumerate(want)] == want
        assert labels.shape == (4, 4)
    assert dec.target_tokens[2] == ["<pad>"] * 4
    labels, lengths = dec._labels, dec._label_lengths

    p = {n: v.double().clone().requires_grad_(True) for n, v in params.items()}
    states = enc.temporal_states.detach().double()
    want = CO.ctc_decoder(p, "decoder", states, enc.lengths, labels, lengths, merge_outputs)
    assert abs(float(dec.cost) - float(want["cost"])) < 1e-4
    assert max_abs(dec.logits, want["logits"].transpose(0, 1)) < 1e-5
    assert dec.train_loss is dec.cost and dec.runtime_loss is dec.cost
    assert torch.equal(dec.decoded, want["decoded"])
    dec.cost.backward()
    want["cost"].backward()
    for name in ("decoder/state_to_word_W", "decoder/state_to_word_b"):
        assert max_abs(arena.get(name).grad, p[name].grad) < 1e-4, name


def test_ctc_decoder_runs_without_references_and_in_the_plain_runner(cpu_model):
    from neuralmonkey_b200.runners import PlainRunner
    seq, enc, dec, _, _ = _model()
    features = [np.ones((n, 4), np.float32) for n in (3, 5)]
    _feed((seq, enc, dec), features, None, train=False)
    assert dec.decoded.shape[1] == 2 and dec.target_tokens is None
    with pytest.raises(ValueError):
        _feed((seq, enc, dec), features, None, train=True)
    PlainRunner(output_series="target", decoder=dec)


def test_beam_width_above_one_is_refused(cpu_model):
    from neuralmonkey_b200.decoders.ctc_decoder import CTCDecoder
    from neuralmonkey_b200.encoders.numpy_stateful_filler import TemporalFiller
    seq = TemporalFiller(name="input_seq", data_id="source", input_size=4)
    with pytest.raises(NotImplementedError, match="ctc_beam_search_decoder"):
        CTCDecoder(name="decoder", encoder=seq, vocabulary=_vocabulary(["a"]), data_id="target", beam_width=4)
    with pytest.raises(TypeError):
        CTCDecoder(name="decoder", encoder=seq, vocabulary=_vocabulary(["a"]), data_id="target", beam_width="1")


@pytest.mark.parametrize("tag,max_length,merge_targets,merge_outputs", [
    ("default", None, False, True), ("merge_targets", None, True, True), ("no_merge_out", 4, False, False)])
def test_ctc_decoder_against_the_reference_run(cpu_model, tag, max_length, merge_targets, merge_outputs):
    """The product's CTCDecoder against the reference's own CTCDecoder run over the TF stand-in
    (tests/golden/make_ctc_golden.py): fed tokens, train_targets, variable names and shapes, time-major logits,
    the summed cost (incl. an ignored sentence) and the time-major, </s>-padded decoding."""
    import os
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.decoders.ctc_decoder import CTCDecoder
    from neuralmonkey_b200.model.stateful import TemporalStateful
    golden = np.load(os.path.join(os.path.dirname(__file__), "golden", "ctc_golden.npz"))
    key = tag + "_"
    states, lengths = torch.from_numpy(golden["states"]), torch.from_numpy(golden["lengths"])

    class Encoder(TemporalStateful):
        temporal_states = property(lambda self: states)
        temporal_mask = property(lambda self: (torch.arange(states.shape[1])[None] < lengths[:, None]).float())
        lengths = property(lambda self: lengths)
        dimension = property(lambda self: states.shape[-1])

    runtime.reset()
    dec = CTCDecoder(name="decoder", encoder=Encoder(), vocabulary=_vocabulary(list(golden["words"])),
                     data_id="target", max_length=max_length, merge_repeated_targets=merge_targets,
                     merge_repeated_outputs=merge_outputs)
    dec.ensure_declared()
    arena = runtime.arena()
    arena.finalize(runtime.device())
    assert sorted(arena.order) == golden[key + "variables"].tolist()
    arena.load_dict({"decoder/state_to_word_W": torch.from_numpy(golden[key + "W"]),
                     "decoder/state_to_word_b": torch.from_numpy(golden[key + "b"])})
    sentences = [s.split() for s in golden["sentences"].tolist()]
    from neuralmonkey_b200.dataset import BatchingScheme, Dataset
    dec.feed_dict(Dataset("toy", {"target": lambda: iter(sentences)}, BatchingScheme(batch_size=len(sentences))),
                  train=True)
    assert dec.target_tokens == golden[key + "padded"].tolist()
    labels, label_lengths = dec.train_targets
    assert labels.shape[1] == int(golden[key + "label_shape"][1])
    flat = [(b, k, int(labels[b, k])) for b in range(labels.shape[0]) for k in range(int(label_lengths[b]))]
    assert [(b, k) for b, k, _ in flat] == [tuple(x) for x in golden[key + "label_indices"].tolist()]
    assert [v for _, _, v in flat] == golden[key + "label_values"].tolist()
    assert max_abs(dec.logits, torch.from_numpy(golden[key + "logits"])) < 1e-5
    assert abs(float(dec.cost) - float(golden[key + "cost"])) < 1e-4
    assert torch.equal(dec.decoded, torch.from_numpy(golden[key + "decoded"]))
