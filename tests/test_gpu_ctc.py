"""CTC on the GPU: the K16 kernels through the C ABI against the fp64 oracle of tests/ctc_oracle.py, the
`TemporalFiller -> RecurrentEncoder -> CTCDecoder` model against the oracle, the captured training step, and the
reference's tests/ctc.ini through bin/neuralmonkey-train and bin/neuralmonkey-run on synthetic features."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import nm_oracle as O
from tests import ctc_oracle as CO
from tests.helpers import max_abs, oracle_params_for

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _labels_for(gen, frames, classes, t_max, merge, kind):
    """Labels of one sentence: empty, one symbol, random with repeats, at the feasibility limit, or too long."""
    if kind == "empty":
        return []
    if kind == "one":
        return [int(torch.randint(0, classes - 1, (1,), generator=gen))]
    if kind in ("limit", "too_long"):
        lab = []
        while CO._required_frames(lab, merge) < frames:
            nxt = int(torch.randint(0, classes - 1, (1,), generator=gen))
            if CO._required_frames(lab + [nxt], merge) > frames:
                nxt = next(c for c in range(classes - 1) if not lab or c != lab[-1])
            lab.append(nxt)
        if kind == "too_long":
            lab.append(lab[-1] if merge else 0)
        return lab
    n = int(torch.randint(1, max(2, frames // 3), (1,), generator=gen))
    lab = [int(x) for x in torch.randint(0, classes - 1, (n,), generator=gen)]
    if n > 1:
        lab[1] = lab[0]                      # a repeat
    return lab


KINDS = ("random", "empty", "one", "limit", "too_long", "random", "limit", "one")


def _case(seed, classes, t_max, merge, bsz=8):
    gen = torch.Generator().manual_seed(seed)
    logits = torch.randn(bsz, t_max, classes, generator=gen) * 3
    frames = torch.randint(max(1, t_max // 2), t_max + 1, (bsz,), generator=gen, dtype=torch.int64)
    frames[0] = t_max
    labs = [_labels_for(gen, int(frames[b]), classes, t_max, merge, KINDS[b % len(KINDS)]) for b in range(bsz)]
    width = max(1, max(len(x) for x in labs))
    labels = torch.zeros(bsz, width, dtype=torch.int64)
    for b, lab in enumerate(labs):
        labels[b, :len(lab)] = torch.tensor(lab, dtype=torch.int64)
    lengths = torch.tensor([len(x) for x in labs], dtype=torch.int32)
    return logits, frames.to(torch.int32), labels, lengths


@pytest.mark.parametrize("merge", [True, False])
@pytest.mark.parametrize("classes,t_max", [(3, 9), (7, 40), (33, 128), (1025, 64), (7, 512)])
def test_ctc_loss_kernels_against_fp64(classes, t_max, merge):
    from neuralmonkey_b200 import ops
    logits, frames, labels, lengths = _case(classes * 7 + t_max, classes, t_max, merge)
    x = logits.cuda().requires_grad_(True)
    loss = ops.ctc_loss(x, frames.cuda(), labels.cuda(), lengths.cuda(), merge)
    g = torch.linspace(0.5, 1.5, logits.shape[0])
    loss.backward(g.cuda())

    x64 = logits.double().requires_grad_(True)
    want = CO.ctc_loss(x64, frames, labels, lengths, merge)
    want.backward(g.double())
    got = loss.detach().cpu().double()
    assert torch.all(torch.abs(got - want.detach()) <= torch.clamp(1e-5 * want.detach().abs(), min=1e-4)), (got, want)
    assert max_abs(x.grad, x64.grad) <= 1e-4
    skipped = want.detach() == 0
    for b in range(logits.shape[0]):
        if skipped[b] and lengths[b] > 0:
            assert float(got[b]) == 0.0 and torch.count_nonzero(x.grad[b]) == 0
        assert torch.count_nonzero(x.grad[b, int(frames[b]):]) == 0
    assert bool(skipped.any()), "the grid must contain an infeasible sentence"

    # deterministic: a second call gives the same bits
    x2 = logits.cuda().requires_grad_(True)
    loss2 = ops.ctc_loss(x2, frames.cuda(), labels.cuda(), lengths.cuda(), merge)
    loss2.backward(g.cuda())
    assert torch.equal(loss2, loss) and torch.equal(x2.grad, x.grad)


def test_ctc_loss_refuses_labels_beyond_the_supported_length():
    from neuralmonkey_b200 import ops
    logits = torch.zeros(1, 4, 3, device="cuda")
    labels = torch.zeros(1, 1024, dtype=torch.int64, device="cuda")
    with pytest.raises(ValueError, match="1023"):
        ops.ctc_loss(logits, torch.tensor([4], dtype=torch.int32, device="cuda"), labels,
                     torch.tensor([2], dtype=torch.int32, device="cuda"), True)


@pytest.mark.parametrize("merge", [True, False])
@pytest.mark.parametrize("classes,t_max", [(3, 9), (7, 300), (1025, 40)])
def test_greedy_decode_is_bit_exact(classes, t_max, merge):
    from neuralmonkey_b200 import ops
    gen = torch.Generator().manual_seed(classes + t_max)
    bsz = 6
    # few distinct values: many argmax ties (the lower index wins) and many repeated frames
    logits = torch.randint(0, 3, (bsz, t_max, classes), generator=gen).float()
    frames = torch.randint(0, t_max + 1, (bsz,), generator=gen, dtype=torch.int32)
    frames[0] = t_max
    ids, lengths = ops.ctc_greedy_decode(logits.cuda(), frames.cuda(), merge)
    want_ids, want_lengths = CO.ctc_greedy_decode(logits, frames, merge)
    assert torch.equal(ids.cpu(), want_ids) and torch.equal(lengths.cpu(), want_lengths)


# -- the whole model --------------------------------------------------------------------------------------
VOCAB = ["yes", "no", "maybe"]


def _model(lr=1e-2, cuda_graph=False, keep_prob=1.0):
    from neuralmonkey_b200 import runtime, tf
    from neuralmonkey_b200.decoders.ctc_decoder import CTCDecoder
    from neuralmonkey_b200.encoders import RecurrentEncoder
    from neuralmonkey_b200.encoders.numpy_stateful_filler import TemporalFiller
    from neuralmonkey_b200.trainers import CrossEntropyTrainer
    from neuralmonkey_b200.vocabulary import Vocabulary
    runtime.reset()
    seq = TemporalFiller(name="input_seq", data_id="source", input_size=6)
    enc = RecurrentEncoder(name="audio_encoder", input_sequence=seq, rnn_layers=[(8, "bidirectional"), (12, "forward")],
                           dropout_keep_prob=keep_prob)
    dec = CTCDecoder(name="decoder", encoder=enc, vocabulary=Vocabulary(VOCAB), data_id="target")
    trainer = CrossEntropyTrainer(decoders=[dec], l2_weight=1e-8, optimizer=tf.AdamOptimizer(learning_rate=lr),
                                  use_cuda_graph=cuda_graph)
    for part in (seq, enc, dec):
        part.ensure_declared()
    arena = runtime.arena()
    arena.finalize(runtime.device())
    return seq, enc, dec, trainer, arena


def _synthetic(seed, n, frames_per_word=3):
    """Sentences over VOCAB and their feature sequences: a word is `frames_per_word` frames of its own pattern plus
    noise, words are separated by a silent frame."""
    rng = np.random.RandomState(seed)
    patterns = np.eye(6, dtype=np.float32)[:len(VOCAB)] * 2
    sents, feats = [], []
    for _ in range(n):
        words = [VOCAB[i] for i in rng.randint(0, len(VOCAB), rng.randint(0, 5))]
        frames = [np.zeros(6, np.float32)]
        for w in words:
            frames += [patterns[VOCAB.index(w)]] * frames_per_word + [np.zeros(6, np.float32)]
        feats.append((np.stack(frames) + 0.1 * rng.randn(len(frames), 6)).astype(np.float32))
        sents.append(words)
    return sents, feats


def _feed(parts, feats, sents, train=True):
    from neuralmonkey_b200.dataset import BatchingScheme, Dataset
    series = {"source": lambda: iter(feats)}
    if sents is not None:
        series["target"] = lambda: iter(sents)
    data = Dataset("toy", series, BatchingScheme(batch_size=len(feats)))
    for part in parts:
        part.feed_dict(data, train=train)


def test_ctc_model_against_the_oracle():
    from neuralmonkey_b200 import ops
    try:
        ops.set_gemm_backend("simt")
        seq, enc, dec, _, arena = _model()
        params = oracle_params_for({"arena": arena}, scale=0.5)
        arena.load_dict(params)
        sents, feats = _synthetic(0, 7)
        sents[1] = ["yes", "yes", "no", "no", "no", "yes", "maybe", "maybe", "yes", "yes", "no", "no", "yes", "no"]
        _feed((seq, enc, dec), feats, sents)
        arena.zero_grad()
        dec.cost.backward()
        arena.fold_autograd_grads()

        p = {n: v.double().clone().requires_grad_(True) for n, v in params.items()}
        oenc = O.recurrent_encoder(p, "audio_encoder", seq.temporal_states.double().cpu(), seq.temporal_mask.cpu(),
                                   [(8, "bidirectional", "GRU"), (12, "forward", "GRU")], False, False, True)
        labels, lengths = dec.train_targets
        want = CO.ctc_decoder(p, "decoder", oenc["temporal_states"], enc.lengths.cpu(), labels.cpu(), lengths.cpu(),
                              True)
        assert float(want["losses"][1]) == 0.0          # more labels than frames: ignored
        assert abs(float(dec.cost) - float(want["cost"])) <= max(1e-4, 1e-5 * abs(float(want["cost"])))
        assert max_abs(dec.logits, want["logits"].transpose(0, 1)) < 2e-5
        assert torch.equal(dec.decoded.cpu(), want["decoded"])
        want["cost"].backward()
        for name in arena.train_names:
            assert max_abs(arena.grad(name), p[name].grad) < 5e-5, name
    finally:
        ops.set_gemm_backend("auto")


def test_captured_training_step_is_bit_identical_to_eager():
    from neuralmonkey_b200 import ops
    try:
        ops.set_gemm_backend("simt")
        results = {}
        for mode in (False, True):
            seq, enc, dec, trainer, arena = _model(cuda_graph=mode)
            arena.load_dict(oracle_params_for({"arena": arena}, scale=0.5))
            sents, feats = _synthetic(5, 6)
            feats = [np.resize(f, (13, 6)) for f in feats]          # one shape: the captured graph is replayed
            losses = []
            for step in range(3):
                _feed((seq, enc, dec), feats, sents[step:] + sents[:step])
                losses.append(trainer.train_step()["losses"][0].item())
            results[mode] = (losses, arena.state_dict())
            if mode:
                assert any(isinstance(v, tuple) for v in trainer._graphs.values()), trainer._graphs
        assert results[True][0] == results[False][0]
        for name, want in results[False][1].items():
            assert torch.equal(results[True][1][name], want), name
    finally:
        ops.set_gemm_backend("auto")


LEARN_STEPS = 150


def test_a_synthetic_task_is_learned():
    """The training labels decode exactly after LEARN_STEPS Adam steps on one batch."""
    seq, enc, dec, trainer, arena = _model(lr=2e-2)
    sents, feats = _synthetic(11, 16)
    for _ in range(LEARN_STEPS):
        _feed((seq, enc, dec), feats, sents)
        trainer.train_step()
    _feed((seq, enc, dec), feats, None, train=False)
    got = dec.vocabulary.vectors_to_sentences(dec.decoded.cpu().numpy())
    assert got == sents


# -- the reference's tests/ctc.ini through the entry points ----------------------------------------------
def feature_reader(files):
    """Feature sequences stored as the arrays of .npz archives, in the order of their names."""
    for path in files:
        with np.load(path) as archive:
            for key in sorted(archive.files):
                yield archive[key]


CTC_INI = """
[main]
name="speech recognition using CTC"
tf_manager=<tf_manager>
output="{out}"
overwrite_output_dir=True

batch_size=4
epochs=5

train_dataset=<train_data>
val_dataset=<val_data>
test_datasets=[<val_data>]

trainer=<trainer>
runners=[<runner>]

evaluation=[("target", evaluators.WER)]

logging_period=1
# ctc.ini validates every "5s"; this toy run is over sooner than that, so it validates every 5 batches
validation_period=5

random_seed=123485

[tf_manager]
class=tf_manager.TensorFlowManager
num_threads=16
num_sessions=1
minimize_metric=True

[train_data]
class=dataset.load
series=["source", "target"]
data=[("{data}/train.npz", tests.test_gpu_ctc.feature_reader), "{data}/train.txt"]

[val_data]
class=dataset.load
series=["source", "target"]
data=[("{data}/test.npz", tests.test_gpu_ctc.feature_reader), "{data}/test.txt"]

[decoder_vocabulary]
class=vocabulary.from_wordlist
path="{data}/yesno.vocab"
contains_header=False
contains_frequencies=False

[input_seq]
class=encoders.numpy_stateful_filler.TemporalFiller
data_id="source"
input_size=39

[audio_encoder]
class=encoders.RecurrentEncoder
input_sequence=<input_seq>
rnn_layers=[(50,"bidirectional"),(100,"forward"),(100,"backward")]
dropout_keep_prob=0.5

[decoder]
class=decoders.ctc_decoder.CTCDecoder
encoder=<audio_encoder>
vocabulary=<decoder_vocabulary>
data_id="target"
name="decoder"

[trainer]
class=trainers.cross_entropy_trainer.CrossEntropyTrainer
decoders=[<decoder>]
l2_weight=1.0e-8

[runner]
class=runners.PlainRunner
decoder=<decoder>
output_series="target"
"""


def _write_ctc_data(path):
    """yes/no sentences of 8 words with 39-dimensional feature sequences (the MFCC + deltas width of ctc.ini)."""
    rng = np.random.RandomState(0)
    os.makedirs(path, exist_ok=True)
    with open(os.path.join(path, "yesno.vocab"), "w") as f:
        f.write("yes\nno\n")
    for split, n in (("train", 12), ("test", 6)):
        arrays, lines = {}, []
        for i in range(n):
            words = [("yes", "no")[k] for k in rng.randint(0, 2, 8)]
            arrays["s{:03d}".format(i)] = rng.randn(rng.randint(40, 80), 39).astype(np.float32)
            lines.append(" ".join(words))
        np.savez(os.path.join(path, split + ".npz"), **arrays)
        with open(os.path.join(path, split + ".txt"), "w") as f:
            f.write("\n".join(lines) + "\n")


def _run(cmd):
    env = dict(os.environ, NEURALMONKEY_STRICT="1")
    return subprocess.run([sys.executable] + cmd, capture_output=True, text=True, timeout=900, cwd=ROOT, env=env)


def test_ctc_ini_trains_and_runs(tmp_path):
    data, out = str(tmp_path / "data"), str(tmp_path / "out")
    _write_ctc_data(data)
    ini = tmp_path / "ctc.ini"
    ini.write_text(CTC_INI.format(out=out, data=data))
    res = _run(["bin/neuralmonkey-train", str(ini)])
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert os.path.exists(os.path.join(out, "variables.data.final"))
    log_text = open(os.path.join(out, "experiment.log")).read()
    assert "target/WER" in log_text

    run_ini = tmp_path / "run.ini"
    run_ini.write_text("""
[main]
test_datasets=[<val_data>]

[batching]
class=dataset.BatchingScheme
batch_size=4

[val_data]
class=dataset.load
series=["source", "target"]
data=[("{data}/test.npz", tests.test_gpu_ctc.feature_reader), "{data}/test.txt"]
outputs=[("target", "{out}/run.out")]
batching=<batching>
""".format(data=data, out=out))
    res = _run(["bin/neuralmonkey-run", str(ini), str(run_ini), "--json", str(tmp_path / "res.json")])
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert "target/WER" in json.load(open(tmp_path / "res.json"))[0]
    assert len(open(os.path.join(out, "run.out")).read().splitlines()) == 6
