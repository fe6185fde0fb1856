"""The sentence classification / regression kernels (csrc/classify.cu) and model parts on the GPU: every kernel
against the fp64 restatement of tests/classifier_oracle.py over a grid of shapes (T = 1, T = filter width, odd
sizes, widths that force the exact GEMM, B up to 512, R from 1 to 32), constructed exact ties, bit-identical repeat
calls, the classifier stack on the device against the same stack over the restatement on the CPU, and the
reference's tests/classifier.ini and tests/regressor.ini through bin/neuralmonkey-train."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import classifier_oracle as CLO
from tests.helpers import training_log_values

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda"


@pytest.fixture
def engine(request):
    from neuralmonkey_b200 import ops
    ops.set_gemm_backend(request.param)
    yield request.param
    ops.set_gemm_backend("auto")


def _mask(b, t, gen):
    """Random lengths in [1, t], the first sentence full length."""
    lengths = torch.randint(1, t + 1, (b,), generator=gen)
    lengths[0] = t
    return (torch.arange(t)[None, :] < lengths[:, None]).float()


def _check(got, want, rtol, atol, what):
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    assert got.shape == want.shape, what
    err = float((got - want).abs().max()) if got.numel() else 0.0
    assert torch.allclose(got, want, rtol=rtol, atol=atol), "{}: max abs err {}".format(what, err)


def _run(fn, inputs, dout, grads):
    """(outputs, gradients of the inputs flagged in `grads`) of sum(out * dout)."""
    leaves = [None if x is None else x.detach().clone().requires_grad_(g) for x, g in zip(inputs, grads)]
    out = fn(*leaves)
    outs = out if isinstance(out, tuple) else (out,)
    sum((o * d).sum() for o, d in zip(outs, dout if isinstance(dout, tuple) else (dout,))).backward()
    return outs, [x.grad if g else None for x, g in zip(leaves, grads)]


POOL_SHAPES = [(1, 1, 1), (3, 7, 5), (4, 13, 33), (2, 50, 600), (512, 50, 64)]


@pytest.mark.parametrize("shape", POOL_SHAPES)
@pytest.mark.parametrize("masked", [True, False])
@pytest.mark.parametrize("kind", ["max", "mean"])
def test_pooling_against_the_oracle(shape, masked, kind):
    from neuralmonkey_b200 import ops
    b, t, d = shape
    gen = torch.Generator().manual_seed(b * 1000 + t * 10 + d)
    x = torch.randn(b, t, d, generator=gen)
    if b > 1:
        x[1] = -x[1].abs() - 0.1                      # an all-negative sentence: pools to 1e-15 where padded
    mask = _mask(b, t, gen) if masked else None
    if masked and b > 1 and t > 1:
        mask[1, t - 1:] = 0                         # sentence 1 is padded: its all-negative values meet the 1e-15
    dy = torch.randn(b, d, generator=gen)
    ours, oracle = (ops.seq_max_pool, CLO.seq_max_pool) if kind == "max" else (ops.seq_mean_pool, CLO.seq_mean_pool)
    (y,), (dx, _) = _run(ours, [x.to(DEV), None if mask is None else mask.to(DEV)], dy.to(DEV), (True, False))
    (y64,), (dx64, _) = _run(oracle, [x.double(), None if mask is None else mask.double()], dy.double(),
                             (True, False))
    # the max is exact; the mean sums T fp32 products in order
    tol = (1e-6, 1e-12) if kind == "max" else (1e-5, 1e-6)
    _check(y, y64, *tol, "forward")
    _check(dx, dx64, *tol, "backward")


def test_max_pool_splits_exact_ties_equally():
    from neuralmonkey_b200 import ops
    gen = torch.Generator().manual_seed(7)
    b, t, d = 64, 21, 37
    x = torch.randint(-2, 3, (b, t, d), generator=gen).float()          # many exact ties
    mask = _mask(b, t, gen)
    mask[2] = 0.0
    mask[2, :5] = 1.0
    x[2] = 0.0          # valid maximum 0 below the padded positions' 1e-15: no gradient reaches the sentence
    dy = torch.randn(b, d, generator=gen)
    (y,), (dx, _) = _run(ops.seq_max_pool, [x.to(DEV), mask.to(DEV)], dy.to(DEV), (True, False))
    (y64,), (dx64, _) = _run(CLO.seq_max_pool, [x.double(), mask.double()], dy.double(), (True, False))
    _check(y, y64, 1e-6, 1e-12, "forward")
    _check(dx, dx64, 1e-6, 1e-12, "backward")
    counts = (x == x.amax(1, keepdim=True)).sum(1)
    assert int(counts.max()) > 3                                          # the grid does tie


def test_empty_batch_is_refused():
    from neuralmonkey_b200 import ops
    with pytest.raises(ValueError, match="mask sum"):
        ops.seq_max_pool(torch.ones(2, 3, 4, device=DEV), torch.zeros(2, 3, device=DEV))


# (B, T, R, D)
ATT_SHAPES = [(1, 1, 1, 1), (3, 7, 1, 5), (5, 13, 32, 33), (4, 64, 8, 301), (512, 50, 30, 64), (2, 512, 32, 20)]


@pytest.mark.parametrize("shape", ATT_SHAPES)
@pytest.mark.parametrize("masked", [True, False])
def test_attentive_pool_against_the_oracle(shape, masked):
    from neuralmonkey_b200 import ops
    b, t, r, d = shape
    gen = torch.Generator().manual_seed(b + t + r + d)
    e, v = torch.randn(b, t, r, generator=gen) * 2, torch.randn(b, t, d, generator=gen)
    mask = _mask(b, t, gen) if masked else None
    dw, dout = torch.randn(b, t, r, generator=gen), torch.randn(b, r, d, generator=gen)

    def run(fn, dev, dtype):
        leaves = [e.to(dev, dtype).requires_grad_(), None if mask is None else mask.to(dev, dtype),
                  v.to(dev, dtype).requires_grad_()]
        w, out = fn(*leaves)
        ((w * dw.to(dev, dtype)).sum() + (out * dout.to(dev, dtype)).sum()).backward()
        return w, out, leaves[0].grad, leaves[2].grad

    got, want = run(ops.attentive_pool, DEV, torch.float32), run(CLO.attentive_pool, "cpu", torch.float64)
    for name, g, w in zip(("weights", "out", "denergies", "dstates"), got, want):
        _check(g, w, 1e-4, 1e-5, name)


def test_attentive_pool_refuses_more_than_32_heads():
    from neuralmonkey_b200 import ops
    with pytest.raises(ValueError, match="R <= 32"):
        ops.attentive_pool(torch.zeros(1, 2, 33, device=DEV), None, torch.zeros(1, 2, 4, device=DEV))


# (B, T, E, width, F): T = 1 = width, T = width, odd E (exact GEMM), the realistic Kim-CNN shape
CONV_SHAPES = [(1, 1, 4, 1, 8), (2, 3, 4, 3, 5), (3, 7, 5, 2, 3), (5, 11, 12, 4, 7), (64, 50, 300, 5, 100)]
TOL = {"auto": 1e-2, "simt": 2e-5}


@pytest.mark.parametrize("engine", ["auto", "simt"], indirect=True)
@pytest.mark.parametrize("shape", CONV_SHAPES)
def test_conv1d_max_pool_against_the_oracle(engine, shape):
    from neuralmonkey_b200 import ops
    b, t, e, width, f = shape
    gen = torch.Generator().manual_seed(b + t + e + width + f)
    x, w, bias = torch.randn(b, t, e, generator=gen), torch.randn(width, e, f, generator=gen) * 0.3, \
        torch.randn(f, generator=gen) * 0.1
    dy = torch.randn(b, f, generator=gen)

    def run(dev, dtype, fn):
        leaves = [a.to(dev, dtype).requires_grad_() for a in (x, w, bias)]
        y = fn(*leaves)
        (y * dy.to(dev, dtype)).sum().backward()
        return [y] + [a.grad for a in leaves]

    got, want = run(DEV, torch.float32, ops.conv1d_max_pool), run("cpu", torch.float64, CLO.conv1d_max_pool)
    for name, g, wv in zip(("out", "dx", "dw", "dbias"), got, want):
        scale = float(wv.detach().abs().max()) or 1.0
        _check(g, wv, 0.0, TOL[engine] * scale, name)


def test_conv1d_refuses_a_batch_shorter_than_the_filter():
    from neuralmonkey_b200 import ops
    with pytest.raises(ValueError, match="shorter than the filter"):
        ops.conv1d_max_pool(torch.zeros(2, 2, 4, device=DEV), torch.zeros(3, 4, 5, device=DEV),
                            torch.zeros(5, device=DEV))


def test_conv1d_splits_ties_of_identical_pad_windows():
    """Identical windows (all-<pad> sentences) tie exactly: the gradient is split among them."""
    from neuralmonkey_b200 import ops
    x = torch.zeros(2, 6, 8)
    x[0, :2] = torch.randn(2, 8)
    w, bias = torch.randn(2, 8, 4) * 0.3, torch.full((4,), 0.5)
    dy = torch.randn(2, 4)
    ops.set_gemm_backend("simt")
    try:
        (y,), (dx, dw, db) = _run(ops.conv1d_max_pool, [x.to(DEV), w.to(DEV), bias.to(DEV)], dy.to(DEV),
                                         (True, True, True))
    finally:
        ops.set_gemm_backend("auto")
    (y64,), (dx64, dw64, db64) = _run(CLO.conv1d_max_pool, [x.double(), w.double(), bias.double()], dy.double(),
                                     (True, True, True))
    for name, g, wv in (("out", y, y64), ("dx", dx, dx64), ("dw", dw, dw64), ("dbias", db, db64)):
        _check(g, wv, 1e-5, 1e-6, name)
    # sentence 1 is all <pad>: its five windows tie, and each gets a fifth of dy through every tap
    assert float(dx[1].abs().sum()) > 0


@pytest.mark.parametrize("shape", [(1, 1), (7, 1), (512, 3), (100, 33)])
def test_squared_error_against_the_oracle(shape):
    from neuralmonkey_b200 import ops
    gen = torch.Generator().manual_seed(shape[0])
    pred, target = torch.randn(*shape, generator=gen), torch.randn(shape[0], generator=gen)
    (loss,), (dpred, _) = _run(ops.squared_error, [pred.to(DEV), target.to(DEV)], torch.tensor(1.5, device=DEV),
                                 (True, False))
    (l64,), (d64, _) = _run(CLO.squared_error, [pred.double(), target.double()], torch.tensor(1.5).double(), (True, False))
    _check(loss, l64, 1e-5, 1e-7, "loss")
    _check(dpred, d64, 1e-5, 1e-7, "dpred")


def test_repeat_backward_calls_are_bit_identical():
    from neuralmonkey_b200 import ops
    gen = torch.Generator().manual_seed(3)
    b, t, r, d = 256, 50, 30, 600
    e, v, mask = torch.randn(b, t, r, generator=gen).to(DEV), torch.randn(b, t, d, generator=gen).to(DEV), \
        _mask(b, t, gen).to(DEV)
    dout = torch.randn(b, r, d, generator=gen).to(DEV)
    w, bias = torch.randn(4, d, 100, generator=gen).to(DEV) * 0.05, torch.zeros(100, device=DEV)
    runs = []
    ops.set_gemm_backend("simt")      # (the tensor-core GEMM's split-K weight gradients add partial tiles atomically)
    for _ in range(2):
        ee, vv = e.clone().requires_grad_(), v.clone().requires_grad_()
        ww, bb = w.clone().requires_grad_(), bias.clone().requires_grad_()
        _, out = ops.attentive_pool(ee, mask, vv)
        pooled = ops.seq_max_pool(vv, mask) + ops.seq_mean_pool(vv, mask)
        pred = pooled[:, :3]
        conv = ops.conv1d_max_pool(vv, ww, bb)
        ((out * dout).sum() + pooled.sum() + ops.squared_error(pred, pooled[:, 5].detach()) + conv.sum()).backward()
        runs.append((out, ee.grad, vv.grad, conv, ww.grad, bb.grad))
    ops.set_gemm_backend("auto")
    for a, b_ in zip(*runs):
        assert torch.equal(a, b_)


# -- model parts ----------------------------------------------------------------------------------------------------
def _build_stack():
    from neuralmonkey_b200.decoders.classifier import Classifier
    from neuralmonkey_b200.decoders.sequence_regressor import SequenceRegressor
    from neuralmonkey_b200.encoders.attentive import AttentiveEncoder
    from neuralmonkey_b200.encoders.pooling import SequenceMaxPooling
    from neuralmonkey_b200.encoders.recurrent import SentenceEncoder
    from neuralmonkey_b200.encoders.sequence_cnn_encoder import SequenceCNNEncoder
    from neuralmonkey_b200.model.gradient_reversal import StatefulView
    from neuralmonkey_b200.vocabulary import Vocabulary
    words = Vocabulary(list("abcdefgh"))
    enc = SentenceEncoder(name="enc", vocabulary=words, data_id="source", embedding_size=12, rnn_size=8)
    att = AttentiveEncoder(name="att", input_sequence=enc, hidden_size=9, num_heads=5, output_size=13)
    maxp = SequenceMaxPooling(name="maxp", input_sequence=enc)
    cnn = SequenceCNNEncoder(name="cnn", vocabulary=words, data_id="source", embedding_size=12,
                             filters=[(2, 8), (3, 4)])
    clf = Classifier(name="clf", encoders=[att, maxp, cnn], vocabulary=Vocabulary(["x", "y", "z"]),
                     data_id="label", layers=[10, 5], dropout_keep_prob=1.0)
    adv = Classifier(name="adv", encoders=[StatefulView(maxp)], vocabulary=Vocabulary(["x", "y", "z"]),
                     data_id="label", layers=[], dropout_keep_prob=1.0)
    reg = SequenceRegressor(name="reg", encoders=[enc], data_id="value", layers=[6], dimension=2)
    return [enc.input_sequence, enc, att, maxp, cnn, clf, adv, reg]


class _Data:
    def __init__(self, series):
        self.series = series

    def __len__(self):
        return len(next(iter(self.series.values())))

    def get_series(self, name):
        return self.series[name]

    def maybe_get_series(self, name):
        return self.series.get(name)


@pytest.mark.parametrize("engine", ["auto", "simt"], indirect=True)
def test_classifier_stack_on_the_device_matches_the_restatement(monkeypatch, engine):
    """The same variables, the same batch: the model parts on the kernels against the model parts over the
    restatement on the CPU (outputs, losses, decisions).  On the exact engine every product is fp32; on `auto` the
    dense products take TF32 operands and the classification layer fp16 ones (fp32 accumulation)."""
    from neuralmonkey_b200 import ops, runtime
    from tests import cpu_ops
    rng = np.random.RandomState(0)
    sentences = [[str(c) for c in rng.choice(list("abcdefgh"), size=rng.randint(3, 9))] for _ in range(37)]
    data = _Data({"source": sentences, "label": [[rng.choice(["x", "y", "z"])] for _ in sentences],
                  "value": [[float(rng.randn())] for _ in sentences]})

    def declare(parts):
        for p in parts:
            p.ensure_declared()
        arena = runtime.arena()
        arena.finalize(runtime.device())
        return arena

    def evaluate(parts):
        for p in parts:
            p.feed_dict(data, train=False)
        enc, att, maxp, cnn, clf, adv, reg = parts[1:]
        return {"att": att.output, "weights": att.attention_weights, "maxp": maxp.output, "cnn": cnn.output,
                "logits": clf.decoded_logits, "logprobs": clf.runtime_logprobs, "loss": clf.cost,
                "adv_loss": adv.cost, "pred": reg.predictions, "mse": reg.cost}

    runtime.reset()
    parts = _build_stack()
    arena = declare(parts)
    variables = {n: arena.get(n).detach().cpu().clone() for n in arena.order}
    got = {k: v.detach().cpu() for k, v in evaluate(parts).items()}
    runtime.reset()
    with monkeypatch.context() as patch:
        for op in cpu_ops.STAND_INS:
            patch.setattr(ops, op, getattr(cpu_ops, op))
        for op in CLO.STAND_INS:
            patch.setattr(ops, op, getattr(CLO, op))
        patch.setattr(runtime, "_device", torch.device("cpu"))
        parts = _build_stack()
        arena = declare(parts)
        arena.load_dict(variables)
        want = evaluate(parts)
        runtime.reset()
    for name in want:
        tol = 1e-4 if engine == "simt" else 2e-2
        _check(got[name], want[name], tol, tol, name)


@pytest.mark.parametrize("engine", ["auto", "simt"], indirect=True)
@pytest.mark.parametrize("tag", CLO.MODEL_CASES)
def test_model_parts_against_the_reference_code(engine, tag):
    """The model parts on the kernels, with the variables of the reference's own graph loaded by name
    (tests/golden/make_classifier_golden.py).  Exact engine: fp32 products; auto: TF32 dense products and, for the
    classifier's output layer, fp16 operands with fp32 accumulation."""
    from neuralmonkey_b200 import runtime
    g = CLO.golden()
    try:
        got = CLO.golden_model_outputs(g, tag, DEV)
        for name, value in got.items():
            want = torch.from_numpy(np.asarray(g[tag + "_" + name] if tag not in ("maxpool", "avgpool")
                                               else g[tag + "_output"]))
            tol = 1e-5 if engine == "simt" or tag in ("maxpool", "avgpool") else 1e-2
            _check(value, want, tol, tol, "{} {}".format(tag, name))
    finally:
        runtime.reset()


class _States:
    """A fixed batch of encoder states for the optimiser-step tests."""

    def __init__(self):
        gen = torch.Generator().manual_seed(5)
        self.states = torch.randn(8, 7, 12, generator=gen)
        self.mask = torch.ones(8, 7)
        self.mask[3, 4:] = 0
        self.mask[5, 2:] = 0
        self.ids = torch.randint(4, 13, (8, 7), generator=gen)
        self.ids[3, 4:] = 0
        self.labels = torch.randint(0, 7, (8,), generator=gen)


def _trainer_stack(batch, adversary):
    from neuralmonkey_b200 import runtime, tf
    from neuralmonkey_b200.decoders.classifier import Classifier
    from neuralmonkey_b200.encoders.attentive import AttentiveEncoder
    from neuralmonkey_b200.encoders.pooling import SequenceMaxPooling
    from neuralmonkey_b200.encoders.sequence_cnn_encoder import SequenceCNNEncoder
    from neuralmonkey_b200.model.gradient_reversal import StatefulView
    from neuralmonkey_b200.model.stateful import TemporalStateful
    from neuralmonkey_b200.trainers import CrossEntropyTrainer
    from neuralmonkey_b200.vocabulary import Vocabulary
    dev = runtime.device()

    class Seq(TemporalStateful):
        temporal_states = property(lambda self: batch.states.to(dev))
        temporal_mask = property(lambda self: batch.mask.to(dev))
        dimension = 12

    seq = Seq()
    att = AttentiveEncoder(name="att", input_sequence=seq, hidden_size=9, num_heads=5, output_size=13)
    maxp = SequenceMaxPooling(name="maxp", input_sequence=seq)
    cnn = SequenceCNNEncoder(name="cnn", vocabulary=Vocabulary(["w{}".format(i) for i in range(9)]),
                             data_id="source", embedding_size=8, filters=[(2, 4), (3, 4)])
    labels = Vocabulary(["l{}".format(i) for i in range(3)])
    clf = Classifier(name="clf", encoders=[att, maxp, cnn], vocabulary=labels, data_id="label", layers=[10, 5],
                     dropout_keep_prob=1.0)
    decoders = [clf]
    if adversary:
        decoders.append(Classifier(name="adv", encoders=[StatefulView(att)], vocabulary=labels, data_id="label",
                                   layers=[], dropout_keep_prob=1.0))
    trainer = CrossEntropyTrainer(decoders=decoders, l2_weight=1e-8, clip_norm=1.0,
                                  optimizer=tf.AdamOptimizer(learning_rate=1e-2))
    for part in trainer.parameterizeds:
        part.ensure_declared()
    runtime.arena().finalize(dev)
    cnn._ids = batch.ids.to(dev)
    for dec in decoders:
        dec._labels = batch.labels.to(dev)
    for part in (att, maxp, cnn) + tuple(decoders):
        part.train_mode = True
    return trainer


@pytest.mark.parametrize("adversary", [False, True])
def test_one_optimiser_step_against_the_restatement(monkeypatch, adversary):
    """One Adam step of a classifier over attentive pooling, max pooling and a Kim CNN: alone (the exact
    single-objective path: the trainer differentiates the cross-entropy SUM and divides by the batch size on the
    device) and with a second classifier behind a gradient-reversal view (the summed objectives).  The updated
    variables on the exact engine against the same step over the restatement on the CPU."""
    from neuralmonkey_b200 import ops, runtime
    from neuralmonkey_b200.trainers.generic_trainer import GenericTrainer
    from tests import cpu_ops
    batch = _States()
    ops.set_gemm_backend("simt")
    try:
        runtime.reset()
        trainer = _trainer_stack(batch, adversary)
        arena = runtime.arena()
        assert (trainer.objectives[0].loss_sum_and_count is not None) and len(trainer.objectives) == 1 + adversary
        before = {n: arena.get(n).detach().cpu().clone() for n in arena.order}
        out = trainer.train_step()
        loss = float(out["losses"][0])
        after = {n: arena.get(n).detach().cpu().clone() for n in arena.order}
    finally:
        ops.set_gemm_backend("auto")
        runtime.reset()
    with monkeypatch.context() as patch:
        for op in cpu_ops.STAND_INS:
            patch.setattr(ops, op, getattr(cpu_ops, op))
        for op in CLO.STAND_INS:
            patch.setattr(ops, op, getattr(CLO, op))
        patch.setattr(runtime, "_device", torch.device("cpu"))
        patch.setattr(GenericTrainer, "_adam_kernel", cpu_ops.adam_kernel)
        try:
            trainer = _trainer_stack(batch, adversary)
            arena = runtime.arena()
            arena.load_dict(before)
            want_loss = float(trainer.train_step()["losses"][0])
            want = {n: arena.get(n).detach().clone() for n in arena.order}
        finally:
            runtime.reset()
    assert abs(loss - want_loss) < 1e-5 * max(1.0, abs(want_loss))
    moved = 0
    for name in want:
        _check(after[name], want[name], 1e-4, 1e-5, name)
        moved += int(not torch.equal(after[name], before[name]))
    assert moved == len(want)         # every variable got a gradient, the adversary's through the reversal too


@pytest.mark.parametrize("name,series,metric", [("classifier", "classification", "classification/Accuracy"),
                                                ("regressor", "regression", "regression/MeanSquaredError")])
def test_reference_ini_trains_unchanged_on_the_gpu(tmp_path, name, series, metric):
    from tests.golden.make_classifier_bundle import unpack
    tree, out = tmp_path / "tree", str(tmp_path / "out")
    unpack(str(tree))
    cmd = [sys.executable, os.path.join(ROOT, "bin", "neuralmonkey-train"), "tests/{}.ini".format(name),
           "-s", 'main.output="{}"'.format(out)]
    env = dict(os.environ, NEURALMONKEY_STRICT="1", PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=str(tree), env=env)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    log_text = open(os.path.join(out, "experiment.log")).read()
    assert "Training finished" in log_text and "Validation (epoch" in log_text
    assert os.path.exists(os.path.join(out, "variables.data.final"))
    assert metric + ": " in log_text
    losses = training_log_values(log_text, series + ("/train_xent" if name == "classifier" else "/mse"))
    assert losses and all(np.isfinite(losses)), log_text[-2000:]
