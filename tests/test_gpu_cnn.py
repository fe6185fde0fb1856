"""The trainable CNN encoder on the GPU: the kernels of csrc/cnn.cu and nm_clip_adadelta_step against the fp64
restatement of tests/cnn_oracle.py, the whole CNNEncoder / CNNTemporalView against it, a captured training step, and
the reference's tests/str.ini through bin/neuralmonkey-train (inputs from tests/golden/reference_experiments_str.json)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import cnn_oracle as CO
from tests.helpers import training_log_values

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def engine(request):
    from neuralmonkey_b200 import ops
    ops.set_gemm_backend(request.param)
    yield request.param
    ops.set_gemm_backend("auto")


def _rel(got: torch.Tensor, want: torch.Tensor) -> float:
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    return float((got - want).abs().max() / want.abs().max().clamp_min(1e-30))


# TF32 operands keep 10 mantissa bits: relative to the largest output, sums of a few thousand products stay well
# inside 1e-2; the exact engine only reorders fp32 sums
TOL = {"auto": 1e-2, "simt": 2e-5}

# (N, H, W, Cin, Cout, k, padding)
CONV_SHAPES = [
    (1, 5, 7, 1, 3, 1, "same"), (2, 9, 11, 1, 4, 3, "valid"), (3, 8, 6, 3, 5, 2, "same"), (2, 7, 9, 6, 70, 2, "valid"),
    (1, 12, 10, 13, 17, 5, "same"), (2, 11, 13, 5, 9, 5, "valid"), (4, 16, 20, 16, 64, 3, "same"),
    (2, 10, 30, 64, 130, 3, "same"), (1, 6, 6, 4, 4, 3, "valid"), (5, 15, 17, 12, 12, 3, "same"),
]


@pytest.mark.parametrize("engine", ["auto", "simt"], indirect=True)
@pytest.mark.parametrize("shape", CONV_SHAPES)
def test_conv2d_forward_and_gradients(engine, shape):
    from neuralmonkey_b200 import ops
    n, h, w, cin, cout, k, pad = shape
    gen = torch.Generator().manual_seed(sum(shape[:6]))
    x = torch.randn(n, h, w, cin, generator=gen)
    wt = torch.randn(k, k, cin, cout, generator=gen) / (k * np.sqrt(cin))
    b = torch.randn(cout, generator=gen)
    xd, wd, bd = (t.cuda().requires_grad_(True) for t in (x, wt, b))
    y = ops.conv2d(xd, wd, bd, pad)
    xr, wr, br = (t.double().requires_grad_(True) for t in (x, wt, b))
    yr = CO.conv2d(xr, wr, br, pad)
    assert y.shape == yr.shape
    assert _rel(y, yr) < TOL[engine]
    g = torch.randn(yr.shape, generator=gen)
    y.backward(g.cuda())
    yr.backward(g.double())
    assert _rel(xd.grad, xr.grad) < TOL[engine]
    assert _rel(wd.grad, wr.grad) < TOL[engine]
    assert _rel(bd.grad, br.grad) < TOL[engine]


@pytest.mark.parametrize("engine", ["auto", "simt"], indirect=True)
def test_conv2d_fused_relu(engine):
    from neuralmonkey_b200 import ops
    gen = torch.Generator().manual_seed(3)
    x, wt, b = torch.randn(2, 6, 8, 4, generator=gen), torch.randn(3, 3, 4, 8, generator=gen), torch.randn(8, generator=gen)
    xd, wd = x.cuda().requires_grad_(True), wt.cuda().requires_grad_(True)
    y = ops.conv2d(xd, wd, b.cuda(), "same", act="relu")
    xr, wr = x.double().requires_grad_(True), wt.double().requires_grad_(True)
    yr = CO.conv2d(xr, wr, b.double(), "same", act="relu")
    assert _rel(y, yr) < TOL[engine]
    y.sum().backward()
    yr.sum().backward()
    assert _rel(xd.grad, xr.grad) < TOL[engine] and _rel(wd.grad, wr.grad) < TOL[engine]


@pytest.mark.parametrize("engine", ["auto", "simt"], indirect=True)
def test_weight_gradient_is_bit_identical_across_calls(engine):
    """Two calls at a shape whose pixel reduction is split over many CTAs give the same bits."""
    from neuralmonkey_b200 import lib, ops
    from neuralmonkey_b200.lib import call, ptr
    gen = torch.Generator().manual_seed(5)
    n, h, w, cin, cout, k = 16, 32, 64, 32, 64, 3
    x = torch.randn(n, h, w, cin, generator=gen).cuda()
    dy = torch.randn(n, h, w, cout, generator=gen).cuda()
    outs = []
    for _ in range(2):
        dw = torch.zeros(k, k, cin, cout, device="cuda")
        db = torch.zeros(cout, device="cuda")
        ws = torch.empty(32 * (k * k * cin + 1) * cout, device="cuda")
        call("nm_conv2d_wgrad", ptr(x), ptr(dy), ptr(dw), ptr(db), ptr(ws), ws.numel(), n, h, w, cin, cout, k, 1, 1,
             1, 1, ops._conv_backend(), lib.stream())
        outs.append((dw, db))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("shape", [(2, 5, 7, 3), (4, 9, 11, 12), (1, 1, 1, 70), (8, 16, 33, 64)])
def test_batch_norm_train_and_eval(shape, relu):
    from neuralmonkey_b200 import ops
    gen = torch.Generator().manual_seed(shape[3])
    c = shape[3]
    x = torch.randn(*shape, generator=gen) * 3 + 2
    gamma, beta = torch.rand(c, generator=gen) + 0.5, torch.randn(c, generator=gen)
    mm, mv = torch.randn(c, generator=gen), torch.rand(c, generator=gen) + 0.5
    for training in (True, False):
        mmd, mvd = mm.cuda(), mv.cuda()
        xd, gd, bd = (t.cuda().requires_grad_(True) for t in (x, gamma, beta))
        y = ops.batch_norm(xd, gd, bd, mmd, mvd, training, relu)
        mmr, mvr = mm.double(), mv.double()
        xr, gr, br = (t.double().requires_grad_(True) for t in (x, gamma, beta))
        yr = CO.batch_norm(xr, gr, br, mmr, mvr, training, relu)
        assert _rel(y, yr) < 1e-5
        assert _rel(mmd, mmr) < 1e-6 and _rel(mvd, mvr) < 1e-6
        g = torch.randn(shape, generator=gen)
        y.backward(g.cuda())
        yr.backward(g.double())
        for got, want in ((xd.grad, xr.grad), (gd.grad, gr.grad), (bd.grad, br.grad)):
            assert _rel(got, want) < 2e-5


@pytest.mark.parametrize("kind", ["max", "avg"])
@pytest.mark.parametrize("k,stride,pad,shape", [
    (2, 2, "valid", (2, 8, 10, 3)), (2, 1, "valid", (3, 7, 9, 5)), (3, 2, "valid", (1, 9, 12, 4)),
    (2, 2, "same", (2, 7, 9, 3)), (3, 1, "same", (2, 6, 5, 2)), (3, 2, "same", (1, 10, 7, 70)),
    (1, 1, "valid", (2, 3, 4, 1))])
def test_pooling_forward_and_backward(kind, k, stride, pad, shape):
    from neuralmonkey_b200 import ops
    gen = torch.Generator().manual_seed(k * 10 + stride)
    x = torch.randn(*shape, generator=gen)
    xd = x.cuda().requires_grad_(True)
    y = ops.pool2d(xd, k, stride, pad, kind)
    xr = x.double().requires_grad_(True)
    yr = CO.pool2d(xr, k, stride, pad, kind)
    assert y.shape == yr.shape and _rel(y, yr) < 1e-6
    g = torch.randn(yr.shape, generator=gen)
    y.backward(g.cuda())
    yr.backward(g.double())
    assert _rel(xd.grad, xr.grad) < 1e-6


def test_max_pool_gradient_goes_to_the_first_maximum():
    from neuralmonkey_b200 import ops
    x = torch.ones(1, 2, 4, 1, device="cuda", requires_grad=True)
    ops.pool2d(x, 2, 2, "valid", "max").sum().backward()
    assert x.grad[0, :, :, 0].tolist() == [[1.0, 0.0, 1.0, 0.0], [0.0, 0.0, 0.0, 0.0]]


@pytest.mark.parametrize("trainer_path", [False, True])
def test_adadelta_step_against_the_oracle(trainer_path):
    """Three steps over four segments.  trainer_path: as the trainer calls it - gradients scaled by 0.5 and divided
    by a device token count, L1 / L2 terms on two of the segments, so the first pass rewrites the gradients before
    the clip and the update."""
    from neuralmonkey_b200 import lib
    from neuralmonkey_b200.lib import call, ptr
    gen = torch.Generator().manual_seed(9)
    sizes = [7, 130, 1000, 64]
    reg = [1, 0, 1, 0]
    off = np.concatenate([[0], np.cumsum(sizes)])
    n = int(off[-1])
    params = torch.randn(n, generator=gen)
    p = {i: params[off[i]:off[i + 1]].double() for i in range(len(sizes))}
    acc = {i: torch.zeros(s, dtype=torch.float64) for i, s in enumerate(sizes)}
    upd = {i: torch.zeros(s, dtype=torch.float64) for i, s in enumerate(sizes)}
    pd, ad, ud = params.cuda(), torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    seg_off = torch.tensor(off, dtype=torch.int64, device="cuda")
    seg_reg = torch.tensor(reg if trainer_path else [0] * len(sizes), dtype=torch.uint8, device="cuda")
    norms = torch.zeros(len(sizes), device="cuda")
    scale, count, l1, l2 = (0.5, 7.0, 1e-3, 0.05) if trainer_path else (1.0, None, 0.0, 0.0)
    denominator = torch.tensor([count], device="cuda") if count is not None else None
    l1l2 = torch.zeros(2, device="cuda")
    for _ in range(3):
        grads = torch.randn(n, generator=gen) * 2
        call("nm_clip_adadelta_step", ptr(pd), ptr(grads.cuda()), ptr(ad), ptr(ud), ptr(seg_off), ptr(seg_reg),
             ptr(norms), n, len(sizes), scale, ptr(denominator), 0.5, 0.95, 1e-6, 1.0, l1, l2, ptr(l1l2), None,
             lib.stream())
        g = {}
        for i in range(len(sizes)):
            g[i] = grads[off[i]:off[i + 1]].double() * scale / (count or 1.0)
            if trainer_path and reg[i]:
                g[i] = g[i] + 2 * l2 * p[i] + l1 * torch.sign(p[i])
        want_l2 = sum(float((p[i] ** 2).sum()) for i in range(len(sizes)) if trainer_path and reg[i])
        CO.adadelta_step(p, g, acc, upd, 0.5, 0.95, 1e-6, 1.0)
    want = torch.cat([p[i] for i in range(len(sizes))])
    assert _rel(pd, want) < 1e-5
    assert _rel(ad, torch.cat([acc[i] for i in range(len(sizes))])) < 1e-5
    assert _rel(ud, torch.cat([upd[i] for i in range(len(sizes))])) < 1e-5
    if trainer_path:
        assert abs(float(l1l2[1]) - want_l2) < 1e-4 * want_l2     # the last step's L2 sum, before its update


# -- the model part ---------------------------------------------------------------------------------------------
STR_SPECS = [("C", 3, 1, "valid", 4), ("M", 2, 2, "same"), ("R", 3, 12), ("A", 2, 1, "same")]
MODEL_CASES = {
    "str": dict(convolutions=STR_SPECS, batch_normalize=True, fully_connected=None, hw=(32, 64), pixel=1),
    "residual_same_channels": dict(convolutions=[("C", 2, 1, "same", 6), ("R", 3, 6), ("M", 2, 2, "valid")],
                                   batch_normalize=True, fully_connected=[10, 5], hw=(12, 14), pixel=3),
    "plain": dict(convolutions=[("C", 5, 1, "same", 8), ("A", 3, 2, "valid"), ("C", 2, 1, "valid", 5)],
                  batch_normalize=False, fully_connected=None, hw=(15, 18), pixel=2),
}


def _encoder(case):
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.encoders.cnn_encoder import CNNEncoder, CNNTemporalView
    runtime.reset()
    cfg = MODEL_CASES[case]
    cnn = CNNEncoder(name="cnn", data_id="images", convolutions=cfg["convolutions"], image_height=cfg["hw"][0],
                     image_width=cfg["hw"][1], pixel_dim=cfg["pixel"], fully_connected=cfg["fully_connected"],
                     batch_normalize=cfg["batch_normalize"], dropout_keep_prob=1.0)
    view = CNNTemporalView(name="view", cnn=cnn)
    cnn.ensure_declared()
    arena = runtime.arena()
    arena.finalize(runtime.device())
    return cfg, cnn, view, arena


def _images(cfg, bsz, seed):
    rng = np.random.RandomState(seed)
    img = rng.randint(0, 256, size=(bsz, cfg["hw"][0], cfg["hw"][1], cfg["pixel"])).astype(np.float32)
    img[:, :, -5:] = 0                      # blank right margin: masked columns
    return img


@pytest.mark.parametrize("engine", ["auto", "simt"], indirect=True)
@pytest.mark.parametrize("case", sorted(MODEL_CASES))
def test_encoder_loss_and_gradients_against_the_oracle(engine, case):
    cfg, cnn, view, arena = _encoder(case)
    gen = torch.Generator().manual_seed(1)
    params = {name: arena.get(name).detach().cpu().clone() for name in arena.order}
    for name in arena.train_names:          # non-trivial BN scales and biases
        params[name] = params[name] + 0.1 * torch.randn(params[name].shape, generator=gen)
    arena.load_dict(params)
    images = _images(cfg, 3, 2)
    cnn.feed_images(torch.from_numpy(images / np.float32(255.0)), train=True)
    view.reset_batch()
    r1 = torch.randn(view.temporal_states.shape, generator=gen)
    r2 = torch.randn(cnn.output.shape, generator=gen)
    loss = (view.temporal_states * r1.cuda()).sum() + (cnn.output * r2.cuda()).sum()
    arena.zero_grad()
    loss.backward()
    arena.fold_autograd_grads()

    p = {n: v.double().clone().requires_grad_(n in arena.train_names) for n, v in params.items()}
    want = CO.cnn_encoder(p, "cnn", cfg["convolutions"], torch.from_numpy(images).double() / 255.0,
                          cfg["batch_normalize"], True, cfg["fully_connected"])
    want_loss = (want["temporal_states"] * r1.double()).sum() + (want["output"] * r2.double()).sum()
    assert torch.equal(view.temporal_mask.cpu(), want["temporal_mask"].float())
    assert torch.equal(cnn.spatial_mask.cpu(), want["spatial_mask"].float())
    assert abs(float(loss) - float(want_loss)) <= TOL[engine] * max(1.0, abs(float(want_loss)))
    want_loss.backward()
    largest = max(float(p[name].grad.abs().max()) for name in arena.train_names)
    for name in arena.train_names:
        got, want = arena.grad(name).double().cpu(), p[name].grad
        if engine == "simt":
            # a convolution bias followed by batch normalization has a gradient of exactly zero; what the kernels
            # give there is rounding of sums over every pixel, measured against the model's largest gradient
            scale = float(want.abs().max()) if float(want.abs().max()) > 1e-9 * largest else largest
            assert float((got - want).abs().max()) < 5 * TOL[engine] * scale, name
        else:
            # TF32 rounding of every convolution operand, compounded through up to five convolutions and four batch
            # normalizations (which divide by the batch's standard deviation).  Per tensor: the error within a
            # quarter of the tensor's own largest gradient and the direction within 2 degrees (cosine > 0.999), which
            # a missing, zero, mis-scaled or mis-routed gradient fails; the arithmetic itself is pinned by the
            # per-kernel tests above and by the exact engine's run of this test.
            if float(want.abs().max()) <= 1e-9 * largest:
                assert float(got.abs().max()) < 0.05 * largest, name   # zero in exact arithmetic (bias before BN)
                continue
            cosine = float((got * want).sum() / (got.norm() * want.norm()))
            assert _rel(got, want) < 0.25 and cosine > 0.999, name
    for name in arena.order:
        if name.endswith(("moving_mean", "moving_variance")):
            assert _rel(arena.get(name), p[name]) < TOL[engine], name


@pytest.mark.parametrize("engine", ["auto", "simt"], indirect=True)
@pytest.mark.parametrize("tag", ["plain", "residual", "str"])
def test_encoder_against_the_reference_code(engine, tag):
    """The kernels behind the model part against the reference's own CNNEncoder (tests/golden/cnn_golden.npz), the
    golden's variables loaded by name, in training (moving statistics included) and inference."""
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.encoders.cnn_encoder import CNNEncoder, CNNTemporalView
    from tests.test_host_cnn import GOLDEN_CASES, OUTPUTS, golden_case
    specs, (h, w, c), bn, fc = GOLDEN_CASES[tag]
    variables, images, outputs, moving = golden_case(tag)
    try:
        for mode in ("train", "eval"):
            runtime.reset()
            cnn = CNNEncoder(name="cnn", data_id="images", convolutions=specs, image_height=h, image_width=w,
                             pixel_dim=c, batch_normalize=bn, fully_connected=fc, dropout_keep_prob=1.0)
            view = CNNTemporalView(name="cnn_in_time", cnn=cnn)
            cnn.ensure_declared()
            arena = runtime.arena()
            arena.finalize(runtime.device())
            arena.load_dict({n: torch.from_numpy(v) for n, v in variables.items()})
            cnn.feed_images(torch.from_numpy((images / 255.0).astype(np.float32)), train=mode == "train")
            got = {"spatial_states": cnn.spatial_states, "spatial_mask": cnn.spatial_mask, "output": cnn.output,
                   "temporal_states": view.temporal_states, "temporal_mask": view.temporal_mask}
            for name in OUTPUTS:
                want = torch.from_numpy(outputs[mode][name])
                if name.endswith("mask"):
                    assert torch.equal(got[name].double().cpu(), want), (mode, name)
                else:
                    assert _rel(got[name], want) < TOL[engine], (mode, name)
            if mode == "train":
                for name, want in moving.items():
                    assert _rel(arena.get(name), torch.from_numpy(want)) < TOL[engine], name
    finally:
        runtime.reset()


def test_str_like_model_captured_step_matches_eager():
    """CNN -> temporal view -> GRU encoder -> attention decoder with Adadelta, exact engine: three steps eager and
    with the step captured as a CUDA graph give the same losses and variables, moving statistics included (within
    the tolerance test_gpu_model.py allows the attention decoder's captured step)."""
    from neuralmonkey_b200 import ops, runtime, tf
    from neuralmonkey_b200.attention import Attention
    from neuralmonkey_b200.dataset import BatchingScheme, Dataset
    from neuralmonkey_b200.decoders.decoder import Decoder
    from neuralmonkey_b200.encoders import RecurrentEncoder
    from neuralmonkey_b200.encoders.cnn_encoder import CNNEncoder, CNNTemporalView
    from neuralmonkey_b200.trainers import CrossEntropyTrainer
    from neuralmonkey_b200.vocabulary import Vocabulary
    words = ["ab", "bca", "c", "abc"]
    rng = np.random.RandomState(4)
    images = [rng.randint(0, 256, size=(32, 64, 1)).astype(np.float64) for _ in range(4)]
    results = {}
    try:
        ops.set_gemm_backend("simt")
        for mode in (False, True):
            runtime.reset()
            cnn = CNNEncoder(name="cnn", data_id="images", convolutions=STR_SPECS, image_height=32, image_width=64,
                             pixel_dim=1, batch_normalize=True)
            view = CNNTemporalView(name="cnn_in_time", cnn=cnn)
            enc = RecurrentEncoder(name="encoder", input_sequence=view, rnn_layers=[(16,)])
            att = Attention(name="attention", encoder=enc)
            dec = Decoder(name="decoder", encoders=[enc], attentions=[att], rnn_size=9, embedding_size=9,
                          data_id="target_chars", max_output_len=5, vocabulary=Vocabulary(list("abc")))
            trainer = CrossEntropyTrainer(decoders=[dec], l2_weight=1e-8, clip_norm=1.0,
                                          optimizer=tf.train.AdadeltaOptimizer(learning_rate=0.5, epsilon=1e-6,
                                                                               rho=0.95),
                                          use_cuda_graph=mode)
            for part in (cnn, view, enc, att, dec):
                part.ensure_declared()
            arena = runtime.arena()
            arena.finalize(runtime.device())
            losses = []
            for step in range(3):
                order = words[step:] + words[:step]
                data = Dataset("toy", {"images": lambda: iter(images),
                                       "target_chars": lambda o=order: iter([list(w) for w in o])},
                               BatchingScheme(batch_size=4))
                for part in (cnn, view, enc, att, dec):
                    part.feed_dict(data, train=True)
                losses.append(trainer.train_step()["losses"][0].item())
            results[mode] = (losses, arena.state_dict())
            if mode:
                assert any(isinstance(v, tuple) for v in trainer._graphs.values()), trainer._graphs
    finally:
        ops.set_gemm_backend("auto")
        runtime.reset()
    assert all(np.isfinite(results[False][0]))
    for a, b in zip(results[True][0], results[False][0]):
        assert abs(a - b) < 1e-5
    for name, want in results[False][1].items():
        assert float((results[True][1][name] - want).abs().max()) < 2e-5, name


def test_reference_str_ini_trains_unchanged_on_the_gpu(tmp_path):
    from tests.golden.make_str_bundle import unpack
    tree, out = tmp_path / "tree", str(tmp_path / "out")
    unpack(str(tree))
    cmd = [sys.executable, os.path.join(ROOT, "bin", "neuralmonkey-train"), "tests/str.ini",
           "-s", 'main.output="{}"'.format(out)]
    env = dict(os.environ, NEURALMONKEY_STRICT="1", PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=str(tree), env=env)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    log_text = open(os.path.join(out, "experiment.log")).read()
    assert "Training finished" in log_text and "Validation (epoch" in log_text
    assert os.path.exists(os.path.join(out, "variables.data.final"))
    losses = training_log_values(log_text, "target_chars/train_xent")
    assert losses and all(np.isfinite(losses)), losses
