"""The convolutional seq2seq encoder's kernels (csrc/glu_conv.cu) and model part on the GPU: every entry point
against fp64 on both engines over a grid of shapes (F = 1 to 1024, T = 1, T < k, even k, B*T above 65,535),
bit-identical repeat calls, the autograd op against autograd over the restatement, the encoder part against the
reference's own code, and the two bpe.ini commands of the reference's tests_run.sh through bin/neuralmonkey-train."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import convs2s_oracle as CSO
from tests.helpers import training_log_values

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda"
ENGINES = {"simt": 1, "tc": 0}          # NM_GEMM_SIMT, NM_GEMM_AUTO
BACKEND_NAME = {"simt": "simt", "tc": "auto"}     # ops.set_gemm_backend: 'auto' runs the convolutions on wgmma
# error allowed relative to the sum of |products| of each output: TF32 operands (cvt.rna, 2^-11 each) and exact fp32
TOL = {"simt": 1e-4, "tc": 2.0 ** -9}
GRID = [(1, 1, 1, 1), (2, 3, 4, 5), (16, 10, 10, 5), (4, 13, 33, 4), (64, 50, 512, 3), (8, 100, 1024, 5),
        (1100, 60, 8, 3), (3, 1, 7, 3), (5, 2, 6, 4)]


def _call(name, *args):
    from neuralmonkey_b200 import lib
    lib.call(name, *args)


def _inputs(b, t, f, k, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(b, t, f, device=DEV, generator=gen)
    w = torch.randn(k, f, 2 * f, device=DEV, generator=gen) * (4.0 / f) ** 0.5
    bias = torch.randn(2 * f, device=DEV, generator=gen)
    dy = torch.randn(b, t, f, device=DEV, generator=gen)
    return x, w, bias, dy


def _within(got, want, bound, what):
    err = (got.double() - want).abs()
    excess = float((err - bound).max())
    assert excess <= 0, "{}: max error {:.3e} over its bound (worst excess {:.3e})".format(what, float(err.max()),
                                                                                          excess)


@pytest.mark.parametrize("engine", list(ENGINES))
@pytest.mark.parametrize("shape", GRID, ids=lambda s: "B{}T{}F{}k{}".format(*s))
def test_entry_points_against_fp64(engine, shape):
    from neuralmonkey_b200 import lib
    b, t, f, k = shape
    backend, tol = ENGINES[engine], TOL[engine]
    x, w, bias, dy = _inputs(b, t, f, k, seed=sum(shape))
    xd, wd, bd, dyd = x.double(), w.double(), bias.double(), dy.double()
    s = lib.stream()

    # forward: z and y
    y = torch.empty_like(x)
    z = torch.empty(b, t, 2 * f, device=DEV)
    _call("nm_glu_conv1d_fwd", x.data_ptr(), w.data_ptr(), bias.data_ptr(), y.data_ptr(), z.data_ptr(), b, t, f, k,
          backend, s)
    z_want = CSO.conv1d_same(xd, wd) + bd
    z_bound = tol * (CSO.conv1d_same(xd.abs(), wd.abs()) + bd.abs()) + 1e-6
    _within(z, z_want, z_bound, "z")
    lin, gate = z_want[..., :f], z_want[..., f:]
    y_want = lin * torch.sigmoid(gate) + xd
    y_bound = z_bound[..., :f] + lin.abs() * 0.25 * z_bound[..., f:] + 1e-6 * (1 + xd.abs())
    _within(y, y_want, y_bound, "y")
    # inference: y alone, the same bits
    y2 = torch.empty_like(x)
    _call("nm_glu_conv1d_fwd", x.data_ptr(), w.data_ptr(), bias.data_ptr(), y2.data_ptr(), None, b, t, f, k,
          backend, s)
    assert torch.equal(y, y2)

    # dZ from dY and the saved z
    dz = torch.empty_like(z)
    _call("nm_glu_conv1d_dz", dy.data_ptr(), z.data_ptr(), dz.data_ptr(), b * t, f, s)
    zs = z.double()
    sg = torch.sigmoid(zs[..., f:])
    dz_want = torch.cat([dyd * sg, dyd * zs[..., :f] * sg * (1 - sg)], -1)
    # 1 - sigmoid is exact in fp32 but carries the rounding of the sigmoid itself (a few 2^-24 absolute)
    _within(dz, dz_want, 1e-5 * dz_want.abs() + 1e-6 * (dyd * zs[..., :f]).abs().repeat(1, 1, 2) + 1e-7, "dz")

    # the data gradient, residual included, and the weight and bias gradients, from the same dz
    dzd = dz.double()
    xv, xa = xd.clone().requires_grad_(), xd.abs().requires_grad_()
    wv, wa = wd.clone().requires_grad_(), wd.abs().requires_grad_()
    (CSO.conv1d_same(xv, wv) * dzd).sum().backward()
    (CSO.conv1d_same(xa, wa) * dzd.abs()).sum().backward()
    dx = torch.empty_like(x)
    _call("nm_glu_conv1d_dgrad", dz.data_ptr(), w.data_ptr(), dy.data_ptr(), dx.data_ptr(), b, t, f, k, backend, s)
    _within(dx, xv.grad + dyd, tol * xa.grad + 1e-6 * (1 + dyd.abs()), "dx")

    ws = torch.empty(int(lib.load().nm_glu_conv1d_wgrad_workspace(b, t, f, k, backend)), device=DEV)
    dw = torch.zeros_like(w)
    db = torch.zeros_like(bias)
    _call("nm_glu_conv1d_wgrad", x.data_ptr(), dz.data_ptr(), dw.data_ptr(), db.data_ptr(), ws.data_ptr(),
          ws.numel(), b, t, f, k, backend, s)
    _within(dw, wv.grad, tol * wa.grad + 1e-6, "dw")
    # the bias gradient is the product with a row of ones: on the tensor cores dz enters it rounded to TF32
    _within(db, dzd.sum((0, 1)), max(tol, 1e-5) * dzd.abs().sum((0, 1)) + 1e-6, "db")

    # repeat calls: identical bits (the weight gradient through a fixed-order reduction)
    dw2, db2 = torch.zeros_like(w), torch.zeros_like(bias)
    _call("nm_glu_conv1d_wgrad", x.data_ptr(), dz.data_ptr(), dw2.data_ptr(), db2.data_ptr(), ws.data_ptr(),
          ws.numel(), b, t, f, k, backend, s)
    dx2 = torch.empty_like(x)
    _call("nm_glu_conv1d_dgrad", dz.data_ptr(), w.data_ptr(), dy.data_ptr(), dx2.data_ptr(), b, t, f, k, backend, s)
    assert torch.equal(dw, dw2) and torch.equal(db, db2) and torch.equal(dx, dx2)


@pytest.mark.parametrize("engine", list(ENGINES))
def test_wgrad_with_the_smallest_workspace_and_accumulation(engine):
    """One workspace slice: the whole position sum in one split; dw and db accumulate (+=) into what they hold."""
    from neuralmonkey_b200 import lib
    b, t, f, k = 6, 40, 24, 3
    backend = ENGINES[engine]
    x, w, bias, dy = _inputs(b, t, f, k, seed=7)
    dz = torch.randn(b, t, 2 * f, device=DEV)
    small = torch.empty((k * f + 1) * 2 * f, device=DEV)
    big = torch.empty(int(lib.load().nm_glu_conv1d_wgrad_workspace(b, t, f, k, backend)), device=DEV)
    outs = []
    for ws in (small, big):
        dw, db = torch.ones_like(w), torch.ones_like(bias)
        _call("nm_glu_conv1d_wgrad", x.data_ptr(), dz.data_ptr(), dw.data_ptr(), db.data_ptr(), ws.data_ptr(),
              ws.numel(), b, t, f, k, backend, lib.stream())
        outs.append((dw - 1, db - 1))
    assert torch.allclose(outs[0][0], outs[1][0], rtol=1e-4, atol=1e-4)
    assert torch.allclose(outs[0][1], outs[1][1], rtol=1e-5, atol=1e-4)


def test_entry_points_refuse_bad_arguments():
    from neuralmonkey_b200 import lib
    x = torch.zeros(2, 3, 4, device=DEV)
    with pytest.raises(ValueError, match="bad sizes"):
        _call("nm_glu_conv1d_fwd", x.data_ptr(), x.data_ptr(), x.data_ptr(), x.data_ptr(), None, 2, 3, 0, 3, 0,
              lib.stream())
    with pytest.raises(ValueError, match="null pointer"):
        _call("nm_glu_conv1d_fwd", x.data_ptr(), None, x.data_ptr(), x.data_ptr(), None, 2, 3, 4, 3, 0, lib.stream())
    with pytest.raises(ValueError, match="workspace"):
        _call("nm_glu_conv1d_wgrad", x.data_ptr(), x.data_ptr(), x.data_ptr(), x.data_ptr(), x.data_ptr(), 3,
              2, 3, 4, 3, 0, lib.stream())


@pytest.mark.parametrize("engine", list(ENGINES))
@pytest.mark.parametrize("shape", [(2, 3, 4, 5), (16, 10, 10, 5), (4, 13, 33, 4), (32, 20, 128, 3)])
def test_autograd_op_against_the_restatement(engine, shape):
    from neuralmonkey_b200 import ops
    b, t, f, k = shape
    tol = TOL[engine]
    x, w, bias, dy = _inputs(b, t, f, k, seed=3 + f)
    ops.set_gemm_backend(BACKEND_NAME[engine])
    try:
        xs, ws, bs = (v.clone().requires_grad_() for v in (x, w, bias))
        y = ops.conv1d_glu_residual(xs, ws, bs)
        y.backward(dy)
        with torch.no_grad():
            y_inf = ops.conv1d_glu_residual(x, w, bias)
    finally:
        ops.set_gemm_backend("auto")
    assert torch.equal(y, y_inf)
    xd, wd, bd = (v.double().requires_grad_() for v in (x, w, bias))
    want = CSO.conv1d_glu_residual(xd, wd, bd)
    want.backward(dy.double())
    # errors relative to each tensor's largest entry: TF32 rounding grows with sqrt(K) for random signs
    rel = 4 * tol * (k * f) ** 0.5
    for what, got, ref in (("y", y, want), ("dx", xs.grad, xd.grad), ("dw", ws.grad, wd.grad),
                           ("db", bs.grad, bd.grad)):
        err = float((got.double() - ref).abs().max())
        assert err <= rel * (1.0 + float(ref.abs().max())), (what, err)


@pytest.mark.parametrize("engine", list(ENGINES))
@pytest.mark.parametrize("tag", CSO.CASES)
def test_encoder_part_against_the_reference_code(engine, tag):
    from neuralmonkey_b200 import ops, runtime
    g = CSO.golden()
    ops.set_gemm_backend(BACKEND_NAME[engine])
    try:
        with torch.no_grad():
            got = CSO.golden_model_outputs(g, tag, DEV)
    finally:
        ops.set_gemm_backend("auto")
        runtime.reset()
    for name, value in got.items():
        want = torch.from_numpy(np.asarray(g[tag + "_" + name])).double()
        assert value.shape == want.shape, (tag, name)
        atol = (1e-4 if engine == "simt" else 2e-2) * (1.0 + float(want.abs().max()))
        assert float((value.double().cpu() - want).abs().max()) <= atol, (tag, name)


def _train(tree, out, extra, strict):
    cmd = [sys.executable, os.path.join(ROOT, "bin", "neuralmonkey-train"), "tests/bpe.ini"] + extra
    if out is not None:
        cmd += ["-s", 'main.output="{}"'.format(out)]
    env = dict(os.environ, NEURALMONKEY_STRICT=strict, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=str(tree), env=env)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]


def test_reference_bpe_commands_train_on_the_gpu(tmp_path):
    """tests_run.sh: bpe.ini, then bpe.ini again with the decoder and attention over the gradient-blocking views of
    the encoder, starting from the first run's variables."""
    from tests.golden.make_bpe_bundle import unpack
    unpack(str(tmp_path))
    _train(tmp_path, None, [], "")
    first = open(os.path.join(tmp_path, "tests/outputs/bpe/experiment.log")).read()
    assert "Training finished" in first and "Validation (epoch" in first
    losses = training_log_values(first, "target_greedy/train_xent")
    assert losses and all(np.isfinite(losses))
    out = str(tmp_path / "frozen")
    _train(tmp_path, out, ["-s", "decoder.encoders=[<encoder_output_frozen>]",
                           "-s", "attention.encoder=<encoder_states_frozen>",
                           "-s", 'main.initial_variables=["tests/outputs/bpe/variables.data"]'], "1")
    second = open(os.path.join(out, "experiment.log")).read()
    assert "Training finished" in second
    losses = training_log_values(second, "target_greedy/train_xent")
    assert losses and all(np.isfinite(losses))


# -- one training step of tests/bpe.ini's model ---------------------------------------------------------------------
def _gpu_step(engine, views, init=None, apply_update=False):
    """One step of bpe.ini's model on the device from `init` (or a fresh draw): (variables before, loss, loss
    gradients per variable, variables after, the optimizer's first slot per variable)."""
    from neuralmonkey_b200 import ops, runtime
    ops.set_gemm_backend(BACKEND_NAME[engine])
    try:
        runtime.reset()
        trainer, parts = CSO.bpe_model(views)
        arena = runtime.arena()
        if init is not None:
            arena.load_dict(init)
        before = {n: arena.get(n).detach().cpu().clone() for n in arena.order}
        CSO.feed_bpe(parts, CSO.bpe_batch())
        loss = float(trainer.train_step(apply_update=apply_update)["losses"][0])
        grads = {n: arena.grad(n).detach().cpu().clone() for n in arena.order}
        after = {n: arena.get(n).detach().cpu().clone() for n in arena.order}
        slot = arena.optimizer_slot(trainer.optimizer)[0]
        accum = {n: slot[arena.variables[n].offset:arena.variables[n].offset + before[n].numel()]
                 .view(before[n].shape).detach().cpu().clone() for n in arena.order}
        return before, loss, grads, after, accum
    finally:
        ops.set_gemm_backend("auto")
        runtime.reset()


@pytest.mark.parametrize("engine", list(ENGINES))
def test_bpe_training_step_against_the_restatement(monkeypatch, engine):
    """The loss and the loss gradient of every variable of bpe.ini's model after one step on the device, against
    the same step over the restatement on the CPU (the stand-ins of tests/cpu_ops.py and tests/convs2s_oracle.py,
    the encoder's layers by autograd over `conv1d_glu_residual`) from the same variables and batch."""
    from neuralmonkey_b200 import ops, runtime
    from tests import cpu_ops
    before, loss, grads, _, _ = _gpu_step(engine, views=False)
    with monkeypatch.context() as patch:
        for op in cpu_ops.STAND_INS:
            patch.setattr(ops, op, getattr(cpu_ops, op))
        for op in CSO.STAND_INS:
            patch.setattr(ops, op, getattr(CSO, op))
        patch.setattr(runtime, "_device", torch.device("cpu"))
        try:
            runtime.reset()
            trainer, parts = CSO.bpe_model(False)
            arena = runtime.arena()
            arena.load_dict(before)
            CSO.feed_bpe(parts, CSO.bpe_batch())
            want_loss = float(trainer.train_step(apply_update=False)["losses"][0])
            want = {n: arena.grad(n).detach().clone() for n in arena.order}
        finally:
            runtime.reset()
    # exact engine: fp32 everywhere; auto: TF32 dense and convolution products, fp16 vocabulary operands
    tol = 1e-4 if engine == "simt" else 3e-2
    assert abs(loss - want_loss) <= tol * max(1.0, abs(want_loss))
    assert sorted(grads) == sorted(want)
    # relative to each variable's largest gradient, with a floor at 1e-4 of the model's largest: at the first step
    # the attention's gradients are some 1e-9, sums of terms that cancel to far below their own rounding
    floor = 1e-4 * max(float(g.abs().max()) for g in want.values())
    for name in want:
        scale = float(want[name].abs().max())
        assert scale > 0, name                      # every variable gets a gradient, the encoder's included
        err = float((grads[name].double() - want[name].double()).abs().max())
        assert err <= tol * max(scale, floor), (name, err, scale)


@pytest.mark.parametrize("engine", list(ENGINES))
def test_bpe_training_step_over_the_gradient_blocking_views(engine):
    """The second command of tests_run.sh: the decoder and the attention over StatefulView / TemporalStatefulView
    of the encoder.  The decoder's and the attention's loss gradients are those of the model without the views; the
    encoder's variables (and its input embeddings) get no part of the cross-entropy gradient, so in the update the
    trainer's L2 term (2 * l2_weight * w, none for biases) is their whole gradient.  Adadelta's first accumulator
    after one step is (1 - rho) * g^2, which holds that gradient at any magnitude (the update itself, lr * g, is
    below the resolution of an fp32 weight)."""
    from tests import cnn_oracle as CO
    before, loss, plain, _, _ = _gpu_step(engine, views=False)
    _, loss_v, blocked, _, _ = _gpu_step(engine, views=True, init=before)
    assert abs(loss_v - loss) <= 1e-6 * abs(loss)
    frozen = [n for n in before if n.startswith(("sentence_encoder/", "encoder_input/"))]
    assert len(frozen) == 10
    for name in before:
        if name in frozen:
            assert float(blocked[name].abs().max()) == 0.0, name
            assert float(plain[name].abs().max()) > 0.0, name
        else:
            scale = float(plain[name].abs().max())
            assert float((blocked[name] - plain[name]).abs().max()) <= 1e-5 * scale, name

    start, _, _, after, accum = _gpu_step(engine, views=True, init=before, apply_update=True)
    for name in frozen:
        w = start[name].double()
        g = {name: 2 * 1e-8 * w if "bias" not in name.lower() else torch.zeros_like(w)}
        p, a, u = {name: w.clone()}, {name: torch.zeros_like(w)}, {name: torch.zeros_like(w)}
        CO.adadelta_step(p, g, a, u, 1e-4, 0.95, 1e-6, 1.0)
        _within(accum[name], a[name], 1e-5 * a[name] + 1e-45, name + " accumulator")
        _within(after[name], p[name], 1e-7 * w.abs() + 1e-30, name)
    moved = [n for n in before if n not in frozen and not torch.equal(after[n], start[n])]
    assert moved, "the decoder's variables did not move"
