"""The character-level sentence encoder on the GPU: the one-row convolution kernels (nm_conv1d_fwd / dgrad / wgrad
through `ops.conv1d`) exactly against fp64 on both engines over widths 1-8 and lengths around the segment size and
the 64- and 128-row tiles; the highway gate kernels against fp64 with bit-identical repeat calls; the encoder and
its gradients against the fp64 restatement of tests/sentence_cnn_oracle.py at the golden cases; one Adam step of a
model of tests/small_sent_cnn.ini's shape against the same step over the CPU stand-ins; and the reference's
tests/small_sent_cnn.ini through `bin/neuralmonkey-train`.

The convolution operands are small integers (|x| <= 1, |w|, |b|, |dy| <= 3): every product and partial sum is an
integer below 2^24, exact in TF32 operands and fp32 sums whatever the order, so both engines must give the fp64
result exactly, as in test_gpu_conv_exact.py."""
import os
import subprocess
import sys

import pytest
import torch

from tests import cpu_ops
from tests import sentence_cnn_oracle as SO

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device"),
              pytest.mark.filterwarnings("ignore:Converting a tensor with requires_grad")]

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENGINES = ("tc", "simt")
SEGMENT = 5
LENGTHS = (1, 2, SEGMENT - 1, SEGMENT, SEGMENT + 1, 63, 64, 65, 450)
CINS = (7, 11, 128)
COUTS = (1, 13, 64, 300)


@pytest.fixture
def engine_backend(request):
    from neuralmonkey_b200 import ops
    ops.set_gemm_backend("simt" if request.param == "simt" else "auto")
    yield request.param
    ops.set_gemm_backend("auto")


def _ints(shape, g, lo=-3, hi=3):
    return torch.randint(lo, hi + 1, shape, device="cuda", generator=g).float()


def _exact(out, want, what):
    assert out.shape == want.shape, what
    bad = out.double() != want
    assert not bad.any(), "{}: {} of {} differ, max |diff| {}".format(what, int(bad.sum()), bad.numel(),
                                                                    float((out.double() - want).abs().max()))


# -- nm_conv1d_fwd / dgrad / wgrad -----------------------------------------------------------------------------------
@pytest.mark.parametrize("engine_backend", ENGINES, indirect=True)
@pytest.mark.parametrize("k", range(1, 9))
def test_conv1d_exact(engine_backend, k):
    """Forward with and without ReLU and with and without a bias, the data gradient (through the ReLU's nm_act_bwd)
    and the weight and bias gradients, equal to fp64 in every element."""
    from neuralmonkey_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(k)
    for t in LENGTHS:
        for cin in CINS:
            for cout in COUTS:
                x = _ints((2, t, cin), g, -1, 1)
                w, b, dy = _ints((k, cin, cout), g), _ints((cout,), g), _ints((2, t, cout), g)
                # without a bias, the epilogue reads no bias and the weight-gradient reduction writes no db
                for act, bias in ((None, True), ("relu", True), ("relu", False)):
                    what = "{} k={} T={} Cin={} Cout={} act={} bias={}".format(engine_backend, k, t, cin, cout, act,
                                                                               bias)
                    xr, wr, br = (a.double().requires_grad_(True) for a in (x, w, b))
                    want = SO.conv1d(xr, wr, br if bias else None, "same", act)
                    want.backward(dy.double())
                    xg, wg, bg = (a.clone().requires_grad_(True) for a in (x, w, b))
                    y = ops.conv1d(xg, wg, bg if bias else None, "same", act)
                    y.backward(dy)
                    _exact(y, want.detach(), what + " y")
                    _exact(xg.grad, xr.grad, what + " dx")
                    _exact(wg.grad, wr.grad, what + " dw")
                    if bias:
                        _exact(bg.grad, br.grad, what + " db")
                    else:
                        assert bg.grad is None, what


def test_conv1d_refusals():
    from neuralmonkey_b200 import lib, ops
    x, w = torch.zeros(1, 4, 3, device="cuda"), torch.zeros(2, 3, 5, device="cuda")
    with pytest.raises(ValueError, match="padding must be 'same'"):
        ops.conv1d(x, w, None, "valid")
    with pytest.raises(ValueError, match="act"):
        ops.conv1d(x, w, None, "same", "tanh")
    with pytest.raises(ValueError, match="do not fit"):
        ops.conv1d(x, torch.zeros(2, 4, 5, device="cuda"), None)
    assert lib.load().nm_conv1d_fwd(None, None, None, None, 1, 4, 3, 5, 2, 0, 0, None) < 0
    assert lib.load().nm_conv1d_wgrad_workspace(1, 0, 3, 5, 2, 0) == -1


# -- nm_highway_fwd / bwd ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 7, 1000, 64 * 80 * 2100 // 64])
def test_highway_gate_against_fp64_and_repeatable(n):
    from neuralmonkey_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(n)
    zh, zt, x, dy = (torch.randn(n, device="cuda", generator=g) * 3 for _ in range(4))
    zh[: n // 10] = 0.0                          # ReLU's gradient at 0 is 0, as TF's
    zhr, ztr, xr = (a.double().requires_grad_(True) for a in (zh, zt, x))
    want = SO.highway_gate(zhr, ztr, xr)
    want.backward(dy.double())
    runs = []
    for _ in range(2):
        a, b, c = (t.clone().requires_grad_(True) for t in (zh, zt, x))
        y = ops.highway_gate(a, b, c)
        y.backward(dy)
        runs.append((y.detach(), a.grad, b.grad, c.grad))
    # a few fp32 roundings of the largest term each output sums or multiplies
    size = zh.double().clamp(min=0).abs() + x.double().abs()
    tol = 1e-6 * (1.0 + size + dy.double().abs() * (1.0 + size))
    for got, ref, name in zip(runs[0], (want.detach(), zhr.grad, ztr.grad, xr.grad), ("y", "dzh", "dzt", "dx")):
        err = (got.double() - ref).abs()
        assert bool((err <= tol).all()), (name, float(err.max()))
    for a, b in zip(*runs):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))


# -- the encoder against the restatement ---------------------------------------------------------------------------
@pytest.fixture
def cuda_dropout(monkeypatch):
    from neuralmonkey_b200.nn import utils

    def mask(shape, keep_prob, train_mode, device):
        if keep_prob >= 1.0 or not train_mode:
            return None
        return SO.feature_dropout_mask(shape, keep_prob).to(device=device, dtype=torch.float32)
    monkeypatch.setattr(utils, "dropout_mask", mask)
    yield
    from neuralmonkey_b200 import runtime
    runtime.reset()


@pytest.mark.parametrize("engine_backend", ENGINES, indirect=True)
@pytest.mark.parametrize("tag", SO.CASES)
def test_encoder_against_the_oracle(cuda_dropout, engine_backend, tag):
    """Outputs against the reference's golden and gradients against the fp64 restatement: to 1e-5 on the exact
    engine, and within TF32 rounding (5e-3 of the scale per convolution or product) on the wgmma engine."""
    g = SO.golden()
    got, grads, dstates = SO.model_case(g, tag, "cuda")
    _, want_grads, want_dstates = SO.oracle_case(g, tag)
    exact = engine_backend == "simt"
    rtol, atol = (1e-5, 1e-6) if exact else (1e-2, 5e-3)
    for name in SO.OUTPUTS:
        want = torch.from_numpy(g[tag + "_" + name])
        scale = max(1.0, float(want.abs().max()))
        assert torch.allclose(got[name], want, rtol=rtol, atol=atol * scale), (
            tag, name, float((got[name] - want).abs().max()))
    gtol = (1e-4, 1e-5) if exact else (2e-2, 1e-2)
    assert sorted(grads) == sorted(want_grads)
    for name, want in list(want_grads.items()) + [("states", want_dstates)]:
        got_g = (dstates if name == "states" else grads[name]).double()
        scale = max(1.0, float(want.abs().max()))
        assert torch.allclose(got_g, want, rtol=gtol[0], atol=gtol[1] * scale), (
            tag, name, float((got_g - want).abs().max()))


# -- one training step of small_sent_cnn.ini's model -----------------------------------------------------------------
def test_adam_step_of_the_ini_model_against_the_cpu_stand_ins(monkeypatch):
    from neuralmonkey_b200 import ops, runtime
    from neuralmonkey_b200.trainers.generic_trainer import GenericTrainer
    g = torch.Generator().manual_seed(5)
    src, tgt = SO.ini_batch(g)
    model = SO.build_ini_model()
    params = {n: (torch.randn(v.shape, generator=g) * 0.3).float() for n, v in model["arena"].state_dict().items()}
    ops.set_gemm_backend("simt")
    try:
        loss_gpu, after_gpu = SO.ini_step(params, src, tgt)
    finally:
        ops.set_gemm_backend("auto")
        runtime.reset()
    with monkeypatch.context() as m:
        for op in cpu_ops.STAND_INS:
            m.setattr(ops, op, getattr(cpu_ops, op))
        for op in SO.STAND_INS:
            m.setattr(ops, op, getattr(SO, op))
        m.setattr(runtime, "_device", torch.device("cpu"))
        m.setattr(GenericTrainer, "_adam_kernel", cpu_ops.adam_kernel)
        try:
            loss_cpu, after_cpu = SO.ini_step(params, src, tgt)
        finally:
            runtime.reset()
    assert abs(loss_gpu - loss_cpu) <= 1e-5 * max(1.0, abs(loss_cpu)), (loss_gpu, loss_cpu)
    assert sorted(after_gpu) == sorted(after_cpu)
    for name in after_cpu:
        moved = (after_cpu[name] - params[name]).abs().max()
        assert torch.allclose(after_gpu[name], after_cpu[name], rtol=1e-4, atol=1e-6), (
            name, float((after_gpu[name] - after_cpu[name]).abs().max()), float(moved))
    assert any(not torch.equal(after_cpu[n], params[n]) for n in params if n.startswith("sentence_encoder/"))


def test_decoding_and_gradient_blocking_views():
    """Greedy decoding (the fused decoder step) and a beam search of one over the encoder agree, and behind the
    gradient-blocking views an Adam step without L2 leaves the encoder's variables as they were."""
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.decoders.beam_search_decoder import BeamSearchDecoder
    g = torch.Generator().manual_seed(3)
    src, tgt = SO.ini_batch(g)
    try:
        model = SO.build_ini_model()
        params = {n: torch.randn(v.shape, generator=g) * 0.3 for n, v in model["arena"].state_dict().items()}
        model["arena"].load_dict(params)
        SO.feed_ini_model(model, src, tgt, False)
        greedy = model["dec"].runtime_symbols.cpu()
        bs = BeamSearchDecoder(name="bs", parent_decoder=model["dec"], beam_size=1, max_steps=10,
                               length_normalization=0.6)
        SO.feed_ini_model(model, src, None, False)
        bs.reset_batch()
        bs.batch_size = src.shape[0]
        ids = bs.outputs.last_search_step_output.token_ids[1:].cpu()
        steps = min(ids.shape[0], greedy.shape[0])
        assert torch.equal(ids[:steps].reshape(steps, -1), greedy[:steps])
        _, after = SO.ini_step(params, src, tgt, views=True, l2_weight=0.0)
    finally:
        runtime.reset()
    encoder = [n for n in params if n.startswith(("sentence_encoder/", "encoder_input/"))]
    assert all(torch.equal(after[n], params[n]) for n in encoder)
    assert any(not torch.equal(after[n], params[n]) for n in params if n.startswith("decoder/"))


# -- the reference's INI ---------------------------------------------------------------------------------------------
def test_small_sent_cnn_ini_trains(tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    from make_sent_cnn_bundle import unpack
    tree, out = tmp_path / "tree", str(tmp_path / "out")
    unpack(str(tree))
    # only the output directory is redirected and the TER evaluation dropped (pyter, third-party, is absent)
    cmd = [sys.executable, os.path.join(ROOT, "bin", "neuralmonkey-train"), "tests/small_sent_cnn.ini",
           "-s", 'main.output="{}"'.format(out), "-s", 'main.evaluation=[("target", evaluators.BLEU)]']
    env = dict(os.environ, NEURALMONKEY_STRICT="1", PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=str(tree), env=env)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    log_text = open(os.path.join(out, "experiment.log")).read()
    assert "Training finished" in log_text and "Validation (epoch" in log_text
    assert os.path.exists(os.path.join(out, "variables.data.final"))
