"""Supervised attention on the device: the K21 kernels (nm_alignment_xent_fwd / _bwd through ops.alignment_xent)
against fp64 at ragged shapes, bit-identical repeat calls, nm_bahdanau_bwd with de_in against fp64 autograd of
attention + alignment loss at the tolerances of tests/test_gpu_bahdanau.py, the whole model against the oracle of
tests/alignment_oracle.py, a learnability check on a copy task, and the reference's tests/alignment.ini."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import alignment_oracle as AO
from tests.helpers import max_abs, rel_err, random_batch, training_log_values
from tests.test_host_alignment import ALIGNMENT_INI_OVERRIDES, unpack_alignment_ini

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# -- the kernels ---------------------------------------------------------------------------------------------------------
def _xent_inputs(bsz, nq, tx, seed):
    g = torch.Generator().manual_seed(seed)
    e = torch.randn(bsz, nq, tx, generator=g) * 3
    a = torch.rand(bsz, nq, tx, generator=g) * (torch.rand(bsz, nq, tx, generator=g) < 0.3)
    a[0, 0] = 0.                                                   # a row with all-zero targets
    pad = (torch.rand(bsz, nq, generator=g) < 0.8).float()
    pad[-1, -1] = 0.                                               # a padded row
    pad[0, 0] = 1.
    return e, a, pad


@pytest.mark.parametrize("tx", [1, 31, 32, 33, 196, 1000])
@pytest.mark.parametrize("nq", [1, 50])
def test_alignment_xent_against_fp64(tx, nq):
    from neuralmonkey_b200 import ops
    e, a, pad = _xent_inputs(7, nq, tx, seed=tx * 100 + nq)
    e64 = e.cuda().double().requires_grad_(True)
    want = AO.alignment_xent(e64, a.cuda().double(), pad.cuda().double())
    grad_scale = 0.7
    (want * grad_scale).backward()
    ec = e.cuda().requires_grad_(True)
    ac, pc = a.cuda(), pad.cuda()
    got = ops.alignment_xent(ec, ac, pc)
    (got * grad_scale).backward()
    assert got.shape == () and torch.isfinite(got)
    assert abs(float(got) - float(want)) <= 1e-5 * abs(float(want)) + 1e-5
    assert max_abs(ec.grad, e64.grad) < 1e-6 * max(1., float(a.sum(-1).max()))
    assert float(ec.grad[-1, -1].abs().max()) == 0. and float(ec.grad[0, 0].abs().max()) == 0.
    # repeat calls: identical bits
    again = ec.detach().clone().requires_grad_(True)
    second = ops.alignment_xent(again, ac, pc)
    (second * grad_scale).backward()
    assert torch.equal(second, got.detach()) and torch.equal(again.grad, ec.grad)


def test_alignment_xent_refuses_bad_arguments():
    from neuralmonkey_b200 import lib, ops
    e = torch.zeros(2, 3, 4, device="cuda")
    with pytest.raises(ValueError):
        ops.alignment_xent(e, torch.zeros(2, 3, 5, device="cuda"), torch.zeros(2, 3, device="cuda"))
    assert lib.load().nm_alignment_xent_fwd(None, None, None, None, None, 2, 3, 4, None) < 0
    assert lib.load().nm_alignment_xent_bwd(None, None, None, None, None, 2, 3, 4, None) < 0


# -- nm_bahdanau_bwd with de_in ------------------------------------------------------------------------------------------
# (B, Tx, NQ, A, C): the en-de training shape, the decoding step, and ragged small shapes from test_gpu_bahdanau.SHAPES
SHAPES = [(256, 50, 50, 600, 600), (40, 33, 1, 14, 10), (40, 33, 51, 14, 10), (264, 9, 13, 14, 10),
          (3, 196, 9, 601, 600), (3, 1, 9, 601, 600), (5, 20, 13, 601, 601)]


@pytest.mark.parametrize("dims", SHAPES)
@pytest.mark.parametrize("use_mask", [True, False])
def test_bahdanau_bwd_with_energy_gradient(dims, use_mask):
    from neuralmonkey_b200 import ops
    bsz, tx, nq, a, c = dims
    g = torch.Generator().manual_seed(bsz + tx + nq)
    keys, values = torch.randn(bsz, tx, a, generator=g), torch.randn(bsz, tx, c, generator=g)
    q = torch.randn(bsz, nq, a, generator=g)
    v, bias = torch.randn(a, generator=g) * 0.3, torch.randn(1, generator=g)
    mask = None
    if use_mask:
        lens = torch.randint(1, tx + 1, (bsz,), generator=g)
        lens[0] = tx
        mask = (torch.arange(tx).unsqueeze(0) < lens.unsqueeze(1)).float()
    dctx = torch.randn(bsz, nq, c, generator=g)
    target = torch.rand(bsz, nq, tx, generator=g)
    pad = (torch.rand(bsz, nq, generator=g) < 0.9).float()
    weight = 0.5

    # fp64 autograd of <ctx, dctx> + weight * alignment loss, a few sentences at a time
    v64 = v.cuda().double().requires_grad_(True)
    b64 = bias.cuda().double().requires_grad_(True)
    ref = {n: [] for n in ("keys", "values", "q")}
    loss64 = 0.
    for s in range(0, bsz, 16):
        k64, val64, q64 = (t[s:s + 16].cuda().double().requires_grad_(True) for t in (keys, values, q))
        m64 = mask[s:s + 16].cuda().double() if mask is not None else None
        ctx, _w, e = AO.bahdanau_attention_energies(k64, val64, m64, q64, v64, b64)
        ali = AO.alignment_xent(e, target[s:s + 16].cuda().double(), pad[s:s + 16].cuda().double())
        ((ctx * dctx[s:s + 16].cuda().double()).sum() + weight * ali).backward()
        loss64 += float(ali)
        for n, t in (("keys", k64), ("values", val64), ("q", q64)):
            ref[n].append(t.grad)
    ref = {n: torch.cat(t) for n, t in ref.items()}
    ref["v"], ref["bias"] = v64.grad, b64.grad

    leaves = [t.clone().cuda().requires_grad_(True) for t in (keys, values, q, v, bias)]
    ctx, _w, e = ops.bahdanau_attention_energies(leaves[0], leaves[1], mask.cuda() if mask is not None else None,
                                                 leaves[2], leaves[3], leaves[4])
    ali = ops.alignment_xent(e, target.cuda(), pad.cuda())
    ((ctx * dctx.cuda()).sum() + weight * ali).backward()
    assert abs(float(ali) - loss64) <= 1e-5 * abs(loss64) + 1e-4
    for name, t in zip(("keys", "values", "q", "v"), leaves):
        assert torch.isfinite(t.grad).all(), name
        assert rel_err(t.grad, ref[name]) < 1e-4, name
    rows = bsz * nq
    assert abs(float(leaves[4].grad) - float(ref["bias"])) < 1e-4 * max(1.0, (rows / 16) ** 0.5)


def test_bahdanau_bwd_without_energy_gradient_is_unchanged():
    """The energies as an unused output: the same bits as `bahdanau_attention`, which passes no de_in (dv and dbias
    are sums of atomic adds over the sentences, so their last bits depend on the order the CTAs finish in)."""
    from neuralmonkey_b200 import ops
    g = torch.Generator().manual_seed(3)
    keys, values, q = (torch.randn(8, 20, 32, generator=g).cuda() for _ in range(3))
    v, bias = torch.randn(32, generator=g).cuda(), torch.randn(1, generator=g).cuda()
    dctx = torch.randn(8, 20, 32, generator=g).cuda()
    grads = []
    for fn in (ops.bahdanau_attention, ops.bahdanau_attention_energies):
        leaves = [t.clone().requires_grad_(True) for t in (keys, values, q, v, bias)]
        out = fn(leaves[0], leaves[1], None, leaves[2], leaves[3], leaves[4])
        (out[0] * dctx).sum().backward()
        grads.append([t.grad for t in leaves])
    for a, b in zip(grads[0][:3], grads[1][:3]):
        assert torch.equal(a, b)
    for a, b in zip(grads[0][3:], grads[1][3:]):
        torch.testing.assert_close(a, b, rtol=1e-6, atol=1e-5)


# -- the model -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rnn_cell,conditional", [("GRU", False), ("NematusGRU", False)])
def test_model_against_the_oracle(rnn_cell, conditional):
    from neuralmonkey_b200 import ops
    from tests.helpers import oracle_params_for
    ops.set_gemm_backend("simt")
    try:
        model = AO.build(rnn_cell=rnn_cell, conditional_gru=conditional, weights=(1., 1e-3))
        params = oracle_params_for(model, seed=7)
        model["arena"].load_dict(params)
        src, tgt = random_batch(6, 8, 7, 40, 50, seed=1)
        rng = np.random.RandomState(0)
        ali = (rng.rand(6, 8, 8) * (rng.rand(6, 8, 8) < 0.4)).astype(np.float32)
        AO.feed(model, src, tgt, ali, train=True)
        p64 = {n: v.double().requires_grad_(True) for n, v in params.items()}
        o_dec, o_ali, o_e = AO.oracle_losses(p64, model["spec"], src, tgt, torch.from_numpy(ali))
        energies = model["dec"].train_attention_energies(model["att"])
        assert max_abs(energies.detach().cpu(), o_e.detach()) < 2e-5
        assert abs(float(model["ali"].cost) - float(o_ali)) <= 2e-5 * abs(float(o_ali)) + 1e-5
        arena = model["arena"]
        arena.zero_grad()
        model["trainer"]._backward()                   # pylint: disable=protected-access
        (o_dec + 1e-3 * o_ali).backward()
        for name, grad in arena.named_grads().items():
            want = p64[name].grad
            want = torch.zeros_like(p64[name]) if want is None else want
            err = float((grad.double().cpu() - want.reshape(grad.shape)).norm())
            assert err <= 2e-4 * float(want.norm()) + 2e-6, (name, err, float(want.norm()))
        # a trainer step, then the run-time alignments
        AO.feed(model, src, tgt, ali, train=True)
        model["trainer"].train_step()
        assert torch.isfinite(model["arena"].params).all()
        AO.feed(model, src, None, None, train=False)
        decoded = model["ali"].decoded
        assert decoded.shape[0] == 6 and decoded.shape[2] == 8
        torch.testing.assert_close(decoded.sum(-1), torch.ones_like(decoded.sum(-1)), rtol=1e-5, atol=1e-5)
    finally:
        ops.set_gemm_backend("auto")


def _copy_batch(rng, bsz, length, vocab):
    """Source and target the same token sequence, and as the reference alignment the REVERSED diagonal: target step
    t onto source position length-1-t, the </s> step onto position 0."""
    src = torch.from_numpy(rng.randint(4, vocab, size=(bsz, length))).long()
    tgt = torch.cat([src.clone(), torch.full((bsz, 1), 2, dtype=torch.long)], 1)
    ali = np.zeros((bsz, length + 1, length), np.float32)
    ali[:, np.arange(length), length - 1 - np.arange(length)] = 1.
    ali[:, length, 0] = 1.
    return src, tgt, ali


def _agreement(model, rng, length, vocab):
    """Share of the (sentence, step) rows whose attention argmax is the reference's position."""
    src, tgt, ali = _copy_batch(rng, 64, length, vocab)
    AO.feed(model, src, tgt, ali, train=True)
    with torch.no_grad():
        w = model["dec"].train_attention_energies(model["att"])
    return float((w.argmax(-1).cpu() == torch.from_numpy(ali).argmax(-1)).float().mean())


def test_alignment_objective_teaches_the_attention():
    """The attention follows the given alignments, not what the task alone would teach it.  A copy task, 300 steps
    at a learning rate of 1e-2, with and without the alignment objective (weight 1); the reference alignment is the
    reversed diagonal.  Trained on the copy task alone, the attention finds the plain diagonal by itself (99 % of
    the steps after 100 updates), so it agrees with the reversed one on almost no step; with the objective it
    agrees on nearly all.  (With diagonal references the two runs end on the same attention, which is why the
    reference here is one the cross-entropy would not find.)"""
    length, vocab, agreements = 10, 24, {}
    for weight in (None, 1.0):
        model = AO.build(vs=vocab, vt=vocab, es=16, he=16, et=16, hd=32, maxout=16, max_len=12, weights=(1., weight),
                         lr=1e-2)
        torch.manual_seed(0)
        rng = np.random.RandomState(0)
        for _ in range(300):
            src, tgt, ali = _copy_batch(rng, 32, length, vocab)
            AO.feed(model, src, tgt, ali, train=True)
            model["trainer"].train_step()
        agreements[weight] = _agreement(model, np.random.RandomState(1), length, vocab)
    assert agreements[1.0] > 0.9 and agreements[None] < 0.3, agreements


# -- the reference's INI ------------------------------------------------------------------------------------------------
def test_alignment_ini_trains_and_runs_on_the_gpu(tmp_path):
    tree, out = tmp_path / "tree", str(tmp_path / "out")
    unpack_alignment_ini(str(tree))
    cmd = [sys.executable, os.path.join(ROOT, "bin", "neuralmonkey-train"), "tests/alignment.ini",
           "-s", 'main.output="{}"'.format(out)]
    for change in ALIGNMENT_INI_OVERRIDES:
        cmd += ["-s", change]
    env = dict(os.environ, NEURALMONKEY_STRICT="1", PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=str(tree), env=env)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    log_text = open(os.path.join(out, "experiment.log")).read()
    assert "Training finished" in log_text and "Validation (epoch" in log_text
    assert os.path.exists(os.path.join(out, "variables.data.final"))
    losses = training_log_values(log_text, "target/train_xent")
    assert losses and all(np.isfinite(losses)), losses
