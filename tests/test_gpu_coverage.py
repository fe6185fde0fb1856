"""nm_coverage_* (through ops.coverage_attention / ops.coverage_fertility) against fp64 autograd of the restatement
in tests/coverage_oracle.py, at K4's tolerances (tests/test_gpu_bahdanau.py): weights 1e-5 and contexts 5e-5
absolute, gradients 1e-4 relative; `cov_out`, the running sum of weights, 1e-5 per step.  Covers the en-de training
and the captioning shapes, query counts 1 to 51, one to 196 keys, odd widths, sentences without a mask and fully
masked ones, and a fertility of ~1e-8 that saturates the tanh.  Then the scan's own properties (one-step calls chain
to the bits of one call, repeat calls give the same bits, refused shapes), the model part against the CPU stand-ins,
and the bahdanau INI with a coverage attention through `neuralmonkey-train` with a greedy and a beam-3 runner."""
import os

import pytest
import torch

from tests import coverage_oracle as CVO
from tests import cpu_ops
from tests.helpers import max_abs, rel_err

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore:Converting a tensor with requires_grad")]

# (B, Tx, NQ, A, C)
SHAPES = ([(256, 50, 50, 600, 600), (32, 196, 16, 512, 512)]             # en-de training, captioning
          + [(6, 33, nq, 40, 24) for nq in (1, 7, 8, 50, 51)]
          + [(3, tx, 9, 64, 48) for tx in (1, 33, 196)]
          + [(5, 20, 13, a, c) for a, c in ((37, 601), (601, 37), (33, 33))])
NAMES = ("keys", "values", "fert", "q", "v", "cw", "cov_in")


def _inputs(dims, use_mask, seed, cov_in=True, all_masked_row=False):
    bsz, tx, nq, a, c = dims
    g = torch.Generator().manual_seed(seed)
    x = {"keys": torch.randn(bsz, tx, a, generator=g), "values": torch.randn(bsz, tx, c, generator=g),
         "fert": 1e-8 + 5 * torch.sigmoid(torch.randn(bsz, tx, generator=g)),
         "q": torch.randn(bsz, nq, a, generator=g), "v": torch.randn(a, generator=g) * 0.3,
         "cw": torch.randn(a, generator=g), "cov_in": torch.rand(bsz, tx, generator=g) * 2 if cov_in else None}
    mask = None
    if use_mask:
        lens = torch.randint(1, tx + 1, (bsz,), generator=g)
        lens[0] = tx
        mask = (torch.arange(tx).unsqueeze(0) < lens.unsqueeze(1)).float()
        if all_masked_row:
            mask[-1] = 0
    douts = (torch.randn(bsz, nq, c, generator=g), torch.randn(bsz, tx, generator=g))
    return x, mask, douts


def _reference(x, mask, douts, chunk=16):
    """fp64 on the device, a few sentences at a time."""
    v64, cw64 = (x[n].cuda().double().requires_grad_(True) for n in ("v", "cw"))
    out = {n: [] for n in ("w", "ctx", "cov_out", "keys", "values", "fert", "q", "cov_in")}
    for s in range(0, x["keys"].shape[0], chunk):
        part = {n: x[n][s:s + chunk].cuda().double().requires_grad_(True)
                for n in ("keys", "values", "fert", "q", "cov_in") if x[n] is not None}
        m = mask[s:s + chunk].cuda().double() if mask is not None else None
        ctx, w, cov = CVO.coverage_attention(part["keys"], part["values"], m, part["fert"], part["q"], v64, cw64,
                                             part.get("cov_in"))
        ((ctx * douts[0][s:s + chunk].cuda().double()).sum()
         + (cov * douts[1][s:s + chunk].cuda().double()).sum()).backward()
        for n, t in (("w", w), ("ctx", ctx.detach()), ("cov_out", cov.detach())):
            out[n].append(t)
        for n, t in part.items():
            out[n].append(t.grad)
    out = {n: torch.cat(t) for n, t in out.items() if t}
    out["v"], out["cw"] = v64.grad, cw64.grad
    return out


def _run(x, mask, douts):
    from neuralmonkey_b200 import ops
    leaves = {n: x[n].clone().cuda().requires_grad_(True) for n in NAMES if x[n] is not None}
    ctx, w, cov = ops.coverage_attention(leaves["keys"], leaves["values"], mask.cuda() if mask is not None else None,
                                         leaves["fert"], leaves["q"], leaves["v"], leaves["cw"], leaves.get("cov_in"))
    ((ctx * douts[0].cuda()).sum() + (cov * douts[1].cuda()).sum()).backward()
    got = {"w": w.detach(), "ctx": ctx.detach(), "cov_out": cov.detach()}
    got.update({n: t.grad for n, t in leaves.items()})
    return got


def _check(got, ref):
    for name in ("w", "ctx", "cov_out"):
        assert torch.isfinite(got[name]).all(), name
    assert max_abs(got["w"], ref["w"]) < 1e-5
    assert max_abs(got["ctx"], ref["ctx"]) < 5e-5
    assert max_abs(got["cov_out"], ref["cov_out"]) < 1e-5 * got["w"].shape[1]
    for name in ("keys", "values", "fert", "q", "v", "cw", "cov_in"):
        if name in ref:
            assert torch.isfinite(got[name]).all(), name
            assert rel_err(got[name], ref[name]) < 1e-4, name


@pytest.mark.parametrize("use_mask", [True, False])
@pytest.mark.parametrize("dims", SHAPES)
def test_coverage_against_fp64(dims, use_mask):
    args = _inputs(dims, use_mask, seed=21)
    _check(_run(*args), _reference(*args))


def test_from_zero_coverage_and_an_all_masked_row():
    args = _inputs((7, 33, 12, 40, 24), True, seed=22, cov_in=False, all_masked_row=True)
    got, ref = _run(*args), _reference(*args)
    _check(got, ref)
    assert float(got["w"][-1].abs().max()) == 0.0 and float(got["ctx"][-1].abs().max()) == 0.0


def _fertility_case(scale, seed=23):
    """Encoder states through ops.coverage_fertility into the scan; `scale` pushes the fertility logits down."""
    g = torch.Generator().manual_seed(seed)
    bsz, tx, nq, a, c = 4, 33, 9, 40, 24
    states = torch.randn(bsz, tx, c, generator=g)
    fw = torch.randn(c, generator=g) * 0.3
    fw[0] = -scale
    states[..., 0] = states[..., 0].abs() + 1.0
    x, mask, douts = _inputs((bsz, tx, nq, a, c), True, seed)
    return states, fw, x, mask, douts


@pytest.mark.parametrize("scale", [0.0, 60.0])
def test_fertility_against_fp64(scale):
    """The fertility op, and the scan over it; at scale 60 the fertility is ~1e-8, so the coverage reaches ~1e8 and
    the tanh saturates."""
    from neuralmonkey_b200 import ops
    states, fw, x, mask, douts = _fertility_case(scale)
    leaves = [t.clone().cuda().requires_grad_(True) for t in (states, fw, x["keys"], x["q"])]
    fert = ops.coverage_fertility(leaves[0], leaves[1], 3)
    ctx, w, cov = ops.coverage_attention(leaves[2], leaves[0], mask.cuda(), fert, leaves[3], x["v"].cuda(),
                                         x["cw"].cuda())
    ((ctx * douts[0].cuda()).sum() + (cov * douts[1].cuda()).sum()).backward()
    ref = [t.cuda().double().requires_grad_(True) for t in (states, fw, x["keys"], x["q"])]
    fert64 = CVO.coverage_fertility(ref[0], ref[1], 3)
    ctx64, w64, cov64 = CVO.coverage_attention(ref[2], ref[0], mask.cuda().double(), fert64, ref[3],
                                               x["v"].cuda().double(), x["cw"].cuda().double())
    ((ctx64 * douts[0].cuda().double()).sum() + (cov64 * douts[1].cuda().double()).sum()).backward()
    if scale:
        assert float(fert.max()) < 2e-8
    assert max_abs(fert, fert64) < 1e-6 * 3
    assert max_abs(w, w64) < 1e-5 and max_abs(ctx, ctx64) < 5e-5
    for got, want, name in zip(leaves, ref, ("states", "fertility_w", "keys", "q")):
        assert torch.isfinite(got.grad).all(), name
        assert rel_err(got.grad, want.grad) < 1e-4, name


def test_one_step_calls_chain_to_one_call():
    """T calls of one step, each from the previous cov_out, give the bits of one T-step call; the gradients chained
    back through cov_out agree with the single call's."""
    from neuralmonkey_b200 import ops
    x, mask, douts = _inputs((32, 50, 20, 600, 600), True, seed=24, cov_in=False)
    dev = {n: x[n].cuda() for n in NAMES if x[n] is not None}
    mask = mask.cuda()
    q = dev["q"].clone().requires_grad_(True)
    ctx, w, cov = ops.coverage_attention(dev["keys"], dev["values"], mask, dev["fert"], q, dev["v"], dev["cw"])
    ((ctx * douts[0].cuda()).sum() + (cov * douts[1].cuda()).sum()).backward()
    q1 = dev["q"].clone().requires_grad_(True)
    running, ctxs, ws = None, [], []
    for t in range(q1.shape[1]):
        c, wt, running = ops.coverage_attention(dev["keys"], dev["values"], mask, dev["fert"], q1[:, t:t + 1],
                                                dev["v"], dev["cw"], running)
        ctxs.append(c)
        ws.append(wt)
    ctx1 = torch.cat(ctxs, 1)
    assert torch.equal(torch.cat(ws, 1), w) and torch.equal(ctx1, ctx) and torch.equal(running, cov)
    ((ctx1 * douts[0].cuda()).sum() + (running * douts[1].cuda()).sum()).backward()
    assert rel_err(q1.grad, q.grad) < 1e-5


def test_repeat_calls_give_the_same_bits():
    args = _inputs((64, 50, 50, 600, 600), True, seed=25)
    first, second = _run(*args), _run(*args)
    for name in first:
        assert torch.equal(first[name], second[name]), name


def test_shapes_beyond_the_plan_are_refused():
    from neuralmonkey_b200 import ops
    x, mask, _ = _inputs((1, 20000, 1, 4, 4), False, seed=26)
    dev = {n: x[n].cuda() for n in NAMES if x[n] is not None}
    with pytest.raises(ValueError, match="shared memory, the limit is 204800"):
        ops.coverage_attention(dev["keys"], dev["values"], None, dev["fert"], dev["q"], dev["v"], dev["cw"])
    x, mask, douts = _inputs((1, 4, 1, 1100, 4), False, seed=26)
    leaves = {n: x[n].cuda().requires_grad_(True) for n in NAMES if x[n] is not None}
    ctx, _w, cov = ops.coverage_attention(leaves["keys"], leaves["values"], None, leaves["fert"], leaves["q"],
                                          leaves["v"], leaves["cw"], leaves["cov_in"])
    with pytest.raises(ValueError, match="A=1100 Tx=4 C=4 need .* shared memory, the limit is 204800"):
        ctx.sum().backward()


# -- the model part ------------------------------------------------------------------------------------------------
def _on(device, monkeypatch):
    from neuralmonkey_b200 import ops, runtime
    if device == "cpu":
        for op in cpu_ops.STAND_INS:
            monkeypatch.setattr(ops, op, getattr(cpu_ops, op))
        for op in CVO.STAND_INS:
            monkeypatch.setattr(ops, op, getattr(CVO, op))
        monkeypatch.setattr(runtime, "_device", torch.device("cpu"))
    else:
        monkeypatch.undo()


def _train_step(rnn_cell):
    from neuralmonkey_b200 import runtime
    dec, att = CVO.build_model(rnn_cell=rnn_cell)
    CVO.randomize()
    CVO.feed(dec, att, train=True, ids=CVO.target_ids())
    arena = runtime.arena()
    arena.zero_grad()
    loss = dec.train_loss
    loss.backward()
    arena.fold_autograd_grads()
    grads = {n: arena.grad(n).detach().double().cpu().clone() for n in arena.order}
    CVO.feed(dec, att, train=False)
    symbols = dec._runtime["symbols"].cpu().clone()
    runtime.reset()
    return float(loss), grads, symbols


@pytest.mark.parametrize("rnn_cell", ["GRU", "NematusGRU"])
def test_training_step_and_greedy_decoding_against_the_cpu(monkeypatch, rnn_cell):
    _on("cpu", monkeypatch)
    want_loss, want_grads, want_symbols = _train_step(rnn_cell)
    _on("cuda", monkeypatch)
    loss, grads, symbols = _train_step(rnn_cell)
    assert abs(loss - want_loss) < 1e-4 * max(1.0, abs(want_loss))
    assert sorted(grads) == sorted(want_grads)
    assert float(grads["coverage/coverage_matrix"].abs().max()) > 0
    assert float(grads["coverage/fertility_matrix"].abs().max()) > 0
    # the dense products of the gradients run in TF32 on the default engine, as in tests/test_gpu_multiattention.py
    for name, g in want_grads.items():
        scale = float(g.abs().max()) + 1e-3
        torch.testing.assert_close(grads[name] / scale, g / scale, rtol=0, atol=1e-2, msg=lambda m, n=name: n + m)
    assert torch.equal(symbols, want_symbols)


def test_bahdanau_ini_with_coverage_trains_and_decodes(monkeypatch, tmp_path):
    """Two epochs with finite losses; the greedy runner and the beam-3 runner both produce outputs."""
    import math
    import re
    from tests.test_host_coverage import run_coverage_ini
    monkeypatch.setenv("NEURALMONKEY_STRICT", "1")
    log_text, out = run_coverage_ini(monkeypatch, tmp_path)
    assert "Training finished" in log_text and "Validation (epoch" in log_text
    losses = [float(v) for v in re.findall(r"train_xent:\s*(\S+)", log_text)]
    assert losses and all(math.isfinite(v) for v in losses)
    assert re.search(r"target_beam", log_text) and os.path.exists(os.path.join(out, "variables.data.final"))
