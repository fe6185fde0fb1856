"""The joint multi-source attention kernels (csrc/joint_attention.cu) against the fp64 restatement of
tests/multiattention_oracle.py, their determinism and their agreement with K4, and the attention-combination
model parts on the GPU against the same model on the CPU stand-ins."""
import itertools

import pytest
import torch

from tests import cpu_ops
from tests import multiattention_oracle as MAO

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore:Converting a tensor with requires_grad")]
DEV = torch.device("cuda")


def _inputs(bsz, segs, j, nq, a, c, masked=True, scale=1.0, seed=0, all_masked_row=False):
    gen = torch.Generator().manual_seed(seed)
    tx = sum(segs)

    def r(*shape):
        return torch.randn(*shape, generator=gen, dtype=torch.float64) * scale
    ends = list(itertools.accumulate(segs))
    inp = dict(keys=r(bsz, tx, a) if tx else None, values=torch.randn(bsz, tx, c, generator=gen,
                                                                      dtype=torch.float64) if tx else None,
               mask=None, seg_ends=ends, seg_bias=r(len(segs)) if tx else None,
               ckeys=r(bsz, nq, j, a) if j else None,
               cvalues=torch.randn(bsz, nq, j, c, generator=gen, dtype=torch.float64) if j else None,
               cand_bias=r(j) if j else None, qproj=r(bsz, nq, a), v=torch.randn(a, generator=gen, dtype=torch.float64))
    if masked and tx:
        lengths = torch.randint(1, tx + 1, (bsz,), generator=gen)
        mask = (torch.arange(tx)[None, :] < lengths[:, None]).double()
        if all_masked_row:
            mask[0] = 0.0
        inp["mask"] = mask
    return inp


def _dev(inp, dtype=torch.float32):
    return {k: (v.to(DEV, dtype) if isinstance(v, torch.Tensor) else v) for k, v in inp.items()}


def _call(fn, inp):
    return fn(inp["keys"], inp["values"], inp["mask"], inp["seg_ends"], inp["seg_bias"], inp["ckeys"],
              inp["cvalues"], inp["cand_bias"], inp["qproj"], inp["v"])


GRID = [
    # (B, segment lengths, J, NQ, A, C)
    (3, [], 1, 1, 16, 8),
    (2, [], 5, 4, 33, 17),
    (3, [1], 0, 3, 40, 24),
    (2, [1], 3, 9, 64, 32),
    (4, [7, 5], 0, 1, 48, 40),
    (3, [7, 5], 1, 17, 128, 96),
    (2, [6, 1, 9], 2, 30, 64, 64),
    (2, [40, 49], 1, 120, 32, 32),          # a long query sequence
    (2, [5, 3], 1, 3, 1024, 1024),          # the widest A and C
    (256, [4, 3], 1, 24, 32, 16),           # a large B * NQ
]


def _variables(inp):
    names = ("keys", "values", "seg_bias", "ckeys", "cvalues", "cand_bias", "qproj", "v")
    return [n for n in names if inp[n] is not None]


@pytest.mark.parametrize("shape", GRID)
def test_forward_and_backward_against_fp64(shape):
    from neuralmonkey_b200 import ops
    bsz, segs, j, nq, a, c = shape
    ref = _inputs(bsz, segs, j, nq, a, c, all_masked_row=bool(segs) and j > 0)
    names = _variables(ref)
    ref64 = {k: (v.clone().requires_grad_() if k in names else v) for k, v in ref.items()}
    want_ctx, want_w = _call(MAO.joint_attention, ref64)
    dctx = torch.randn(want_ctx.shape, generator=torch.Generator().manual_seed(9), dtype=torch.float64)
    (want_ctx * dctx).sum().backward()
    got = _dev(ref)
    got = {k: (v.clone().requires_grad_() if k in names else v) for k, v in got.items()}
    ctx, w = _call(ops.joint_attention, got)
    (ctx * dctx.to(DEV, torch.float32)).sum().backward()
    torch.testing.assert_close(w.double().cpu(), want_w, rtol=1e-4, atol=2e-5)
    torch.testing.assert_close(ctx.double().cpu(), want_ctx, rtol=1e-4, atol=5e-5)
    for n in names:
        scale = float(ref64[n].grad.abs().max()) + 1e-6
        torch.testing.assert_close(got[n].grad.double().cpu() / scale, ref64[n].grad / scale, rtol=0, atol=2e-4,
                                   msg=lambda m, n=n: "{}: {}".format(n, m))


@pytest.mark.parametrize("masked", [True, False])
def test_outside_the_fast_tanh_range(masked):
    from neuralmonkey_b200 import ops
    ref = _inputs(2, [5, 4], 2, 6, 32, 16, masked=masked, scale=30.0, seed=3)
    ref["keys"][0, 0, 0] = 50.0
    ref["qproj"][0, 0, 0] = -49.5
    ref["ckeys"][1, 2, 1, 3] = 45.0
    want_ctx, want_w = _call(MAO.joint_attention, ref)
    ctx, w = _call(ops.joint_attention, _dev(ref))
    torch.testing.assert_close(w.double().cpu(), want_w, rtol=1e-4, atol=2e-5)
    torch.testing.assert_close(ctx.double().cpu(), want_ctx, rtol=1e-4, atol=1e-4)


def test_repeat_calls_give_identical_bits():
    from neuralmonkey_b200 import ops
    ref = _inputs(64, [40, 60], 1, 30, 64, 64, seed=5)
    outs = []
    for _ in range(3):
        got = {k: (v.clone().requires_grad_() if k in _variables(ref) else v) for k, v in _dev(ref).items()}
        ctx, w = _call(ops.joint_attention, got)
        ctx.sum().backward()
        outs.append([ctx.detach(), w] + [got[n].grad for n in _variables(ref)])
    for other in outs[1:]:
        for x, y in zip(outs[0], other):
            assert torch.equal(x, y)


@pytest.mark.parametrize("masked", [True, False])
def test_agrees_with_bahdanau_at_one_segment(masked):
    """J = 0, one segment and seg_bias = bias is K4's computation."""
    from neuralmonkey_b200 import ops
    ref = _dev(_inputs(4, [23], 0, 7, 96, 80, masked=masked, seed=7))
    names = ["keys", "values", "qproj", "v", "seg_bias"]
    a = {k: (v.clone().requires_grad_() if k in names else v) for k, v in ref.items()}
    b = {k: (v.clone().requires_grad_() if k in names else v) for k, v in ref.items()}
    ctx, w = _call(ops.joint_attention, a)
    ctx_k4, w_k4 = ops.bahdanau_attention(b["keys"], b["values"], b["mask"], b["qproj"], b["v"], b["seg_bias"])
    torch.testing.assert_close(w, w_k4, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(ctx, ctx_k4, rtol=1e-5, atol=1e-5)
    dctx = torch.randn_like(ctx)
    (ctx * dctx).sum().backward()
    (ctx_k4 * dctx).sum().backward()
    for n in names:
        torch.testing.assert_close(a[n].grad, b[n].grad, rtol=1e-4, atol=1e-5)


def test_shapes_beyond_the_plan_are_refused():
    from neuralmonkey_b200 import ops
    ref = _dev(_inputs(1, [9] * 9, 0, 1, 8, 8))
    with pytest.raises(ValueError, match="segments"):
        _call(ops.joint_attention, ref)
    ref = _dev(_inputs(1, [6000], 0, 1, 1024, 8, masked=False))
    with pytest.raises(ValueError, match="shared memory"):
        _call(ops.joint_attention, ref)


# -- the model parts ------------------------------------------------------------------------------------------------
def _on(device, monkeypatch):
    from neuralmonkey_b200 import ops, runtime
    if device == "cpu":
        for op in cpu_ops.STAND_INS:
            monkeypatch.setattr(ops, op, getattr(cpu_ops, op))
        for op in MAO.STAND_INS:
            monkeypatch.setattr(ops, op, getattr(MAO, op))
        monkeypatch.setattr(runtime, "_device", torch.device("cpu"))
    else:
        monkeypatch.undo()


def _randomize():
    from neuralmonkey_b200 import runtime
    gen = torch.Generator().manual_seed(3)
    with torch.no_grad():
        for name in runtime.arena().order:
            t = runtime.arena().get(name)
            t.copy_((torch.randn(t.shape, generator=gen) * 0.5).to(t.device))


def _train_step(kind, share, sentinel, stepwise):
    from neuralmonkey_b200 import runtime
    dec, wrapper, children = MAO.build_model(kind, share, sentinel)
    _randomize()
    MAO.feed(dec, [wrapper] + children, train=True, ids=MAO.target_ids())
    dec._stepwise = stepwise
    arena = runtime.arena()
    arena.zero_grad()
    loss = dec.train_loss
    loss.backward()
    arena.fold_autograd_grads()
    grads = {n: arena.grad(n).detach().double().cpu().clone() for n in arena.order}
    MAO.feed(dec, [wrapper] + children, train=False)
    symbols = dec._runtime["symbols"].cpu().clone()
    runtime.reset()
    return float(loss), grads, symbols


@pytest.mark.parametrize("kind,share,sentinel,stepwise", [
    ("flat", False, True, False), ("flat", True, False, False), ("flat", False, True, True),
    ("hier", False, True, False), ("hier", True, True, False), ("hier", False, False, True)])
def test_training_step_and_greedy_decoding_against_the_cpu(monkeypatch, kind, share, sentinel, stepwise):
    _on("cpu", monkeypatch)
    want_loss, want_grads, want_symbols = _train_step(kind, share, sentinel, stepwise)
    _on("cuda", monkeypatch)
    loss, grads, symbols = _train_step(kind, share, sentinel, stepwise)
    assert abs(loss - want_loss) < 1e-4 * max(1.0, abs(want_loss))
    assert sorted(grads) == sorted(want_grads)
    # the default engine runs the dense products of the gradients in TF32 (10-bit mantissa), as in
    # tests/test_gpu_convs2s.py; the attention kernels themselves are held to fp32 tolerances above
    for name, g in want_grads.items():
        scale = float(g.abs().max()) + 1e-3
        torch.testing.assert_close(grads[name] / scale, g / scale, rtol=0, atol=1e-2, msg=lambda m, n=name: n + m)
    assert torch.equal(symbols, want_symbols)


@pytest.mark.parametrize("name", ["flat-multiattention", "hier-multiattention"])
def test_reference_ini_trains_unchanged(monkeypatch, tmp_path, name):
    """tests/{flat,hier}-multiattention.ini through `neuralmonkey-train` on the kernels (the batches of the
    hierarchical INI as the reference makes them: see tests/test_host_multiattention.py)."""
    import os
    import sys
    from neuralmonkey_b200 import runtime
    from tests.golden.make_multiattention_bundle import unpack
    from tests.test_host_multiattention import INI_CHANGES
    unpack(str(tmp_path / "tree"))
    monkeypatch.chdir(tmp_path / "tree")
    monkeypatch.setenv("NEURALMONKEY_STRICT", "1")
    out = str(tmp_path / name)
    argv = ["neuralmonkey-train", "tests/{}.ini".format(name), "-s", 'main.output="{}"'.format(out)]
    monkeypatch.setattr(sys, "argv", argv + INI_CHANGES.get(name, []))
    try:
        from neuralmonkey_b200.train import main
        main()
    finally:
        runtime.reset()
    log_text = open(os.path.join(out, "experiment.log")).read()
    assert "Training finished" in log_text and "Validation (epoch" in log_text
    if name == "flat-multiattention":
        assert "target_fss_beam_2:" in log_text and "target_fss_beam_2/beam_search_score" in log_text


# exact fp32 products: the kernels' tolerance; the default engine runs the dense projections (query, keys, vector
# projections, the children's key projections) on TF32 tensor cores, 10-bit mantissas, as tests/test_gpu_convs2s.py
GOLDEN_TOL = {"simt": (1e-4, 2e-5), "auto": (1e-2, 2e-3)}


@pytest.mark.parametrize("engine", list(GOLDEN_TOL))
@pytest.mark.parametrize("tag", MAO.CASES)
def test_model_part_against_the_reference_code(tag, engine):
    """The wrappers on the kernels against the reference's own combination.py (tests/golden)."""
    import numpy as np
    from neuralmonkey_b200 import ops, runtime
    from tests.test_host_multiattention import _golden_outputs
    g = MAO.golden()
    previous = ops.gemm_backend()
    ops.set_gemm_backend(engine)
    try:
        ctx, weights, stepped, hist = _golden_outputs(g, tag)
    finally:
        ops._GEMM_BACKEND = previous
        runtime.reset()
    rtol, atol = GOLDEN_TOL[engine]
    for got in (ctx, stepped):
        np.testing.assert_allclose(got, g[tag + "_contexts"], rtol=rtol, atol=atol)
    for got in (weights, hist):
        np.testing.assert_allclose(got, g[tag + "_weights"], rtol=rtol, atol=atol)


def test_backward_outside_the_fast_tanh_range():
    """The two-SFU branch of the key-gradient kernel against fp64 gradients."""
    from neuralmonkey_b200 import ops
    ref = _inputs(2, [5, 4], 2, 6, 32, 16, scale=30.0, seed=3)
    ref["keys"][0, 0, 0] = 50.0
    ref["qproj"][0, 0, 0] = -49.5
    names = _variables(ref)
    ref64 = {k: (v.clone().requires_grad_() if k in names else v) for k, v in ref.items()}
    want_ctx, _ = _call(MAO.joint_attention, ref64)
    dctx = torch.randn(want_ctx.shape, generator=torch.Generator().manual_seed(4), dtype=torch.float64)
    (want_ctx * dctx).sum().backward()
    got = {k: (v.clone().requires_grad_() if k in names else v) for k, v in _dev(ref).items()}
    ctx, _ = _call(ops.joint_attention, got)
    (ctx * dctx.to(DEV, torch.float32)).sum().backward()
    for n in names:
        scale = float(ref64[n].grad.abs().max()) + 1e-6
        torch.testing.assert_close(got[n].grad.double().cpu() / scale, ref64[n].grad / scale, rtol=0, atol=2e-4,
                                   msg=lambda m, n=n: "{}: {}".format(n, m))
