"""The exact-fp32 attention core (csrc/mha.cu) at every boundary where `nm_mha_fwd` / `nm_mha_bwd` choose between
the tiled kernels and the row kernels, against fp64 autograd of the reference's semantics
(attention/scaled_dot_product.py:160-214): causal entries are REPLACED by -1e9, padded keys get E*m + (1-m)*(-1e9),
softmax, then (softmax * drop) . V.  Also the engine switch of `ops.mha_core`, and one Transformer training step
with attention dropout whose 7-token decoder runs on the row kernels.

Tiled kernels: dh % 8 == 0, dh <= 128, 8 <= Tq <= 256, Tk <= 256, NJ = 8 / 16 / 32 key columns per thread at
Tk <= 64 / 128 / 256; the backward also needs the dK/dV block's Tq * (2 dh + 66) floats within 200 KB.  Row
kernels: everything else, one CTA of 128 threads per query row, striding over keys and head features."""
import pytest
import torch

from tests.helpers import max_abs, rel_err
from tests.test_gpu_mha_tc import _reference
from tests.test_gpu_transformer import _setup, feed_transformer

pytestmark = pytest.mark.gpu

# (B, Tq, Tk, heads, dh), named after the path each one pins
SHAPES = {
    "row_step_tk300": (2, 1, 300, 4, 16),       # a single-query decoding step; more keys than threads
    "row_step_tk1000": (2, 1, 1000, 2, 64),     # ... and more than the tiled kernels' 256
    "row_tq5": (3, 5, 5, 2, 16),                # fewer than 8 queries
    "row_tq7": (2, 7, 7, 4, 8),                 # test_gpu_transformer.py's toy decoder
    "row_dh50": (2, 20, 20, 6, 50),             # dh % 8 != 0
    "row_dh256": (1, 12, 12, 1, 256),           # more head features than threads
    "tile_tk1": (2, 16, 1, 2, 16),              # a single key
    "tile_smallest": (2, 8, 8, 4, 8),
    "tile_nj8_tk64": (2, 40, 64, 2, 32),
    "tile_nj16_tk65": (2, 40, 65, 2, 32),
    "tile_nj16_tk128": (2, 40, 128, 2, 32),
    "tile_nj32_tk129": (2, 40, 129, 2, 32),
    "tile_nj32_tk256": (2, 40, 256, 2, 32),
    "row_tk257": (2, 40, 257, 2, 32),
    "row_tq257": (1, 257, 100, 2, 64),
    "tile_tq256_tk256": (1, 256, 256, 2, 64),
    "tilefwd_rowbwd_dh120": (1, 200, 100, 2, 120),   # the dK/dV block exceeds 200 KB: row backward
    "tilefwd_rowbwd_dh128": (1, 200, 100, 2, 128),
    "tile_tq9": (2, 9, 9, 4, 8),                # a ragged second block of query rows
    "tile_tq33_tk70": (3, 33, 70, 2, 16),
    "tile_tq64_tk130": (2, 64, 130, 8, 64),
}
CASES = [pytest.param(shape, causal, id=name + ("_causal" if causal else ""))
         for name, shape in SHAPES.items() for causal in (False, True) if not causal or shape[1] == shape[2]]
KEEP = 0.7


def _key_mask(bsz, tk, g):
    """Ragged lengths (full, empty, half) over the batch, and holes in sentence 0 as a key mask may have them
    (key 0 stays, so only the empty sentence has a row with every key masked)."""
    lens = [tk, 0, max(1, tk // 2)]
    mask = torch.stack([(torch.arange(tk) < lens[b % 3]).float() for b in range(bsz)])
    holes = (torch.rand(tk, generator=g) < 0.8).float()
    holes[0] = 1.0
    mask[0] *= holes
    return mask


def _run(backend, q, k, v, mask, causal, heads, drop, dout):
    """ops.mha_core forward and backward on `backend`: (context, weights, dq, dk, dv, weights are a view of
    padded storage)."""
    from neuralmonkey_b200 import ops
    ops.set_gemm_backend(backend)
    try:
        qd, kd, vd = (t.clone().cuda().requires_grad_(True) for t in (q, k, v))
        out, probs = ops.mha_core(qd, kd, vd, None if mask is None else mask.cuda(), causal, heads,
                                  None if drop is None else drop.cuda())
        out.backward(dout.cuda())
        torch.cuda.synchronize()
        return (out.detach().cpu(), probs.cpu(), qd.grad.cpu(), kd.grad.cpu(), vd.grad.cpu(),
                probs._base is not None)
    finally:
        ops.set_gemm_backend("auto")


def _inputs(shape, causal, use_drop, masked, q_scale, seed):
    bsz, tq, tk, heads, dh = shape
    g = torch.Generator().manual_seed(seed)
    q, k, v = (torch.randn(bsz, t, heads * dh, generator=g) for t in (tq, tk, tk))
    mask = _key_mask(bsz, tk, g) if masked else None
    drop = (torch.rand(bsz, heads, tq, tk, generator=g) < KEEP).float() / KEEP if use_drop else None
    dout = torch.randn(bsz, tq, heads * dh, generator=g)
    return q * q_scale, k, v, mask, causal, heads, drop, dout


def _fp64(q, k, v, mask, causal, heads, drop, dout):
    q64, k64, v64 = (t.double().requires_grad_(True) for t in (q, k, v))
    ref, p = _reference(q64, k64, v64, mask, causal, heads, drop)
    ref.backward(dout.double())
    return ref.detach(), p.detach(), q64.grad, k64.grad, v64.grad


@pytest.mark.parametrize("q_scale", [1.0, 10.0])
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("use_drop", [False, True])
@pytest.mark.parametrize("shape,causal", CASES)
def test_exact_attention_against_fp64(shape, causal, use_drop, masked, q_scale):
    """q_scale 10 gives energies of +-50, so every softmax depends on its max subtraction."""
    bsz, tq, tk, heads, dh = shape
    args = _inputs(shape, causal, use_drop, masked, q_scale, seed=tq * 1009 + tk * 31 + dh)
    out, probs, dq, dk, dv, _ = _run("simt", *args)
    ref, p, dq64, dk64, dv64 = _fp64(*args)
    # With dropout the context sums terms up to 1/0.7 times larger, and dP carries the same factor.  An fp32
    # energy (a dh-term dot product) is off by a few ulps of its own size, and the context moves by that error
    # times |v|: 10x larger energies, 10x the bar on the context.  The weights themselves stay small where
    # the error is large, and the gradients are held to a relative bar.
    tol, gtol = (1e-4, 1e-4) if use_drop else (1e-5 * q_scale, 2e-5)
    err = max_abs(probs, p)
    assert err < 1e-5, ("probabilities", err)
    err = max_abs(out, ref)
    assert err < tol, ("context", err)
    for name, got, want in (("dq", dq, dq64), ("dk", dk, dk64), ("dv", dv, dv64)):
        err = rel_err(got, want)
        assert err < gtol, (name, err)
        err = max_abs(got, want)   # a single key has a constant softmax: dq = dk = 0 exactly
        assert err <= gtol * float(want.abs().max()), (name + " elementwise", err)
    if masked and bsz > 1:
        # sentence 1 has no keys: uniform weights, and no gradient reaches its queries or keys
        assert max_abs(probs[1], torch.full_like(probs[1], 1.0 / tk)) < 1e-6 / tk
        assert float(dq[1].abs().max()) == 0.0 and float(dk[1].abs().max()) == 0.0
        assert float(dq64[1].abs().max()) == 0.0 and float(dk64[1].abs().max()) == 0.0
    if not use_drop:
        # multiplying by 1.0 is exact: the dropout instances of both kernel families reproduce every bit
        q, k, v, mask, _, _, _, dout = args
        ones = _run("simt", q, k, v, mask, causal, heads, torch.ones(bsz, heads, tq, tk), dout)
        for name, a, b in zip(("context", "weights", "dq", "dk", "dv"), ones, (out, probs, dq, dk, dv)):
            assert torch.equal(a, b), name


@pytest.mark.parametrize("use_drop", [False, True])
@pytest.mark.parametrize("shape,tensor_cores", [((2, 40, 128, 2, 32), True), ((2, 40, 129, 2, 32), False),
                                                ((2, 7, 7, 4, 32), False)])
def test_engine_switch_of_mha_core(shape, tensor_cores, use_drop):
    """On the default engine ops.mha_core takes the tensor cores up to 128 keys and from 8 queries on, and the
    exact kernels otherwise: each case against fp64 with its own engine's bar (test_gpu_mha_tc.py's for TF32)."""
    from neuralmonkey_b200 import ops
    bsz, tq, tk, heads, dh = shape
    assert ops._mha_on_tensor_cores(bsz, tq, tk, heads, dh) == tensor_cores
    args = _inputs(shape, False, use_drop, True, 1.0, seed=tk)
    auto = _run("auto", *args)
    ref, p, dq64, dk64, dv64 = _fp64(*args)
    # the tensor-core engine returns its weights as a view of [Tq, Tk] storage padded to multiples of 32
    assert auto[5] == tensor_cores
    if tensor_cores:
        assert max_abs(auto[1], p) < 2e-3, "probabilities"
        assert rel_err(auto[0], ref) < 3e-3, "context"
        for name, got, want in (("dq", auto[2], dq64), ("dk", auto[3], dk64), ("dv", auto[4], dv64)):
            assert rel_err(got, want) < 5e-3, name
    else:
        exact = _run("simt", *args)
        for name, a, b in zip(("context", "weights", "dq", "dk", "dv"), auto, exact):
            assert torch.equal(a, b), name
        tol, gtol = (1e-4, 1e-4) if use_drop else (1e-5, 2e-5)
        assert max_abs(auto[1], p) < 1e-5, "probabilities"
        assert max_abs(auto[0], ref) < tol, "context"
        for name, got, want in (("dq", auto[2], dq64), ("dk", auto[3], dk64), ("dv", auto[4], dv64)):
            assert rel_err(got, want) < gtol, name


def _transformer_step(backend, keep_prob):
    """One training step of test_gpu_transformer.py's toy model (5 sentences of 8 source and 7 target tokens,
    d = 32 over 4 heads) with every attention-dropout keep probability set to `keep_prob`.  The encoder's
    self-attention (8 x 8) runs on the tiled kernels; the decoder's self- and encoder-attention (7 queries) on the
    row kernels.  Returns (loss, gradients, parameters after the update)."""
    from neuralmonkey_b200 import ops
    try:
        model, _params, src, tgt = _setup(backend)
        enc, dec = model["enc"], model["dec"]
        enc.attention_dropout_keep_prob = keep_prob
        dec.self_att_dropout_keep_prob = keep_prob
        dec.attention_dropout_keep_prob = [keep_prob for _ in dec.encoders]
        feed_transformer(model, src, tgt, train=True)
        loss = float(model["trainer"].train_step()["losses"][0])
        torch.cuda.synchronize()
        return loss, model["arena"].named_grads(), model["arena"].state_dict()
    finally:
        ops.set_gemm_backend("auto")


@pytest.mark.parametrize("backend", ["simt", "auto"])
def test_transformer_step_with_attention_dropout(backend, monkeypatch):
    from neuralmonkey_b200.attention import scaled_dot_product
    loss, grads, _ = _transformer_step(backend, 0.9)
    assert torch.isfinite(torch.tensor(loss))
    for name, grad in grads.items():
        assert bool(torch.isfinite(grad).all()), name
    base_loss, base_grads, base_params = _transformer_step(backend, 1.0)
    assert loss != base_loss, "the attention dropout masks were not applied"
    # Gradients summed by atomic adds in no fixed order (the embedding table's: a repeated token adds into the
    # same row) may change their last bits from one run to the next.  A second run without dropout finds them.
    again_loss, again_grads, _ = _transformer_step(backend, 1.0)
    assert again_loss == base_loss
    atomic = {name for name, grad in base_grads.items() if not torch.equal(grad, again_grads[name])}
    if backend == "simt":   # every gradient behind the attention core is compared bit for bit
        assert not any(n.endswith(("query_proj/kernel", "keys_proj/kernel", "vals_proj/kernel")) for n in atomic)
    # all-ones masks: the dropout kernels must reproduce the run without dropout bit for bit
    monkeypatch.setattr(scaled_dot_product, "dropout_mask",
                        lambda shape, keep_prob, train_mode, device: torch.ones(shape, device=device))
    ones_loss, ones_grads, ones_params = _transformer_step(backend, 0.9)
    assert ones_loss == base_loss
    for name in base_grads:
        if name in atomic:
            assert rel_err(ones_grads[name], base_grads[name]) < 1e-5, name
        else:
            assert torch.equal(ones_grads[name], base_grads[name]), name
            assert torch.equal(ones_params[name], base_params[name]), name
