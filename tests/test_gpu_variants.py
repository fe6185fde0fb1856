"""The step-wise model variants (SURVEY.md 8(f) N4: Nematus GRU cell, conditional GRU, nematus / mlp
deep outputs, nematus initial state) on the GPU against the oracle.

Their host logic is also checked on the CPU over stand-in operations
(tests/test_host_model_cpu.py::test_decoder_and_encoder_variants)."""
import pytest
import torch

from oracle import nm_oracle as O
from tests.helpers import feed, max_abs, oracle_params_for, random_batch
from tests.test_host_model_cpu import _build_variant, check_label_smoothing, check_multi_source

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("backend,tol", [("simt", 5e-5), ("auto", 1e-2)])
@pytest.mark.parametrize("cell,conditional,out_proj,enc_proj,enc_cell", [
    ("NematusGRU", True, "nematus", "nematus", "NematusGRU"),
    ("GRU", True, "mlp", "linear", "GRU"),
    ("NematusGRU", False, "maxout", "linear", "NematusGRU"),
    ("LSTM", False, "maxout", "linear", "LSTM")])
def test_variants_against_oracle(cell, conditional, out_proj, enc_proj, enc_cell, backend, tol):
    from neuralmonkey_b200 import ops
    try:
        ops.set_gemm_backend(backend)
        model = _build_variant(cell, conditional, out_proj, enc_proj, enc_cell)
        params = oracle_params_for(model)
        model["arena"].load_dict(params)
        src, tgt = random_batch(5, 8, 7, 30, 40, seed=1)
        feed(model, src, tgt, train=True)
        enc, dec = model["enc"], model["dec"]
        spec = O.RNNDecoderSpec("decoder", "attention", 10, out_proj, False, cell, conditional, enc_proj, 8, 2)
        p64 = {n: v.double().requires_grad_(True) for n, v in params.items()}

        def oracle_encoder(pp):
            seq = O.embedded_sequence(pp, "sentence_encoder_input", [src])
            return O.recurrent_encoder(pp, "sentence_encoder", seq["temporal_states"], seq["temporal_mask"],
                                       [(5, "bidirectional", enc_cell)])
        odec = O.decoder_train(p64, spec, oracle_encoder(p64), tgt.t())
        assert max_abs(enc.temporal_states, oracle_encoder(p64)["temporal_states"]) < tol
        assert max_abs(dec.train_output_states, odec["train_output_states"]) < tol
        assert abs(float(dec.train_loss) - float(odec["train_loss"])) < max(tol, 1e-5)
        arena = model["arena"]
        arena.zero_grad()
        dec.train_loss.backward()
        odec["train_loss"].backward()
        gtol = 3e-4 if backend == "simt" else 2e-2
        for name, grad in arena.named_grads().items():
            want = p64[name].grad
            want = torch.zeros_like(p64[name]) if want is None else want
            err = float((grad.double().cpu() - want.reshape(grad.shape)).norm())
            assert err <= gtol * float(want.norm()) + 1e-6, (name, err, float(want.norm()))
        feed(model, src, tgt, train=False)
        og = O.decoder_greedy(params, spec, oracle_encoder(params))
        assert max_abs(dec.runtime_logits, og["runtime_logits"]) < 10 * tol
        if backend == "simt":
            assert bool((dec.runtime_symbols.cpu() == og["output_symbols"]).all())
        out = model["trainer"].train_step()          # one optimizer step through the arena
        assert float(out["losses"][0]) > 0.0
    finally:
        ops.set_gemm_backend("auto")


# The exact engine pins the arithmetic (1e-3 on every gradient).  With TF32 products over d = 24 toy
# dimensions the LayerNorm-scale gradients (sums of dy * x_hat over few, small terms) carry several percent
# of rounding noise, so the tensor-core run only guards against gross errors.
@pytest.mark.parametrize("backend,tol,gtol", [("simt", 1e-4, 1e-3), ("auto", 3e-2, 3e-1)])
@pytest.mark.parametrize("strategy", ["serial", "parallel", "flat", "hierarchical"])
def test_multi_source_transformer_decoder(strategy, backend, tol, gtol):
    from neuralmonkey_b200 import ops
    try:
        ops.set_gemm_backend(backend)

        def grads_of(model):
            return model["arena"].named_grads()
        check_multi_source(strategy, grads_of, tol, gtol)
    finally:
        ops.set_gemm_backend("auto")


@pytest.mark.parametrize("backend,tol,gtol", [("simt", 5e-5, 3e-4), ("auto", 1e-2, 2e-2)])
@pytest.mark.parametrize("tie", [False, True])
def test_label_smoothing(tie, backend, tol, gtol):
    from neuralmonkey_b200 import ops
    try:
        ops.set_gemm_backend(backend)
        check_label_smoothing(tie, tol, gtol)
    finally:
        ops.set_gemm_backend("auto")


def test_var_scopes_through_the_optimizer_kernel():
    """var_scopes on the GPU: the variables outside the scopes keep their bits (values and Adam moments),
    the ones inside move - the restriction rides on the kernel's lazy flag and a gradient mask."""
    from neuralmonkey_b200 import ops, tf
    from neuralmonkey_b200.trainers import CrossEntropyTrainer
    from tests.helpers import build_bahdanau
    try:
        ops.set_gemm_backend("simt")
        cfg = dict(vs=60, vt=70, es=11, he=7, et=9, hd=8, out=9, maxout=True, max_len=10, supress_unk=True)
        model = build_bahdanau(**cfg)
        scoped = CrossEntropyTrainer(decoders=[model["dec"]], optimizer=tf.AdamOptimizer(learning_rate=1e-2),
                                     var_scopes=["decoder"], l2_weight=1e-3, clip_norm=1.0)
        arena = model["arena"]
        arena.load_dict(oracle_params_for(model))
        src, tgt = random_batch(6, 8, 7, cfg["vs"], cfg["vt"], seed=0)
        before = arena.state_dict()
        for _ in range(2):
            feed(model, src, tgt, train=True)
            scoped.train_step()
        after = arena.state_dict()
        for name in arena.train_names:
            if name.startswith("decoder"):
                assert not torch.equal(before[name], after[name]), name
            else:
                assert torch.equal(before[name], after[name]), name
        assert float(arena.adam_m.abs().sum()) > 0.0
    finally:
        ops.set_gemm_backend("auto")


@pytest.mark.parametrize("b,tq,tk,heads,dh,causal", [(2, 9, 9, 4, 8, True), (3, 33, 70, 2, 16, False),
                                                     (2, 64, 130, 8, 64, False)])
def test_attention_dropout_in_the_mha_kernels(b, tq, tk, heads, dh, causal):
    """ops.mha_core with a drop mask (nm_mha_fwd_drop / nm_mha_bwd_drop): context and the gradients of
    q, k, v against fp64 autograd of softmax(E) * mask . V."""
    from neuralmonkey_b200 import ops
    g = torch.Generator().manual_seed(5)
    d = heads * dh
    q, k, v = (torch.randn(b, t, d, generator=g) * 0.5 for t in (tq, tk, tk))
    if causal:
        k, v = k[:, :tq], v[:, :tq]
        tk = tq
    key_mask = (torch.rand(b, tk, generator=g) < 0.8).float()
    key_mask[:, 0] = 1.0
    drop = (torch.rand(b, heads, tq, tk, generator=g) < 0.7).float() / 0.7
    qd, kd, vd = (x.cuda().requires_grad_(True) for x in (q, k, v))
    out, probs = ops.mha_core(qd, kd, vd, key_mask.cuda(), causal, heads, drop.cuda())
    dout = torch.randn(b, tq, d, generator=g)
    out.backward(dout.cuda())
    q64, k64, v64 = (x.double().requires_grad_(True) for x in (q, k, v))

    def split(x):
        return x.reshape(b, x.shape[1], heads, dh).transpose(1, 2)
    e = split(q64) @ split(k64).transpose(-1, -2) / dh ** 0.5
    if causal:
        e = torch.where(torch.tril(torch.ones(tq, tk, dtype=torch.bool)), e, torch.full_like(e, -1e9))
    m = key_mask.double()[:, None, None, :]
    e = e * m + (1 - m) * -1e9
    w = torch.softmax(e, -1)
    ref = ((w * drop.double()) @ split(v64)).transpose(1, 2).reshape(b, tq, d)
    ref.backward(dout.double())
    assert max_abs(out, ref) < 1e-4 and max_abs(probs, w) < 1e-5
    for got, ref_grad in ((qd.grad, q64.grad), (kd.grad, k64.grad), (vd.grad, v64.grad)):
        assert float((got.cpu().double() - ref_grad).norm()) <= 1e-4 * float(ref_grad.norm()) + 1e-7
