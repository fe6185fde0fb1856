"""GPU parity tests of what was added in the CPU-only part of round 2: an RNN decoder with scaled-dot attention
OBJECTS (attention.ScaledDotProdAttention / MultiHeadAttention, tests/post-edit.ini's topology) - training pass,
greedy loop, beam search -, optimizer state per optimizer object, and the sampling loop, against the oracle.

Written after round 2's GPU budget was spent: the host composition is checked on the CPU over stand-in
operations (tests/test_host_model_cpu.py::test_rnn_decoder_with_scaled_dot_attention_objects) and every
operation it calls is GPU-verified in other compositions (the Transformer decoder's cross-attention makes the same
`ops.mha_core` call), but THIS test has never run.  It is therefore opt-in - `NMB200_RUN_UNRUN_GPU_TESTS=1` -
so that the default suite holds only tests that have been seen green on a GPU; `bench.py` runs it in a
separate process and records the outcome under `extra_workloads.late_gpu_checks`."""
import os

import pytest
import torch

from oracle import nm_oracle as O
from tests.helpers import max_abs, oracle_params_for, random_batch
from tests.test_host_model_cpu import _post_edit_feed, _post_edit_model, _post_edit_oracle

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(os.environ.get("NMB200_RUN_UNRUN_GPU_TESTS", "0") != "1",
                                 reason="never run on a GPU yet: opt in with NMB200_RUN_UNRUN_GPU_TESTS=1")]


@pytest.mark.parametrize("backend,tol", [("simt", 5e-5), ("auto", 1e-2)])
@pytest.mark.parametrize("heads", [3, 1])
def test_rnn_decoder_with_scaled_dot_attention_objects_on_the_gpu(heads, backend, tol):
    from neuralmonkey_b200 import ops
    try:
        ops.set_gemm_backend(backend)
        model = _post_edit_model(heads)
        arena, dec = model["arena"], model["dec"]
        params = oracle_params_for(model)
        arena.load_dict(params)
        src, tgt = random_batch(5, 8, 7, model["vs"], model["vt"], seed=4)
        trans, _ = random_batch(5, 8, 7, model["vt"], model["vt"], seed=5)
        _post_edit_feed(model, src, trans, tgt, train=True)
        p64 = {n: v.double().requires_grad_(True) for n, v in params.items()}
        spec = O.RNNDecoderSpec("decoder", None, 8, "tanh", False)
        enc, attend = _post_edit_oracle(p64, heads, src, trans)
        odec = O.decoder_train(p64, spec, enc, tgt.t(), attend=attend)
        assert max_abs(dec.train_output_states, odec["train_output_states"]) < tol
        assert abs(float(dec.train_loss) - float(odec["train_loss"])) < max(tol, 1e-5)
        arena.zero_grad()
        dec.train_loss.backward()
        odec["train_loss"].backward()
        arena.fold_autograd_grads()        # what plain autograd left in `.grad` joins the flat buffer, as in a trainer step
        gtol = 3e-4 if backend == "simt" else 2e-2
        for name, grad in arena.named_grads().items():
            want = p64[name].grad
            want = torch.zeros_like(p64[name]) if want is None else want
            err = float((grad.double().cpu() - want.reshape(grad.shape)).norm())
            assert err <= gtol * float(want.norm()) + 1e-6, (name, err, float(want.norm()))
        _post_edit_feed(model, src, trans, tgt, train=False)
        enc, attend = _post_edit_oracle(params, heads, src, trans)
        og = O.decoder_greedy(params, spec, enc, tgt.t(), attend=attend)
        assert dec.decode_engine is None
        assert max_abs(dec.runtime_logits, og["runtime_logits"]) < 10 * tol
        if backend == "simt":
            assert bool((dec.runtime_symbols.cpu() == og["output_symbols"]).all())
        _post_edit_feed(model, src, trans, tgt, train=True)
        out = model["trainer"].train_step()
        assert float(out["losses"][0]) > 0.0
    finally:
        ops.set_gemm_backend("auto")


def test_beam_search_over_the_rnn_decoder_with_attention_objects_on_the_gpu():
    """Beam search around that decoder (no fused engine: the step-wise loop, keys / values tiled to the beam)
    against the oracle's beam search on the exact engine: token ids bit-exact."""
    from neuralmonkey_b200 import ops
    from neuralmonkey_b200.decoders import BeamSearchDecoder
    heads, beam, bsz = 3, 3, 4
    try:
        ops.set_gemm_backend("simt")
        model = _post_edit_model(heads)
        params = oracle_params_for(model)
        model["arena"].load_dict(params)
        src, _tgt = random_batch(bsz, 8, 7, model["vs"], model["vt"], seed=4)
        trans, _ = random_batch(bsz, 8, 7, model["vt"], model["vt"], seed=5)
        bs = BeamSearchDecoder(name="bs", parent_decoder=model["dec"], beam_size=beam, max_steps=7,
                               length_normalization=1.0)
        bs.use_cuda_graph = False
        _post_edit_feed(model, src, trans, None, train=False)
        bs.reset_batch()
        bs.batch_size = bsz
        got = bs.outputs.last_search_step_output
        spec = O.RNNDecoderSpec("decoder", None, 8, "tanh", False)
        enc, attend = _post_edit_oracle(params, heads, src, trans, beam=beam)
        emb = params["decoder/word_embeddings"]
        prev0 = O.decoder_initial_state(params, spec, enc["output"]).repeat_interleave(beam, 0)

        def run(embedded, prev):
            output, cell, _c, _w = O.decoder_step(params, spec, embedded, prev, None, None, None, attend)
            return cell, torch.log_softmax(O.state_to_logits(params, spec, output), -1)

        prev1, first = run(emb[torch.full((bsz * beam,), O.START, dtype=torch.int64)], prev0)
        want = O.beam_search(lambda prev, words, _f: run(emb[words], prev), prev1, first, beam, 7, 1.0,
                             lambda st, idx: st[idx])
        assert bool((got.token_ids[1:].cpu() == want["token_ids"]).all())
        assert max_abs(got.scores, want["scores"]) < 1e-3
    finally:
        ops.set_gemm_backend("auto")


def test_two_optimizers_keep_their_own_state_on_the_gpu():
    """Two trainers with an optimizer each alternating on one model: the second optimizer's moments live in its
    own buffers handed to `nm_clip_adam_step`, bias corrections follow each optimizer's own update count -
    against two oracle Adam states (tests/test_host_model_cpu.py::test_every_optimizer_keeps_its_own_adam_state is
    the same check over the stand-in kernel)."""
    from neuralmonkey_b200 import ops, runtime, tf
    from neuralmonkey_b200.trainers import CrossEntropyTrainer
    from tests.helpers import build_bahdanau, feed, oracle_spec
    toy = dict(vs=60, vt=70, es=11, he=7, et=9, hd=8, out=9, maxout=True, max_len=10, supress_unk=True)
    lrs = (1e-2, 3e-3)
    try:
        ops.set_gemm_backend("simt")
        model = build_bahdanau(**toy, lr=lrs[0])
        second = CrossEntropyTrainer(decoders=[model["dec"]], optimizer=tf.AdamOptimizer(learning_rate=lrs[1]))
        trainers = [model["trainer"], second]
        params = oracle_params_for(model)
        model["arena"].load_dict(params)
        src, tgt = random_batch(6, 8, 7, toy["vs"], toy["vt"], seed=3)
        p32 = {n: v.clone() for n, v in params.items()}
        shared_p = {n: v.clone() for n, v in params.items()}
        states, shared = [O.AdamState(p32), O.AdamState(p32)], O.AdamState(shared_p)
        spec = oracle_spec(True, 10, True)
        for which in (0, 0, 1, 0, 1):
            feed(model, src, tgt, train=True)
            loss = float(trainers[which].train_step()["losses"][0])
            ref = O.train_step(p32, spec, "sentence_encoder", src, tgt.t(), states[which], lr=lrs[which])
            O.train_step(shared_p, spec, "sentence_encoder", src, tgt.t(), shared, lr=lrs[which])
            assert abs(loss - float(ref["loss"])) < 1e-3
        got = model["arena"].state_dict()
        assert max(max_abs(got[n], p32[n]) for n in p32) < 2e-3          # see the CPU test for the scale of the noise
        assert max(max_abs(got[n], shared_p[n]) for n in p32) > 3e-3     # one shared state would be this far off
        assert runtime.global_step() == 5 and [t.optimizer.steps for t in trainers] == [3, 2]
        slots = model["arena"].optimizer_slots
        assert len(slots) == 2 and slots[1][1].data_ptr() != model["arena"].adam_m.data_ptr()
    finally:
        ops.set_gemm_backend("auto")


def test_sampling_loop_on_the_gpu():
    """decoding_loop(sample=True, temperature) over the real step kernels: a very low temperature reproduces the
    greedy symbols, a temperature divides the logits of the histories, sampled rows stay <pad> once finished."""
    from neuralmonkey_b200 import ops
    from tests.helpers import build_bahdanau, feed
    toy = dict(vs=60, vt=70, es=11, he=7, et=9, hd=8, out=9, maxout=True, max_len=10, supress_unk=True)
    try:
        ops.set_gemm_backend("simt")
        model = build_bahdanau(**toy)
        model["arena"].load_dict(oracle_params_for(model))
        src, tgt = random_batch(6, 8, 7, toy["vs"], toy["vt"], seed=3)
        feed(model, src, tgt, train=False)
        dec = model["dec"]
        greedy = dec.decoding_loop(train_mode=False)
        g_logits = torch.stack(greedy.histories.logits, 0)
        g_symbols = torch.stack(greedy.histories.output_symbols, 0)
        warm = dec.decoding_loop(train_mode=False, temperature=2.0)
        assert bool((torch.stack(warm.histories.output_symbols, 0) == g_symbols).all())
        assert max_abs(torch.stack(warm.histories.logits, 0), g_logits / 2.0) < 1e-5
        torch.manual_seed(0)
        cold = dec.decoding_loop(train_mode=False, sample=True, temperature=1e-4)
        assert bool((torch.stack(cold.histories.output_symbols, 0) == g_symbols).all())
        torch.manual_seed(1)
        drawn = dec.decoding_loop(train_mode=False, sample=True)
        sym = torch.stack(drawn.histories.output_symbols, 0).cpu()
        ended = torch.cumsum((sym == 2).to(torch.int64), 0) > 0
        assert bool((sym[1:][ended[:-1]] == 0).all())
    finally:
        ops.set_gemm_backend("auto")
