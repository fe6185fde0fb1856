"""The HOST side of the model parts, run on the CPU over stand-in operations (tests/cpu_ops.py) and
compared with the oracle: which tensors go to which operation, variable names, teacher forcing, the
decoding loops, beam-search bookkeeping, and the step-wise decoder / encoder variants.  The CUDA
kernels are not involved here (tests/test_gpu_*.py test those through the C ABI); what this guards is
the Python around them, which can regress without a GPU in the loop."""
import pytest
import torch

from oracle import nm_oracle as O
from tests import cpu_ops
from tests.helpers import (build_bahdanau, feed, max_abs, oracle_params_for, oracle_spec, random_batch,
                           training_log_values)

pytestmark = pytest.mark.filterwarnings("ignore:Converting a tensor with requires_grad")

TOY = dict(vs=60, vt=70, es=11, he=7, et=9, hd=8, out=9, maxout=True, max_len=10, supress_unk=True)


@pytest.fixture
def cpu_model(monkeypatch):
    from neuralmonkey_b200 import ops, runtime
    for name in cpu_ops.STAND_INS:
        monkeypatch.setattr(ops, name, getattr(cpu_ops, name))
    monkeypatch.setattr(runtime, "_device", torch.device("cpu"))
    yield
    runtime.reset()


def _grads(model):
    return {n: model["arena"].get(n).grad for n in model["arena"].train_names}


def test_bahdanau_training_pass_and_gradients(cpu_model):
    model = build_bahdanau(**TOY)
    params = oracle_params_for(model)
    model["arena"].load_dict(params)
    src, tgt = random_batch(6, 8, 7, TOY["vs"], TOY["vt"], seed=0)
    feed(model, src, tgt, train=True)
    enc, dec = model["enc"], model["dec"]
    spec = oracle_spec(True, 10, True)
    p = {n: v.clone().requires_grad_(True) for n, v in params.items()}
    oenc = O.sentence_encoder(p, "sentence_encoder", src)
    odec = O.decoder_train(p, spec, oenc, tgt.t())
    assert max_abs(enc.temporal_states, oenc["temporal_states"]) < 1e-5
    assert max_abs(dec.train_output_states, odec["train_output_states"]) < 1e-5
    assert max_abs(dec.train_xents, odec["train_xents"]) < 1e-4
    assert abs(float(dec.train_loss) - float(odec["train_loss"])) < 1e-5
    dec.train_loss.backward()
    odec["train_loss"].backward()
    for name, grad in _grads(model).items():
        want = p[name].grad if p[name].grad is not None else torch.zeros_like(p[name])
        got = grad if grad is not None else torch.zeros_like(p[name])
        assert float((got - want.reshape(got.shape)).norm()) <= 1e-4 * float(want.norm()) + 1e-7, name


def test_bahdanau_greedy_decoding(cpu_model):
    model = build_bahdanau(**TOY)
    params = oracle_params_for(model)
    model["arena"].load_dict(params)
    src, tgt = random_batch(6, 8, 7, TOY["vs"], TOY["vt"], seed=3)
    feed(model, src, tgt, train=False)
    dec = model["dec"]
    og = O.decoder_greedy(params, oracle_spec(True, 10, True), O.sentence_encoder(params, "sentence_encoder", src),
                          tgt.t())
    assert dec.runtime_logits.shape == og["runtime_logits"].shape
    keep = torch.ones(TOY["vt"], dtype=torch.bool)
    keep[3] = False
    assert max_abs(dec.runtime_logits[..., keep], og["runtime_logits"][..., keep]) < 1e-4
    assert bool((dec.runtime_symbols == og["output_symbols"]).all())
    assert bool((dec.runtime_mask == og["runtime_mask"]).all())


@pytest.mark.parametrize("beam,bsz", [(3, 1), (4, 3)])
def test_beam_search_over_the_rnn_decoder(cpu_model, beam, bsz):
    from neuralmonkey_b200.decoders import BeamSearchDecoder
    from neuralmonkey_b200.runners.beamsearch_runner import select_hypotheses
    model = build_bahdanau(**TOY)
    params = oracle_params_for(model)
    model["arena"].load_dict(params)
    src, _tgt = random_batch(bsz, 8, 7, TOY["vs"], TOY["vt"], seed=9)
    bs = BeamSearchDecoder(name="bs", parent_decoder=model["dec"], beam_size=beam, max_steps=8,
                           length_normalization=1.0)
    bs.use_cuda_graph = False
    feed(model, src, None, train=False)
    bs.reset_batch()
    bs.batch_size = bsz
    out = bs.outputs
    spec = oracle_spec()
    oenc = O.sentence_encoder(params, "sentence_encoder", src)
    states = oenc["temporal_states"].repeat_interleave(beam, 0)
    mask = oenc["temporal_mask"].repeat_interleave(beam, 0)
    hidden = O.bahdanau_precompute(params, "attention", states)
    emb = params["decoder/word_embeddings"]
    prev0 = O.decoder_initial_state(params, spec, oenc["output"]).repeat_interleave(beam, 0)

    def run(embedded, prev):
        output, cell, _c, _w = O.decoder_step(params, spec, embedded, prev, hidden, states, mask)
        return cell, torch.log_softmax(O.state_to_logits(params, spec, output), -1)

    prev1, first = run(emb[torch.full((bsz * beam,), O.START, dtype=torch.int64)], prev0)
    want = O.beam_search(lambda prev, words, _f: run(emb[words], prev), prev1, first, beam, 8, 1.0,
                         lambda st, idx: st[idx])
    got = out.last_search_step_output
    assert bool((got.token_ids[1:] == want["token_ids"]).all())
    assert max_abs(got.scores, want["scores"]) < 1e-4
    assert bool((out.last_search_state.lengths == want["lengths"]).all())
    assert bool((out.last_search_state.finished.to(torch.bool) == want["finished"]).all())
    words, _loss = select_hypotheses(got.scores.numpy(), got.token_ids.numpy(), 1,
                                     model["dec"].vocabulary.index_to_word)
    assert len(words) == bsz


def _transformer(tie=True, supress_unk=False, bsz=5, seed=0):
    from tests.test_gpu_transformer import CFG, build_transformer
    model = build_transformer(**CFG, tie=tie, supress_unk=supress_unk)
    params = oracle_params_for(model, scale=0.2)
    for name in params:
        if name.endswith("gamma"):
            params[name] = 1.0 + params[name]
    model["arena"].load_dict(params)
    src, tgt = random_batch(bsz, 8, 7, CFG["vs"], CFG["vt"], seed=seed)
    return model, params, src, tgt, CFG


@pytest.mark.parametrize("tie", [True, False])
def test_transformer_training_pass_and_gradients(cpu_model, tie):
    from tests.test_gpu_transformer import feed_transformer, oracle_encoder
    model, params, src, tgt, cfg = _transformer(tie=tie, supress_unk=not tie)
    feed_transformer(model, src, tgt, train=True)
    enc, dec = model["enc"], model["dec"]
    spec = O.TransformerDecoderSpec("decoder", cfg["depth"], cfg["heads"], cfg["heads"], cfg["max_len"], tie, not tie)
    p = {n: v.clone().requires_grad_(True) for n, v in params.items()}
    oenc = oracle_encoder(p, src, cfg)
    odec = O.transformer_decoder_train(p, spec, oenc, tgt)
    assert max_abs(enc.temporal_states, oenc["states"]) < 5e-5
    assert max_abs(dec.train_output_states.transpose(0, 1), odec["states"]) < 5e-5
    assert abs(float(dec.train_loss) - float(odec["loss"])) < 1e-4
    dec.train_loss.backward()
    odec["loss"].backward()
    for name, grad in _grads(model).items():
        want = p[name].grad if p[name].grad is not None else torch.zeros_like(p[name])
        got = grad if grad is not None else torch.zeros_like(p[name])
        assert float((got - want.reshape(got.shape)).norm()) <= 1e-3 * float(want.norm()) + 1e-6, name


@pytest.mark.parametrize("kv_cache", [True, False])
def test_transformer_greedy_and_beam_search(cpu_model, kv_cache):
    from neuralmonkey_b200.decoders import BeamSearchDecoder
    from tests.test_gpu_transformer import _oracle_transformer_beam, feed_transformer, oracle_encoder
    model, params, src, tgt, cfg = _transformer(seed=2, bsz=3)
    model["dec"].use_kv_cache = kv_cache
    feed_transformer(model, src, tgt, train=False)
    dec = model["dec"]
    spec = O.TransformerDecoderSpec("decoder", cfg["depth"], cfg["heads"], cfg["heads"], cfg["max_len"], True, False)
    oenc = oracle_encoder(params, src, cfg)
    og = O.transformer_decoder_greedy(params, spec, oenc)
    assert dec.runtime_logits.shape == og["logits"].shape
    assert max_abs(dec.runtime_logits, og["logits"]) < 2e-4
    assert bool((dec.runtime_symbols == og["symbols"]).all())
    assert bool((dec.runtime_mask == og["mask"]).all())
    bs = BeamSearchDecoder(name="bs", parent_decoder=dec, beam_size=4, max_steps=7, length_normalization=0.6)
    bs.use_cuda_graph = False
    feed_transformer(model, src, None, train=False)
    bs.reset_batch()
    bs.batch_size = 3
    out = bs.outputs
    want = _oracle_transformer_beam(params, spec, oenc, 4, 7, 0.6)
    assert bool((out.last_search_step_output.token_ids[1:] == want["token_ids"]).all())
    assert max_abs(out.last_search_step_output.scores, want["scores"]) < 2e-4
    assert bool((out.last_search_state.lengths == want["lengths"]).all())


def _build_variant(cell, conditional, out_proj, enc_proj, enc_cell):
    from neuralmonkey_b200 import runtime, tf
    from neuralmonkey_b200.attention import Attention
    from neuralmonkey_b200.decoders import Decoder
    from neuralmonkey_b200.decoders.encoder_projection import nematus_projection
    from neuralmonkey_b200.decoders.output_projection import maxout_output, mlp_output, nematus_output
    from neuralmonkey_b200.encoders import SentenceEncoder
    from neuralmonkey_b200.trainers import CrossEntropyTrainer
    from neuralmonkey_b200.vocabulary import Vocabulary
    runtime.reset()
    src_vocab = Vocabulary(["s{}".format(i) for i in range(26)])
    tgt_vocab = Vocabulary(["t{}".format(i) for i in range(36)])
    enc = SentenceEncoder(name="sentence_encoder", vocabulary=src_vocab, data_id="source", embedding_size=6,
                          rnn_size=5, max_input_len=10, rnn_cell=enc_cell)
    att = Attention(name="attention", encoder=enc)
    projection = {"maxout": maxout_output, "nematus": nematus_output, "mlp": lambda n: mlp_output([11, n])}[out_proj](9)
    dec = Decoder(encoders=[enc], vocabulary=tgt_vocab, data_id="target", name="decoder", max_output_len=10,
                  rnn_size=10 if enc_proj == "concat" else 8, embedding_size=9, attentions=[att],
                  output_projection=projection, rnn_cell=cell, conditional_gru=conditional,
                  encoder_projection=nematus_projection() if enc_proj == "nematus" else None)
    trainer = CrossEntropyTrainer(decoders=[dec], optimizer=tf.AdamOptimizer(learning_rate=1e-3))
    for part in trainer.parameterizeds:
        part.ensure_declared()
    runtime.arena().finalize(runtime.device())
    return {"enc": enc, "att": att, "dec": dec, "trainer": trainer, "arena": runtime.arena()}


@pytest.mark.parametrize("cell,conditional,out_proj,enc_proj,enc_cell", [
    ("NematusGRU", True, "nematus", "nematus", "NematusGRU"),      # tests/small.ini / tests/nematus.ini
    ("GRU", True, "mlp", "linear", "GRU"),
    ("NematusGRU", False, "maxout", "linear", "NematusGRU"),
    ("LSTM", False, "maxout", "linear", "LSTM")])
def test_decoder_and_encoder_variants(cpu_model, cell, conditional, out_proj, enc_proj, enc_cell):
    """The step-wise variants (nn/variants.py, decoders/decoder.py `_variant_step`): the Nematus cell in
    encoder and decoder, the conditional GRU, nematus / mlp deep outputs, the nematus initial state -
    training pass, every gradient, greedy decoding and beam search against the oracle, whose
    restatement of these variants is pinned to the reference's own code."""
    from neuralmonkey_b200.decoders import BeamSearchDecoder
    model = _build_variant(cell, conditional, out_proj, enc_proj, enc_cell)
    params = oracle_params_for(model)
    model["arena"].load_dict(params)
    src, tgt = random_batch(5, 8, 7, 30, 40, seed=1)
    feed(model, src, tgt, train=True)
    enc, dec = model["enc"], model["dec"]
    spec = O.RNNDecoderSpec("decoder", "attention", 10, out_proj, False, cell, conditional, enc_proj, 8, 2)
    p = {n: v.clone().requires_grad_(True) for n, v in params.items()}

    def oracle_encoder(pp):
        seq = O.embedded_sequence(pp, "sentence_encoder_input", [src])
        return O.recurrent_encoder(pp, "sentence_encoder", seq["temporal_states"], seq["temporal_mask"],
                                   [(5, "bidirectional", enc_cell)])
    oenc = oracle_encoder(p)
    odec = O.decoder_train(p, spec, oenc, tgt.t())
    assert max_abs(enc.temporal_states, oenc["temporal_states"]) < 1e-5
    assert max_abs(enc.output, oenc["output"]) < 1e-5
    assert max_abs(dec.train_output_states, odec["train_output_states"]) < 1e-5
    assert max_abs(dec.train_rnn_outputs, odec["rnn_outputs"]) < 1e-5
    assert abs(float(dec.train_loss) - float(odec["train_loss"])) < 1e-5
    dec.train_loss.backward()
    odec["train_loss"].backward()
    for name, grad in _grads(model).items():
        want = p[name].grad if p[name].grad is not None else torch.zeros_like(p[name])
        got = grad if grad is not None else torch.zeros_like(p[name])
        assert float((got - want.reshape(got.shape)).norm()) <= 1e-4 * float(want.norm()) + 1e-7, name
    # greedy decoding and a beam search step through the same `_variant_step`
    feed(model, src, tgt, train=False)
    og = O.decoder_greedy(params, spec, oracle_encoder(params))
    assert max_abs(dec.runtime_logits, og["runtime_logits"]) < 1e-4
    assert bool((dec.runtime_symbols == og["output_symbols"]).all())
    bs = BeamSearchDecoder(name="bs", parent_decoder=dec, beam_size=3, max_steps=6, length_normalization=1.0)
    bs.use_cuda_graph = False
    feed(model, src[:1], None, train=False)
    bs.reset_batch()
    bs.batch_size = 1
    out = bs.outputs
    oenc1 = {k: v[:1] for k, v in oracle_encoder(params).items()}
    states, mask = oenc1["temporal_states"].repeat_interleave(3, 0), oenc1["temporal_mask"].repeat_interleave(3, 0)
    hidden = O.bahdanau_precompute(params, "attention", states)
    emb = params["decoder/word_embeddings"]

    def run(embedded, prev):
        output, cell_out, _c, _w = O.decoder_step(params, spec, embedded, prev, hidden, states, mask)
        return cell_out, torch.log_softmax(O.state_to_logits(params, spec, output), -1)

    prev0 = O.decoder_initial_state(params, spec, oenc1["output"], oenc1, 1).repeat_interleave(3, 0)
    prev1, first = run(emb[torch.full((3,), O.START, dtype=torch.int64)], prev0)
    want = O.beam_search(lambda prev, words, _f: run(emb[words], prev), prev1, first, 3, 6, 1.0,
                         lambda st, idx: tuple(x[idx] for x in st) if isinstance(st, tuple) else st[idx])
    assert bool((out.last_search_step_output.token_ids[1:] == want["token_ids"]).all())
    assert max_abs(out.last_search_step_output.scores, want["scores"]) < 1e-4


def test_variant_configurations_build(cpu_model):
    """A decoder with Nematus GRU cells, the conditional GRU and a maxout output, and a GRU decoder with the
    Nematus output projection, build like any other configuration."""
    assert _build_variant("NematusGRU", True, "maxout", "linear", "GRU") is not None
    assert _build_variant("GRU", False, "nematus", "linear", "GRU") is not None


def _cli(monkeypatch, module, argv):
    import importlib
    import sys
    monkeypatch.setattr(sys, "argv", argv)
    importlib.import_module(module).main()


@pytest.mark.parametrize("which", ["bahdanau", "transformer"])
def test_experiments_end_to_end_on_the_cpu(cpu_model, monkeypatch, tmp_path, which):
    """The INIs of tests/test_gpu_cli.py through `neuralmonkey_b200.train.main` / `run.main` in this
    process, on the CPU over the stand-in operations: configuration, datasets and bucketing, feeding, the
    training loop with validation, runners, evaluators, writers, checkpoints, the `.best` bookkeeping,
    loading the variables back for neuralmonkey-run.  (The GPU test runs the same INIs through the real
    entry points; this one keeps the host side honest between GPU sessions.)"""
    import json
    import os
    from neuralmonkey_b200.trainers.generic_trainer import GenericTrainer
    from tests import test_gpu_cli as cli
    monkeypatch.setattr(GenericTrainer, "_adam_kernel", cpu_ops.adam_kernel)
    monkeypatch.setenv("NEURALMONKEY_STRICT", "1")
    data, out = str(tmp_path / "data"), str(tmp_path / "out")
    cli._write_data(data)
    ini = tmp_path / "exp.ini"
    template = cli.INI if which == "bahdanau" else cli.TRANSFORMER_INI
    if which == "bahdanau":     # a per-part checkpoint, written whenever validation finds a new best score
        assert 'name="bahdanau_decoder"\n' in template
        template = template.replace('name="bahdanau_decoder"\n',
                                    'name="bahdanau_decoder"\nsave_checkpoint="{out}/decoder.part"\n')
    ini.write_text(template.format(out=out, data=data, epochs=2))
    _cli(monkeypatch, "neuralmonkey_b200.train", ["neuralmonkey-train", str(ini)])
    log_text = open(os.path.join(out, "experiment.log")).read()
    assert "Validation (epoch" in log_text
    for name in ("experiment.ini", "original.ini", "variables.data.best", "variables.data.final"):
        assert os.path.exists(os.path.join(out, name)), name
    if which == "bahdanau":
        assert os.path.exists(os.path.join(out, "variables.data"))
        import torch
        part = torch.load(os.path.join(out, "decoder.part"))["variables"]
        best = torch.load(os.path.join(out, open(os.path.join(out, "variables.data.best")).read().strip()))
        assert part and all(n.startswith("bahdanau_decoder") for n in part)
        assert all(torch.equal(v, best["variables"][n]) for n, v in part.items())
        assert "Variables of 'bahdanau_decoder' saved to" in log_text
        losses = training_log_values(log_text, "target/train_xent")
        assert len(losses) >= 2 and losses[-1] < losses[0], losses
        assert len(open(os.path.join(out, "val.out")).read().splitlines()) == 30
        run_ini = tmp_path / "run.ini"
        run_ini.write_text("""
[main]
test_datasets=[<val_data>]

[batching]
class=dataset.BatchingScheme
batch_size=7

[val_data]
class=dataset.load
series=["source", "target"]
data=["{data}/val.src", "{data}/val.tgt"]
outputs=[("target", "{out}/run.out")]
batching=<batching>
""".format(data=data, out=out))
        _cli(monkeypatch, "neuralmonkey_b200.run",
             ["neuralmonkey-run", str(ini), str(run_ini), "--json", str(tmp_path / "res.json")])
        results = json.load(open(tmp_path / "res.json"))
        assert "target/BLEU" in results[0] and "target/runtime_xent" in results[0]
        assert len(open(os.path.join(out, "run.out")).read().splitlines()) == 30
    else:
        assert "target_beam.rank001/BLEU" in log_text and "beam_search_score" in log_text


def test_captioning_model_with_the_frozen_vgg_encoder(cpu_model, monkeypatch):
    from neuralmonkey_b200.trainers.generic_trainer import GenericTrainer
    from tests.test_gpu_imagenet import _params, build_captioning
    monkeypatch.setattr(GenericTrainer, "_adam_kernel", cpu_ops.adam_kernel)
    model = build_captioning()
    params = _params(model)
    enc, att, dec = model["enc"], model["att"], model["dec"]
    images = torch.randn(3, 32, 32, 3, generator=torch.Generator().manual_seed(2))
    _src, tgt = random_batch(3, 4, 6, 50, 50, seed=3)
    enc.feed_images(images, train=True)
    att.reset_batch()
    att.train_mode, att.batch_size = True, 3
    dec.feed_ids(tgt, 3, train=True)
    oenc = O.vgg_features(params, "vgg_16", images, "vgg_16/conv5/conv5_3")
    assert max_abs(enc.spatial_states, oenc["spatial_states"]) < 1e-4 * float(oenc["spatial_states"].abs().max())
    odec = O.decoder_train(params, O.RNNDecoderSpec("decoder", "attention", 8, "tanh", False), oenc, tgt.t())
    assert abs(float(dec.train_loss) - float(odec["train_loss"])) < 1e-4
    arena = model["arena"]
    assert not any(n.startswith("vgg_16") for n in arena.train_names)
    before = arena.state_dict()
    model["trainer"].train_step()
    after = arena.state_dict()
    assert all(torch.equal(before[n], after[n]) for n in before if n.startswith("vgg_16"))
    assert not torch.equal(before["decoder/state_to_word_W"], after["decoder/state_to_word_W"])


@pytest.mark.parametrize("strategy", ["serial", "parallel", "flat", "hierarchical"])
def test_multi_source_transformer_decoder(cpu_model, strategy):
    """Two Transformer encoders under one decoder with each attention_combination_strategy: training
    pass, gradients and greedy decoding against the oracle (whose four strategies are pinned to the
    reference's own code)."""
    check_multi_source(strategy, _grads, 5e-5, 1e-3)


def check_multi_source(strategy, grads_of, tol, gtol):
    from neuralmonkey_b200 import runtime, tf
    from neuralmonkey_b200.decoders import TransformerDecoder
    from neuralmonkey_b200.encoders import TransformerEncoder
    from neuralmonkey_b200.model.sequence import EmbeddedSequence
    from neuralmonkey_b200.trainers import CrossEntropyTrainer
    from neuralmonkey_b200.vocabulary import Vocabulary
    runtime.reset()
    dim, ff, depth, heads = 24, 40, 2, 4
    vocabs = [Vocabulary(["a{}".format(i) for i in range(26)]), Vocabulary(["b{}".format(i) for i in range(20)])]
    tgt_vocab = Vocabulary(["t{}".format(i) for i in range(36)])
    seqs = [EmbeddedSequence(name="input_{}".format(i), vocabulary=v, data_id="source_{}".format(i),
                             embedding_size=dim, max_length=9, scale_embeddings_by_depth=True)
            for i, v in enumerate(vocabs)]
    encs = [TransformerEncoder(name="encoder_{}".format(i), input_sequence=s, ff_hidden_size=ff, depth=depth,
                               n_heads=heads) for i, s in enumerate(seqs)]
    heads_enc = 4 if strategy == "flat" else [4, 2]
    dec = TransformerDecoder(name="decoder", encoders=encs, vocabulary=tgt_vocab, data_id="target",
                             ff_hidden_size=ff, n_heads_self=heads, n_heads_enc=heads_enc, depth=depth,
                             max_output_len=8, embedding_size=dim, tie_embeddings=True,
                             attention_combination_strategy=strategy,
                             n_heads_hier=3 if strategy == "hierarchical" else None)
    trainer = CrossEntropyTrainer(decoders=[dec], optimizer=tf.AdamOptimizer(learning_rate=1e-3))
    for part in trainer.parameterizeds:
        part.ensure_declared()
    runtime.arena().finalize(runtime.device())
    model = {"arena": runtime.arena()}
    params = oracle_params_for(model, scale=0.2)
    for name in params:
        if name.endswith("gamma"):
            params[name] = 1.0 + params[name]
    model["arena"].load_dict(params)
    src_a, tgt = random_batch(4, 7, 6, 30, 40, seed=5)
    src_b, _ = random_batch(4, 5, 6, 24, 40, seed=6)

    def feed_all(train, targets):
        for seq, enc, src in zip(seqs, encs, (src_a, src_b)):
            seq.feed_ids([src], train=train)
            enc.reset_batch()
            enc.train_mode, enc.batch_size = train, 4
        dec.feed_ids(targets, 4, train=train)

    def oracle_encoders(pp):
        outs = []
        for i, src in enumerate((src_a, src_b)):
            emb = pp["input_{}/embedding_matrix_0".format(i)]
            mask = (src != 0).to(emb.dtype)
            outs.append(O.transformer_encoder(pp, "encoder_{}".format(i), emb[src] * (mask * dim ** 0.5).unsqueeze(-1),
                                              mask, depth, heads))
        return [o["states"] for o in outs], [o["mask"] for o in outs]

    spec = O.TransformerDecoderSpec("decoder", depth, heads, heads, 8, True, False)
    kw = dict(strategy=strategy, heads_enc=[4, 4] if strategy == "flat" else [4, 2],
              heads_hier=3 if strategy == "hierarchical" else None)
    feed_all(True, tgt)
    p = {n: v.clone().requires_grad_(True) for n, v in params.items()}
    states, masks = oracle_encoders(p)
    emb = p["decoder/word_embeddings"]
    go = torch.full((4, 1), O.START, dtype=torch.int64)
    want = O.transformer_decoder_stack(p, spec, emb[torch.cat([go, tgt[:, :-1]], 1)], (tgt != 0).to(emb.dtype),
                                       states, masks, **kw)
    assert max_abs(dec.train_output_states.transpose(0, 1), want) < tol
    logp = torch.log_softmax(O.transformer_logits(p, spec, want), -1)
    tmask = (tgt != 0).to(emb.dtype)
    want_loss = (-(logp.gather(2, tgt.unsqueeze(2)).squeeze(2)) * tmask).sum() / tmask.sum()
    assert abs(float(dec.train_loss) - float(want_loss)) < max(1e-4, tol)
    dec.train_loss.backward()
    want_loss.backward()
    for name, grad in grads_of(model).items():
        ref = p[name].grad if p[name].grad is not None else torch.zeros_like(p[name])
        got = grad.cpu() if grad is not None else torch.zeros_like(p[name])
        assert float((got - ref.reshape(got.shape)).norm()) <= gtol * float(ref.norm()) + 1e-6, name
    if tol > 1e-3:
        return                      # tensor-core engines: near-ties may flip an argmax
    # greedy decoding: the product re-runs the prefix (or uses its KV cache for serial / parallel)
    feed_all(False, tgt)
    states, masks = oracle_encoders(params)
    seq = torch.zeros(4, 0, dim)
    mask_seq = torch.zeros(4, 0)
    finished = torch.zeros(4, dtype=torch.bool)
    symbols = torch.full((4,), O.START, dtype=torch.int64)
    table = params["decoder/word_embeddings"]
    for step in range(dec.runtime_symbols.shape[0]):
        seq = torch.cat([seq, table[symbols].unsqueeze(1)], 1)
        mask_seq = torch.cat([mask_seq, (~finished).float().unsqueeze(1)], 1)
        out = O.transformer_decoder_stack(params, spec, seq, mask_seq, states, masks, **kw)[:, -1]
        symbols = O.transformer_logits(params, spec, out).argmax(-1) * (~finished).long()
        finished = finished | (symbols == O.END)
        assert bool((dec.runtime_symbols[step].cpu() == symbols).all()), step


@pytest.mark.parametrize("tie", [False, True])
def test_label_smoothing_follows_the_reference(cpu_model, tie):
    """label_smoothing as the reference computes it (SURVEY.md trap 14, pinned in
    test_oracle_vs_reference_code.py): ONE scalar - the mean over all positions, padding included, of the
    smoothed cross-entropy - times the mask.  The product adds eps * (logit_target - mean logit) to the
    fused plain cross-entropy; loss and every gradient against the oracle."""
    check_label_smoothing(tie, 1e-5, 1e-4)


def check_label_smoothing(tie, tol, gtol):
    from neuralmonkey_b200 import runtime, tf
    from neuralmonkey_b200.attention import Attention
    from neuralmonkey_b200.decoders import Decoder
    from neuralmonkey_b200.encoders import SentenceEncoder
    from neuralmonkey_b200.trainers import CrossEntropyTrainer
    from neuralmonkey_b200.vocabulary import Vocabulary
    runtime.reset()
    src_vocab = Vocabulary(["s{}".format(i) for i in range(26)])
    tgt_vocab = Vocabulary(["t{}".format(i) for i in range(36)])
    enc = SentenceEncoder(name="sentence_encoder", vocabulary=src_vocab, data_id="source", embedding_size=6,
                          rnn_size=5, max_input_len=10)
    att = Attention(name="attention", encoder=enc)
    dec = Decoder(encoders=[enc], vocabulary=tgt_vocab, data_id="target", name="decoder", max_output_len=10,
                  rnn_size=8, embedding_size=8, attentions=[att], label_smoothing=0.1, tie_embeddings=tie,
                  supress_unk=False)
    trainer = CrossEntropyTrainer(decoders=[dec], optimizer=tf.AdamOptimizer(learning_rate=1e-3))
    for part in trainer.parameterizeds:
        part.ensure_declared()
    runtime.arena().finalize(runtime.device())
    model = {"enc": enc, "att": att, "dec": dec, "arena": runtime.arena()}
    params = oracle_params_for(model)
    model["arena"].load_dict(params)
    src, tgt = random_batch(5, 8, 7, 30, 40, seed=1)
    feed(model, src, tgt, train=True)
    p = {n: v.clone().requires_grad_(True) for n, v in params.items()}
    if tie:      # the oracle's RNN decoder reads state_to_word_W / b: the transposed embeddings, zero bias
        p["decoder/state_to_word_W"] = p["decoder/word_embeddings"].t()
        p["decoder/state_to_word_b"] = torch.zeros(40)
    spec = O.RNNDecoderSpec("decoder", "attention", 10, "tanh", False)
    odec = O.decoder_train(p, spec, O.sentence_encoder(p, "sentence_encoder", src), tgt.t(), label_smoothing=0.1)
    assert max_abs(dec.train_xents, odec["train_xents"]) < tol
    assert abs(float(dec.train_loss) - float(odec["train_loss"])) < tol
    model["arena"].zero_grad()
    dec.train_loss.backward()
    odec["train_loss"].backward()
    for name in model["arena"].train_names:
        view = model["arena"].get(name)   # CPU stand-ins leave gradients in .grad, the real ops in the arena
        got = ((view.grad if view.grad is not None else torch.zeros_like(view)) + model["arena"].grad(name)).cpu()
        want = p[name].grad if p[name].grad is not None else torch.zeros_like(p[name])
        assert float((got - want.reshape(got.shape)).norm()) <= gtol * float(want.norm()) + 1e-7, name


def _two_sessions(model, params_a, params_b, runners, batch_feed):
    """A TensorFlowManager with two sessions holding params_a / params_b, executed on the fed batch."""
    from neuralmonkey_b200.tf_manager import TensorFlowManager
    manager = TensorFlowManager(num_sessions=2, num_threads=1)
    arena = model["arena"]
    for index, params in enumerate((params_a, params_b)):
        arena.load_dict(params)
        manager._session_buffers()[index].copy_(arena.params.detach())

    class _Feed:                      # the manager feeds through `feed_dict`; the test feeds tensors directly
        def feed_dict(self, _batch, _train):
            batch_feed()
    return manager.execute(None, {_Feed()}, runners, train=False, compute_losses=False, summaries=False)


def test_greedy_runner_over_two_sessions(cpu_model):
    """GreedyRunner with num_sessions = 2 (runner.py:33-62): every session decodes on its own, the
    fetched log-probabilities are combined with logaddexp per step and the argmax is decoded."""
    import numpy as np
    from neuralmonkey_b200.runners import GreedyRunner
    model = build_bahdanau(**TOY)
    params_a, params_b = oracle_params_for(model, seed=7), oracle_params_for(model, seed=8)
    src, tgt = random_batch(5, 8, 7, TOY["vs"], TOY["vt"], seed=3)
    runner = GreedyRunner(output_series="target", decoder=model["dec"])
    result, = _two_sessions(model, params_a, params_b, [runner], lambda: feed(model, src, tgt, train=False))
    spec = oracle_spec(True, 10, True)
    logprobs = [O.decoder_greedy(p, spec, O.sentence_encoder(p, "sentence_encoder", src))["runtime_logprobs"].numpy()
                for p in (params_a, params_b)]
    steps = logprobs[0].shape[0]
    summed = [np.logaddexp(logprobs[0][t], logprobs[1][t]) if t < logprobs[1].shape[0] else logprobs[0][t]
              for t in range(steps)]
    want = model["dec"].vocabulary.vectors_to_sentences([np.argmax(s, axis=1) for s in summed])
    assert result.outputs["target"] == want
    # the ensemble of a model with itself decodes what the model decodes
    same, = _two_sessions(model, params_a, params_a, [runner], lambda: feed(model, src, tgt, train=False))
    single = model["dec"].vocabulary.vectors_to_sentences([np.argmax(s, axis=1) for s in logprobs[0]])
    assert same.outputs["target"] == single


@pytest.mark.parametrize("parent", ["rnn", "transformer"])
def test_beam_search_over_two_sessions(cpu_model, parent):
    """BeamSearchRunner with num_sessions = 2 (beamsearch_runner.py:44-118): one beam, each session steps
    its own decoder, next-token log-probabilities averaged in probability space.  Against the oracle's
    beam search over a pair of decoders, and the reference's own check (tests/tests_run.sh:40-50): the
    ensemble of a model with itself scores what the single model scores."""
    import math
    from neuralmonkey_b200.decoders import BeamSearchDecoder
    from neuralmonkey_b200.runners import BeamSearchRunner
    beam, max_steps, alpha = 3, 6, 1.0
    if parent == "rnn":
        model = build_bahdanau(**TOY)
        params_a, params_b = oracle_params_for(model, seed=7), oracle_params_for(model, seed=8)
        src, _ = random_batch(1, 8, 7, TOY["vs"], TOY["vt"], seed=9)
        feeder = lambda: feed(model, src, None, train=False)
        spec = oracle_spec()

        def session(p):
            oenc = O.sentence_encoder(p, "sentence_encoder", src)
            states, mask = oenc["temporal_states"].repeat_interleave(beam, 0), oenc["temporal_mask"].repeat_interleave(beam, 0)
            hidden = O.bahdanau_precompute(p, "attention", states)
            emb = p["decoder/word_embeddings"]

            def run(words, prev, _finished=None):
                output, cell, _c, _w = O.decoder_step(p, spec, emb[words], prev, hidden, states, mask)
                return cell, torch.log_softmax(O.state_to_logits(p, spec, output), -1)
            prev0 = O.decoder_initial_state(p, spec, oenc["output"]).repeat_interleave(beam, 0)
            return run, prev0
    else:
        from tests.test_gpu_transformer import feed_transformer, oracle_encoder
        model, params_a, src, _tgt, cfg = _transformer(seed=2, bsz=2)
        params_b = oracle_params_for(model, scale=0.2, seed=11)
        for name in params_b:
            if name.endswith("gamma"):
                params_b[name] = 1.0 + params_b[name]
        model["dec"].use_kv_cache = True
        feeder = lambda: feed_transformer(model, src, None, train=False)
        spec = O.TransformerDecoderSpec("decoder", cfg["depth"], cfg["heads"], cfg["heads"], cfg["max_len"], True, False)

        def session(p):
            oenc = oracle_encoder(p, src, cfg)
            states, emask = oenc["states"].repeat_interleave(beam, 0), oenc["mask"].repeat_interleave(beam, 0)
            emb = p["decoder/word_embeddings"]

            def run(words, prev, finished=None):      # prev = (sequence so far, its key mask)
                live = torch.ones(len(words)) if finished is None else (~finished).to(emb.dtype)
                seq = torch.cat([prev[0], emb[words].unsqueeze(1)], 1)
                mask = torch.cat([prev[1], live.unsqueeze(1)], 1)
                out = O.transformer_decoder_stack(p, spec, seq, mask, states, emask)
                return (seq, mask), torch.log_softmax(O.transformer_logits(p, spec, out[:, -1]), -1)
            rows = states.shape[0]
            return run, (torch.zeros(rows, 0, emb.shape[1]), torch.zeros(rows, 0))
    bs = BeamSearchDecoder(name="bs", parent_decoder=model["dec"], beam_size=beam, max_steps=max_steps,
                           length_normalization=alpha)
    bs.use_cuda_graph = False
    runner = BeamSearchRunner(output_series="target", decoder=bs, rank=1)

    def feed_all():
        feeder()
        bs.reset_batch()
        bs.batch_size = src.shape[0]

    def oracle_ensemble(param_sets):
        sessions = [session(p) for p in param_sets]
        rows = src.shape[0] * beam
        start = torch.full((rows,), O.START, dtype=torch.int64)
        firsts = [run(start, prev0) for run, prev0 in sessions]
        average = lambda lps: torch.logsumexp(torch.stack(lps, 0), 0) - math.log(len(lps))

        def step_fn(states, words, finished):
            outs = [run(words, st, finished) for (run, _p), st in zip(sessions, states)]
            return [o[0] for o in outs], average([o[1] for o in outs])

        def gather(states, idx):
            return [tuple(x[idx] for x in st) if isinstance(st, tuple) else st[idx] for st in states]
        return O.beam_search(step_fn, [f[0] for f in firsts], average([f[1] for f in firsts]), beam, max_steps,
                             alpha, gather)

    result, = _two_sessions(model, params_a, params_b, [runner], feed_all)
    want = oracle_ensemble([params_a, params_b])
    vocab = model["dec"].vocabulary
    for b in range(src.shape[0]):
        toks = []
        for t in want["token_ids"][:, b, 0].tolist():
            if t == O.END:
                break
            toks.append(vocab.index_to_word[t])
        assert result.outputs["target"][b] == toks
    assert abs(result.losses["target/beam_search_score"] - float(want["scores"][:, 0].sum())) < 1e-3
    # the reference's ensemble test: a model ensembled with itself scores what it scores alone
    twice, = _two_sessions(model, params_a, params_a, [runner], feed_all)
    model["arena"].load_dict(params_a)
    feed_all()
    alone = runner.get_executable(compute_losses=False, summaries=False, num_sessions=1)
    alone.execute()
    assert twice.outputs["target"] == alone.result.outputs["target"]
    assert abs(twice.losses["target/beam_search_score"] - alone.result.losses["target/beam_search_score"]) < 1e-4


def test_ensemble_of_a_model_with_itself_through_neuralmonkey_run(cpu_model, monkeypatch, tmp_path):
    """The reference's ensemble check (tests/tests_run.sh:40-50) end to end: train the Transformer +
    beam search experiment, then `neuralmonkey-run` it once alone and once as an ensemble of two copies
    of the same variables (tf_manager.num_sessions=2, `variables=[v, v]` in the datasets INI): the
    beam-search scores and the BLEU agree."""
    import json
    import os
    from neuralmonkey_b200.trainers.generic_trainer import GenericTrainer
    from tests import test_gpu_cli as cli
    monkeypatch.setattr(GenericTrainer, "_adam_kernel", cpu_ops.adam_kernel)
    data, out = str(tmp_path / "data"), str(tmp_path / "out")
    cli._write_data(data)
    ini = tmp_path / "exp.ini"
    text = cli.TRANSFORMER_INI.format(out=out, data=data, epochs=1)
    ini.write_text(text)
    _cli(monkeypatch, "neuralmonkey_b200.train", ["neuralmonkey-train", str(ini)])
    variables = os.path.join(out, "variables.data.final")
    ensemble_ini = tmp_path / "ensemble.ini"
    assert "num_sessions=1" in text
    ensemble_ini.write_text(text.replace("num_sessions=1", "num_sessions=2"))
    results = {}
    for name, config, files in (("single", ini, [variables]), ("ensemble", ensemble_ini, [variables, variables])):
        run_ini = tmp_path / (name + "_data.ini")
        run_ini.write_text("""
[main]
test_datasets=[<val_data>]
variables={files}

[batching]
class=dataset.BatchingScheme
batch_size=10

[val_data]
class=dataset.load
series=["source", "target"]
data=["{data}/val.src", "{data}/val.tgt"]
batching=<batching>
""".format(files=json.dumps(files), data=data))
        _cli(monkeypatch, "neuralmonkey_b200.run",
             ["neuralmonkey-run", str(config), str(run_ini), "--json", str(tmp_path / (name + ".json"))])
        results[name] = json.load(open(tmp_path / (name + ".json")))[0]
    key = "target_beam.rank001/beam_search_score"
    assert key in results["single"]
    assert abs(results["single"][key] - results["ensemble"][key]) < 1e-3 * max(1.0, abs(results["single"][key]))
    assert results["single"]["target_beam.rank001/BLEU-4"] == pytest.approx(results["ensemble"]["target_beam.rank001/BLEU-4"])


def test_var_scopes_restrict_the_update(cpu_model, monkeypatch):
    """GenericTrainer(var_scopes=[...]) (generic_trainer.py:196-205): only variables whose name starts
    with one of the scopes are in `var_list` and move; the segment flags / gradient mask handed to the
    optimizer kernel exclude exactly the others."""
    from neuralmonkey_b200 import runtime, tf
    from neuralmonkey_b200.trainers import CrossEntropyTrainer
    from neuralmonkey_b200.trainers.generic_trainer import GenericTrainer
    monkeypatch.setattr(GenericTrainer, "_adam_kernel", cpu_ops.adam_kernel)
    model = build_bahdanau(**TOY)
    scoped = CrossEntropyTrainer(decoders=[model["dec"]], optimizer=tf.AdamOptimizer(learning_rate=1e-2),
                                 var_scopes=["decoder", "attention/attn_sim"])
    arena = model["arena"]
    arena.load_dict(oracle_params_for(model))
    names = arena.train_names
    assert scoped.var_list == [n for n in names if n.startswith("decoder") or n.startswith("attention/attn_sim")]
    flags, mask = scoped._scope_restriction(arena.seg_reg)
    for i, name in enumerate(names):
        inside = name in scoped.var_list
        assert int(flags[i]) == (int(arena.seg_reg[i]) if inside else 2), name
        lo, hi = int(arena.seg_off[i]), int(arena.seg_off[i + 1])
        assert float(mask[lo:hi].min()) == float(mask[lo:hi].max()) == (1.0 if inside else 0.0)
    src, tgt = random_batch(6, 8, 7, TOY["vs"], TOY["vt"], seed=0)
    before = arena.state_dict()
    feed(model, src, tgt, train=True)
    scoped.train_step()
    after = arena.state_dict()
    for name in names:
        moved = not torch.equal(before[name], after[name])
        assert moved == (name in scoped.var_list and not name.endswith("attn_bias")) or name.endswith("attn_bias"), name


def test_attention_dropout_rides_into_the_fused_core(cpu_model, monkeypatch):
    """attention(..., attention_dropout_keep_prob < 1) in train mode: the mask drawn for the weights
    [batch, heads, time_q, time_k] is handed to the attention core, which applies it between the softmax
    and the values - against the oracle with the same mask (whose placement is pinned to the reference)."""
    import types
    from neuralmonkey_b200.attention import scaled_dot_product as sdp
    g = torch.Generator().manual_seed(4)
    dim, heads = 12, 3
    kernels = {n: torch.randn(dim, dim, generator=g) * 0.3 for n in ("query_proj", "keys_proj", "vals_proj", "output_proj")}
    part = types.SimpleNamespace(var=lambda name: kernels[name.split("/")[1]].requires_grad_(True), train_mode=True)
    q, k = torch.randn(2, 5, dim, generator=g), torch.randn(2, 7, dim, generator=g)
    key_mask = torch.tensor([[1, 1, 1, 1, 1, 0, 0], [1, 1, 1, 0, 0, 0, 0]], dtype=torch.float32)
    mask = (torch.rand(2, heads, 5, 7, generator=g) < 0.8).float() / 0.8
    seen = {}

    def fixed_mask(shape, keep_prob, train_mode, device):
        seen["shape"], seen["keep"] = tuple(shape), keep_prob
        return mask
    monkeypatch.setattr(sdp, "dropout_mask", fixed_mask)
    ctx, _w = sdp.attention(part, "s", q, k, k, key_mask, heads, False, 0.8, True, False)
    assert seen == {"shape": (2, heads, 5, 7), "keep": 0.8}
    p = {"s/{}/kernel".format(n): v.detach() for n, v in kernels.items()}
    want, _ = O.multihead_attention(p, "s", q, k, k, key_mask, heads, drop_mask=mask)
    assert max_abs(ctx, want) < 1e-5
    # evaluation mode: no mask at all
    ctx_eval, _ = sdp.attention(part, "s", q, k, k, key_mask, heads, False, 0.8, False, False)
    assert max_abs(ctx_eval, O.multihead_attention(p, "s", q, k, k, key_mask, heads)[0]) < 1e-5


@pytest.mark.parametrize("case", ["space", "cross"])
def test_transformer_encoder_options_against_the_reference_run(cpu_model, case):
    """The PRODUCT's TransformerEncoder (over stand-in ops) against the outputs of the REFERENCE's
    TransformerEncoder executed over the numpy TF stand-in (tests/golden/tf_shim_golden.npz), with the
    variables the reference drew under its own names loaded into the arena: the target-space embedding,
    projection biases, no position signal, cross-attention to another encoder."""
    import os
    import types
    import numpy as np
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.encoders import TransformerEncoder
    from neuralmonkey_b200.model.stateful import TemporalStateful
    golden = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tf_shim_golden.npz"))
    name = "tx_" + case
    runtime.reset()

    class Sequence(TemporalStateful):
        def __init__(self, states, mask):
            self._states, self._mask = torch.from_numpy(states), torch.from_numpy(mask)
        temporal_states = property(lambda self: self._states)
        temporal_mask = property(lambda self: self._mask)
        dimension = property(lambda self: self._states.shape[-1])

    inputs = Sequence(golden["tx_in"], golden["tx_mask"])
    opts = (dict(target_space_id=5, use_att_transform_bias=True) if case == "space" else
            dict(use_positional_encoding=False, n_cross_att_heads=2,
                 input_for_cross_attention=Sequence(golden["tx_other"], golden["tx_other_mask"])))
    enc = TransformerEncoder(name=name, input_sequence=inputs, ff_hidden_size=20, depth=2, n_heads=3, **opts)
    enc.ensure_declared()
    arena = runtime.arena()
    arena.finalize(runtime.device())
    reference_vars = {k[4:]: torch.from_numpy(golden[k]) for k in golden.files if k.startswith("xv::" + name + "/")}
    assert set(arena.order) == set(reference_vars)           # the same variables under the same names
    arena.load_dict(reference_vars)
    enc.reset_batch()
    enc.train_mode, enc.batch_size = False, 3
    assert max_abs(enc.temporal_states, torch.from_numpy(golden[name + "_states"])) < 3e-5
    assert max_abs(enc.output, torch.from_numpy(golden[name + "_output"])) < 1e-4


def _golden():
    import os
    import numpy as np
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tf_shim_golden.npz"))


@pytest.mark.parametrize("tag,layers,residual,layer_norm,final_norm,scale", [
    ("sentence", [(4, "bidirectional")], False, False, True, False),
    ("deep", [(4, "forward"), (4, "backward"), (2, "bidirectional"), (3, "bidirectional")], True, True, True, True),
    ("plain", [(3, "backward"), (3, "forward")], True, False, False, False),
    ("nematus", [(4, "bidirectional", "NematusGRU"), (3, "forward", "NematusGRU")], False, False, True, False),
    ("mixed", [(4, "forward", "LSTM"), (4, "backward", "NematusGRU"), (3, "bidirectional", "NematusGRU"),
               (2, "bidirectional", "LSTM")], True, True, True, False)])
def test_recurrent_encoder_against_the_reference_run(cpu_model, tag, layers, residual, layer_norm, final_norm, scale):
    """The PRODUCT's EmbeddedFactorSequence + RecurrentEncoder against the outputs of the REFERENCE's classes
    run over the TF stand-in, the reference's variables loaded under the reference's names."""
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.encoders import RecurrentEncoder
    from neuralmonkey_b200.model.sequence import EmbeddedFactorSequence
    from neuralmonkey_b200.vocabulary import Vocabulary
    golden = _golden()
    name = "re_" + tag
    runtime.reset()
    factors = [torch.from_numpy(f) for f in golden[name + "_ids"]]
    sizes = [golden["ev::{}_input/embedding_matrix_{}".format(name, i)].shape for i in range(len(factors))]
    seq = EmbeddedFactorSequence(name=name + "_input",
                                 vocabularies=[Vocabulary(["w{}".format(j) for j in range(s[0] - 4)]) for s in sizes],
                                 data_ids=["f{}".format(i) for i in range(len(factors))],
                                 embedding_sizes=[s[1] for s in sizes], scale_embeddings_by_depth=scale)
    # the generator drove RecurrentEncoder.rnn directly, past the constructor's check that residual layers
    # have one width (which the product's constructor repeats): set the flag after construction
    enc = RecurrentEncoder(name=name, input_sequence=seq, rnn_layers=layers, add_residual=False,
                           add_layer_norm=layer_norm, include_final_layer_norm=final_norm)
    enc.add_residual = residual
    enc.ensure_declared()
    arena = runtime.arena()
    arena.finalize(runtime.device())
    reference_vars = {k[4:]: torch.from_numpy(golden[k]) for k in golden.files
                      if k.startswith("ev::" + name + "/") or k.startswith("ev::" + name + "_input/")}
    assert set(arena.order) == set(reference_vars)
    arena.load_dict(reference_vars)
    seq.feed_ids(factors, train=False)
    enc.reset_batch()
    enc.train_mode, enc.batch_size = False, factors[0].shape[0]
    assert max_abs(seq.temporal_states, torch.from_numpy(golden[name + "_embedded"])) < 1e-6
    assert max_abs(enc.temporal_states, torch.from_numpy(golden[name + "_states"])) < 1e-5
    assert max_abs(enc.output, torch.from_numpy(golden[name + "_output"])) < 1e-5


def _stub_encoder(states, mask, output):
    from neuralmonkey_b200.model.stateful import TemporalStatefulWithOutput

    class Encoder(TemporalStatefulWithOutput):
        temporal_states = property(lambda self: states)
        temporal_mask = property(lambda self: mask)
        output = property(lambda self: output)
        dimension = property(lambda self: states.shape[-1])
    return Encoder()


@pytest.mark.parametrize("prefix,tag,cell,conditional,out_proj,enc_proj,hsz,esz", [
    ("r", "maxout", "GRU", False, "maxout", "linear", 7, 5),
    ("r", "tanh", "GRU", False, "tanh", "linear", 6, 6),
    ("v", "nematus", "NematusGRU", True, "nematus", "nematus", 7, 5),
    ("v", "cond_gru", "GRU", True, "mlp", "concat", 10, 5),
    ("v", "nematus_plain", "NematusGRU", False, "maxout", "empty", 7, 5),
    ("v", "lstm", "LSTM", False, "maxout", "linear", 7, 5)])
def test_attention_decoder_against_the_reference_run(cpu_model, prefix, tag, cell, conditional, out_proj, enc_proj,
                                                     hsz, esz):
    """The PRODUCT's Attention + Decoder (training pass and greedy loop, over stand-in ops) against the outputs
    of the REFERENCE's Attention + Decoder run over the TF stand-in - default configuration and every N4
    variant - with the reference's variables loaded under the reference's names."""
    golden = _golden()
    key = "{}d_{}_".format(prefix, tag)
    g = lambda n: torch.from_numpy(golden[key + n])
    _att, dec, feed_all = _reference_decoder(prefix, tag, cell, conditional, out_proj, enc_proj, hsz, esz)
    feed_all(True)
    assert max_abs(dec.train_logits, g("train_logits")) < 2e-5
    assert abs(float(dec.train_loss) - float(golden[key + "train_loss"])) < 2e-5
    feed_all(False)
    run_logits = g("run_logits")
    assert dec.runtime_logits.shape == run_logits.shape
    assert max_abs(dec.runtime_logits, run_logits) < 2e-5
    assert bool((dec.runtime_symbols == g("run_symbols")).all())


def _reference_decoder(prefix, tag, cell, conditional, out_proj, enc_proj, hsz, esz, use_mask=None):
    """Attention + Decoder of the product holding the variables of one reference run (tf_shim_golden.npz)."""
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.attention import Attention
    from neuralmonkey_b200.decoders import Decoder
    from neuralmonkey_b200.decoders.encoder_projection import nematus_projection
    from neuralmonkey_b200.decoders.output_projection import maxout_output, mlp_output, nematus_output
    from neuralmonkey_b200.vocabulary import Vocabulary
    golden = _golden()
    dname, aname, key = "{}d_{}".format(prefix, tag), "{}a_{}".format(prefix, tag), "{}d_{}_".format(prefix, tag)
    varkey = "{}v::".format(prefix)
    runtime.reset()
    g = lambda n: torch.from_numpy(golden[key + n])
    table = g("table")
    if use_mask is None:
        use_mask = not (prefix == "r" and tag == "tanh")
    mask = g("mask") if use_mask else torch.ones(g("states").shape[:2])
    encoder = _stub_encoder(g("states"), mask, g("enc_out"))
    vocab = Vocabulary(["t{}".format(i) for i in range(table.shape[0] - 4)])
    att = Attention(name=aname, encoder=encoder, state_size=8)
    projection = {"maxout": lambda: maxout_output(esz), "tanh": lambda: None, "nematus": lambda: nematus_output(esz),
                  "mlp": lambda: mlp_output([9, esz])}[out_proj]()
    gold = g("gold").t().contiguous()
    dec = Decoder(encoders=[] if enc_proj == "empty" else [encoder], vocabulary=vocab, data_id="target", name=dname,
                  max_output_len=gold.shape[1] if prefix == "v" else 6, rnn_size=None if enc_proj == "concat" else hsz,
                  embedding_size=esz, attentions=[att], output_projection=projection, rnn_cell=cell,
                  conditional_gru=conditional,
                  encoder_projection=nematus_projection() if enc_proj == "nematus" else None)
    for part in (att, dec):
        part.ensure_declared()
    arena = runtime.arena()
    arena.finalize(runtime.device())
    reference_vars = {k[4:]: torch.from_numpy(golden[k]) for k in golden.files
                      if k.startswith(varkey + dname + "/") or k.startswith(varkey + aname + "/")}
    reference_vars[dname + "/word_embeddings"] = table
    reference_vars[dname + "/state_to_word_W"], reference_vars[dname + "/state_to_word_b"] = g("w"), g("b")
    assert set(arena.order) == set(reference_vars), set(arena.order) ^ set(reference_vars)
    arena.load_dict({n: v.reshape(arena.variables[n].shape) for n, v in reference_vars.items()})
    bsz = gold.shape[0]

    def feed_all(train):
        att.reset_batch()
        att.train_mode, att.batch_size = train, bsz
        dec.feed_ids(gold, bsz, train=train)

    return att, dec, feed_all


@pytest.mark.parametrize("search,dtag,out_proj,hsz,esz,use_mask", [
    ("rnn", "beam", "maxout", 7, 5, True), ("rnn1", "beam1", "tanh", 6, 6, True), ("rnn2", "beam2", "tanh", 6, 6, False)])
def test_beam_search_over_the_rnn_decoder_against_the_reference_run(cpu_model, search, dtag, out_proj, hsz, esz,
                                                                    use_mask):
    """The PRODUCT's BeamSearchDecoder over its attention Decoder against BeamSearchDecoder.outputs of the
    REFERENCE run to the end over the reference's Decoder (one sentence; early </s>, max_steps reached)."""
    from neuralmonkey_b200.decoders import BeamSearchDecoder
    golden = _golden()
    pre = "bsearch_{}_".format(search)
    g = lambda n: torch.from_numpy(golden[pre + n])
    _att, dec, feed_all = _reference_decoder("r", dtag, "GRU", False, out_proj, "linear", hsz, esz, use_mask)
    bs = BeamSearchDecoder(name="bs", parent_decoder=dec, beam_size=int(golden[pre + "beam"]),
                           max_steps=int(golden[pre + "max_steps"]), length_normalization=float(golden[pre + "alpha"]))
    bs.use_cuda_graph = False
    feed_all(False)
    bs.reset_batch()
    bs.batch_size = 1
    out = bs.outputs
    assert bool((out.last_search_step_output.token_ids == g("token_ids")).all())
    assert max_abs(out.last_search_step_output.scores, g("scores")) < 2e-5
    assert bool((out.last_search_state.lengths == g("lengths")).all())
    assert bool((out.last_search_state.finished.to(torch.bool) == g("finished")).all())


def test_transformer_decoder_against_the_reference_run(cpu_model):
    """The PRODUCT's TransformerDecoder - training pass, greedy loop (with and without the KV cache) and a
    whole beam search through BeamSearchDecoder - against the REFERENCE's TransformerDecoder /
    BeamSearchDecoder.outputs run over the TF stand-in, the reference's variables under its names."""
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.decoders import BeamSearchDecoder, TransformerDecoder
    from neuralmonkey_b200.vocabulary import Vocabulary
    golden = _golden()
    g = lambda n: torch.from_numpy(golden[n])
    runtime.reset()
    encoder = _stub_encoder(g("tenc_states"), g("tenc_mask"), g("tenc_output"))
    vocab = Vocabulary(["t{}".format(i) for i in range(golden["tloop_table"].shape[0] - 4)])
    dec = TransformerDecoder(name="tdec", encoders=[encoder], vocabulary=vocab, data_id="target", ff_hidden_size=20,
                             n_heads_self=3, n_heads_enc=2, depth=2, max_output_len=6, embedding_size=12,
                             tie_embeddings=True)
    dec.ensure_declared()
    arena = runtime.arena()
    arena.finalize(runtime.device())
    reference_vars = {k[4:]: g(k) for k in golden.files if k.startswith("tv::tdec/")}
    reference_vars["tdec/word_embeddings"] = g("tloop_table")
    assert set(arena.order) == set(reference_vars), set(arena.order) ^ set(reference_vars)
    arena.load_dict(reference_vars)
    gold = g("tloop_gold").t().contiguous()
    dec.feed_ids(gold, 3, train=True)
    assert max_abs(dec.train_logits, g("tloop_train_logits")) < 5e-5
    for kv_cache, table, case in ((True, "tloop_table", "run"), (False, "tloop_table", "run"),
                                  (True, "tloop_table_eos", "run_eos")):
        arena.load_dict({"tdec/word_embeddings": g(table)})
        dec.use_kv_cache = kv_cache
        dec.feed_ids(gold, 3, train=False)
        assert bool((dec.runtime_symbols == g("tloop_{}_symbols".format(case))).all())
        assert bool((dec.runtime_mask == g("tloop_{}_mask".format(case))).all())
        assert max_abs(dec.runtime_logits, g("tloop_{}_logits".format(case))) < 5e-5
    for tag, table in (("tr", "tloop_table"), ("tr_eos", "tloop_table_eos")):
        arena.load_dict({"tdec/word_embeddings": g(table)})
        pre = "bsearch_{}_".format(tag)
        bs = BeamSearchDecoder(name="bs_" + tag, parent_decoder=dec, beam_size=int(golden[pre + "beam"]),
                               max_steps=int(golden[pre + "max_steps"]),
                               length_normalization=float(golden[pre + "alpha"]))
        bs.use_cuda_graph = False
        dec.feed_ids(None, 3, train=False)
        bs.reset_batch()
        bs.batch_size = 3
        out = bs.outputs
        # slot 0 of the reference's history is the first step's greedy symbol - and so is the product's
        assert bool((out.last_search_step_output.token_ids == g(pre + "token_ids")).all())
        assert max_abs(out.last_search_step_output.scores, g(pre + "scores")) < 2e-5
        assert bool((out.last_search_state.lengths == g(pre + "lengths")).all())
        assert bool((out.last_search_state.finished.to(torch.bool) == g(pre + "finished")).all())


@pytest.mark.parametrize("strategy", ["serial", "parallel", "flat", "hierarchical"])
def test_multi_source_decoder_layers_against_the_reference_run(cpu_model, strategy):
    """The PRODUCT's TransformerDecoder layer stack over two encoders, each combination strategy, against
    the REFERENCE's TransformerDecoder.layer run over the TF stand-in (variables and names the reference's)."""
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.decoders import TransformerDecoder
    from neuralmonkey_b200.vocabulary import Vocabulary
    golden = _golden()
    g = lambda n: torch.from_numpy(golden[n])
    name = "tms_" + strategy
    runtime.reset()
    encoders = [_stub_encoder(g("ms_enc_a"), g("ms_mask_a"), g("ms_enc_a").sum(1)),
                _stub_encoder(g("ms_enc_b"), g("ms_mask_b"), g("ms_enc_b").sum(1))]
    dec = TransformerDecoder(name=name, encoders=encoders, vocabulary=Vocabulary(["a", "b", "c"]), data_id="target",
                             ff_hidden_size=20, n_heads_self=3, n_heads_enc=3 if strategy == "flat" else [3, 2],
                             depth=2, max_output_len=6, embedding_size=12, tie_embeddings=True,
                             attention_combination_strategy=strategy,
                             n_heads_hier=4 if strategy == "hierarchical" else None)
    dec.ensure_declared()
    arena = runtime.arena()
    arena.finalize(runtime.device())
    reference_vars = {k[4:]: g(k) for k in golden.files if k.startswith("mv::" + name + "/")}
    assert set(arena.order) - {name + "/word_embeddings"} == set(reference_vars)
    arena.load_dict(reference_vars)
    dec.reset_batch()
    dec.train_mode, dec.batch_size = False, 3
    assert max_abs(dec._stack(g("ms_in"), g("ms_mask")), g(name + "_states")) < 3e-5


def _deterministic_dropout(monkeypatch):
    """The deterministic mask of tests/golden/tf_numpy_shim.feature_dropout_mask in place of the random one,
    in every module that draws dropout masks."""
    import numpy as np
    from neuralmonkey_b200.attention import scaled_dot_product
    from neuralmonkey_b200.decoders import decoder as decoder_module
    from neuralmonkey_b200.nn import utils

    def mask(shape, keep_prob, train_mode, device):
        if keep_prob >= 1.0 or not train_mode:
            return None
        pattern = torch.from_numpy(np.where(np.arange(int(shape[-1])) % 2 == 0, 1.0 / keep_prob, 0.0).astype(np.float32))
        return pattern.expand(tuple(int(d) for d in shape)).clone()
    for module in (utils, scaled_dot_product, decoder_module):
        monkeypatch.setattr(module, "dropout_mask", mask)


def test_dropout_placement_against_the_reference_run(cpu_model, monkeypatch):
    """WHERE dropout is applied.  The reference's RecurrentEncoder + Attention + Decoder ran in training
    mode with keep_prob 0.5 and a deterministic mask in place of tf.nn.dropout (every second entry of the
    last axis dropped); the product runs with the same mask.  Equal outputs pin the placement traps: the
    initial state dropped twice (inside the linear projection and again in `initial_state`), the attention
    queried with the undropped cell output, the dropped output fed back as the next state, dropout on the
    attention states, on the contexts and inside the maxout projection, on embeddings and encoder layers."""
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.attention import Attention
    from neuralmonkey_b200.decoders import Decoder
    from neuralmonkey_b200.decoders.output_projection import maxout_output
    from neuralmonkey_b200.encoders import RecurrentEncoder
    from neuralmonkey_b200.model.sequence import EmbeddedFactorSequence
    from neuralmonkey_b200.vocabulary import Vocabulary
    _deterministic_dropout(monkeypatch)
    golden = _golden()
    g = lambda n: torch.from_numpy(golden[n])
    runtime.reset()
    seq = EmbeddedFactorSequence(name="dr_enc_input", vocabularies=[Vocabulary(["w{}".format(i) for i in range(5)])],
                                 data_ids=["f0"], embedding_sizes=[6])
    enc = RecurrentEncoder(name="dr_enc", input_sequence=seq, rnn_layers=[(4, "bidirectional"), (8, "forward")],
                           add_residual=True, dropout_keep_prob=0.5)
    att = Attention(name="dr_att", encoder=enc, state_size=7, dropout_keep_prob=0.5)
    dec = Decoder(encoders=[enc], vocabulary=Vocabulary(["t{}".format(i) for i in range(8)]), data_id="target",
                  name="dr_dec", max_output_len=5, dropout_keep_prob=0.5, embedding_size=5, rnn_size=6,
                  attentions=[att], output_projection=maxout_output(5, 0.5))
    for part in (enc, att, dec):
        part.ensure_declared()
    arena = runtime.arena()
    arena.finalize(runtime.device())
    reference_vars = {k[4:]: g(k) for k in golden.files if k.startswith("dv::")}
    assert set(arena.order) == set(reference_vars), set(arena.order) ^ set(reference_vars)
    arena.load_dict({n: v.reshape(arena.variables[n].shape) for n, v in reference_vars.items()})
    seq.feed_ids([g("dr_ids")], train=True)
    for part in (enc, att):
        part.reset_batch()
        part.train_mode, part.batch_size = True, 3
    dec.feed_ids(g("dr_gold").t().contiguous(), 3, train=True)
    assert max_abs(enc.temporal_states, g("dr_enc_states")) < 1e-5
    assert max_abs(enc.output, g("dr_enc_output")) < 1e-5
    assert max_abs(dec.initial_state, g("dr_dec_initial_state")) < 1e-5
    assert max_abs(dec.train_logits, g("dr_dec_train_logits")) < 5e-5
    assert abs(float(dec.train_loss) - float(golden["dr_dec_train_loss"])) < 5e-5


def test_transformer_dropout_placement_against_the_reference_run(cpu_model, monkeypatch):
    """The same for the Transformer: embedded inputs, every sublayer's output, the feed-forward activations
    and the ATTENTION WEIGHTS (self, masked self and encoder attention) under keep_prob 0.5 with the
    deterministic mask - encoder states, the decoder's training logits and loss against the reference run."""
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.decoders import TransformerDecoder
    from neuralmonkey_b200.encoders import TransformerEncoder
    from neuralmonkey_b200.model.sequence import EmbeddedSequence
    from neuralmonkey_b200.vocabulary import Vocabulary
    _deterministic_dropout(monkeypatch)
    golden = _golden()
    g = lambda n: torch.from_numpy(golden[n])
    runtime.reset()
    seq = EmbeddedSequence(name="dt_input", vocabulary=Vocabulary(["w{}".format(i) for i in range(5)]), data_id="f0",
                           embedding_size=12, scale_embeddings_by_depth=True)
    enc = TransformerEncoder(name="dt_enc", input_sequence=seq, ff_hidden_size=20, depth=2, n_heads=3,
                             dropout_keep_prob=0.5, attention_dropout_keep_prob=0.5)
    dec = TransformerDecoder(name="dt_dec", encoders=[enc], vocabulary=Vocabulary(["t{}".format(i) for i in range(7)]),
                             data_id="target", ff_hidden_size=20, n_heads_self=3, n_heads_enc=2, depth=2,
                             max_output_len=4, embedding_size=12, tie_embeddings=True, dropout_keep_prob=0.5,
                             attention_dropout_keep_prob=0.5, self_attention_dropout_keep_prob=0.5)
    for part in (enc, dec):
        part.ensure_declared()
    arena = runtime.arena()
    arena.finalize(runtime.device())
    reference_vars = {k[4:]: g(k) for k in golden.files if k.startswith("dw::")}
    assert set(arena.order) == set(reference_vars), set(arena.order) ^ set(reference_vars)
    arena.load_dict(reference_vars)
    seq.feed_ids([g("dt_ids")], train=True)
    enc.reset_batch()
    enc.train_mode, enc.batch_size = True, 3
    dec.feed_ids(g("dt_gold").t().contiguous(), 3, train=True)
    assert max_abs(enc.temporal_states, g("dt_enc_states")) < 3e-5
    assert max_abs(dec.train_logits, g("dt_dec_train_logits")) < 1e-4
    assert abs(float(dec.train_loss) - float(golden["dt_dec_train_loss"])) < 1e-4


def test_xent_and_plain_runners(cpu_model):
    """XentRunner: `train_xents` rows as the output series, their mean as the loss (xent_runner.py:13-35).
    PlainRunner: `decoder.decoded` - argmax over the non-<pad> symbols - through the vocabulary
    (plain_runner.py:20-58)."""
    import numpy as np
    from neuralmonkey_b200.runners import PlainRunner, XentRunner
    model = build_bahdanau(**TOY)
    params = oracle_params_for(model)
    model["arena"].load_dict(params)
    src, tgt = random_batch(5, 8, 7, TOY["vs"], TOY["vt"], seed=3)
    spec = oracle_spec(True, 10, True)
    oenc = O.sentence_encoder(params, "sentence_encoder", src)
    feed(model, src, tgt, train=False)
    exe = XentRunner(output_series="xents", decoder=model["dec"]).get_executable(compute_losses=True, num_sessions=1)
    exe.execute()
    want = O.decoder_train(params, spec, oenc, tgt.t())["train_xents"].numpy()
    assert np.abs(np.array(exe.result.outputs["xents"]) - want).max() < 1e-4
    assert abs(exe.result.losses["xents/xent"] - float(want.mean())) < 1e-5
    plain = PlainRunner(output_series="target", decoder=model["dec"]).get_executable(compute_losses=True, num_sessions=1)
    plain.execute()
    og = O.decoder_greedy(params, spec, oenc, tgt.t())
    assert plain.result.outputs["target"] == model["dec"].vocabulary.vectors_to_sentences(og["decoded"].numpy())
    assert sorted(plain.result.losses) == ["target/runtime_loss", "target/train_loss"]


def test_numpy_fillers_feed_precomputed_features(cpu_model, tmp_path):
    """SpatialFiller (1x1 conv projections named as tf.layers numbers them), StatefulFiller and TemporalFiller
    (encoders/numpy_stateful_filler.py of the reference) through the numpy readers, under the attention decoder."""
    import numpy as np
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.attention import Attention
    from neuralmonkey_b200.dataset import BatchingScheme, Dataset
    from neuralmonkey_b200.decoders import Decoder
    from neuralmonkey_b200.encoders.numpy_stateful_filler import SpatialFiller, StatefulFiller, TemporalFiller
    from neuralmonkey_b200.readers.numpy_reader import from_file_list, single_tensor
    from neuralmonkey_b200.readers.string_vector_reader import FloatVectorReader, get_string_vector_reader
    from neuralmonkey_b200.vocabulary import Vocabulary
    from tests.helpers import oracle_params_for

    rng = np.random.RandomState(5)
    maps = rng.randn(3, 2, 3, 6).astype(np.float32)
    names = []
    for i, m in enumerate(maps):
        np.savez(tmp_path / "m{}.npz".format(i), m)
        names.append("m{}".format(i))
    (tmp_path / "list.txt").write_text("\n".join(names) + "\n")
    read = from_file_list(str(tmp_path), [2, 3, 6], suffix=".npz")
    loaded = list(read([str(tmp_path / "list.txt")]))
    assert np.array_equal(np.stack(loaded), maps)
    with pytest.raises(ValueError):
        list(from_file_list(str(tmp_path), [2, 3, 5], suffix=".npz")([str(tmp_path / "list.txt")]))
    np.save(tmp_path / "a.npy", maps[:2])
    np.save(tmp_path / "b.npy", maps[2:])
    assert np.array_equal(single_tensor([str(tmp_path / "a.npy"), str(tmp_path / "b.npy")]), maps)
    (tmp_path / "vec.txt").write_text("1 2   3.5\n\n 4 -5e3 6\n")
    vecs = list(FloatVectorReader([str(tmp_path / "vec.txt")]))
    assert [v.tolist() for v in vecs] == [[1.0, 2.0, 3.5], [4.0, -5000.0, 6.0]] and vecs[0].dtype == np.float32
    with pytest.raises(ValueError):
        list(get_string_vector_reader(np.int32, columns=2)([str(tmp_path / "vec.txt")]))

    runtime.reset()
    vocab = Vocabulary(["t{}".format(i) for i in range(20)])
    enc = SpatialFiller(name="maps", input_shape=[2, 3, 6], data_id="maps", projection_dim=5, ff_hidden_dim=7)
    vec = StatefulFiller(name="vec", dimension=4, data_id="vec", output_shape=3)
    plain = SpatialFiller(name="plain", input_shape=[2, 3, 6], data_id="maps")
    seq = TemporalFiller(name="seq", data_id="seq", input_size=2, max_input_len=3)
    att = Attention(name="attention", encoder=enc, state_size=6)
    dec = Decoder(encoders=[enc, vec], vocabulary=vocab, data_id="target", name="decoder", max_output_len=5,
                  rnn_size=8, embedding_size=8, attentions=[att])
    for part in (enc, vec, plain, seq, att, dec):
        part.ensure_declared()
    arena = runtime.arena()
    arena.finalize(runtime.device())
    assert {"maps/conv2d/kernel", "maps/conv2d/bias", "maps/conv2d_1/kernel", "maps/conv2d_1/bias",
            "vec/dense/kernel", "vec/dense/bias"} <= set(arena.train_names)
    assert not any(n.startswith(("plain/", "seq/")) for n in arena.train_names)
    assert float(arena.get("maps/conv2d/bias").abs().max()) == 0.0          # tf.layers defaults
    limit = (6.0 / (6 + 7)) ** 0.5
    assert 0.5 * limit < float(arena.get("maps/conv2d/kernel").abs().max()) <= limit
    params = oracle_params_for({"arena": arena}, scale=0.3)
    arena.load_dict(params)

    sequences = [rng.randn(n, 2).astype(np.float32) for n in (4, 1, 2)]
    vectors = rng.randn(3, 4).astype(np.float32)
    data = Dataset("toy", {"maps": lambda: iter(maps), "vec": lambda: iter(vectors), "seq": lambda: iter(sequences)},
                   BatchingScheme(batch_size=3))
    for part in (enc, vec, plain, seq):
        part.feed_dict(data, train=True)
    k1, b1 = params["maps/conv2d/kernel"].reshape(6, 7), params["maps/conv2d/bias"]
    k2, b2 = params["maps/conv2d_1/kernel"].reshape(7, 5), params["maps/conv2d_1/bias"]
    want = torch.relu(torch.from_numpy(maps) @ k1 + b1) @ k2 + b2
    assert max_abs(enc.spatial_states, want) < 1e-5 and enc.dimension == 5
    assert max_abs(enc.output, want.mean(dim=(1, 2))) < 1e-5
    assert tuple(enc.spatial_mask.shape) == (3, 2, 3) and float(enc.spatial_mask.min()) == 1.0
    assert torch.equal(plain.spatial_states.cpu(), torch.from_numpy(maps)) and plain.dimension == 6
    want_vec = torch.from_numpy(vectors) @ params["vec/dense/kernel"] + params["vec/dense/bias"]
    assert max_abs(vec.output, want_vec) < 1e-5
    assert tuple(seq.temporal_states.shape) == (3, 3, 2)                      # clipped to max_input_len
    assert seq.temporal_mask.cpu().tolist() == [[1, 1, 1], [1, 0, 0], [1, 1, 0]]
    assert float(seq.temporal_states[1, 1:].abs().max()) == 0.0

    _src, tgt = random_batch(3, 4, 5, 20, 20, seed=4)
    att.reset_batch()
    att.train_mode, att.batch_size = True, 3
    dec.feed_ids(tgt, 3, train=True)
    # the initial state projects the concatenated outputs of both encoders (encoder_projection.py:47-73)
    oenc = {"output": torch.cat([want.mean(dim=(1, 2)), want_vec], dim=1),
            "temporal_states": want.reshape(3, 6, 5), "temporal_mask": torch.ones(3, 6)}
    odec = O.decoder_train(params, O.RNNDecoderSpec("decoder", "attention", 8, "tanh", False), oenc, tgt.t())
    assert abs(float(dec.train_loss) - float(odec["train_loss"])) < 1e-4
    float(dec.train_loss)
    dec.train_loss.backward()
    arena.fold_autograd_grads()
    runtime.reset()


def test_recurrent_encoder_over_a_temporal_filler(cpu_model):
    """`RecurrentEncoder(input_sequence=<TemporalFiller>)` - the encoder of the reference's audio INIs
    (tests/audio-classifier.ini:53-62, tests/ctc.ini:55-64) - against the oracle on ragged numeric sequences."""
    import numpy as np
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.dataset import BatchingScheme, Dataset
    from neuralmonkey_b200.encoders import RecurrentEncoder
    from neuralmonkey_b200.encoders.numpy_stateful_filler import TemporalFiller
    from tests.helpers import oracle_params_for
    runtime.reset()
    seq = TemporalFiller(name="input_seq", data_id="features", input_size=4)
    enc = RecurrentEncoder(name="encoder", input_sequence=seq, rnn_layers=[(5, "bidirectional"), (6, "backward")])
    for part in (seq, enc):
        part.ensure_declared()
    arena = runtime.arena()
    arena.finalize(runtime.device())
    params = oracle_params_for({"arena": arena}, scale=0.3)
    arena.load_dict(params)
    rng = np.random.RandomState(1)
    series = [rng.randn(n, 4).astype(np.float32) for n in (5, 2, 3)]
    data = Dataset("toy", {"features": lambda: iter(series)}, BatchingScheme(batch_size=3))
    seq.feed_dict(data, train=False)
    enc.feed_dict(data, train=False)
    want = O.recurrent_encoder(params, "encoder", seq.temporal_states, seq.temporal_mask,
                               [(5, "bidirectional", "GRU"), (6, "backward", "GRU")], False, False, True)
    assert max_abs(enc.temporal_states, want["temporal_states"]) < 1e-5
    assert max_abs(enc.output, want["output"]) < 1e-5
    assert torch.equal(enc.temporal_mask.cpu(), seq.temporal_mask.cpu())
    runtime.reset()


def test_every_optimizer_keeps_its_own_adam_state(cpu_model, monkeypatch, tmp_path):
    """Several trainers on one model (tests/bahdanau.ini: trainer1, trainer2, greedy_trainer): every
    tf.train.AdamOptimizer object owns its moment slots and beta-power accumulators, while ONE global step
    counts the updates of all of them (generic_trainer.py:56-57,183-195).  Two alternating trainers here against
    two oracle Adam states; then the whole state through a checkpoint into a fresh model."""
    from neuralmonkey_b200 import runtime, tf
    from neuralmonkey_b200.tf_manager import TensorFlowManager
    from neuralmonkey_b200.trainers import CrossEntropyTrainer
    from neuralmonkey_b200.trainers.generic_trainer import GenericTrainer
    monkeypatch.setattr(GenericTrainer, "_adam_kernel", cpu_ops.adam_kernel)
    lrs = (1e-2, 3e-3)
    src, tgt = random_batch(6, 8, 7, TOY["vs"], TOY["vt"], seed=3)

    def make():
        model = build_bahdanau(**TOY, lr=lrs[0])
        second = CrossEntropyTrainer(decoders=[model["dec"]], optimizer=tf.AdamOptimizer(learning_rate=lrs[1]))
        return model, [model["trainer"], second]

    def step(model, trainer):
        feed(model, src, tgt, train=True)
        return float(trainer.train_step()["losses"][0])

    model, trainers = make()
    params = oracle_params_for(model)
    model["arena"].load_dict(params)
    p32 = {n: v.clone() for n, v in params.items()}
    shared_p = {n: v.clone() for n, v in params.items()}     # what ONE state for both trainers would give
    states, shared = [O.AdamState(p32), O.AdamState(p32)], O.AdamState(shared_p)
    spec = oracle_spec(TOY["maxout"], TOY["max_len"], TOY["supress_unk"])
    order = [0, 0, 1, 0, 1]
    for which in order:
        loss = step(model, trainers[which])
        ref = O.train_step(p32, spec, "sentence_encoder", src, tgt.t(), states[which], lr=lrs[which])
        O.train_step(shared_p, spec, "sentence_encoder", src, tgt.t(), shared, lr=lrs[which])
        assert abs(loss - float(ref["loss"])) < 1e-4
    arena = model["arena"]
    got = arena.state_dict()
    # Adam moves every element by about lr per step whatever the gradient's size, so rounding noise on the
    # near-zero gradients shows up at a few per cent of one step (the same with a single trainer); sharing the
    # state between the optimizers would show up at the size of a step
    assert max(max_abs(got[n], p32[n]) for n in p32) < 1e-3
    assert max(max_abs(got[n], shared_p[n]) for n in p32) > 3e-3
    assert runtime.global_step() == len(order)
    assert [t.optimizer.steps for t in trainers] == [3, 2] == [s.t for s in states]
    slots = arena.optimizer_slots
    assert len(slots) == 2 and slots[0][1] is arena.adam_m and slots[1][1] is not arena.adam_m
    for (opt, m, _v), st in zip(slots, states):
        flat = arena.moment_dict(m)
        assert max(max_abs(flat[n], st.m[n]) for n in flat) < 1e-5

    # checkpoint -> fresh model: moments of both optimizers, their update counts and the global step resume
    path = str(tmp_path / "variables.data")
    manager = TensorFlowManager(num_sessions=1, num_threads=1)
    manager.save(path)
    next_losses = [step(model, trainers[1]), step(model, trainers[0])]
    want = model["arena"].state_dict()

    model2, trainers2 = make()
    manager2 = TensorFlowManager(num_sessions=1, num_threads=1)
    manager2.restore(path)
    assert runtime.global_step() == len(order)
    # the continued run uses its trainers in the same order of first use as the run that wrote the file
    # (slot 0 = first optimizer that ever stepped): here trainer 0 first, as above
    trainers2[0].optimizer.steps, trainers2[1].optimizer.steps = 0, 0
    model2["arena"].optimizer_slot(trainers2[0].optimizer)
    model2["arena"].optimizer_slot(trainers2[1].optimizer)
    assert [t.optimizer.steps for t in trainers2] == [3, 2]
    again = [step(model2, trainers2[1]), step(model2, trainers2[0])]
    assert max(abs(a - b) for a, b in zip(again, next_losses)) < 1e-6
    got = model2["arena"].state_dict()
    assert max(max_abs(got[n], want[n]) for n in want) < 1e-6


@pytest.mark.parametrize("kind", ["rnn", "transformer"])
def test_decoding_loop_with_sampling_and_temperature(cpu_model, kind):
    """`decoding_loop(train_mode=False, sample=..., temperature=...)` / `get_body` (autoregressive.py:442-562,
    the RL trainer's sampling pass): a temperature divides the logits that enter the histories and leaves the
    greedy symbols alone; sampled symbols follow softmax(logits / temperature) - at a very low temperature they
    ARE the greedy symbols, at temperature 1 their first-step frequencies match the first-step distribution -
    finished hypotheses emit <pad> and stay finished."""
    if kind == "rnn":
        model = build_bahdanau(**TOY)
        model["arena"].load_dict(oracle_params_for(model))
        src, tgt = random_batch(6, 8, 7, TOY["vs"], TOY["vt"], seed=3)
        feed(model, src, tgt, train=False)
    else:
        from tests.test_gpu_transformer import feed_transformer
        model, _params, src, tgt, _cfg = _transformer(seed=2, bsz=3)
        feed_transformer(model, src, tgt, train=False)
    dec = model["dec"]
    greedy = dec.decoding_loop(train_mode=False)
    g_logits = torch.stack(greedy.histories.logits, 0)
    g_symbols = torch.stack(greedy.histories.output_symbols, 0)
    assert bool((g_symbols == dec.runtime_symbols).all())

    warm = dec.decoding_loop(train_mode=False, temperature=2.0)
    assert bool((torch.stack(warm.histories.output_symbols, 0) == g_symbols).all())
    assert max_abs(torch.stack(warm.histories.logits, 0), g_logits / 2.0) < 1e-6

    torch.manual_seed(0)
    cold = dec.decoding_loop(train_mode=False, sample=True, temperature=1e-4)
    c_symbols = torch.stack(cold.histories.output_symbols, 0)
    assert c_symbols.shape == g_symbols.shape and bool((c_symbols == g_symbols).all())

    torch.manual_seed(1)
    first = []
    for _ in range(300):
        drawn = dec.decoding_loop(train_mode=False, sample=True)
        sym = torch.stack(drawn.histories.output_symbols, 0)
        mask = torch.stack(drawn.histories.output_mask, 0)
        first.append(sym[0])
        # once </s> (2) was emitted the hypothesis is finished: <pad> (0) afterwards, mask off from that step on
        ended = torch.cumsum((sym == 2).to(torch.int64), 0) > 0
        assert bool((sym[1:][ended[:-1]] == 0).all()) and bool((mask == ~ended).all())
    first = torch.stack(first, 0)                                   # [draws, batch]
    probs = torch.softmax(g_logits[0], dim=-1)                      # the first step does not depend on the draw
    vocab = probs.shape[-1]
    for b in range(first.shape[1]):
        freq = torch.bincount(first[:, b], minlength=vocab).to(torch.float32) / first.shape[0]
        assert float((freq - probs[b]).abs().sum()) < 0.6           # total variation of 300 draws over V=70: ~0.4
        assert float(freq[3]) == 0.0 or not getattr(dec, "supress_unk", False)   # <unk> carries -1e9

    with pytest.raises(NotImplementedError):
        dec.get_body(train_mode=True)
    with pytest.raises(ValueError):
        dec.decoding_loop(train_mode=False, temperature=0.0)


def _post_edit_model(heads=3, keep=1.0):
    """tests/post-edit.ini's topology: two recurrent encoders, a MultiHeadAttention whose keys come from one and
    whose values from the other, a ScaledDotProdAttention over the first, one GRU decoder over both."""
    from neuralmonkey_b200 import runtime, tf
    from neuralmonkey_b200.attention import ScaledDotProdAttention
    from neuralmonkey_b200.attention.scaled_dot_product import MultiHeadAttention
    from neuralmonkey_b200.decoders import Decoder
    from neuralmonkey_b200.encoders import SentenceEncoder
    from neuralmonkey_b200.trainers import CrossEntropyTrainer
    from neuralmonkey_b200.vocabulary import Vocabulary
    runtime.reset()
    vs, vt = 40, 50
    src_vocab = Vocabulary(["s{}".format(i) for i in range(vs - 4)])
    tgt_vocab = Vocabulary(["t{}".format(i) for i in range(vt - 4)])
    src = SentenceEncoder(name="src_encoder", vocabulary=src_vocab, data_id="source", embedding_size=7,
                          rnn_size=6, max_input_len=9)
    trans = SentenceEncoder(name="trans_encoder", vocabulary=tgt_vocab, data_id="translated", embedding_size=5,
                            rnn_size=6, max_input_len=9)
    mha = MultiHeadAttention(name="attention_trans_encoder", n_heads=heads, keys_encoder=src,
                             values_encoder=trans, dropout_keep_prob=keep)
    sdp = ScaledDotProdAttention(name="attention_source_encoder", keys_encoder=src)
    dec = Decoder(encoders=[trans, src], attentions=[mha, sdp], vocabulary=tgt_vocab, data_id="edits",
                  name="decoder", max_output_len=8, rnn_size=12, embedding_size=12)
    trainer = CrossEntropyTrainer(decoders=[dec], optimizer=tf.AdamOptimizer(learning_rate=1e-3))
    for part in trainer.parameterizeds:
        part.ensure_declared()
    runtime.arena().finalize(runtime.device())
    return {"src": src, "trans": trans, "mha": mha, "sdp": sdp, "dec": dec, "trainer": trainer,
            "arena": runtime.arena(), "vs": vs, "vt": vt}


def _post_edit_feed(model, src_ids, trans_ids, tgt_ids, train):
    bsz = src_ids.shape[0]
    model["src"].input_sequence.feed_ids([src_ids], train=train)
    model["trans"].input_sequence.feed_ids([trans_ids], train=train)
    for part in (model["src"], model["trans"], model["mha"], model["sdp"]):
        part.reset_batch()
        part.train_mode = train
        part.batch_size = bsz
    model["dec"].feed_ids(tgt_ids, bsz, train=train)


def _post_edit_oracle(p, heads, src_ids, trans_ids, beam=1):
    so = O.sentence_encoder(p, "src_encoder", src_ids)
    to = O.sentence_encoder(p, "trans_encoder", trans_ids)
    rep = (lambda x: x.repeat_interleave(beam, 0)) if beam > 1 else (lambda x: x)
    keys, kmask, values = rep(so["temporal_states"]), rep(so["temporal_mask"]), rep(to["temporal_states"])
    attend = [lambda q: O.multihead_attention_step(p, "decoder/attention_decoder", q, keys, values, kmask, heads),
              lambda q: O.multihead_attention_step(p, "decoder/attention_decoder", q, keys, keys, kmask, 1)]
    enc = {"output": torch.cat([to["output"], so["output"]], 1)}
    return enc, attend


@pytest.mark.parametrize("heads", [3, 1])
def test_rnn_decoder_with_scaled_dot_attention_objects(cpu_model, heads):
    """`attention.ScaledDotProdAttention` / `attention.scaled_dot_product.MultiHeadAttention` as the attentions of
    an RNN decoder (scaled_dot_product.py:246-402; tests/factored.ini, tests/post-edit.ini): variables (the head
    projections belong to the decoder's step scope), the hoisted training pass with every gradient, the greedy
    loop with its per-head histories, and beam search over the tiled keys - against the oracle."""
    from neuralmonkey_b200.decoders import BeamSearchDecoder
    model = _post_edit_model(heads)
    arena, dec = model["arena"], model["dec"]
    proj = sorted(n for n in arena.order if "_proj/" in n)
    want_proj = ["decoder/attention_decoder/{}_proj/kernel".format(k) for k in ("keys", "output", "query", "vals")]
    assert proj == (want_proj if heads > 1 else [])
    assert not any(n.startswith("attention_") for n in arena.order)      # the attention objects own nothing
    assert model["mha"].context_vector_size == 12 and model["sdp"].context_vector_size == 12
    params = oracle_params_for(model)
    arena.load_dict(params)
    src, tgt = random_batch(5, 8, 7, model["vs"], model["vt"], seed=4)
    trans, _ = random_batch(5, 8, 7, model["vt"], model["vt"], seed=5)      # keys and values: one time axis

    _post_edit_feed(model, src, trans, tgt, train=True)
    p = {n: v.clone().requires_grad_(True) for n, v in params.items()}
    spec = O.RNNDecoderSpec("decoder", None, 8, "tanh", False)
    enc, attend = _post_edit_oracle(p, heads, src, trans)
    odec = O.decoder_train(p, spec, enc, tgt.t(), attend=attend)
    assert max_abs(dec.train_output_states, odec["train_output_states"]) < 1e-5
    assert abs(float(dec.train_loss) - float(odec["train_loss"])) < 1e-5
    for i in range(heads):      # [time, batch, keys] per head, like a stepped loop's history
        assert max_abs(model["mha"].histories["decoder_train_head{}".format(i)],
                       odec["attention_weights"][0][:, :, i]) < 1e-5
    assert max_abs(model["sdp"].histories["decoder_train_head0"], odec["attention_weights"][1][:, :, 0]) < 1e-5
    dec.train_loss.backward()
    odec["train_loss"].backward()
    for name, grad in _grads(model).items():
        want = p[name].grad if p[name].grad is not None else torch.zeros_like(p[name])
        got = grad if grad is not None else torch.zeros_like(p[name])
        assert float((got - want.reshape(got.shape)).norm()) <= 1e-4 * float(want.norm()) + 1e-7, name

    _post_edit_feed(model, src, trans, tgt, train=False)
    enc, attend = _post_edit_oracle(params, heads, src, trans)
    og = O.decoder_greedy(params, spec, enc, tgt.t(), attend=attend)
    assert dec.decode_engine is None            # the fused step kernel covers the Bahdanau attention only
    assert max_abs(dec.runtime_logits, og["runtime_logits"]) < 1e-4
    assert bool((dec.runtime_symbols == og["output_symbols"]).all())
    steps = dec.runtime_symbols.shape[0]
    for i in range(heads):
        assert tuple(model["mha"].histories["decoder_run_head{}".format(i)].shape) == (steps, 5, src.shape[1])

    beam, bsz = 3, 4
    bs = BeamSearchDecoder(name="bs", parent_decoder=dec, beam_size=beam, max_steps=7, length_normalization=1.0)
    bs.use_cuda_graph = False
    _post_edit_feed(model, src[:bsz], trans[:bsz], None, train=False)
    bs.reset_batch()
    bs.batch_size = bsz
    out = bs.outputs
    enc, attend = _post_edit_oracle(params, heads, src[:bsz], trans[:bsz], beam=beam)
    emb = params["decoder/word_embeddings"]
    prev0 = O.decoder_initial_state(params, spec, enc["output"]).repeat_interleave(beam, 0)

    def run(embedded, prev):
        output, cell, _c, _w = O.decoder_step(params, spec, embedded, prev, None, None, None, attend)
        return cell, torch.log_softmax(O.state_to_logits(params, spec, output), -1)

    prev1, first = run(emb[torch.full((bsz * beam,), O.START, dtype=torch.int64)], prev0)
    want = O.beam_search(lambda prev, words, _f: run(emb[words], prev), prev1, first, beam, 7, 1.0,
                         lambda st, idx: st[idx])
    got = out.last_search_step_output
    assert bool((got.token_ids[1:] == want["token_ids"]).all())
    assert max_abs(got.scores, want["scores"]) < 1e-4


def test_scaled_dot_attention_objects_validate_their_sizes(cpu_model):
    """The checks `attention()` makes on the first query (scaled_dot_product.py:148-169) are made when the
    decoder announces its query size."""
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.attention import ScaledDotProdAttention
    from neuralmonkey_b200.attention.scaled_dot_product import MultiHeadAttention
    from neuralmonkey_b200.decoders import Decoder
    from neuralmonkey_b200.encoders import SentenceEncoder
    from neuralmonkey_b200.vocabulary import Vocabulary
    runtime.reset()
    vocab = Vocabulary(["a", "b"])
    enc = SentenceEncoder(name="enc", vocabulary=vocab, data_id="source", embedding_size=4, rnn_size=6,
                          max_input_len=5)
    with pytest.raises(ValueError, match="greater than zero"):
        MultiHeadAttention(name="a0", n_heads=0, keys_encoder=enc)
    with pytest.raises(ValueError, match="keep prob"):
        ScaledDotProdAttention(name="a1", keys_encoder=enc, dropout_keep_prob=0.0)

    def decoder(att, size):
        return Decoder(encoders=[enc], attentions=[att], vocabulary=vocab, data_id="target", name="dec" + att.name,
                       max_output_len=5, rnn_size=size, embedding_size=size)
    with pytest.raises(ValueError, match="do not match in the last dimension"):
        decoder(ScaledDotProdAttention(name="a2", keys_encoder=enc), 10)
    with pytest.raises(ValueError, match="divisible by the number of heads"):
        decoder(MultiHeadAttention(name="a3", n_heads=5, keys_encoder=enc), 12)
    att = ScaledDotProdAttention(name="a4", keys_encoder=enc)
    feedables, params = decoder(att, 12).get_dependencies()
    assert att in params and enc in params and att in feedables


def test_gradient_blocking_views_freeze_the_encoder(cpu_model):
    """model.gradient_blocking.{StatefulView,TemporalStatefulView} (tests/bpe.ini, second run of tests_run.sh):
    a decoder and an attention over VIEWS of the encoder compute what they compute over the encoder itself,
    their own gradients are unchanged, and nothing reaches the encoder's variables; the wrapped encoder is still
    found as a dependency (variables declared, batches fed)."""
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.attention import Attention
    from neuralmonkey_b200.decoders import Decoder
    from neuralmonkey_b200.decoders.output_projection import maxout_output
    from neuralmonkey_b200.encoders import SentenceEncoder
    from neuralmonkey_b200.model.gradient_blocking import SpatialStatefulView, StatefulView, TemporalStatefulView
    from neuralmonkey_b200.trainers import CrossEntropyTrainer
    from neuralmonkey_b200.vocabulary import Vocabulary

    plain = build_bahdanau(**TOY)
    params = oracle_params_for(plain)
    plain["arena"].load_dict(params)
    src, tgt = random_batch(6, 8, 7, TOY["vs"], TOY["vt"], seed=0)
    feed(plain, src, tgt, train=True)
    want_loss = float(plain["dec"].train_loss)
    plain["dec"].train_loss.backward()
    want = {n: (g.clone() if g is not None else None) for n, g in _grads(plain).items()}

    runtime.reset()
    src_vocab = Vocabulary(["s{}".format(i) for i in range(TOY["vs"] - 4)])
    tgt_vocab = Vocabulary(["t{}".format(i) for i in range(TOY["vt"] - 4)])
    enc = SentenceEncoder(name="sentence_encoder", vocabulary=src_vocab, data_id="source",
                          embedding_size=TOY["es"], rnn_size=TOY["he"], max_input_len=TOY["max_len"])
    att = Attention(name="attention", encoder=TemporalStatefulView(enc))
    dec = Decoder(encoders=[StatefulView(enc)], vocabulary=tgt_vocab, data_id="target", name="decoder",
                  max_output_len=TOY["max_len"], rnn_size=TOY["hd"], embedding_size=TOY["et"], attentions=[att],
                  output_projection=maxout_output(TOY["out"]), supress_unk=True)
    trainer = CrossEntropyTrainer(decoders=[dec])
    feedables, parameterizeds = trainer.get_dependencies()
    assert enc in parameterizeds and enc in feedables and enc.input_sequence in feedables
    for part in parameterizeds:
        part.ensure_declared()
    runtime.arena().finalize(runtime.device())
    frozen = {"enc": enc, "att": att, "dec": dec, "trainer": trainer, "arena": runtime.arena()}
    assert sorted(frozen["arena"].order) == sorted(params)
    frozen["arena"].load_dict(params)
    feed(frozen, src, tgt, train=True)
    assert abs(float(dec.train_loss) - want_loss) < 1e-6
    dec.train_loss.backward()
    for name, grad in _grads(frozen).items():
        upstream = name.startswith("sentence_encoder")
        if upstream:
            assert grad is None or float(grad.abs().max()) == 0.0, name
        elif want[name] is not None:
            assert max_abs(grad, want[name]) < 1e-6, name
    assert any(n.startswith("sentence_encoder") and want[n] is not None and float(want[n].abs().max()) > 0
               for n in want)
    view = TemporalStatefulView(enc)
    assert view.dimension == enc.dimension and view.temporal_mask is enc.temporal_mask
    assert not view.temporal_states.requires_grad and enc.temporal_states.requires_grad
    from neuralmonkey_b200.model.stateful import SpatialStateful
    assert issubclass(SpatialStatefulView, SpatialStateful)
    with pytest.raises(TypeError, match="blocked_object"):
        StatefulView("not a stateful object")


@pytest.mark.parametrize("tag,heads", [("h3", 3), ("h1", 1)])
def test_scaled_dot_attention_objects_against_the_reference_run(cpu_model, tag, heads):
    """The PRODUCT's Decoder with MultiHeadAttention + ScaledDotProdAttention against the REFERENCE's classes run
    over the TF stand-in (tests/golden/make_tf_shim_golden.py, `rnn_multihead_case`): the reference's variables
    under the reference's names (the name sets must be equal: head projections in the decoder's step scope),
    training logits / loss, the greedy loop, per-head attention histories under the reference's keys."""
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.attention import ScaledDotProdAttention
    from neuralmonkey_b200.attention.scaled_dot_product import MultiHeadAttention
    from neuralmonkey_b200.decoders import Decoder
    from neuralmonkey_b200.vocabulary import Vocabulary
    golden = _golden()
    dname, pre = "md_" + tag, "md_{}_".format(tag)
    g = lambda n: torch.from_numpy(golden[pre + n])
    runtime.reset()
    keys_enc = _stub_encoder(g("keys"), g("mask"), g("enc_out1"))
    vals_enc = _stub_encoder(g("values"), g("mask"), g("enc_out0"))
    table = g("table")
    vocab = Vocabulary(["t{}".format(i) for i in range(table.shape[0] - 4)])
    mha = MultiHeadAttention(name="ma_" + tag, n_heads=heads, keys_encoder=keys_enc, values_encoder=vals_enc)
    sdp = ScaledDotProdAttention(name="sa_" + tag, keys_encoder=keys_enc)
    gold = g("gold").t().contiguous()
    dec = Decoder(encoders=[vals_enc, keys_enc], vocabulary=vocab, data_id="target", name=dname,
                  max_output_len=gold.shape[1], rnn_size=12, embedding_size=12, attentions=[mha, sdp])
    for part in (mha, sdp, dec):
        part.ensure_declared()
    arena = runtime.arena()
    arena.finalize(runtime.device())
    reference_vars = {k[4:]: torch.from_numpy(golden[k]) for k in golden.files if k.startswith("mv::" + dname + "/")}
    reference_vars[dname + "/word_embeddings"] = table
    reference_vars[dname + "/state_to_word_W"], reference_vars[dname + "/state_to_word_b"] = g("w"), g("b")
    assert set(arena.order) == set(reference_vars), set(arena.order) ^ set(reference_vars)
    arena.load_dict({n: v.reshape(arena.variables[n].shape) for n, v in reference_vars.items()})
    assert [mha.context_vector_size, sdp.context_vector_size] == golden[pre + "context_sizes"].tolist()
    bsz = gold.shape[0]

    def feed_all(train):
        for att in (mha, sdp):
            att.reset_batch()
            att.train_mode, att.batch_size = train, bsz
        dec.feed_ids(gold, bsz, train=train)

    feed_all(True)
    assert max_abs(dec.train_logits, g("train_logits")) < 2e-5
    assert abs(float(dec.train_loss) - float(golden[pre + "train_loss"])) < 2e-5
    for i in range(heads):
        assert max_abs(mha.histories["{}_train_head{}".format(dname, i)], g("train_mha_head{}".format(i))) < 1e-5
    assert max_abs(sdp.histories[dname + "_train_head0"], g("train_sdp_head0")) < 1e-5
    feed_all(False)
    assert dec.runtime_logits.shape == g("run_logits").shape
    assert max_abs(dec.runtime_logits, g("run_logits")) < 2e-5
    assert bool((dec.runtime_symbols == g("run_symbols")).all())
    for i in range(heads):
        assert max_abs(mha.histories["{}_run_head{}".format(dname, i)], g("run_mha_head{}".format(i))) < 1e-5
    assert max_abs(sdp.histories[dname + "_run_head0"], g("run_sdp_head0")) < 1e-5
    assert sorted(list(mha.histories) + list(sdp.histories)) == sorted(golden[pre + "history_keys"].tolist())


def test_training_losses_are_read_when_somebody_looks(cpu_model, monkeypatch):
    """The executable of a trainer hands out its losses as a mapping that converts the device values on first
    access (so the training loop does not wait for the device after every step); what it then shows is THAT
    step's loss and regularisation sums, whatever ran since."""
    from neuralmonkey_b200.learning_utils import evaluation, join_execution_results
    from neuralmonkey_b200.trainers.generic_trainer import GenericTrainer
    monkeypatch.setattr(GenericTrainer, "_adam_kernel", cpu_ops.adam_kernel)
    model = build_bahdanau(**TOY, l2=1e-3, lr=1e-2)
    model["arena"].load_dict(oracle_params_for(model))
    src, tgt = random_batch(6, 8, 7, TOY["vs"], TOY["vt"], seed=3)
    results, eager = [], []
    for _ in range(3):
        feed(model, src, tgt, train=True)
        executable = model["trainer"].get_executable()
        executable.execute()
        results.append(executable.result)
        eager.append((float(model["dec"].train_loss), float(model["trainer"]._l1l2[1])))
    assert all(r.losses._values is None for r in results)            # nothing was converted yet
    name = model["trainer"].objectives[0].name
    for result, (loss, l2) in zip(results, eager):
        assert list(result.losses) == [name, "L1", "L2"] and len(result.losses) == 3
        assert result.losses[name] == pytest.approx(loss, rel=1e-6)
        assert result.losses["L2"] == pytest.approx(l2, rel=1e-6)     # this step's sum, not the last step's
    assert eager[0][1] != eager[2][1] and eager[0][0] > eager[2][0]
    joined = join_execution_results(results)
    assert joined.losses[name] == pytest.approx(sum(l for l, _ in eager) / 3, rel=1e-6)
    assert evaluation([], {}, results[:1], {})[name] == pytest.approx(eager[0][0], rel=1e-6)
    assert dict(results[0].losses) == results[0].losses._values
