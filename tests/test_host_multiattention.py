"""Attention combination on the CPU: the model parts over the stand-in of `ops.joint_attention` against the
restatement of the reference's per-step `attention()` (tests/multiattention_oracle.py), variable names, shapes and
initializers, constructor errors, and the sentinel's inputs in the decoder's training and decoding paths.  The
kernels are tested in tests/test_gpu_multiattention.py."""
import itertools

import numpy as np

import pytest
import torch

from tests import cnn_oracle as CO
from tests import cpu_ops
from tests import multiattention_oracle as MAO

pytestmark = [pytest.mark.filterwarnings("ignore:Converting a tensor with requires_grad")]
CASES = list(itertools.product(("flat", "hier"), (False, True), (False, True)))
STEP = "decoder/attention_decoder/attention_combination"


@pytest.fixture
def cpu_model(monkeypatch):
    from neuralmonkey_b200 import ops, runtime
    for op in cpu_ops.STAND_INS:
        monkeypatch.setattr(ops, op, getattr(cpu_ops, op))
    for op in MAO.STAND_INS:
        monkeypatch.setattr(ops, op, getattr(MAO, op))
    monkeypatch.setattr(runtime, "_device", torch.device("cpu"))
    yield
    runtime.reset()


def _var(wrapper):
    from neuralmonkey_b200 import runtime

    def var(name):
        if name.startswith("step/"):
            return runtime.arena().get(STEP + name[4:]).detach()
        return wrapper.var(name).detach()
    return var


def _randomize():
    from neuralmonkey_b200 import runtime
    gen = torch.Generator().manual_seed(3)
    with torch.no_grad():
        for name in runtime.arena().order:
            t = runtime.arena().get(name)
            t.copy_(torch.randn(t.shape, generator=gen) * 0.5)


@pytest.mark.parametrize("kind,share,sentinel", CASES)
def test_model_part_against_the_restated_reference(cpu_model, kind, share, sentinel):
    dec, wrapper, children = MAO.build_model(kind, share, sentinel)
    _randomize()
    MAO.feed(dec, [wrapper] + children, train=False)
    gen = torch.Generator().manual_seed(1)
    bsz, steps = len(MAO.LENGTHS), 3
    queries = torch.randn(bsz, steps, dec.rnn_size, generator=gen)
    prev = torch.randn(bsz, steps, dec.rnn_size, generator=gen)
    inp = torch.randn(bsz, steps, dec.embedding_size, generator=gen)
    with torch.no_grad():
        ctx, weights = wrapper.attention_sequence(queries, prev, inp)
    text, mask, image = (torch.from_numpy(a) for a in MAO.encoder_states())
    states = [text, image.reshape(bsz, -1, MAO.SPATIAL_DIM)]
    masks = [mask, torch.ones(bsz, states[1].shape[1])]
    var = _var(wrapper)
    state = wrapper.initial_loop_state()
    for t in range(steps):
        if kind == "flat":
            want_ctx, want_w = MAO.flat_step(var, "step", states, masks, queries[:, t], prev[:, t], inp[:, t],
                                             share, sentinel)
        else:
            child_ctx = [c.attention_sequence(queries[:, t:t + 1])[0][:, 0].detach() for c in children]
            want_ctx, want_w = MAO.hier_step(var, "step", [c.name for c in children], child_ctx, queries[:, t],
                                             prev[:, t], inp[:, t], share, sentinel)
        torch.testing.assert_close(ctx[:, t], want_ctx, rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(weights[:, t], want_w, rtol=1e-5, atol=1e-6)
        with torch.no_grad():      # the stepped interface gives the same numbers and keeps the histories
            step_ctx, state = wrapper.attention(queries[:, t], prev[:, t], inp[:, t], state)
        torch.testing.assert_close(step_ctx, want_ctx, rtol=1e-5, atol=1e-6)
    hist = state.weights if kind == "flat" else state.loop_state.weights
    assert hist.shape == (steps, bsz, weights.shape[-1])
    wrapper.finalize_loop("k", state)
    assert wrapper.histories["k"].shape == hist.shape
    if kind == "hier":
        assert all("k" in c.histories for c in children)


@pytest.mark.parametrize("kind,share,sentinel", CASES)
def test_variable_names_shapes_and_initializers(cpu_model, kind, share, sentinel):
    from neuralmonkey_b200 import runtime
    dec, wrapper, children = MAO.build_model(kind, share, sentinel, attention_state_size=8)
    arena = runtime.arena()
    names = {n: tuple(arena.get(n).shape) for n in arena.order}
    a, r, e = 8, dec.rnn_size, dec.embedding_size
    want = {"combination/attn_v": (1, 1, a), STEP + "/dense/kernel": (r, a), STEP + "/dense/bias": (a,)}
    if kind == "flat":
        dims = [MAO.TEMPORAL_DIM, MAO.SPATIAL_DIM]
        for scope in ["logits_projections"] + ([] if share else ["context_projections"]):
            for i, d in enumerate(dims):
                want["combination/{}/proj_matrix_{}".format(scope, i)] = (d, a)
                want["combination/{}/proj_bias_{}".format(scope, i)] = (a,)
        for i in range(2):
            want["combination/attn_bias_{}".format(i)] = ()
    else:
        for c in children:
            want["{}/{}_logit/vector_bias".format(STEP, c.name)] = ()
            want["{}/{}_logit/vector_projection/kernel".format(STEP, c.name)] = (c.context_vector_size, a)
            if not share:
                want["{}/{}_logit/vector_ctx_proj/kernel".format(STEP, c.name)] = (c.context_vector_size, a)
                want["{}/proj_attn_{}/kernel".format(STEP, c.name)] = (c.context_vector_size, a)
        if sentinel and not share:
            want[STEP + "/proj_sentinel/kernel"] = (r, a)
    if sentinel:
        want[STEP + "/sentinel/dense/kernel"] = (r + e, r)
        want[STEP + "/sentinel/dense/bias"] = (r,)
        want[STEP + "/sentinel_logit/vector_bias"] = ()
        want[STEP + "/sentinel_logit/vector_projection/kernel"] = (r, a)
        if not share:
            want[STEP + "/sentinel_logit/vector_ctx_proj/kernel"] = (r, a)
    for name, shape in want.items():
        assert names.get(name) == shape, (name, names.get(name))
    assert not [n for n in names if "context_projections" in n or "ctx_proj" in n or "proj_attn" in n] or not share
    # attn_v and the encoder projections are N(0, 0.001); biases start at zero
    assert 0 < float(arena.get("combination/attn_v").std()) < 0.01
    for n in names:
        if n.startswith(("combination/attn_bias", "combination/logits_projections/proj_bias")) or \
                n.endswith(("vector_bias", "dense/bias")) and n.startswith(STEP):
            assert float(arena.get(n).abs().max()) == 0.0, n


def test_constructor_errors(cpu_model):
    from neuralmonkey_b200.attention.combination import FlatMultiAttention, HierarchicalMultiAttention
    with pytest.raises(ValueError, match="at least one encoder"):
        FlatMultiAttention(name="f", encoders=[], attention_state_size=4)
    with pytest.raises(ValueError, match="at least one attention"):
        HierarchicalMultiAttention(name="h", attentions=[], attention_state_size=4, use_sentinels=False,
                                   share_attn_projections=False)
    with pytest.raises(ValueError, match="positive"):
        FlatMultiAttention(name="f", encoders=[], attention_state_size=0)
    with pytest.raises(TypeError, match="encoders"):
        FlatMultiAttention(name="f", encoders=[object()], attention_state_size=4)
    with pytest.raises(TypeError):
        HierarchicalMultiAttention(name="h", attentions=[], attention_state_size=4)   # no defaults for the flags
    dec, wrapper, _ = MAO.build_model("flat", False, True)
    MAO.feed(dec, [wrapper], train=False)
    with pytest.raises(ValueError, match="sentinel"):
        wrapper.attention_sequence(torch.zeros(3, 1, dec.rnn_size))


def _record(monkeypatch):
    """Every (queries, previous outputs, inputs) the sentinel is computed from."""
    from neuralmonkey_b200.attention.combination import MultiAttention
    seen = []
    original = MultiAttention._sentinel

    def spy(self, queries, prev_outputs, inputs):
        seen.append((queries.detach().clone(), prev_outputs.detach().clone(), inputs.detach().clone()))
        return original(self, queries, prev_outputs, inputs)
    monkeypatch.setattr(MultiAttention, "_sentinel", spy)
    return seen


@pytest.mark.parametrize("kind", ["flat", "hier"])
def test_sentinel_inputs_in_every_decoder_path(cpu_model, monkeypatch, kind):
    """All-steps training hands step t the initial state (t = 0) or the previous dropped cell output and the
    step's embedded input, as `next_state` does at run time; the step-wise pass computes the same loss."""
    dec, wrapper, children = MAO.build_model(kind, False, True)
    _randomize()
    ids = MAO.target_ids()
    MAO.feed(dec, [wrapper] + children, train=True, ids=ids)
    seen = _record(monkeypatch)
    loss = float(dec.train_loss)
    (queries, prev, inp), = seen
    cells = dec.train_rnn_outputs.transpose(0, 1).detach()
    torch.testing.assert_close(prev[:, 0], dec.initial_state.detach())
    torch.testing.assert_close(prev[:, 1:], cells[:, :-1])
    torch.testing.assert_close(inp, dec.embed_input_symbols(dec._train_step_inputs_bm).detach())

    # the same loss step by step (the path of conditional / LSTM / Nematus decoders)
    seen.clear()
    MAO.feed(dec, [wrapper] + children, train=True, ids=ids)
    monkeypatch.setattr(dec, "_stepwise", True)
    assert abs(float(dec.train_loss) - loss) < 1e-5
    assert len(seen) == ids.shape[1]
    torch.testing.assert_close(seen[0][1][:, 0], dec.initial_state.detach())
    torch.testing.assert_close(torch.cat([s[1] for s in seen[1:]], 1), cells[:, :-1])
    monkeypatch.setattr(dec, "_stepwise", False)

    # greedy decoding: next_state hands attention() the previous output, starting at the initial state
    seen.clear()
    MAO.feed(dec, [wrapper] + children, train=False)
    assert dec.decode_engine is None         # no fused step for multi-source decoders
    symbols = dec._runtime["symbols"]
    assert symbols.shape[1] == len(MAO.LENGTHS) and len(seen) == symbols.shape[0]
    torch.testing.assert_close(seen[0][1][:, 0], dec.initial_state.detach())
    assert "decoder_run" in wrapper.histories


def test_beam_rows_are_repeated_beam_minor(cpu_model):
    dec, wrapper, _ = MAO.build_model("flat", False, False)
    _randomize()
    MAO.feed(dec, [wrapper], train=False)
    gen = torch.Generator().manual_seed(4)
    bsz, beam = len(MAO.LENGTHS), 2
    queries = torch.randn(bsz, 1, dec.rnn_size, generator=gen)
    with torch.no_grad():
        ctx, _ = wrapper.attention_sequence(queries)
        tiled, _ = wrapper.attention_sequence(queries.repeat_interleave(beam, 0))
    torch.testing.assert_close(tiled, ctx.repeat_interleave(beam, 0))
    with pytest.raises(ValueError, match="query rows"):
        wrapper.attention_sequence(torch.zeros(bsz + 1, 1, dec.rnn_size))


# The reference's bucketing measures every series of a row, images included, although its scheme names them in
# `ignore_series` (the TODO of its dataset.py:521): a 32-row image exceeds every boundary, so each instance of the
# hierarchical INI lands in the overflow bucket of size 1 and the epoch has 10 batches, enough to reach
# validation_period=5.  This package honours `ignore_series` and would make 4 batches of the same 10 sentences, so
# the run asks for the batches the reference makes.
INI_CHANGES = {"hier-multiattention": ["-s", "batch_scheme.bucket_batch_sizes=[1, 1, 1, 1, 1, 1]"]}


@pytest.mark.parametrize("name", ["flat-multiattention", "hier-multiattention"])
def test_reference_ini_trains_unchanged(monkeypatch, tmp_path, name):
    """The reference's tests/{flat,hier}-multiattention.ini through `neuralmonkey-train` over the stand-ins: four
    decoders under one trainer, four wrappers sharing two child attentions (hier), a SpatialFiller (flat) or a
    CNNEncoder (hier) beside the sentence encoder, and the flat INI's beam-2 runner."""
    import os
    import sys
    from neuralmonkey_b200 import ops, runtime
    from neuralmonkey_b200.trainers.generic_trainer import GenericTrainer
    from tests.golden.make_multiattention_bundle import unpack
    for op in cpu_ops.STAND_INS:
        monkeypatch.setattr(ops, op, getattr(cpu_ops, op))
    for op in MAO.STAND_INS:
        monkeypatch.setattr(ops, op, getattr(MAO, op))
    for op in ("conv2d", "batch_norm", "pool2d"):          # the hierarchical INI's CNNEncoder
        monkeypatch.setattr(ops, op, getattr(CO, op))
    monkeypatch.setattr(runtime, "_device", torch.device("cpu"))
    monkeypatch.setattr(GenericTrainer, "_adam_kernel", cpu_ops.adam_kernel)
    monkeypatch.setenv("NEURALMONKEY_STRICT", "1")
    unpack(str(tmp_path / "tree"))
    monkeypatch.chdir(tmp_path / "tree")
    out = str(tmp_path / name)
    argv = ["neuralmonkey-train", "tests/{}.ini".format(name), "-s", 'main.output="{}"'.format(out)]
    argv += INI_CHANGES.get(name, [])
    monkeypatch.setattr(sys, "argv", argv)
    try:
        from neuralmonkey_b200.train import main
        main()
    finally:
        runtime.reset()
    log_text = open(os.path.join(out, "experiment.log")).read()
    assert "Training finished" in log_text and "Validation (epoch" in log_text
    assert os.path.exists(os.path.join(out, "variables.data.final"))
    if name == "flat-multiattention":      # the beam-2 runner over the sentinel wrapper's decoder decoded
        assert "target_fss_beam_2:" in log_text and "target_fss_beam_2/beam_search_score" in log_text


# -- against the reference's own combination.py ------------------------------------------------------------------------
@pytest.mark.parametrize("tag", MAO.CASES)
def test_restatement_against_the_reference_code(tag):
    g = MAO.golden()
    for step in range(g[tag + "_queries"].shape[0]):
        ctx, w = MAO.restated_golden_step(g, tag, step)
        np.testing.assert_allclose(ctx.numpy(), g[tag + "_contexts"][step], rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(w.numpy(), g[tag + "_weights"][step], rtol=1e-5, atol=1e-6)


def _golden_outputs(g, tag):
    """(all steps through attention_sequence, stepped attention()) of the model part for the golden case."""
    from neuralmonkey_b200 import runtime
    dec, wrapper, _children = MAO.golden_model(g, tag)
    dev = runtime.device()

    def arr(name):      # [steps, B, .] -> [B, steps, .]
        return torch.from_numpy(np.asarray(g[tag + "_" + name])).to(dev).transpose(0, 1).contiguous()
    queries, prev, inp = arr("queries"), arr("prev"), arr("inputs")
    with torch.no_grad():
        ctx, weights = wrapper.attention_sequence(queries, prev, inp)
        state = wrapper.initial_loop_state()
        stepped = []
        for t in range(queries.shape[1]):
            c, state = wrapper.attention(queries[:, t], prev[:, t], inp[:, t], state)
            stepped.append(c)
    hist = state.weights if tag.startswith("flat") else state.loop_state.weights
    return (ctx.transpose(0, 1).cpu().numpy(), weights.transpose(0, 1).cpu().numpy(),
            torch.stack(stepped).cpu().numpy(), hist.cpu().numpy())


@pytest.mark.parametrize("tag", MAO.CASES)
def test_model_part_against_the_reference_code(cpu_model, tag):
    g = MAO.golden()
    ctx, weights, stepped, hist = _golden_outputs(g, tag)
    for got in (ctx, stepped):
        np.testing.assert_allclose(got, g[tag + "_contexts"], rtol=1e-5, atol=1e-6)
    for got in (weights, hist):
        np.testing.assert_allclose(got, g[tag + "_weights"], rtol=1e-5, atol=1e-6)
