"""Coverage attention on the CPU: the restatement and the model part over the stand-ins of `ops.coverage_attention` /
`ops.coverage_fertility` (tests/coverage_oracle.py) against the reference's own `coverage.py`, the running coverage
in every decoder path (all-steps training, the step-wise variants, `differentiable_loop`, beam search), the
hierarchical combination's refusal, and the bahdanau INI with a coverage attention.  The kernels are tested in
tests/test_gpu_coverage.py."""
import os
import sys

import numpy as np
import pytest
import torch

from tests import coverage_oracle as CVO
from tests import cpu_ops

pytestmark = [pytest.mark.filterwarnings("ignore:Converting a tensor with requires_grad")]


def _stand_ins(monkeypatch):
    from neuralmonkey_b200 import ops, runtime
    for op in cpu_ops.STAND_INS:
        monkeypatch.setattr(ops, op, getattr(cpu_ops, op))
    for op in CVO.STAND_INS:
        monkeypatch.setattr(ops, op, getattr(CVO, op))
    monkeypatch.setattr(runtime, "_device", torch.device("cpu"))


@pytest.fixture
def cpu_model(monkeypatch):
    from neuralmonkey_b200 import runtime
    _stand_ins(monkeypatch)
    yield
    runtime.reset()


# -- against the reference's own coverage.py --------------------------------------------------------------------------
@pytest.mark.parametrize("tag", CVO.CASES)
def test_restatement_against_the_reference_code(tag):
    g = CVO.golden()
    fert, steps = CVO.restated_golden(g, tag)
    np.testing.assert_allclose(fert.numpy(), g[tag + "_fertility"], rtol=1e-5, atol=1e-6)
    for q, (ctx, w, e) in enumerate(steps):
        np.testing.assert_allclose(e.numpy(), g[tag + "_energies"][q], rtol=1e-5, atol=1e-5)
        np.testing.assert_allclose(w.numpy(), g[tag + "_weights"][q], rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(ctx.numpy(), g[tag + "_contexts"][q], rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("tag", CVO.CASES)
def test_model_part_against_the_reference_code(cpu_model, tag):
    """Variables loaded BY NAME: the part declares exactly the reference's (no attn_bias), of the same shapes."""
    from neuralmonkey_b200 import runtime
    g = CVO.golden()
    variables = CVO.golden_variables(g, tag)
    state_size = variables["coverage/attn_similarity_v"].shape[0]
    dec, att = CVO.build_model(states=(g[tag + "_text"], g[tag + "_mask"]), max_fertility=int(g[tag + "_max_fertility"]),
                               state_size=None if state_size == CVO.DIM else state_size)
    arena = runtime.arena()
    ours = sorted(n for n in arena.order if n.startswith("coverage/"))
    assert ours == sorted(variables) and "coverage/attn_bias" not in ours
    for name, value in variables.items():
        assert tuple(arena.get(name).shape) == value.shape, name
    arena.load_dict({n: torch.from_numpy(v) for n, v in variables.items()})
    CVO.feed(dec, att, train=False)
    queries = torch.from_numpy(g[tag + "_queries"]).transpose(0, 1).contiguous()
    with torch.no_grad():
        ctx, weights = att.attention_sequence(queries)
        state = att.initial_loop_state()
        stepped = []
        for q in range(queries.shape[1]):
            c, state = att.attention(queries[:, q], None, None, state)
            stepped.append(c)
    np.testing.assert_allclose(att.fertility.detach().numpy(), g[tag + "_fertility"], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(ctx.transpose(0, 1).numpy(), g[tag + "_contexts"], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(torch.stack(stepped).numpy(), g[tag + "_contexts"], rtol=1e-5, atol=1e-6)
    for got in (weights.transpose(0, 1), state.weights):
        np.testing.assert_allclose(got.numpy(), g[tag + "_weights"], rtol=1e-5, atol=1e-6)
    att.finalize_loop("k", state)
    assert att.histories["k"].shape == state.weights.shape


# -- the running coverage in the decoder's paths -------------------------------------------------------------------------
def _spy(monkeypatch, att):
    """Record every coverage_scan call of `att`: (queries, coverage in, contexts, weights, coverage out)."""
    calls = []
    scan = type(att).coverage_scan

    def spy(self, queries, coverage):
        ctx, w, cov = scan(self, queries, coverage)
        calls.append((queries.detach(), coverage, ctx.detach(), w, cov))
        return ctx, w, cov
    monkeypatch.setattr(type(att), "coverage_scan", spy)
    return calls, scan


def test_training_pass_equals_stepping_attention(cpu_model, monkeypatch):
    """The default GRU pass attends all steps in one scan; stepping `attention()` over the same queries gives the
    same contexts and weights, and the pass records its weights under `decoder_train`."""
    dec, att = CVO.build_model()
    CVO.randomize()
    calls, _ = _spy(monkeypatch, att)
    CVO.feed(dec, att, train=True, ids=CVO.target_ids())
    loss = dec.train_loss
    assert len(calls) == 1 and calls[0][1] is None
    queries, _, ctx, weights, _ = calls[0]
    assert queries.shape[1] == CVO.target_ids().shape[1]
    with torch.no_grad():
        state = att.initial_loop_state()
        for q in range(queries.shape[1]):
            c, state = att.attention(queries[:, q], None, None, state)
            torch.testing.assert_close(c, ctx[:, q], rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(state.weights, weights.transpose(0, 1), rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(att.histories["decoder_train"], weights.transpose(0, 1))
    _check_gradients(loss)


def _check_gradients(loss):
    """The loss reaches both coverage variables (fertility_matrix only through the running coverage)."""
    from neuralmonkey_b200 import runtime
    names = ("coverage/coverage_matrix", "coverage/fertility_matrix")
    grads = torch.autograd.grad(loss, [runtime.arena().get(n) for n in names])
    for name, grad in zip(names, grads):
        assert float(grad.abs().max()) > 0, name


def _check_chain(calls, steps):
    """`steps` one-step calls, each continuing from the running sum the one before returned, whose weights equal one
    scan over all their queries from zero coverage."""
    assert len(calls) == steps and calls[0][1] is None
    for prev, nxt in zip(calls, calls[1:]):
        assert nxt[1] is prev[4]
    queries = torch.cat([c[0] for c in calls], 1)
    return queries, torch.cat([c[2] for c in calls], 1), torch.cat([c[3] for c in calls], 1)


@pytest.mark.parametrize("cell,conditional", [("NematusGRU", False), ("NematusGRU", True), ("LSTM", False),
                                              ("GRU", True)])
def test_stepwise_training_carries_coverage(cpu_model, monkeypatch, cell, conditional):
    dec, att = CVO.build_model(rnn_cell=cell, conditional_gru=conditional)
    CVO.randomize()
    calls, scan = _spy(monkeypatch, att)
    ids = CVO.target_ids()
    CVO.feed(dec, att, train=True, ids=ids)
    loss = dec.train_loss
    queries, ctx, weights = _check_chain(calls, ids.shape[1])
    with torch.no_grad():
        want_ctx, want_w, _ = scan(att, queries, None)
    torch.testing.assert_close(ctx, want_ctx, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(weights, want_w, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(att.histories["decoder_train"], weights.transpose(0, 1))
    _check_gradients(loss)


def test_differentiable_loop_carries_coverage(cpu_model, monkeypatch):
    dec, att = CVO.build_model()
    CVO.randomize()
    calls, scan = _spy(monkeypatch, att)
    CVO.feed(dec, att, train=True, ids=CVO.target_ids())
    out = dec.differentiable_loop()
    queries, _ctx, weights = _check_chain(calls, out["states"].shape[0])
    with torch.no_grad():
        torch.testing.assert_close(weights, scan(att, queries, None)[1], rtol=1e-5, atol=1e-6)
    nll, _ = dec.loop_nll(out["states"], out["symbols"])
    _check_gradients(nll.sum())


def test_greedy_decoding_carries_coverage(cpu_model, monkeypatch):
    """Decoding steps through `next_state` (the fused step engine takes only a plain Attention)."""
    dec, att = CVO.build_model()
    CVO.randomize()
    assert dec.decode_engine is None
    calls, _ = _spy(monkeypatch, att)
    CVO.feed(dec, att, train=False)
    symbols = dec.runtime_symbols
    _queries, _ctx, weights = _check_chain(calls, len(calls))
    assert symbols.shape[0] == len(calls)
    torch.testing.assert_close(att.histories["decoder_run"], weights.transpose(0, 1))


def _beam(dec, att, beam, max_steps):
    from neuralmonkey_b200.decoders.beam_search_decoder import BeamSearchDecoder
    bs = BeamSearchDecoder(name="bs", parent_decoder=dec, beam_size=beam, max_steps=max_steps,
                           length_normalization=1.0)
    CVO.feed(dec, att, train=False)
    bs.reset_batch()
    bs.batch_size = dec.batch_size
    return bs, bs.outputs


def _forced_logprob_sums(bs, token_ids):
    """Each final hypothesis scored on its own: rows b*k+j follow hypothesis (b, j) from the start symbol with no
    re-ordering, summing the log-probabilities of its words up to and including </s>."""
    from neuralmonkey_b200.vocabulary import END_TOKEN_INDEX
    parent = bs.parent_decoder
    steps, bsz, k = token_ids.shape
    words = token_ids.reshape(steps, bsz * k)
    with torch.no_grad():
        init = bs.get_initial_loop_state()
        logprobs = init.search_state.prev_logprobs.reshape(bsz * k, -1)
        dec_ls = init.decoder_loop_state
        total = torch.zeros(bsz * k)
        alive = torch.ones(bsz * k, dtype=torch.bool)
        for t in range(steps):
            total += torch.where(alive, logprobs[torch.arange(bsz * k), words[t]], torch.zeros(()))
            alive &= words[t] != END_TOKEN_INDEX
            feed = dec_ls.feedables._replace(embedded_input=parent.embed_input_symbols(words[t]))
            dec_ls, lp, _ = bs._decoder_step(dec_ls._replace(feedables=feed))
            logprobs = lp.reshape(bsz * k, -1)
    return total.view(bsz, k)


def test_beam_search_reorders_the_coverage(cpu_model, monkeypatch):
    """Beam 3 over a batch of 2: every final hypothesis' log-probability equals that hypothesis scored on its own.
    Without re-ordering the running coverage with the selected beams it does not."""
    from neuralmonkey_b200.decoders.decoder import Decoder
    text, mask = CVO.encoder_states(5)
    dec, att = CVO.build_model(states=(text[:2], mask[:2]), max_fertility=1)
    CVO.randomize(scale=1.0, seed=5)
    bs, out = _beam(dec, att, 3, 4)
    token_ids = out.last_search_step_output.token_ids[1:]
    want = _forced_logprob_sums(bs, token_ids)
    torch.testing.assert_close(out.last_search_state.logprob_sum, want, rtol=1e-5, atol=1e-5)

    monkeypatch.setattr(Decoder, "reorder_attention_states", lambda self, histories, gather: histories)
    bs, out = _beam(dec, att, 3, 4)
    want = _forced_logprob_sums(bs, out.last_search_step_output.token_ids[1:])
    assert float((out.last_search_state.logprob_sum - want).abs().max()) > 1e-3


def test_hierarchical_combination_refuses_a_coverage_child(cpu_model):
    from neuralmonkey_b200.attention import Attention, CoverageAttention
    from neuralmonkey_b200.attention.combination import HierarchicalMultiAttention
    dec, att = CVO.build_model()
    plain = Attention(name="plain", encoder=att.encoder)
    with pytest.raises(ValueError, match="CoverageAttention"):
        HierarchicalMultiAttention(name="hier", attentions=[plain, att], attention_state_size=4,
                                   use_sentinels=False, share_attn_projections=False)
    assert isinstance(att, CoverageAttention)


# -- the bahdanau INI with a coverage attention ----------------------------------------------------------------------
BEAM_SECTIONS = """
[bs_decoder]
class=decoders.beam_search_decoder.BeamSearchDecoder
name="beam_search_decoder"
parent_decoder=<decoder>
length_normalization=0.6
max_steps=10
beam_size=3

[beam_runner]
class=runners.beamsearch_runner.BeamSearchRunner
output_series="target_beam"
decoder=<bs_decoder>
"""


def write_coverage_ini(tree: str) -> str:
    """tests/bahdanau.ini of the reference with its [attention] a CoverageAttention and a beam-3 runner added;
    returns the INI's path relative to `tree`."""
    from tests.golden.make_reference_bundle import unpack
    unpack(tree)
    text = open(os.path.join(tree, "tests", "bahdanau.ini"), encoding="utf-8").read()
    for old, new in (("class=attention.Attention\n", "class=attention.coverage.CoverageAttention\nmax_fertility=3\n"),
                     ("runners=[<runner>, ", "runners=[<runner>, <beam_runner>, ")):
        assert old in text
        text = text.replace(old, new)
    with open(os.path.join(tree, "tests", "coverage.ini"), "w", encoding="utf-8") as handle:
        handle.write(text + BEAM_SECTIONS)
    return "tests/coverage.ini"


def run_coverage_ini(monkeypatch, tmp_path, extra=()):
    from neuralmonkey_b200 import runtime
    ini = write_coverage_ini(str(tmp_path / "tree"))
    monkeypatch.chdir(tmp_path / "tree")
    out = str(tmp_path / "coverage")
    argv = ["neuralmonkey-train", ini, "-s", 'main.output="{}"'.format(out),
            "-s", 'val_data_no_target.outputs=[("encoded", "{0}/encoded"), ("debugtensors", "{0}/debugtensors")]'
            .format(out)] + list(extra)
    monkeypatch.setattr(sys, "argv", argv)
    try:
        from neuralmonkey_b200.train import main
        main()
    finally:
        runtime.reset()
    return open(os.path.join(out, "experiment.log")).read(), out


def test_bahdanau_ini_with_coverage_trains(monkeypatch, tmp_path):
    from neuralmonkey_b200.trainers.generic_trainer import GenericTrainer
    _stand_ins(monkeypatch)
    monkeypatch.setattr(GenericTrainer, "_adam_kernel", cpu_ops.adam_kernel)
    monkeypatch.setenv("NEURALMONKEY_STRICT", "1")
    log_text, out = run_coverage_ini(monkeypatch, tmp_path, ["-s", "main.epochs=1"])
    assert "Training finished" in log_text and "Validation (epoch" in log_text
    assert "target_beam" in log_text
    assert os.path.exists(os.path.join(out, "variables.data.final"))
