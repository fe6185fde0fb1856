"""The reinforcement-learning kernels and objectives on the GPU.

* `nm_sentence_ngram_reward` against the golden vectors of the reference's own sentence_bleu / sentence_gleu
  (tests/golden/make_rl_golden.py), within 1 fp32 ulp, on contiguous and strided inputs.
* `nm_sample_logits_step`: chi-square goodness of fit at V = 70 and 32000 and two temperatures, <unk> never drawn,
  the finished bookkeeping, bit-identical draws for identical keys and fresh draws the next training step.
* ReinforceObjective / SelfCriticalObjective losses and every parameter gradient against fp64 autograd through the
  oracle fed with the symbols the loop chose (it then reproduces the loop exactly), on the exact engine.
* With dropout, the logits that are differentiated choose the loop's greedy symbols: the gradient saw the loop's
  dropout masks.
* The reference's tests/rl.ini and tests/self-critical.ini train unchanged through `neuralmonkey-train`."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from scipy import stats

from oracle import nm_oracle as O
from tests import rl_oracle
from tests.helpers import build_bahdanau, feed, oracle_params_for, oracle_spec, random_batch, training_log_values

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore:Converting a tensor with requires_grad")]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "rl_golden.npz")
CASES = ("small", "ragged", "long", "large_ids", "quirks", "unequal")
TOY = dict(vs=60, vt=70, es=11, he=7, et=9, hd=8, out=9, maxout=True, max_len=10, supress_unk=True)


def _ulps(got: np.ndarray, want: np.ndarray) -> int:
    a, b = got.astype(np.float32).view(np.int32).astype(np.int64), want.astype(np.float32).view(np.int32)
    return int(np.abs(a - b).max()) if a.size else 0


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("layout", ["contiguous", "strided"])
def test_reward_kernel_matches_the_reference(case, layout):
    from neuralmonkey_b200 import ops
    g = np.load(GOLDEN)
    refs, hyps = torch.from_numpy(g[case + "_refs"]), torch.from_numpy(g[case + "_hyps"])
    if layout == "contiguous":
        r, h = refs.cuda(), hyps.cuda()
    else:       # batch-major storage read time-major, and every second row of a wider buffer
        r = refs.t().contiguous().cuda().t()
        wide = torch.full((hyps.shape[0], 2 * hyps.shape[1]), 99, dtype=torch.int64)
        wide[:, ::2] = hyps
        h = wide.cuda()[:, ::2]
    assert not (layout == "strided" and r.is_contiguous())
    for mode in ("bleu", "gleu"):
        got = ops.sentence_ngram_reward(r, h, mode).cpu().numpy()
        assert _ulps(got, g["{}_{}".format(case, mode)]) <= 1, (mode, got, g["{}_{}".format(case, mode)])


def test_reward_functions_take_device_tensors_and_arrays():
    from neuralmonkey_b200.trainers.self_critical_objective import sentence_bleu, sentence_gleu
    g = np.load(GOLDEN)
    refs, hyps = g["small_refs"], g["small_hyps"]
    dev = sentence_bleu(torch.from_numpy(refs).cuda(), torch.from_numpy(hyps).cuda())
    assert dev.is_cuda and dev.dtype == torch.float32
    assert torch.equal(dev, sentence_bleu(refs, hyps))
    assert _ulps(sentence_gleu(refs, hyps).cpu().numpy(), rl_oracle.sentence_gleu(refs, hyps)) <= 1


def _draw(logits_row, rows, temperature, unk=-1, step=0, sample=0, finished=None):
    from neuralmonkey_b200 import ops
    lg = logits_row.reshape(1, -1).expand(rows, -1)           # every row reads the same logits (stride 0)
    fin = torch.zeros(rows, dtype=torch.bool, device="cuda") if finished is None else finished
    return ops.sample_logits_step(lg, temperature, fin, unk, step, sample)


@pytest.mark.parametrize("vocab", [70, 32000])
@pytest.mark.parametrize("temperature", [1.0, 0.5])
def test_sampler_chi_square(vocab, temperature):
    from neuralmonkey_b200 import runtime
    runtime.reset()
    torch.manual_seed(5)
    runtime.dropout_state()
    logits = (torch.randn(vocab, generator=torch.Generator().manual_seed(vocab)) * 2.0).cuda()
    n = 1 << 20
    symbols, _ = _draw(logits, n, temperature)
    counts = torch.bincount(symbols, minlength=vocab).cpu().double().numpy()
    probs = torch.softmax(logits.double().cpu() / temperature, 0).numpy()
    expected = probs * n
    # categories with fewer than 5 expected draws are pooled (the chi-square approximation needs it)
    small = expected < 5
    obs = np.append(counts[~small], counts[small].sum())
    exp = np.append(expected[~small], expected[small].sum())
    if exp[-1] == 0:
        obs, exp = obs[:-1], exp[:-1]
    _, pval = stats.chisquare(obs, exp)
    assert pval > 1e-4, (vocab, temperature, pval)


def test_sampler_bookkeeping_unk_and_keys():
    from neuralmonkey_b200 import runtime
    runtime.reset()
    torch.manual_seed(11)
    logits = torch.zeros(80, device="cuda")
    logits[3] = 5.0                                            # <unk> would be the favourite
    sym, fin = _draw(logits, 1 << 18, 1.0, unk=3)
    assert not bool((sym == 3).any()) and bool((sym == 2).any())
    assert torch.equal(fin, sym == 2)
    # finished rows emit <pad> and stay finished
    finished = torch.arange(1 << 12, device="cuda") % 2 == 0
    sym2, fin2 = _draw(logits, 1 << 12, 1.0, unk=3, finished=finished)
    assert bool((sym2[finished] == 0).all()) and bool(fin2[finished].all())
    assert torch.equal(fin2[~finished], sym2[~finished] == 2)
    # identical keys: bit-identical; another loop step, sample or training step: different draws
    a, _ = _draw(logits, 4096, 0.7, unk=3, step=4, sample=1)
    b, _ = _draw(logits, 4096, 0.7, unk=3, step=4, sample=1)
    assert torch.equal(a, b)
    for other in (_draw(logits, 4096, 0.7, unk=3, step=5, sample=1)[0],
                  _draw(logits, 4096, 0.7, unk=3, step=4, sample=2)[0]):
        assert float((other != a).double().mean()) > 0.5
    runtime.advance_dropout()
    c, _ = _draw(logits, 4096, 0.7, unk=3, step=4, sample=1)
    assert float((c != a).double().mean()) > 0.5


def test_sampler_never_draws_a_negligible_column():
    """A column 30 above all others takes all but ~3e-9 of the mass per draw: 2^20 draws must all be it.  (A uniform
    that could reach 1.0 gives its column an infinite score, whatever its logit, once in 2^24 elements.)"""
    from neuralmonkey_b200 import runtime
    runtime.reset()
    torch.manual_seed(13)
    logits = torch.zeros(32000, device="cuda")
    logits[1234] = 30.0
    for temperature in (1.0, 0.5):
        sym, _ = _draw(logits, 1 << 20, temperature)
        assert int((sym != 1234).sum()) == 0, temperature


# -- objectives against fp64 autograd ------------------------------------------------------------------------------
def _record_loops(monkeypatch, dec):
    """The symbols every differentiable loop of the decoder chose."""
    from neuralmonkey_b200.decoders.decoder import Decoder
    seen = []
    original = Decoder.differentiable_loop

    def recording(self, *args, **kwargs):
        out = original(self, *args, **kwargs)
        if self is dec:
            seen.append({k: v.detach().cpu() for k, v in out.items()})
        return out
    monkeypatch.setattr(Decoder, "differentiable_loop", recording)
    return seen


def _toy(seed, end_bias=3.0, builder=None):
    from neuralmonkey_b200 import ops
    ops.set_gemm_backend("simt")                 # the exact engine: the oracle comparison is in fp64
    model = build_bahdanau(**TOY) if builder is None else builder()
    params = oracle_params_for(model)
    if "decoder/state_to_word_b" in params:
        params["decoder/state_to_word_b"][2] += end_bias     # rows finish at different steps
    model["arena"].load_dict(params)
    return model, params


def _check_grads(model, p64, loss64, tol=3e-4):
    loss64.backward()
    model["arena"].fold_autograd_grads()        # what the trainer does after its backward pass
    for name, grad in model["arena"].named_grads().items():
        want = p64[name].grad
        want = torch.zeros_like(p64[name]) if want is None else want
        err = float((grad.double().cpu() - want.reshape(grad.shape)).norm())
        assert err <= tol * float(want.norm()) + 1e-6, (name, err, float(want.norm()))


def _words_reward(hyps, refs):
    return float(len(hyps[0])) / (1 + len(refs[0])) + (0.5 if hyps[0][:1] == refs[0][:1] else 0.0)


def _host_reward(vocab, ref_ids, hyp_ids):
    def words(row):
        out = []
        for i in row:
            if int(i) in (0, 2):
                break
            out.append(vocab.index_to_word[int(i)])
        return " ".join(out).replace("@@ ", "").split(" ")
    return np.array([_words_reward([words(h)], [words(r)]) for r, h in zip(ref_ids.t(), hyp_ids.t())], np.float32)


REINFORCE = {"bandit": dict(subtract_baseline=True), "mrt": dict(normalize=True, alpha=0.5, sample_size=2),
             "reinforce": dict(sample_size=2, temperature=0.5), "mixed": dict(sample_size=2, ce_smoothing=0.5)}


@pytest.mark.parametrize("mode", sorted(REINFORCE))
def test_reinforce_objective_loss_and_gradients(monkeypatch, mode):
    from neuralmonkey_b200 import ops
    from neuralmonkey_b200.trainers.rl_trainer import ReinforceObjective
    try:
        model, params = _toy(seed=3)
        dec = model["dec"]
        src, tgt = random_batch(6, 8, 7, TOY["vs"], TOY["vt"], seed=3)
        feed(model, src, tgt, train=True)
        cfg = REINFORCE[mode]
        obj = ReinforceObjective(dec, _words_reward, **cfg)
        loops = _record_loops(monkeypatch, dec)
        model["arena"].zero_grad()
        loss = obj.loss
        loss.backward()
        assert obj.loss is loss and len(loops) == cfg.get("sample_size", 1)
        temperature = cfg.get("temperature", 1.0)
        p64 = {n: v.double().requires_grad_(True) for n, v in params.items()}
        enc = O.sentence_encoder(p64, "sentence_encoder", src)
        spec = oracle_spec(True, 10, True)
        rewards, logprobs = [], []
        for loop in loops:
            sym = loop["symbols"]
            logits = O.decoder_train(p64, spec, enc, sym)["train_logits"]
            assert logits.shape[0] == sym.shape[0]
            lp = torch.log_softmax(logits / temperature, -1).gather(2, sym.unsqueeze(-1)).squeeze(-1)
            logprobs.append(lp.sum(0))
            rewards.append(_host_reward(dec.vocabulary, tgt.t(), sym))
        rewards = np.stack(rewards)
        if cfg.get("subtract_baseline"):
            rewards = rewards - np.float32(rewards.sum(dtype=np.float32) / np.float32(rewards.size))
        logprobs = torch.stack(logprobs)
        if cfg.get("normalize"):
            logprobs = torch.softmax(logprobs * cfg["alpha"], 0)
        want = (-torch.from_numpy(rewards).double() * logprobs).sum(0).mean()
        if cfg.get("ce_smoothing"):
            want = want + cfg["ce_smoothing"] * O.decoder_train(p64, spec, enc, tgt.t())["train_loss"]
        assert abs(float(loss) - float(want)) <= 1e-3 * abs(float(want)) + 1e-6, (float(loss), float(want))
        _check_grads(model, p64, want)
    finally:
        ops.set_gemm_backend("auto")


def _self_critical_check(model, params, src, tgt, loops, loss, spec, oracle_encoder, ltol=1e-3, gtol=3e-4):
    """The expected loss from the oracle alone: its greedy loop gives the scored symbols and the mask, its
    teacher-forced passes the NLL and the baseline hypothesis."""
    p64 = {n: v.double().requires_grad_(True) for n, v in params.items()}
    enc = oracle_encoder(p64)
    (loop,) = loops
    with torch.no_grad():
        greedy = O.decoder_greedy({n: v.detach() for n, v in p64.items()}, spec, enc)
    sym, mask = greedy["output_symbols"], greedy["runtime_mask"].double()
    argmax = greedy["runtime_logits"].argmax(-1)                       # unmasked, as runtime_argmax
    assert torch.equal(sym, loop["symbols"]) and torch.equal(argmax, loop["argmax"])
    assert float(mask.sum()) > 0, "every row finished at the first step: nothing to score"
    logits = O.decoder_train(p64, spec, enc, sym)["train_logits"]
    nll = -torch.log_softmax(logits, -1).gather(2, argmax.unsqueeze(-1)).squeeze(-1)
    train_decoded = O.decoder_train(p64, spec, enc, tgt.t())["train_logits"].argmax(-1)
    refs = tgt.t().numpy()
    diff = rl_oracle.sentence_bleu(refs, argmax.numpy()) - rl_oracle.sentence_bleu(refs, train_decoded.numpy())
    want = -(torch.from_numpy(diff).double() * nll * mask).sum() / mask.sum()
    assert abs(float(loss) - float(want)) <= ltol * abs(float(want)) + 1e-6, (float(loss), float(want))
    _check_grads(model, p64, want, gtol)
    return float(loss)


def test_self_critical_objective_loss_and_gradients(monkeypatch):
    from neuralmonkey_b200 import ops
    from neuralmonkey_b200.trainers.self_critical_objective import SelfCriticalObjective, sentence_bleu
    try:
        losses = []
        for fn in (sentence_bleu, rl_oracle.sentence_bleu):
            model, params = _toy(seed=5, end_bias=1.0)
            dec = model["dec"]
            src, tgt = random_batch(8, 8, 7, TOY["vs"], TOY["vt"], seed=5)
            feed(model, src, tgt, train=True)
            loops = _record_loops(monkeypatch, dec)
            model["arena"].zero_grad()
            loss = SelfCriticalObjective(dec, fn).loss
            loss.backward()
            losses.append(_self_critical_check(model, params, src, tgt, loops, loss, oracle_spec(True, 10, True),
                                               lambda p: O.sentence_encoder(p, "sentence_encoder", src)))
            monkeypatch.undo()
        # the device and the host BLEU give the same loss (the rewards agree within 1 fp32 ulp)
        assert abs(losses[0] - losses[1]) <= 1e-6 * abs(losses[1]) + 1e-9, losses
    finally:
        ops.set_gemm_backend("auto")


def test_self_critical_over_an_lstm_decoder(monkeypatch):
    from neuralmonkey_b200 import ops
    from neuralmonkey_b200.trainers.self_critical_objective import SelfCriticalObjective, sentence_bleu
    from tests.test_gpu_variants import _build_variant
    try:
        model, params = _toy(seed=7, end_bias=0.0,
                             builder=lambda: _build_variant("LSTM", False, "maxout", "linear", "LSTM"))
        dec = model["dec"]
        src, tgt = random_batch(5, 8, 7, 30, 40, seed=7)
        feed(model, src, tgt, train=True)
        spec = O.RNNDecoderSpec("decoder", "attention", 10, "maxout", False, "LSTM", False, "linear", 8, 2)

        def oracle_encoder(pp):
            seq = O.embedded_sequence(pp, "sentence_encoder_input", [src])
            return O.recurrent_encoder(pp, "sentence_encoder", seq["temporal_states"], seq["temporal_mask"],
                                       [(5, "bidirectional", "LSTM")])
        loops = _record_loops(monkeypatch, dec)
        model["arena"].zero_grad()
        loss = SelfCriticalObjective(dec, sentence_bleu).loss
        loss.backward()
        _self_critical_check(model, params, src, tgt, loops, loss, spec, oracle_encoder)
    finally:
        ops.set_gemm_backend("auto")


def test_self_critical_on_the_default_engine(monkeypatch):
    """The same check through the default engine's fp16 vocabulary projection, whose backward carries the per-row
    upstream gradient - here signed and data-dependent - scaled by its largest magnitude; the tolerances of the
    default-engine decoder gradient tests."""
    from neuralmonkey_b200 import ops
    from neuralmonkey_b200.trainers.self_critical_objective import SelfCriticalObjective, sentence_bleu
    model, params = _toy(seed=5, end_bias=1.0)
    ops.set_gemm_backend("auto")
    dec = model["dec"]
    src, tgt = random_batch(8, 8, 7, TOY["vs"], TOY["vt"], seed=5)
    feed(model, src, tgt, train=True)
    loops = _record_loops(monkeypatch, dec)
    model["arena"].zero_grad()
    loss = SelfCriticalObjective(dec, sentence_bleu).loss
    loss.backward()
    _self_critical_check(model, params, src, tgt, loops, loss, oracle_spec(True, 10, True),
                         lambda p: O.sentence_encoder(p, "sentence_encoder", src), ltol=1e-2, gtol=2e-2)


def test_dropout_masks_of_the_loop_reach_the_gradient():
    """keep_prob = 0.5: the logits that `loop_nll` differentiates choose the greedy loop's symbols, which they
    only do when they were computed under the same dropout masks."""
    model = build_bahdanau(**TOY)
    dec = model["dec"]
    dec.dropout_keep_prob = 0.5
    model["arena"].load_dict(oracle_params_for(model))
    src, tgt = random_batch(16, 8, 7, TOY["vs"], TOY["vt"], seed=9)
    feed(model, src, tgt, train=True)
    loop = dec.differentiable_loop(sample=False)
    _nll, argmax = dec.loop_nll(loop["states"], loop["argmax"])
    assert torch.equal(argmax, loop["argmax"])
    with torch.no_grad():
        again = dec.differentiable_loop(sample=False)       # other masks, other states
    assert not torch.equal(again["states"], loop["states"])


def test_objective_steps_at_the_en_de_shape():
    """The en-de bench model (B = 256, T = 50, H = 300, V = 32000) on the default engine.  First the case that
    once poisoned the parameters: </s> wins every first step, the greedy loop stops with no unmasked position, and
    the self-critical loss is 0 (the reference's 0 / 0 gave NaN, the update spread it, and the next step's argmax
    over NaN logits was no token id).  Then loops of their full 50 steps (</s> pushed down): self-critical and
    REINFORCE training steps with finite losses and parameters."""
    sys.path.insert(0, ROOT)
    import bench_models as bm
    from neuralmonkey_b200.evaluators.gleu import GLEUEvaluator
    from neuralmonkey_b200.trainers.generic_trainer import GenericTrainer
    from neuralmonkey_b200.trainers.objective import CostObjective
    from neuralmonkey_b200.trainers.rl_trainer import ReinforceObjective
    from neuralmonkey_b200.trainers.self_critical_objective import SelfCriticalObjective, sentence_bleu
    try:
        model = bm.build_ende(cuda_graph=False)
        dec = model.decoder
        src, tgt = bm.synthetic_ids(256, 50, 32000, seed=1), bm.synthetic_ids(256, 50, 32000, seed=2)
        sc = GenericTrainer([CostObjective(dec, 0.5), SelfCriticalObjective(dec, sentence_bleu, weight=0.5)],
                            l2_weight=1e-8, clip_norm=1.0)
        with torch.no_grad():
            dec.decoding_b[2] = 1e3
        bm.feed_ende(model, src, tgt, train=True)
        out = sc.train_step()
        assert float(out["losses"][1]) == 0.0
        assert bool(torch.isfinite(model.arena.params).all())
        with torch.no_grad():
            dec.decoding_b[2] = -1e3
        rl = GenericTrainer([ReinforceObjective(dec, GLEUEvaluator(), subtract_baseline=True, sample_size=2,
                                                ce_smoothing=0.5)], l2_weight=1e-8, clip_norm=1.0)
        for trainer in (sc, sc, rl):
            bm.feed_ende(model, src, tgt, train=True)
            out = trainer.train_step()
            assert all(np.isfinite(float(v)) for v in out["losses"]), out["losses"]
        assert bool(torch.isfinite(model.arena.params).all())
        with torch.no_grad():
            assert dec.differentiable_loop(sample=False)["symbols"].shape == (50, 256)
    finally:
        bm.cleanup()


# -- the reference's experiments -----------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["rl", "self-critical"])
def test_reference_rl_ini_trains_unchanged_on_the_gpu(tmp_path, name):
    tree, out = tmp_path / "tree", str(tmp_path / "out")
    for bundle in ("reference_experiments.json", "reference_experiments_rl.json"):
        with open(os.path.join(ROOT, "tests", "golden", bundle), encoding="utf-8") as handle:
            for rel, text in json.load(handle)["files"].items():
                (tree / rel).parent.mkdir(parents=True, exist_ok=True)
                (tree / rel).write_text(text, encoding="utf-8")
    cmd = [sys.executable, os.path.join(ROOT, "bin", "neuralmonkey-train"), "tests/{}.ini".format(name),
           "-s", 'main.output="{}"'.format(out)]
    if name == "self-critical":                 # pyter's TER: third-party, absent
        cmd += ["-s", 'main.evaluation=[("target", evaluators.BLEU)]']
    env = dict(os.environ, NEURALMONKEY_STRICT="1", PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=str(tree), env=env)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    log_text = open(os.path.join(out, "experiment.log")).read()
    assert "Training finished" in log_text and "Validation (epoch" in log_text
    assert os.path.exists(os.path.join(out, "variables.data.final"))
    losses = training_log_values(log_text, "target/train_xent")
    assert losses and all(np.isfinite(losses)), losses
