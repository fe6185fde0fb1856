"""The host side of the reinforcement-learning objectives, without a GPU.

* The fp64 restatement of the index-based rewards (tests/rl_oracle.py) and `evaluators.gleu.GLEUEvaluator` against
  the golden vectors the reference's own code produced (tests/golden/make_rl_golden.py).
* `ReinforceObjective` / `SelfCriticalObjective` over the CPU stand-ins of tests/cpu_ops.py, with the two new
  operations (`sentence_ngram_reward`, `sample_logits_step`) stood in below: the baseline across steps, normalize /
  alpha, ce_smoothing, unmasked against masked sums, one baseline update per step, and the refusals.  The
  expected values come from the oracle's teacher-forced pass fed with the symbols the loop chose."""
import os

import numpy as np
import pytest
import torch

from oracle import nm_oracle as O
from tests import cpu_ops, rl_oracle
from tests.helpers import build_bahdanau, feed, oracle_params_for, oracle_spec, random_batch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "rl_golden.npz")
CASES = ("small", "ragged", "long", "large_ids", "quirks", "unequal")
pytestmark = pytest.mark.filterwarnings("ignore:Converting a tensor with requires_grad")
TOY = dict(vs=60, vt=70, es=11, he=7, et=9, hd=8, out=9, maxout=True, max_len=10, supress_unk=True)


@pytest.mark.parametrize("case", CASES)
def test_reward_restatement_matches_the_reference(case):
    g = np.load(GOLDEN)
    refs, hyps = g[case + "_refs"], g[case + "_hyps"]
    assert np.array_equal(rl_oracle.sentence_bleu(refs, hyps), g[case + "_bleu"])
    assert np.array_equal(rl_oracle.sentence_gleu(refs, hyps), g[case + "_gleu"])


def test_gleu_evaluator_matches_the_reference():
    from neuralmonkey_b200.evaluators.gleu import GLEUEvaluator
    g = np.load(GOLDEN)
    hyps = [str(s).split(" ") for s in g["eval_hyps"]]
    refs = [str(s).split(" ") for s in g["eval_refs"]]
    for n, dedup in ((4, False), (2, False), (4, True)):
        key = "eval_n{}_{}".format(n, "dedup" if dedup else "plain")
        ev = GLEUEvaluator(n=n, deduplicate=dedup)
        assert ev.name == str(g[key + "_name"])
        assert [ev([h], [r]) for h, r in zip(hyps, refs)] == list(g[key + "_sentence"])
        assert ev(hyps, refs) == float(g[key + "_corpus"])


# -- stand-ins of the two new operations -------------------------------------------------------------------------
def sentence_ngram_reward(references, hypotheses, mode):
    fn = rl_oracle.sentence_bleu if mode == "bleu" else rl_oracle.sentence_gleu
    return torch.from_numpy(fn(references.numpy(), hypotheses.numpy()))


def sample_logits_step(logits, temperature, finished, unk_index, loop_step, sample_index):
    gen = torch.Generator().manual_seed(1000 * sample_index + loop_step)
    u = torch.rand(logits.shape, generator=gen, dtype=torch.float64)
    score = logits.double() / temperature - torch.log(-torch.log(u))
    if unk_index >= 0:
        score[:, unk_index] = -float("inf")
    symbols = score.argmax(1) * (~finished).to(torch.int64)
    return symbols, finished | (symbols == 2)


@pytest.fixture
def cpu_model(monkeypatch):
    from neuralmonkey_b200 import ops, runtime
    for name in cpu_ops.STAND_INS:
        monkeypatch.setattr(ops, name, getattr(cpu_ops, name))
    monkeypatch.setattr(ops, "sentence_ngram_reward", sentence_ngram_reward)
    monkeypatch.setattr(ops, "sample_logits_step", sample_logits_step)
    monkeypatch.setattr(runtime, "_device", torch.device("cpu"))
    yield
    runtime.reset()


def _model(seed=0, bsz=6, end_bias=0.0, scale=1.0):
    model = build_bahdanau(**TOY)
    params = oracle_params_for(model, scale=scale)
    params["decoder/state_to_word_b"][2] += end_bias          # </s> more likely: rows finish at different steps
    model["arena"].load_dict(params)
    src, tgt = random_batch(bsz, 8, 7, TOY["vs"], TOY["vt"], seed=seed)
    feed(model, src, tgt, train=True)
    return model, params, src, tgt


def _oracle_logprobs(params, src, symbols, temperature=1.0):
    """[T, B] fp64 log-probabilities of `symbols` under the oracle's pass fed with them (it reproduces the loop)."""
    p = {n: v.double() for n, v in params.items()}
    enc = O.sentence_encoder(p, "sentence_encoder", src)
    logits = O.decoder_train(p, oracle_spec(True, 10, True), enc, symbols)["train_logits"]
    return torch.log_softmax(logits / temperature, -1).gather(2, symbols.unsqueeze(-1)).squeeze(-1), logits


def _words_reward(hyps, refs):
    """A reward over words that depends on both sentences: what the objective hands an evaluator."""
    return float(len(hyps[0])) / (1 + len(refs[0])) + (0.5 if hyps[0][:1] == refs[0][:1] else 0.0)


def _expected_reward(vocab, ref_ids, hyp_ids):
    def words(row):
        out = []
        for i in row:
            if int(i) in (0, 2):
                break
            out.append(vocab.index_to_word[int(i)])
        return " ".join(out).replace("@@ ", "").split(" ")
    return np.array([_words_reward([words(h)], [words(r)]) for r, h in zip(ref_ids.t(), hyp_ids.t())], np.float32)


def _run_loops(dec, sample_size, temperature):
    """The symbols the objective's loops choose, replayed with the same stand-in sampler."""
    out = []
    for s in range(sample_size):
        with torch.no_grad():
            out.append(dec.differentiable_loop(sample=True, temperature=temperature, sample_index=s)["symbols"])
    return out


@pytest.mark.parametrize("mode", ["plain", "baseline", "normalize", "mixed"])
def test_reinforce_objective_against_the_oracle(cpu_model, mode):
    from neuralmonkey_b200.trainers.rl_trainer import ReinforceObjective
    cfg = {"plain": dict(), "baseline": dict(subtract_baseline=True, sample_size=2),
           "normalize": dict(normalize=True, alpha=0.7, sample_size=3, temperature=0.5),
           "mixed": dict(ce_smoothing=0.5, sample_size=2, subtract_baseline=True)}[mode]
    model, params, src, tgt = _model(seed=4)
    dec = model["dec"]
    obj = ReinforceObjective(dec, _words_reward, **cfg)
    temperature, size = cfg.get("temperature", 1.0), cfg.get("sample_size", 1)
    counter = reward_sum = np.float32(0.0)
    for step in range(3):
        if step:
            src, tgt = random_batch(6, 8, 7, TOY["vs"], TOY["vt"], seed=4 + step)
            feed(model, src, tgt, train=True)
        symbols = _run_loops(dec, size, temperature)
        loss = obj.loss
        assert obj.loss is loss                          # read twice: one loss, one baseline update
        rewards = np.stack([_expected_reward(dec.vocabulary, tgt.t(), s) for s in symbols])
        logprobs = torch.stack([_oracle_logprobs(params, src, s, temperature)[0].sum(0) for s in symbols])
        if cfg.get("subtract_baseline"):
            counter = np.float32(counter + np.float32(6 * size))
            reward_sum = np.float32(reward_sum + rewards.sum(dtype=np.float32))
            rewards = rewards - reward_sum / max(counter, np.float32(1))
            assert obj.reward_counter == counter and obj.reward_sum == reward_sum
        if cfg.get("normalize"):
            logprobs = torch.softmax(logprobs * cfg["alpha"], 0)
        want = (-torch.from_numpy(rewards).double() * logprobs).sum(0).mean()
        if cfg.get("ce_smoothing"):
            p = {n: v.double() for n, v in params.items()}
            enc = O.sentence_encoder(p, "sentence_encoder", src)
            want = want + cfg["ce_smoothing"] * O.decoder_train(p, oracle_spec(True, 10, True), enc,
                                                                tgt.t())["train_loss"]
        assert abs(float(loss) - float(want)) <= 1e-4 * abs(float(want)) + 1e-5, (step, float(loss), float(want))


def test_reinforce_sums_every_step_unmasked(cpu_model):
    """The sentence log-probability includes </s> and the <pad> steps after it (rl_trainer.py:138-140)."""
    from neuralmonkey_b200.trainers.rl_trainer import ReinforceObjective
    model, params, src, _tgt = _model(seed=11, end_bias=3.0, scale=0.3)
    dec = model["dec"]
    symbols = _run_loops(dec, 1, 1.0)[0]
    assert bool((symbols == 0).any()), "the batch should contain rows that finished early"
    obj = ReinforceObjective(dec, lambda hyps, refs: 1.0)
    lp = _oracle_logprobs(params, src, symbols)[0]
    assert abs(float(obj.loss) - float(-lp.sum(0).mean())) < 1e-5


@pytest.mark.parametrize("reward", ["device", "host"])
def test_self_critical_objective_against_the_oracle(cpu_model, reward):
    from neuralmonkey_b200.trainers.self_critical_objective import SelfCriticalObjective, sentence_bleu
    model, params, src, tgt = _model(seed=6)
    dec = model["dec"]
    fn = sentence_bleu if reward == "device" else rl_oracle.sentence_bleu
    obj = SelfCriticalObjective(dec, fn, weight=0.5)
    loss = obj.loss
    assert obj.loss is loss and obj.weight == 0.5
    p = {n: v.double() for n, v in params.items()}
    enc = O.sentence_encoder(p, "sentence_encoder", src)
    spec = oracle_spec(True, 10, True)
    greedy = O.decoder_greedy(p, spec, enc)
    symbols, mask = greedy["output_symbols"], greedy["runtime_mask"].double()
    argmax = greedy["runtime_logits"].argmax(-1)             # unmasked, as runtime_argmax
    nll = -torch.log_softmax(O.decoder_train(p, spec, enc, symbols)["train_logits"], -1).gather(
        2, argmax.unsqueeze(-1)).squeeze(-1)
    train_decoded = O.decoder_train(p, spec, enc, tgt.t())["train_logits"].argmax(-1)
    refs = tgt.t().numpy()
    diff = rl_oracle.sentence_bleu(refs, argmax.numpy()) - rl_oracle.sentence_bleu(refs, train_decoded.numpy())
    want = -(torch.from_numpy(diff).double() * nll * mask).sum() / mask.sum()
    assert bool((argmax * mask.long() == symbols * mask.long()).all())
    assert abs(float(loss) - float(want)) <= 1e-4 * abs(float(want)) + 1e-6, (float(loss), float(want))


def test_self_critical_loss_is_zero_when_every_row_finishes_at_once(cpu_model):
    """</s> wins every first step: no unmasked position is left, and the loss is 0 with zero gradients instead of
    the reference's 0 / 0."""
    from neuralmonkey_b200.trainers.self_critical_objective import SelfCriticalObjective, sentence_bleu
    model, _params, _src, _tgt = _model(seed=6, end_bias=1e3, scale=0.3)
    loss = SelfCriticalObjective(model["dec"], sentence_bleu).loss
    assert float(loss) == 0.0
    loss.backward()
    for name in model["arena"].train_names:
        grad = model["arena"].get(name).grad
        assert grad is None or bool(torch.isfinite(grad).all()), name


def test_refusals(cpu_model, monkeypatch):
    from neuralmonkey_b200 import distributed
    from neuralmonkey_b200.trainers.generic_trainer import GenericTrainer
    from neuralmonkey_b200.trainers.rl_trainer import ReinforceObjective, rl_objective
    from neuralmonkey_b200.trainers.self_critical_objective import SelfCriticalObjective, sentence_gleu
    model, _params, _src, _tgt = _model()
    dec = model["dec"]
    for make in (lambda d: ReinforceObjective(d, _words_reward), lambda d: SelfCriticalObjective(d, sentence_gleu)):
        with pytest.raises(TypeError):
            make(object())
        obj = make(dec)
        with pytest.raises(ValueError, match="use_cuda_graph"):
            GenericTrainer([obj], use_cuda_graph=True)
        GenericTrainer([obj])
        monkeypatch.setattr(distributed, "world_size", lambda: 2)
        with pytest.raises(RuntimeError, match="one rank"):
            _ = obj.loss
        monkeypatch.setattr(distributed, "world_size", lambda: 1)
    obj = rl_objective(dec, _words_reward, sample_size=2)
    assert isinstance(obj, ReinforceObjective) and obj.sample_size == 2
    with pytest.raises(ValueError):
        ReinforceObjective(dec, _words_reward, sample_size=0)


def test_trainer_step_sums_cross_entropy_and_self_critical(cpu_model, monkeypatch):
    """self-critical.ini's trainer: CostObjective + SelfCriticalObjective, each weighted 0.5, one update."""
    from neuralmonkey_b200.trainers.generic_trainer import GenericTrainer
    from neuralmonkey_b200.trainers.objective import CostObjective
    from neuralmonkey_b200.trainers.self_critical_objective import SelfCriticalObjective, sentence_bleu
    monkeypatch.setattr(GenericTrainer, "_adam_kernel", cpu_ops.adam_kernel)
    model, _params, _src, _tgt = _model(seed=2)
    dec = model["dec"]
    sc = SelfCriticalObjective(dec, sentence_bleu, weight=0.5)
    trainer = GenericTrainer([CostObjective(dec, 0.5), sc])
    before = model["arena"].params.clone()
    out = trainer.train_step()
    assert len(out["losses"]) == 2 and all(np.isfinite(float(v)) for v in out["losses"])
    assert float(out["losses"][1]) == float(sc.loss)
    assert not torch.equal(before, model["arena"].params)


@pytest.mark.parametrize("name", ["rl", "self-critical"])
def test_reference_rl_ini_trains_on_the_cpu(cpu_model, monkeypatch, tmp_path, name):
    """tests/rl.ini and tests/self-critical.ini of the reference through `neuralmonkey-train` over the stand-ins;
    self-critical.ini's TER evaluation is dropped (pyter is absent)."""
    import json
    import sys
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.trainers.generic_trainer import GenericTrainer
    from tests.golden.make_reference_bundle import unpack
    monkeypatch.setattr(GenericTrainer, "_adam_kernel", cpu_ops.adam_kernel)
    monkeypatch.setenv("NEURALMONKEY_STRICT", "1")
    tree = tmp_path / "tree"
    unpack(str(tree))
    with open(os.path.join(os.path.dirname(GOLDEN), "reference_experiments_rl.json"), encoding="utf-8") as handle:
        for rel, text in json.load(handle)["files"].items():
            (tree / rel).write_text(text, encoding="utf-8")
    monkeypatch.chdir(tree)
    out = str(tmp_path / name)
    argv = ["neuralmonkey-train", "tests/{}.ini".format(name), "-s", 'main.output="{}"'.format(out)]
    if name == "self-critical":
        argv += ["-s", 'main.evaluation=[("target", evaluators.BLEU)]']
    monkeypatch.setattr(sys, "argv", argv)
    try:
        from neuralmonkey_b200.train import main
        main()
    finally:
        runtime.reset()
    log_text = open(os.path.join(out, "experiment.log")).read()
    assert "Training finished" in log_text and "Validation (epoch" in log_text
    assert os.path.exists(os.path.join(out, "variables.data.final"))
