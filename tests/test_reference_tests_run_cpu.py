"""The in-scope part of the reference's own integration script, tests/tests_run.sh, command by command and with
the INIs TRULY unchanged - output directories included: the commands run from a scratch directory into which
the reference's `tests/*.ini` and `tests/data` files are unpacked from the bundles under tests/golden/, so
`neuralmonkey-run` finds what `neuralmonkey-train` wrote where the INI says.  On the CPU over the stand-in
operations (tests/cpu_ops.py); what is exercised is the whole host side of both entry points.

    bin/neuralmonkey-train tests/transformer.ini
    bin/neuralmonkey-run tests/transformer.ini tests/test_data.ini
    NM_EXPERIMENT_NAME=small bin/neuralmonkey-train tests/small.ini        (pyter's TER dropped: third-party, absent)
    NM_EXPERIMENT_NAME='"small"' bin/neuralmonkey-run tests/small.ini tests/test_data.ini --json ... ["target/bleu"]
    bin/neuralmonkey-train tests/beamsearch.ini
    score_single   = neuralmonkey-run tests/beamsearch.ini tests/test_data_ensembles_single.ini --json ...
    score_ensemble = neuralmonkey-run tests/beamsearch_ensembles.ini tests/test_data_ensembles_duplicate.ini --json ...
    "${score_single:0:8}" == "${score_ensemble:0:8}"
    bin/neuralmonkey-run tests/beamsearch_ensembles.ini tests/test_data_ensembles_all.ini

(The other training commands of the script that are on the hot path - bahdanau, post-edit, factored,
language-model - are in tests/test_reference_inis_cpu.py.)"""
import importlib
import json
import os
import sys

import pytest
import torch

from tests import cpu_ops
from tests.golden.make_reference_bundle import unpack

pytestmark = [pytest.mark.filterwarnings("ignore:Converting a tensor with requires_grad")]


@pytest.fixture
def scratch_tree(monkeypatch, tmp_path):
    from neuralmonkey_b200 import ops, runtime
    from neuralmonkey_b200.trainers.generic_trainer import GenericTrainer
    for op in cpu_ops.STAND_INS:
        monkeypatch.setattr(ops, op, getattr(cpu_ops, op))
    monkeypatch.setattr(runtime, "_device", torch.device("cpu"))
    monkeypatch.setattr(GenericTrainer, "_adam_kernel", cpu_ops.adam_kernel)
    monkeypatch.setenv("NEURALMONKEY_STRICT", "1")
    tests_dir = tmp_path / "tests"
    (tests_dir / "outputs").mkdir(parents=True)
    unpack(str(tmp_path))
    monkeypatch.chdir(tmp_path)

    def command(kind, *argv):
        monkeypatch.setattr(sys, "argv", ["neuralmonkey-" + kind] + list(argv))
        try:
            importlib.import_module("neuralmonkey_b200." + kind).main()
        finally:
            runtime.reset()

    yield command, tmp_path
    runtime.reset()


def _first_result(path, key):
    with open(path) as handle:
        return json.load(handle)[0][key]


def test_transformer_train_then_run(scratch_tree):
    command, root = scratch_tree
    command("train", "tests/transformer.ini")
    command("run", "tests/transformer.ini", "tests/test_data.ini")
    written = (root / "tests" / "outputs" / "tmpout-val10.tc.de").read_text().splitlines()
    assert len(written) == 10          # test_data.ini: both datasets write the ten sentences of val10


def test_small_with_the_experiment_name_from_the_environment(scratch_tree, monkeypatch):
    command, root = scratch_tree
    monkeypatch.setenv("NM_EXPERIMENT_NAME", "small")
    command("train", "tests/small.ini", "-s", 'main.evaluation=[("target", $bleu), ("target", evaluators.ChrF3)]')
    assert (root / "tests" / "outputs" / "small" / "variables.data.final").exists()
    monkeypatch.setenv("NM_EXPERIMENT_NAME", '"small"')
    out = str(root / "small.json")
    command("run", "tests/small.ini", "tests/test_data.ini", "-s",
            'main.evaluation=[("target", $bleu), ("target", evaluators.ChrF3)]', "--json", out)
    assert isinstance(_first_result(out, "target/bleu"), float)


def test_an_ensemble_of_a_model_with_itself_scores_what_the_model_scores(scratch_tree):
    command, root = scratch_tree
    command("train", "tests/beamsearch.ini")
    single, ensemble = str(root / "single.json"), str(root / "ensemble.json")
    command("run", "tests/beamsearch.ini", "tests/test_data_ensembles_single.ini", "--json", single)
    command("run", "tests/beamsearch_ensembles.ini", "tests/test_data_ensembles_duplicate.ini", "--json", ensemble)
    key = "target_beam.rank001/beam_search_score"
    score_single, score_ensemble = _first_result(single, key), _first_result(ensemble, key)
    assert str(score_single)[:8] == str(score_ensemble)[:8], (score_single, score_ensemble)
    command("run", "tests/beamsearch_ensembles.ini", "tests/test_data_ensembles_all.ini")
