"""The reference's OWN experiment INIs for the hot path (tests/{bahdanau,transformer,beamsearch,small,
factored,post-edit,language-model}.ini of the reference, the ones its `tests/tests_run.sh` trains), unchanged, through this package's
`neuralmonkey-train` entry point - on the CPU over the stand-in operations of tests/cpu_ops.py.
What is exercised is everything but the kernels: the INI grammar with variables and environment
substitution, `class=` resolution against this package, constructor signatures and validation, datasets
with bucketing, vocabularies, the training loop with validation, runners, evaluators, checkpoints.
The INIs and their toy corpora come from the bundles under tests/golden/ (make_reference_bundle.py), unpacked
into a scratch tree.  Only the output locations are redirected, and `evaluators.TER` (third-party pyter, absent
here as TensorFlow is) is dropped from small.ini's evaluation list."""
import os
import sys

import numpy as np
import pytest
import torch

from tests import cpu_ops
from tests.golden.make_reference_bundle import unpack

pytestmark = [pytest.mark.filterwarnings("ignore:Converting a tensor with requires_grad")]

CASES = {
    "bahdanau": ['val_data_no_target.outputs=[("encoded", "{out}/encoded"), ("debugtensors", "{out}/debugtensors")]'],
    "transformer": [],
    "beamsearch": [],
    "small": ['main.evaluation=[("target", $bleu), ("target", evaluators.ChrF3)]'],
    # FactoredEncoder + attention.ScaledDotProdAttention as the RNN decoder's attention object
    "factored": [],
    # two encoders (GRU and LSTM), MultiHeadAttention (3 heads, keys and values from different encoders) +
    # ScaledDotProdAttention on one decoder, the edit-operation pre/postprocessors; pyter's TER dropped
    "post-edit": ['main.evaluation=[("target", <bleu>)]'],
    # an RNN decoder without encoders, word2vec-initialised embeddings, XentRunner + PerplexityEvaluator
    "language-model": [],
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_reference_ini_trains_unchanged(monkeypatch, tmp_path, name):
    from neuralmonkey_b200 import ops, runtime
    from neuralmonkey_b200.trainers.generic_trainer import GenericTrainer
    for op in cpu_ops.STAND_INS:
        monkeypatch.setattr(ops, op, getattr(cpu_ops, op))
    monkeypatch.setattr(runtime, "_device", torch.device("cpu"))
    monkeypatch.setattr(GenericTrainer, "_adam_kernel", cpu_ops.adam_kernel)
    monkeypatch.setenv("NEURALMONKEY_STRICT", "1")        # as tests_run.sh: warnings are errors
    monkeypatch.setenv("NM_EXPERIMENT_NAME", "small")     # small.ini reads it from the environment
    unpack(str(tmp_path / "tree"))
    monkeypatch.chdir(tmp_path / "tree")                  # the INIs name their data relative to the tree
    out = str(tmp_path / name)
    argv = ["neuralmonkey-train", "tests/{}.ini".format(name), "-s", 'main.output="{}"'.format(out)]
    for change in CASES[name]:
        argv += ["-s", change.format(out=out)]
    monkeypatch.setattr(sys, "argv", argv)
    try:
        from neuralmonkey_b200.train import main
        main()
    finally:
        runtime.reset()
    log_text = open(os.path.join(out, "experiment.log")).read()
    assert "Training finished" in log_text and "Validation (epoch" in log_text
    assert os.path.exists(os.path.join(out, "variables.data.final"))
    if name == "bahdanau":
        assert os.path.exists(os.path.join(out, "encoded.npy"))
    if name == "beamsearch":
        assert "beam_search_score" in log_text
    if name == "language-model":
        assert "xents/perplexity" in log_text


_FEATURES_INI = """
[main]
name="captioning over pre-extracted feature maps"
tf_manager=<tf_manager>
output="{out}"
overwrite_output_dir=True
batch_size=2
epochs=2
train_dataset=<train_data>
val_dataset=<val_data>
trainer=<trainer>
runners=[<runner>]
postprocess=None
evaluation=[("target", evaluators.BLEU)]
logging_period=1
validation_period=5
random_seed=1234

[tf_manager]
class=tf_manager.TensorFlowManager
num_threads=4
num_sessions=1

[numpy_reader]
class=readers.numpy_reader.from_file_list
prefix="tests/data/flickr30k"
shape=[8, 8, 2048]

[train_data]
class=dataset.load
series=["target", "images"]
data=["tests/data/flickr30k/train.de", ("tests/data/flickr30k/train_images.npz.txt", <numpy_reader>)]

[val_data]
class=dataset.load
series=["target", "images"]
data=["tests/data/flickr30k/val.de", ("tests/data/flickr30k/val_images.npz.txt", <numpy_reader>)]

[imagenet]
class=encoders.numpy_stateful_filler.SpatialFiller
name="imagenet"
input_shape=[8, 8, 2048]
data_id="images"
projection_dim=6
ff_hidden_dim=9

[decoder_vocabulary]
class=vocabulary.from_wordlist
path="tests/data/decoder_vocab.tsv"

[attention]
class=attention.Attention
name="attention"
encoder=<imagenet>
state_size=5

[decoder]
class=decoders.decoder.Decoder
name="decoder"
attentions=[<attention>]
encoders=[<imagenet>]
rnn_size=3
embedding_size=3
dropout_keep_prob=0.5
data_id="target"
max_output_len=3
vocabulary=<decoder_vocabulary>

[trainer]
class=trainers.cross_entropy_trainer.CrossEntropyTrainer
decoders=[<decoder>]
l2_weight=1.0e-8
clip_norm=1.0

[runner]
class=runners.GreedyRunner
decoder=<decoder>
output_series="target"
"""


def test_captioning_over_the_reference_feature_files(monkeypatch, tmp_path):
    """The image half of the reference's tests/flat-multiattention.ini - `readers.numpy_reader.from_file_list`
    over the flickr30k sample's file lists into a `SpatialFiller` - under the attention decoder of the hot path
    (the FlatMultiAttention wrapper of that INI is outside it).  The 8 x 8 x 2048 feature maps are seeded
    stand-ins written in the layout of the reference's .npz files (one `arr_0` array each)."""
    from neuralmonkey_b200 import ops, runtime
    from neuralmonkey_b200.trainers.generic_trainer import GenericTrainer
    for op in cpu_ops.STAND_INS:
        monkeypatch.setattr(ops, op, getattr(cpu_ops, op))
    monkeypatch.setattr(runtime, "_device", torch.device("cpu"))
    monkeypatch.setattr(GenericTrainer, "_adam_kernel", cpu_ops.adam_kernel)
    monkeypatch.setenv("NEURALMONKEY_STRICT", "1")
    tree = tmp_path / "tree"
    unpack(str(tree))
    flickr = tree / "tests" / "data" / "flickr30k"
    g = np.random.default_rng(30)
    for listing in ("train_images.npz.txt", "val_images.npz.txt"):
        for name in (flickr / listing).read_text().split():
            np.savez(str(flickr / name), g.standard_normal((8, 8, 2048)).astype(np.float32))
    monkeypatch.chdir(tree)
    out = str(tmp_path / "features")
    ini = tmp_path / "features.ini"
    ini.write_text(_FEATURES_INI.format(out=out))
    monkeypatch.setattr(sys, "argv", ["neuralmonkey-train", str(ini)])
    try:
        from neuralmonkey_b200.train import main
        main()
        names = set(runtime.arena().names) if hasattr(runtime.arena(), "names") else set()
    finally:
        runtime.reset()
    log_text = open(os.path.join(out, "experiment.log")).read()
    assert "Training finished" in log_text and "Validation (epoch" in log_text and "target/BLEU" in log_text
    assert os.path.exists(os.path.join(out, "variables.data.final"))
    saved = torch.load(os.path.join(out, "variables.data.final"), weights_only=False) \
        if not names else None
    keys = names or set(saved.get("variables", saved).keys())
    assert {"imagenet/conv2d/kernel", "imagenet/conv2d_1/kernel"} <= keys
