"""Host-side logic that needs no GPU: vocabulary, padding, arena layout, sharding."""
import json
import os
import subprocess
import sys

import pytest
import torch

from tests.helpers import training_log_values

from neuralmonkey_b200 import distributed
from neuralmonkey_b200.params import ParameterArena, normal_initializer, zeros_initializer
from neuralmonkey_b200.vocabulary import (END_TOKEN, PAD_TOKEN, Vocabulary, from_wordlist, pad_batch,
                                          sentence_mask)


def test_pad_batch_matches_reference_rules():
    # longest + </s>, truncated to max_length; </s> is cut off when the sentence is too long
    out = pad_batch([["a", "b", "c"], ["d"]], max_length=3, add_end_symbol=True)
    assert out == [["a", "b", "c"], ["d", END_TOKEN, PAD_TOKEN]]
    out = pad_batch([["a", "b"], []], add_end_symbol=True)
    assert out == [["a", "b", END_TOKEN], [END_TOKEN, PAD_TOKEN, PAD_TOKEN]]
    out = pad_batch([["a"]], add_start_symbol=True)
    assert out == [["<s>", "a"]]


def test_vocabulary_roundtrip_and_unknowns(tmp_path):
    path = tmp_path / "vocab.tsv"
    path.write_text("word\tcount\n<pad>\t0\n<s>\t0\n</s>\t0\n<unk>\t0\nhello\t5\nworld\t3\n")
    vocab = from_wordlist(str(path))
    assert len(vocab) == 6 and vocab.index_to_word[4] == "hello"
    ids = vocab.strings_to_indices([["hello", "zzz", "</s>", "<pad>"]])
    assert ids.tolist() == [[4, 3, 2, 0]] and ids.dtype == torch.int64
    assert sentence_mask(ids).tolist() == [[1.0, 1.0, 1.0, 0.0]]
    import numpy as np
    sents = vocab.vectors_to_sentences(np.array([[4], [5], [2], [4]]))
    assert sents == [["hello", "world"]]


def test_arena_layout_is_aligned_and_trainables_first():
    arena = ParameterArena()
    arena.declare("frozen/w", [3, 5], normal_initializer(), trainable=False)
    arena.declare("a/kernel", [7, 9], normal_initializer())
    arena.declare("a/bias", [9], zeros_initializer())
    arena.declare("a/kernel", [7, 9], normal_initializer())  # AUTO_REUSE: same shape is fine
    with pytest.raises(ValueError):
        arena.declare("a/kernel", [7, 8], normal_initializer())
    arena.finalize(torch.device("cpu"))
    offs = arena.seg_off.tolist()
    assert offs[0] == 0 and all(o % ParameterArena.ALIGN == 0 for o in offs)
    assert arena.train_names == ["a/bias", "a/kernel"]   # sorted by name, whatever the declaration order
    assert arena.seg_reg.tolist() == [0, 1]       # biases are not regularised
    assert arena.variables["frozen/w"].offset >= arena.trainable_size
    assert arena.get("a/kernel").requires_grad and not arena.get("frozen/w").requires_grad
    assert arena.get("a/kernel").nm_grad.shape == (7, 9)
    assert arena.allreduce_view.numel() == arena.trainable_size + ParameterArena.STAT_SLOTS


def test_arena_is_independent_of_declaration_order(tmp_path):
    """Data-parallel ranks declare variables in whatever order their sets iterate: layout, initial
    values and checkpoints must come out the same."""
    from neuralmonkey_b200.params import orthogonal_initializer
    decls = [("dec/state_to_word_W", [6, 32], normal_initializer()), ("dec/state_to_word_b", [32], zeros_initializer()),
             ("enc/gates/kernel", [8, 8], orthogonal_initializer()), ("enc/emb", [30, 4], normal_initializer(0.1))]
    arenas = []
    for order in (decls, decls[::-1], [decls[2], decls[0], decls[3], decls[1]]):
        arena = ParameterArena()
        for name, shape, init in order:
            arena.declare(name, shape, init)
        arena.finalize(torch.device("cpu"), seed=11)
        arenas.append(arena)
    for other in arenas[1:]:
        assert other.train_names == arenas[0].train_names
        assert torch.equal(other.params, arenas[0].params)
    first = arenas[0]
    w, b = first.variables["dec/state_to_word_W"], first.variables["dec/state_to_word_b"]
    assert b.offset == w.offset + w.numel          # the bias segment directly follows its weight matrix
    # Adam moments survive a save / restore keyed by variable name
    first.adam_m.uniform_(-1, 1)
    moments = first.moment_dict(first.adam_m)
    arenas[1].load_moments(arenas[1].adam_m, moments)
    restored = arenas[1].moment_dict(arenas[1].adam_m)
    assert all(torch.equal(restored[n], moments[n]) for n in moments)


def test_shard_bounds_cover_everything_once():
    for n in (0, 1, 7, 256, 257):
        for ranks in (1, 2, 3, 8):
            b = distributed.shard_bounds(n, ranks)
            assert b[0] == 0 and b[-1] == n and len(b) == ranks + 1
            sizes = [b[i + 1] - b[i] for i in range(ranks)]
            assert max(sizes) - min(sizes) <= 1


_GLOO_WORKER = r"""
import os, sys, torch
sys.path.insert(0, {root!r})
from neuralmonkey_b200 import distributed
from neuralmonkey_b200.params import ParameterArena, normal_initializer
distributed.init_from_env(backend="gloo")
r, n = distributed.rank(), distributed.world_size()
arena = ParameterArena()
arena.declare("w", [4, 3], normal_initializer())
arena.finalize(torch.device("cpu"))
# each rank contributes grad = rank+1 everywhere, loss_sum = 10*(rank+1), count = rank+2
arena.grads.fill_(float(r + 1))
arena.stats[0] = 10.0 * (r + 1)
arena.stats[1] = float(r + 2)
distributed.all_reduce_sum(arena.allreduce_view)
exp = sum(range(1, n + 1))
assert torch.all(arena.grads == exp), arena.grads
assert float(arena.stats[0]) == 10.0 * exp and float(arena.stats[1]) == exp + n
items = list(range(11))
mine = distributed.shard(items)
gathered = [None] * n
torch.distributed.all_gather_object(gathered, list(mine))
assert sum(gathered, []) == items
print("rank", r, "ok")
"""


def test_two_rank_gloo_allreduce_of_the_exchange_buffer(tmp_path):
    """world_size-2 CPU run of the data-parallel exchange (gradients + loss sum + count)."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = tmp_path / "worker.py"
    script.write_text(_GLOO_WORKER.format(root=root))
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
           "--master-addr", "127.0.0.1", "--master-port", "29611", str(script)]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=240, env=env)
    assert res.returncode == 0, res.stdout + res.stderr
    assert res.stdout.count("ok") == 2


def test_bench_reference_arm_prints_the_contract_line():
    """`bench.py --impl reference` (the oracle timed on the host cores) prints exactly one JSON line on
    stdout carrying the keys the driver reads."""
    import json
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    # 16 sentences per step instead of the whole 256-sentence batch: the line's shape is what is checked here
    res = subprocess.run([sys.executable, "bench.py", "--impl", "reference", "--steps", "1", "--warmup", "0",
                          "--batch", "16"], capture_output=True, text=True, timeout=600, cwd=root)
    assert res.returncode == 0, res.stderr[-2000:]
    lines = [l for l in res.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, res.stdout
    line = json.loads(lines[0])
    for key in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better",
                "scaling", "vs_baseline", "dtype", "data", "config", "cpu_baseline", "e2e"):
        assert key in line, key
    assert line["impl"] == "reference" and line["value"] > 0 and "workload" in line["config"]
    assert line["config"]["per_gpu_batch"] == 16 and line["cpu_sample_sentences_per_step"] == 16
    assert "value_with_4_threads" in line["cpu_baseline"]
    assert line["cpu_baseline"]["kind"] == "port" and line["cpu_baseline"]["value"] == line["value"]
    assert line["e2e"]["value"] == line["value"] and line["e2e"]["h2d_bytes_per_step"] == 0
    assert line["e2e"]["d2h_bytes_per_step"] == 0


def test_arena_folds_gradients_left_by_plain_autograd():
    arena = ParameterArena()
    arena.declare("a/kernel", [3, 4], normal_initializer())
    arena.declare("a/bias", [4], zeros_initializer())
    arena.finalize(torch.device("cpu"))
    kernel = arena.get("a/kernel")
    (kernel * 2.0).sum().backward()              # a torch expression on a parameter: gradient in .grad
    arena.grad("a/kernel").fill_(1.0)            # something an op already accumulated
    assert arena.fold_autograd_grads() == 1
    assert kernel.grad is None and torch.equal(arena.grad("a/kernel"), torch.full((3, 4), 3.0))
    assert arena.fold_autograd_grads() == 0


def test_checkpoint_averaging_script(tmp_path):
    """scripts/avg_checkpoints.py (the reference's command line): the mean of every variable."""
    import subprocess
    import sys
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    paths = []
    for i in range(3):
        path = str(tmp_path / "variables.data.{}".format(i))
        torch.save({"variables": {"a/kernel": torch.full((2, 3), float(i)), "a/bias": torch.arange(3.0) * i},
                    "adam_m": {}, "adam_v": {}}, path)
        paths.append(path)
    out = str(tmp_path / "variables.data.avg")
    res = subprocess.run([sys.executable, os.path.join(root, "scripts", "avg_checkpoints.py")] + paths + [out],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    avg = torch.load(out)["variables"]
    assert torch.equal(avg["a/kernel"], torch.full((2, 3), 1.0)) and torch.equal(avg["a/bias"], torch.arange(3.0))
    res = subprocess.run([sys.executable, os.path.join(root, "scripts", "avg_checkpoints.py"),
                          str(tmp_path / "nope"), out], capture_output=True, text=True)
    assert res.returncode != 0 and "do not exist" in res.stderr


_DP_WORKER = r"""
import os, sys, torch
sys.path.insert(0, {root!r})
from neuralmonkey_b200 import distributed, ops, runtime
from neuralmonkey_b200.trainers.generic_trainer import GenericTrainer
from tests import cpu_ops
from tests.helpers import build_bahdanau, feed, oracle_params_for, random_batch
for name in cpu_ops.STAND_INS:
    setattr(ops, name, getattr(cpu_ops, name))
runtime._device = torch.device("cpu")
GenericTrainer._adam_kernel = cpu_ops.adam_kernel
world = int(os.environ.get("WORLD_SIZE", "1"))
if world > 1:
    distributed.init_from_env(backend="gloo")
cfg = dict(vs=60, vt=70, es=11, he=7, et=9, hd=8, out=9, maxout=True, max_len=10, supress_unk=True)
model = build_bahdanau(**cfg, lr=1e-2, clip=1.0, l2=1e-3)
model["arena"].load_dict(oracle_params_for(model))
losses = []
for step in range(3):
    src, tgt = random_batch(8, 8, 7, cfg["vs"], cfg["vt"], seed=40 + step)
    if world > 1:                         # every rank takes its slice of the SAME global batch
        lo, hi = distributed.shard_bounds(8, world)[distributed.rank():distributed.rank() + 2]
        src, tgt = src[lo:hi], tgt[lo:hi]
    feed(model, src, tgt, train=True)
    losses.append(float(model["trainer"].train_step()["losses"][0]))
if world > 1:
    # the decoder-side ranges were exchanged from inside the backward pass, in every step
    assert getattr(model["trainer"], "early_exchanges", 0) == 3, getattr(model["trainer"], "early_exchanges", 0)
    _enc, early, late = model["trainer"]._exchange_plan()
    assert early and late and sum(hi - lo for lo, hi in early + late) == model["arena"].trainable_size
if distributed.rank() == 0:
    torch.save({{"params": model["arena"].state_dict(), "losses": losses}}, {out!r} + str(world))
print("rank", distributed.rank(), "done")
"""


def test_two_rank_data_parallel_training_equals_the_single_process_run(tmp_path):
    """SURVEY.md 8(e): the global batch split by sentence over 2 ranks (gloo, CPU stand-in ops), un-normalised
    loss sums and token counts all-reduced with the gradients, the division by the GLOBAL count inside the
    optimizer step - three steps give the losses and parameters of one process on the whole batch."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = tmp_path / "dp_worker.py"
    script.write_text(_DP_WORKER.format(root=root, out=str(tmp_path / "result")))
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    single = subprocess.run([sys.executable, str(script)], capture_output=True, text=True, timeout=300,
                            env=dict(env, WORLD_SIZE="1"), cwd=root)
    assert single.returncode == 0, single.stdout + single.stderr
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
           "--master-addr", "127.0.0.1", "--master-port", "29613", str(script)]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=300, env=env, cwd=root)
    assert res.returncode == 0, res.stdout + res.stderr
    one, two = torch.load(str(tmp_path / "result1")), torch.load(str(tmp_path / "result2"))
    assert one["losses"] == pytest.approx(two["losses"], abs=1e-5)
    for name, want in one["params"].items():
        if name.endswith("attn_bias"):
            continue
        assert float((two["params"][name] - want).abs().max()) < 2e-5, name


_DP_CLI_WORKER = r"""
import os, sys, torch
sys.path.insert(0, {root!r})
from neuralmonkey_b200 import ops, runtime
from neuralmonkey_b200.trainers.generic_trainer import GenericTrainer
from tests import cpu_ops
for name in cpu_ops.STAND_INS:
    setattr(ops, name, getattr(cpu_ops, name))
runtime._device = torch.device("cpu")
GenericTrainer._adam_kernel = cpu_ops.adam_kernel
from neuralmonkey_b200 import distributed
distributed.init_from_env(backend="gloo")     # CPU tensors: gloo even where a GPU (and with it NCCL) is present
sys.argv = ["neuralmonkey-train", {ini!r}]
from neuralmonkey_b200.train import main
main()
"""


def test_two_rank_training_through_the_entry_point(tmp_path):
    """`torchrun --nproc-per-node 2 neuralmonkey-train INI` (gloo, CPU stand-in ops): every rank takes its
    share of each batch, rank 0 alone logs, validates and writes the checkpoints and outputs."""
    from tests import test_gpu_cli as cli
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    data, out = str(tmp_path / "data"), str(tmp_path / "out")
    cli._write_data(data)
    ini = tmp_path / "exp.ini"
    ini.write_text(cli.INI.format(out=out, data=data, epochs=2))
    script = tmp_path / "worker.py"
    script.write_text(_DP_CLI_WORKER.format(root=root, ini=str(ini)))
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", NEURALMONKEY_STRICT="1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
           "--master-addr", "127.0.0.1", "--master-port", "29617", str(script)]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=env, cwd=root)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    log_text = open(os.path.join(out, "experiment.log")).read()
    assert "Validation (epoch" in log_text and "Training finished" in log_text
    losses = training_log_values(log_text, "target/train_xent")
    assert len(losses) >= 2 and losses[-1] < losses[0], losses
    assert len(open(os.path.join(out, "val.out")).read().splitlines()) == 30
    assert os.path.exists(os.path.join(out, "variables.data.final"))


def test_data_parallel_training_never_hands_a_rank_an_empty_shard(monkeypatch):
    """A batch with fewer sentences than ranks (the remainder of an epoch, a flushed bucket) is held over
    and merged into the next one: every executed batch gives every rank >= 1 sentence, identically on all
    ranks; nothing hangs in the all-reduce."""
    from argparse import Namespace
    from neuralmonkey_b200 import learning_utils
    from neuralmonkey_b200.dataset import BatchingScheme, Dataset

    def batch(ids):
        rows = [["w{}".format(i)] for i in ids]
        return Dataset("b", {"source": (lambda r=rows: iter(r))}, BatchingScheme(batch_size=8))

    sizes = [5, 2, 3, 1, 6, 2]                  # world = 4: the 2-, 3-, 1- and final 2-sentence batches are short
    batches, nxt = [], 0
    for n in sizes:
        batches.append(batch(range(nxt, nxt + n)))
        nxt += n

    class Trainer:
        feedables = set()

    class Manager:
        best_score, best_score_epoch, best_score_batch = 0.0, 0, 0
        executed = []

        def initialize_model_parts(self, _executors):
            pass

        def execute(self, local, _feedables, _trainers, train=False, summaries=True):
            Manager.executed.append([row[0] for row in local.get_series("source")])

    for rank in range(4):
        Manager.executed = []
        monkeypatch.setattr(distributed, "world_size", lambda: 4)
        monkeypatch.setattr(distributed, "rank", lambda r=rank: r)
        cfg = Namespace(runners=[], trainers=[Trainer()], postprocess=None, initial_variables=None,
                        tf_manager=Manager(), epochs=1, train_dataset=Namespace(batches=lambda: iter(batches)),
                        train_start_offset=0, log_timer=lambda step, last: False,
                        val_timer=lambda step, last: False, val_datasets=[], main_metric="x")
        learning_utils.training_loop(cfg)
        # executed global batches: [5], [2+3], [1+6]; the last 2 sentences (< 4 ranks) are dropped
        assert [len(x) for x in Manager.executed] == {0: [2, 2, 2], 1: [1, 1, 2], 2: [1, 1, 2], 3: [1, 1, 1]}[rank]
        assert all(len(x) > 0 for x in Manager.executed)
    # rank 0's shards are the leading sentences of the merged batches
    assert Manager.executed is not None


def test_shutdown_releases_what_was_registered_first_and_is_idempotent():
    """distributed.shutdown(): cleanups (a trainer's CUDA graphs that captured collectives) run before the
    process group would be destroyed, newest first, once; without a process group the rest is a no-op."""
    from neuralmonkey_b200 import distributed
    order = []
    first, second = (lambda: order.append("first")), (lambda: order.append("second"))
    distributed.register_cleanup(first)
    distributed.register_cleanup(second)
    distributed.register_cleanup(first)              # registered once
    distributed.shutdown()
    distributed.shutdown()
    assert order == ["second", "first"]


def test_weight_gradient_window_stays_shut_without_a_gpu_and_while_profiling(monkeypatch):
    """ops.weight_grad_stream(): the second stream is a GPU affair (the trainer opens the window only for CUDA
    arenas) and yields to the per-call profiler, whose times assume calls that do not overlap."""
    from neuralmonkey_b200 import lib, ops
    ran = []
    ops.weight_grad_stream(False)
    ops._off_the_chain(lambda: ran.append(1))        # window shut: runs in place, keeps nothing alive
    assert ran == [1] and not ops._wg["keep"]
    ops.join_weight_grads()                           # nothing to wait for
    monkeypatch.setenv("NMB200_WGRAD_STREAM", "0")
    ops.weight_grad_stream(True)
    assert ops._wg["open"] is False
    monkeypatch.setenv("NMB200_WGRAD_STREAM", "1")
    monkeypatch.setattr(lib, "_profile", {})          # as between profile_start() and profile_stop()
    ops.weight_grad_stream(True)
    assert ops._wg["open"] is False


def test_dropout_helper_on_the_cpu_with_a_residual():
    """nn.utils.dropout off the GPU (the stand-in path of the host tests): identity when inactive, mask product
    plus the residual otherwise."""
    import torch
    from neuralmonkey_b200.nn import utils
    x, res = torch.ones(4, 6), torch.full((4, 6), 2.0)
    assert utils.dropout(x, 1.0, True) is x and utils.dropout(x, 0.5, False) is x
    assert torch.equal(utils.dropout(x, 1.0, True, residual=res), x + res)
    torch.manual_seed(0)
    y = utils.dropout(x, 0.5, True, residual=res)
    assert set(y.unique().tolist()) <= {2.0, 4.0}     # 0 or 1 / keep_prob, plus the residual


def test_model_part_save_and_load(tmp_path, monkeypatch):
    """The reference's tests/test_model_part.py::test_save_and_load restated without sessions: a part with
    `save_checkpoint` / `load_checkpoint` files stores the variables of ITS scope and restores them into a
    freshly initialised model; other parts' variables are neither written nor touched
    (model/parameterized.py:98-125, tf_manager.py:279-289, learning_utils.py:146-159)."""
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.encoders import SentenceEncoder
    from neuralmonkey_b200.tf_manager import TensorFlowManager
    from neuralmonkey_b200.vocabulary import Vocabulary

    # relative file names: SentenceEncoder derives its input sequence's files as "input_" + name
    # (encoders/recurrent.py:279-280), which only works for those
    monkeypatch.chdir(tmp_path)
    path = "enc.ckpt"

    def make(seed):
        runtime.reset()
        vocabulary = Vocabulary(["a", "b"])
        enc = SentenceEncoder(name="enc", vocabulary=vocabulary, data_id="data_id", embedding_size=10,
                              rnn_size=20, max_input_len=30, save_checkpoint=path, load_checkpoint=path)
        other = SentenceEncoder(name="other", vocabulary=vocabulary, data_id="data_id", embedding_size=10,
                                rnn_size=20, max_input_len=30)
        for part in (enc, other):
            for dep in part.get_dependencies()[1]:
                dep.ensure_declared()
        runtime.arena().finalize(torch.device("cpu"), seed=seed)
        return enc, other

    class _Runner:          # what initialize_model_parts looks at
        def __init__(self, *parts):
            self.parameterizeds = set()
            for p in parts:
                self.parameterizeds |= p.get_dependencies()[1]

    enc, other = make(seed=1)
    first = runtime.arena().state_dict()
    TensorFlowManager(num_sessions=1, num_threads=1).initialize_model_parts([_Runner(enc, other)], save=True)
    stored = torch.load(path)["variables"]
    # tf.get_collection(..., scope="enc") is a regex match at the start of the name: `enc_input/...` is covered
    mine = [n for n in first if n.startswith("enc/") or n.startswith("enc_input/")]
    assert any(n.startswith("enc/") for n in mine) and any(n.startswith("enc_input/") for n in mine)
    assert sorted(stored) == sorted(mine)                   # nothing of `other/`
    assert sorted(torch.load("input_enc.ckpt")["variables"]) == sorted(n for n in first if n.startswith("enc_input/"))

    enc, other = make(seed=2)
    second = runtime.arena().state_dict()
    assert any(not torch.equal(first[n], second[n]) for n in mine)
    TensorFlowManager(num_sessions=1, num_threads=1).initialize_model_parts([_Runner(enc, other)])
    now = runtime.arena().state_dict()
    assert all(torch.equal(now[n], first[n]) for n in mine)
    assert all(torch.equal(now[n], second[n]) for n in now if n.startswith("other"))

    # a checkpoint that lacks one of the part's variables is an error, as with Saver.restore
    del stored[mine[0]]
    torch.save({"variables": stored}, path)
    try:
        enc.load()
    except KeyError as exc:
        assert mine[0] in str(exc)
    else:
        raise AssertionError("a missing variable must be reported")
    try:
        TensorFlowManager(num_sessions=1, num_threads=1).initialize_model_parts([object()])
    except TypeError:
        pass
    else:
        raise AssertionError("executors without `parameterizeds` must be refused")
    runtime.reset()


def test_word2vec_files_and_the_perplexity_evaluator(tmp_path):
    """util/word2vec.py (vocabulary + embedding initialiser from a word2vec text file: special tokens first,
    zeros unless the file has them) and evaluators.PerplexityEvaluator (2 ** mean of the non-zero
    cross-entropies), as tests/language-model.ini uses them; compared with what the reference's module loads
    from its sample file."""
    import numpy as np
    from neuralmonkey_b200.evaluators import PerplexityEvaluator
    from neuralmonkey_b200.util import word2vec
    path = tmp_path / "toy.w2v"
    path.write_text("3 2\nhello 0.5 -1\n</s> 0.25 0.75\nworld 2 3\n")
    w2v = word2vec.Word2Vec(str(path))
    assert w2v.vocabulary.index_to_word == ["<pad>", "<s>", "</s>", "<unk>", "hello", "world"]
    assert w2v.embeddings.tolist() == [[0, 0], [0, 0], [0.25, 0.75], [0, 0], [0.5, -1], [2, 3]]
    assert word2vec.word2vec_vocabulary(w2v) is w2v.vocabulary
    init = word2vec.get_word2vec_initializer(w2v)
    assert init([6, 2], None).tolist() == w2v.embeddings.tolist()
    with pytest.raises(ValueError, match="do not match"):
        init([6, 3], None)
    arena = ParameterArena()
    arena.declare("decoder/word_embeddings", [6, 2], init)
    arena.finalize(torch.device("cpu"))
    assert arena.get("decoder/word_embeddings").tolist() == w2v.embeddings.tolist()

    ppl = PerplexityEvaluator("perplexity")
    assert ppl([[1.0, 3.0, 0.0], [2.0, 0.0, 0.0]], [[], []]) == 2 ** 2.0
    assert ppl([[0.0]], [[]]) != ppl([[0.0]], [[]])          # NaN: nothing counted
    # the reference's own loader on its sample file (tests/golden/make_word2vec_golden.py)
    golden = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    with open(os.path.join(golden, "reference_experiments_late.json"), encoding="utf-8") as handle:
        (tmp_path / "sample.w2v").write_text(json.load(handle)["files"]["tests/data/sample.w2v"])
    with open(os.path.join(golden, "word2vec_golden.json"), encoding="utf-8") as handle:
        theirs = json.load(handle)
    ours = word2vec.Word2Vec(str(tmp_path / "sample.w2v"))
    assert np.array_equal(np.array(theirs["embeddings"], dtype=ours.embeddings.dtype), ours.embeddings)
    assert theirs["index_to_word"] == ours.vocabulary.index_to_word


def test_model_part_reuse_shares_variables():
    """The reference's tests/test_model_part.py::test_reuse restated without sessions: a part built with
    `reuse=<other part>` lives in the other part's variable scope - same variables, one copy in the arena - while
    an independent part of the same shape gets its own, differently initialised ones (parameterized.py:44-60)."""
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.model.sequence import EmbeddedSequence
    from neuralmonkey_b200.vocabulary import Vocabulary
    runtime.reset()
    vocabulary = Vocabulary(["a", "b"])
    seq1 = EmbeddedSequence(name="seq1", vocabulary=vocabulary, data_id="id", embedding_size=10)
    seq2 = EmbeddedSequence(name="seq2", vocabulary=vocabulary, embedding_size=10, data_id="id")
    seq3 = EmbeddedSequence(name="seq3", vocabulary=vocabulary, data_id="id", embedding_size=10, reuse=seq1)
    for part in (seq1, seq2, seq3):
        part.ensure_declared()
    arena = runtime.arena()
    arena.finalize(torch.device("cpu"))
    assert sorted(arena.order) == ["seq1/embedding_matrix_0", "seq2/embedding_matrix_0"]
    first, second, third = seq1.embedding_matrix, seq2.embedding_matrix, seq3.embedding_matrix
    assert not torch.equal(first, second)
    assert torch.equal(first, third) and first.data_ptr() == third.data_ptr()
    # a reusing part may not bring its own initialisers (parameterized.py:52-56)
    with pytest.raises(ValueError, match="Cannot use initializers in model part"):
        EmbeddedSequence(name="seq4", vocabulary=vocabulary, data_id="id", embedding_size=10, reuse=seq1,
                         initializers=[("embedding_matrix_0", zeros_initializer())])
    runtime.reset()


def test_dropout_helper_as_the_reference_unit_test():
    """neuralmonkey/tests/test_nn_utils.py restated: invalid keep probabilities raise (tf.nn.dropout's check, in
    either mode), the dropped share follows 1 - keep_prob with the survivors scaled by 1 / keep_prob, and nothing
    happens outside training."""
    from neuralmonkey_b200.nn.utils import dropout
    var = torch.ones(10000)
    for kprob in (-1, 2, 0):
        for mode in (True, False):
            with pytest.raises(ValueError):
                dropout(var, kprob, mode)
    torch.manual_seed(0)
    for kprob in (0.1, 0.7):
        dropped = dropout(var, kprob, True)
        assert abs(int((dropped == 0.0).sum()) - 10000 * (1 - kprob)) < 500
        assert float(dropped.max()) == pytest.approx(1.0 / kprob)
    assert float(dropout(var, 0.1, False).sum()) == 10000
    assert dropout(var, 1.0, True) is var


def test_bench_realistic_length_batches_are_well_formed():
    """`bench.py --lengths realistic` (SURVEY.md 8(d)): lengths ~ N(0.6 T, 0.2 T) clipped to [1, T], rows are
    tokens, (target: </s>,) padding; one full-length sentence keeps the padded shape fixed; the fixed-length batches
    of the headline are what they were (same generator draws)."""
    import bench
    src, tgt = bench.synthetic_batch(256, 5, realistic=True)
    fixed_src, fixed_tgt = bench.synthetic_batch(256, 5)
    assert src.shape == fixed_src.shape == (256, 50) and tgt.shape == (256, 50)
    assert bool((fixed_src >= 4).all()) and bool((fixed_tgt[:, :-1] >= 4).all()) and bool((fixed_tgt[:, -1] == 2).all())
    src_len, tgt_len = (src != 0).sum(1), (tgt != 0).sum(1)
    assert int(src_len[0]) == 50 and int(tgt_len[0]) == 50 and int(src_len.min()) >= 1 and int(tgt_len.min()) >= 1
    assert 25 < float(src_len.float().mean()) < 35 and 25 < float(tgt_len.float().mean()) < 35
    for b in range(256):
        n, m = int(src_len[b]), int(tgt_len[b])
        assert bool((src[b, :n] >= 4).all()) and bool((src[b, n:] == 0).all())
        assert bool((tgt[b, :m - 1] >= 4).all()) and int(tgt[b, m - 1]) == 2 and bool((tgt[b, m:] == 0).all())
        assert bool((src[b, :n] == fixed_src[b, :n]).all())       # the same ids, cut


def test_ini_loop_bench_tool_over_the_stand_in_operations():
    """tools/ini_loop_bench.py (`neuralmonkey-train` on a synthetic corpus on disk, timed from inside the loop):
    its host logic over the CPU stand-ins at toy dims - one JSON line on stdout, the step / token bookkeeping."""
    import json
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    res = subprocess.run([sys.executable, os.path.join(root, "tools", "ini_loop_bench.py"), "--standins", "--rnn", "16",
                          "--vocab", "300", "--sentences", "160", "--batch", "16", "--skip", "3"],
                         capture_output=True, text=True, timeout=600, cwd=root)
    assert res.returncode == 0, res.stderr[-2000:]
    lines = [l for l in res.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, res.stdout
    line = json.loads(lines[0])
    assert line["steps"] == 7 and line["value"] > 0 and line["unit"] == "tokens/s"
    assert line["value"] == pytest.approx(7 * 16 * 50 / (line["ms_per_step"] * 7 * 1e-3), rel=1e-6)
    assert "Training finished" in res.stderr
